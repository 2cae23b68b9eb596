"""Phase trace of the fused FC kernel: median cycles per phase and per tile round, from the clock64 stamps of a trace build.

    make -C bitnetmcu_b200/csrc clean && make -C bitnetmcu_b200/csrc EXTRA=-DBNM_FC_TRACE
    python tools/fc_phase_trace.py [model] [--batch N]

(or point BNM_LIB_PATH at a trace build kept elsewhere).  Runs `batch` random images (default 2^20) through the model (default
the fc fixture), a few warm-up launches first, then one traced launch, and prints per consumer warpgroup and for the producer:
  full wait     mbar_wait on full[] (the tile's stage has not landed yet)
  issue L       (stamp) the warpgroup starts issuing layer L's wgmma: ReLUNorm ends before it, the issue runs after it
  mma wait L    wgmma.wait_group of layer L (cycles the warpgroup blocks on its own tensor-core work)
  round         one slot's cycles from one full-wait begin to the next (a tile's whole trip through the slot)
  period        cycles between consecutive tiles finished by the warpgroup
and per CTA the tiles in compute (sum of tile residencies, full-wait end to epilogue end, over the traced window, halved because
two warpgroups share a tile) and the SM clock over the launch (clock64 against %globaltimer)."""
import argparse
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

FULL_BEGIN, FULL_END, WAIT_BEGIN, WAIT_END, EPI_END, EMPTY_BEGIN, EMPTY_END, ISSUE = range(1, 9)


def read_trace(path):
    raw = open(path, "rb").read()
    ctas, writers, events = np.frombuffer(raw, np.uint32, 3)
    off = 12
    hdr = np.frombuffer(raw, np.uint64, ctas * 4, off).reshape(ctas, 4)
    off += hdr.nbytes
    count = np.frombuffer(raw, np.uint32, ctas * writers, off).reshape(ctas, writers)
    off += count.nbytes
    off = (off - 12 + 15) // 16 * 16 + 12   # ulonglong2 alignment inside the struct
    ev = np.frombuffer(raw, np.uint64, ctas * writers * events * 2, off).reshape(ctas, writers, events, 2)
    return hdr, count, ev


def label(code):
    """event code -> short name: full< full> issueL wait<L wait>L epi (L = layer, from 1; issueL: its wgmma issue starts)"""
    kind, layer = code & 0xff, (code >> 12) & 0xf
    return {FULL_BEGIN: "full<", FULL_END: "full>", WAIT_BEGIN: f"wait<{layer + 1}", WAIT_END: f"wait>{layer + 1}",
            EPI_END: "epi", ISSUE: f"issue{layer + 1}"}.get(kind, str(kind))


def med(xs):
    return float(np.median(xs)) if len(xs) else float("nan")


def consumer_tiles(evs):
    """events of one consumer warpgroup -> per slot, list of tiles {fb, fe, waits: {layer: cycles}, epi}"""
    tiles, cur = {}, {}
    for t, code in evs:
        kind, slot, layer = code & 0xff, (code >> 8) & 0xf, (code >> 12) & 0xf
        if kind == FULL_BEGIN:
            cur[slot] = {"fb": t, "waits": {}, "wb": None}
        elif slot not in cur:
            continue
        elif kind == FULL_END:
            cur[slot]["fe"] = t
        elif kind == WAIT_BEGIN:
            cur[slot]["wb"] = t
        elif kind == WAIT_END and cur[slot]["wb"] is not None:
            cur[slot]["waits"][layer] = t - cur[slot]["wb"]
        elif kind == EPI_END:
            cur[slot]["epi"] = t
            tiles.setdefault(slot, []).append(cur.pop(slot))
    return tiles


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("model", nargs="?", default="fc")
    ap.add_argument("--batch", type=int, default=1 << 20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()

    import torch
    from bitnetmcu_b200.engine import Engine
    from bitnetmcu_b200.model import Model

    eng = Engine(Model.load(os.path.join(ROOT, "tests", "golden", "models", args.model + ".bnm")))
    x = torch.randint(-128, 128, (args.batch, eng.img_bytes), dtype=torch.int8, device="cuda")
    lo = torch.empty((args.batch, eng.n_classes), dtype=torch.int32, device="cuda")
    la = torch.empty(args.batch, dtype=torch.int32, device="cuda")
    for _ in range(args.warmup):
        eng.infer_device(x, lo, la)
    torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "trace.bin")
        os.environ["BNM_FC_TRACE_OUT"] = path
        eng.infer_device(x, lo, la)
        torch.cuda.synchronize()
        del os.environ["BNM_FC_TRACE_OUT"]
        if not os.path.exists(path):
            sys.exit("no trace written: the library is not a BNM_FC_TRACE build")
        hdr, count, ev = read_trace(path)
    eng.close()
    print(f"model {args.model}, batch {args.batch}")
    report(hdr, count, ev)


def report(hdr, count, ev):
    n_ctas, n_writers = count.shape
    print(f"traced CTAs 0..{n_ctas - 1}")
    rows = {"full wait": [], "round": [], "period": []}
    mma, steps, wg_cycles = {}, {}, [0, 0]
    full_share, in_compute, clocks, empty_waits, empty_share = [], [], [], [], []
    for c in range(n_ctas):
        gt0, clk0, gt1, clk1 = (int(v) for v in hdr[c])
        if gt1 > gt0:
            clocks.append((clk1 - clk0) / (gt1 - gt0))
        resid, t_lo, t_hi = 0, None, None
        for w in range(n_writers - 1):
            n = int(count[c, w])
            if n == 0:
                continue
            evs = [(int(t), int(code)) for t, code in ev[c, w, :n]]
            tiles = consumer_tiles(evs)
            all_tiles = sorted((tt for ts in tiles.values() for tt in ts if "fe" in tt), key=lambda tt: tt["epi"])
            if not all_tiles:
                continue
            lo_t, hi_t = all_tiles[0]["fb"], all_tiles[-1]["epi"]
            t_lo = lo_t if t_lo is None else min(t_lo, lo_t)
            t_hi = hi_t if t_hi is None else max(t_hi, hi_t)
            full_share.append(sum(tt["fe"] - tt["fb"] for tt in all_tiles) / max(1, hi_t - lo_t))
            for tt in all_tiles:
                rows["full wait"].append(tt["fe"] - tt["fb"])
                for l, cyc in tt["waits"].items():
                    mma.setdefault(l, []).append(cyc)
                resid += tt["epi"] - tt["fe"]
            for ts in tiles.values():
                rows["round"] += [b["fb"] - a["fb"] for a, b in zip(ts, ts[1:])]
            epis = [tt["epi"] for tt in all_tiles]
            rows["period"] += list(np.diff(epis))
            # time between consecutive stamps of the warpgroup (whatever the slot), by the pair of events
            for (t0, c0), (t1, c1) in zip(evs, evs[1:]):
                steps.setdefault((label(c0), label(c1)), []).append(t1 - t0)
            wg_cycles[0] += evs[-1][0] - evs[0][0]
            wg_cycles[1] += len(all_tiles)
        if t_hi is not None and t_hi > t_lo:
            in_compute.append(resid / 2 / (t_hi - t_lo))
        n = int(count[c, n_writers - 1])
        evs = [(int(t), int(code) & 0xff) for t, code in ev[c, n_writers - 1, :n]]
        waits = [b[0] - a[0] for a, b in zip(evs, evs[1:]) if a[1] == EMPTY_BEGIN and b[1] == EMPTY_END]
        empty_waits += waits
        if len(evs) > 1:
            empty_share.append(sum(waits) / max(1, evs[-1][0] - evs[0][0]))
    print(f"SM clock over the launch: {med(clocks):.3f} GHz (median over traced CTAs)")
    print("consumer warpgroups, cycles per tile (median over traced tiles):")
    print(f"  full wait           {med(rows['full wait']):8.0f}   share of the warpgroup's time {100 * med(full_share):.1f} %")
    for l in sorted(mma):
        print(f"  mma wait layer {l + 1}    {med(mma[l]):8.0f}")
    print(f"  round (per slot)    {med(rows['round']):8.0f}")
    print(f"  period (per wg)     {med(rows['period']):8.0f}")
    print(f"tiles in compute per SM: {med(in_compute):.2f}")
    print("consumer warpgroups, time between consecutive stamps (cycles per tile = mean x count / tiles):")
    per_tile = max(1, wg_cycles[1])
    for (a, b), xs in sorted(steps.items(), key=lambda kv: -sum(kv[1])):
        tot = sum(xs)
        if tot < 0.005 * wg_cycles[0]:
            continue
        print(f"  {a:>10} -> {b:<10} median {med(xs):7.0f}   per tile {tot / per_tile:7.0f}   share {100 * tot / max(1, wg_cycles[0]):5.1f} %")
    print(f"producer: empty wait median {med(empty_waits):.0f} cycles per tile, share of its time {100 * med(empty_share):.1f} %")


if __name__ == "__main__":
    main()
