"""Fixed cost per launch of the fused FC kernel: t(n) = a + n / r fitted to back-to-back launches at 2^18 .. 2^23 images.

    python tools/launch_overhead.py [model] [--steps 20] [--rounds 3]
    BNM_LIB_PATH=<BNM_FC_TRACE build> python tools/launch_overhead.py [model] --trace

Timing run (product build): device-resident int8 images in two buffers alternated per launch (each larger than the 50 MB
L2 from 2^18 images up) and double-buffered outputs, as bench.py does.  Every round visits every size and, per size, the
launch arms in turn: BNM_OPT_LAUNCH_OVERLAP 0, 1 and 2 on one stream, and mode 0 alternating between two streams.  An arm
is `steps` launches between two CUDA events after three warm-up launches; the median over rounds is kept.  The least-squares
fit over the sizes gives per arm the steady rate r (G images/s) and the fixed cost a (us per launch).  The card's name,
power limit and the SM clock sampled over the timed region are printed with the numbers.

Trace run (a BNM_FC_TRACE build; every traced launch synchronises, so it runs alone): one launch per size up to 2^22 (the
trace buffer's 2048 events per warpgroup hold 124 tiles) after warm-up, and per traced CTA
  start -> full>    kernel entry to the first pass of a full barrier (prologue: barriers, weights; then the first tile's load)
  issue -> end      the last layer-1 issue of the CTA (its last tile enters compute) to its last epilogue (the drain)
  last load         the producer's last TMA issue, from kernel entry
  CTA span          kernel entry to exit
so that `a` splits into launch gap + prologue + ramp (start -> full>) and drain (issue -> end)."""
import argparse
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

SIZES = [1 << k for k in range(18, 24)]
ARMS = ("mode 0", "mode 1", "mode 2", "mode 0, two streams")


def card():
    """name, power limit and maximum SM clock of the visible device, as nvidia-smi reports them"""
    try:
        import torch
        from bench import ClockSampler
        sel = ClockSampler.device_selector(torch.cuda.current_device())
        out = subprocess.run(["nvidia-smi", "-i", sel, "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or "nvidia-smi: no output"
    except Exception as ex:
        return f"nvidia-smi unavailable: {ex}"


def fit(ns, us):
    """least-squares t = a + n / r: (a in us, r in G images/s)"""
    slope, a = np.polyfit(np.asarray(ns, float), np.asarray(us, float), 1)
    return a, 1e-3 / slope


def timing(eng, args):
    import torch
    from bench import ClockSampler
    from bitnetmcu_b200 import _lib
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    res = {(arm, n): [] for arm in ARMS for n in SIZES}
    sampler = ClockSampler(ClockSampler.device_selector(torch.cuda.current_device()))
    sampler.start()
    time.sleep(0.3)
    t0 = time.perf_counter()
    for _ in range(args.rounds):
        for n in SIZES:
            g = torch.Generator(device="cuda").manual_seed(n)
            x = [torch.randint(-128, 128, (n, eng.img_bytes), dtype=torch.int8, device="cuda", generator=g) for _ in range(2)]
            lo = [torch.empty((n, eng.n_classes), dtype=torch.int32, device="cuda") for _ in range(2)]
            la = [torch.empty(n, dtype=torch.int32, device="cuda") for _ in range(2)]
            for arm in ARMS:
                two = arm.endswith("two streams")
                eng.set_option(_lib.OPT_LAUNCH_OVERLAP, 0 if two else int(arm[5]))

                def launch(i):
                    eng.infer_device(x[i & 1], lo[i & 1], la[i & 1], streams[i & 1].cuda_stream if two else None)
                for i in range(3):
                    launch(i)
                torch.cuda.synchronize()
                a, b0, b1 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
                if two:
                    a.record(streams[0]); streams[1].wait_event(a)
                else:
                    a.record()
                for i in range(args.steps):
                    launch(i)
                if two:
                    b0.record(streams[0]); b1.record(streams[1])
                else:
                    b0.record(); b1 = b0
                torch.cuda.synchronize()
                res[(arm, n)].append(max(a.elapsed_time(b0), a.elapsed_time(b1)) / args.steps * 1e3)
            del x, lo, la
            torch.cuda.empty_cache()
    t1 = time.perf_counter()
    clocks = sampler.stop(t0, t1, "the timed launches")
    if sampler.proc:
        sampler.proc.wait(timeout=10)
    eng.set_option(_lib.OPT_LAUNCH_OVERLAP, 0)

    print(f"card: {card()}; SM clock over the timed launches: median {clocks.get('sm_mhz')} MHz "
          f"(max {clocks.get('sm_max_mhz')}), power draw max {clocks.get('power_w_max')} W, throttle reasons {clocks.get('reasons')}")
    print(f"{args.steps} launches per arm and size, median of {args.rounds} rounds; us per launch (G images/s)")
    print(f"{'images':>9} " + " ".join(f"{arm:>24}" for arm in ARMS))
    med = {k: float(np.median(v)) for k, v in res.items()}
    for n in SIZES:
        print(f"{n:>9} " + " ".join(f"{med[(arm, n)]:>12.2f} ({n / med[(arm, n)] * 1e-3:6.3f} G)" for arm in ARMS))
    print("fit t(n) = a + n / r over the sizes:")
    for arm in ARMS:
        a, r = fit(SIZES, [med[(arm, n)] for n in SIZES])
        t20 = med[(arm, 1 << 20)]
        print(f"  {arm:<22} a = {a:6.2f} us   r = {r:6.3f} G images/s   a / t(2^20) = {100 * a / t20:4.1f} %")


def trace(eng, args):
    import torch
    from fc_phase_trace import EMPTY_END, EPI_END, FULL_END, ISSUE, read_trace
    print(f"card: {card()}")
    print("per traced CTA, us: start -> full> | issue -> end | last load | CTA span (tiles of the CTA)")
    for n in SIZES[:-1]:
        x = torch.randint(-128, 128, (n, eng.img_bytes), dtype=torch.int8, device="cuda")
        lo = torch.empty((n, eng.n_classes), dtype=torch.int32, device="cuda")
        la = torch.empty(n, dtype=torch.int32, device="cuda")
        for _ in range(3):
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
        del x, lo, la
        n_ctas, n_writers = count.shape
        rows = []
        for c in range(n_ctas):
            gt0, clk0, gt1, clk1 = (int(v) for v in hdr[c])
            ghz = (clk1 - clk0) / max(1, gt1 - gt0)
            us = lambda clk: (clk - clk0) / ghz * 1e-3
            cons = [(int(t), int(code)) for w in range(n_writers - 1) for t, code in ev[c, w, :int(count[c, w])]]
            prod = [(int(t), int(code)) for t, code in ev[c, n_writers - 1, :int(count[c, n_writers - 1])]]
            first_full = min((t for t, code in cons if code & 0xff == FULL_END), default=None)
            last_issue = max((t for t, code in cons if code & 0xff == ISSUE and (code >> 12) & 0xf == 0), default=None)
            last_epi = max((t for t, code in cons if code & 0xff == EPI_END), default=None)
            last_load = max((t for t, code in prod if code & 0xff == EMPTY_END), default=None)
            if first_full is None or last_issue is None or last_epi is None:
                continue
            tiles = sum(1 for _, code in prod if code & 0xff == EMPTY_END)
            rows.append((us(first_full), (last_epi - last_issue) / ghz * 1e-3, us(last_load) if last_load else float("nan"),
                         (gt1 - gt0) * 1e-3, tiles))
        print(f"  {n:>8} images: " + "   ".join(f"{a:5.2f} | {d:5.2f} | {l:6.1f} | {s:6.1f} ({t})" for a, d, l, s, t in rows))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("model", nargs="?", default="fc")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--trace", action="store_true", help="per-CTA prologue and drain from a BNM_FC_TRACE build")
    args = ap.parse_args()
    from bitnetmcu_b200.engine import Engine
    from bitnetmcu_b200.model import Model
    eng = Engine(Model.load(os.path.join(ROOT, "tests", "golden", "models", args.model + ".bnm")))
    print(f"model {args.model}, fused kernel {'trace' if args.trace else 'timing'} run")
    (trace if args.trace else timing)(eng, args)
    eng.close()


if __name__ == "__main__":
    main()
