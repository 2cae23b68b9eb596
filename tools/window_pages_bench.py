"""Window scan of a stack of pages against what a caller does without the stacked entries, alternated in one process.

Cases, each timed with CUDA events over back-to-back calls on one stream:
  * labels:   one bnm_scan_windows_device call on the whole stack against a loop of bnm_infer_windows_device_f32, one call per
              page (labels only);
  * top-5:    bnm_scan_windows_topk_device (k = 5, classes and scores) against bnm_scan_windows_device writing every window's
              logits, then torch.topk over them;
  * emulator: bnm_emulate_windows_device (labels) against the pages unfolded plane by plane, up to 2^20 windows at a time, into a
              float buffer (1 KB per window written and read again), then bnm_emulate_batch_device on it.
Stacks: 64 pages of 1024 x 1024 (every case) and 16 pages of 4096 x 4096 (labels), strides 1, 4 and 16.  Models: FC 4bitsym-64, a
64-wide 4bitsym model with 37 classes (random weights: speed does not depend on them) and CNN-48.  Each round times every variant,
the rounds rotate which goes first, the report is the median over rounds.  Every row checks that the variants' outputs are equal:
labels, or the top-5 scores and classes (classes against a stable sort of the logits, ties to the lower class).  Prints the card
name, its power limit and SM clocks.

    python tools/window_pages_bench.py [--rounds 3] [--steps 2]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bitnetmcu_b200 import pack  # noqa: E402
from bitnetmcu_b200.engine import Engine, window_grid  # noqa: E402
from bitnetmcu_b200.model import Model  # noqa: E402
from window_bench import card, events_ms  # noqa: E402

CHUNK = 1 << 20
K = 5


def timed(variants, rounds, steps):
    """{name: median ms per call}, {name: [min, max]} of alternated rounds"""
    names = list(variants)
    ms = {k: [] for k in names}
    for r in range(rounds):
        for k in names[r % len(names):] + names[:r % len(names)]:
            ms[k].append(events_ms(variants[k], steps, 1))
    torch.cuda.synchronize()
    return {k: float(np.median(v)) for k, v in ms.items()}, {k: [min(v), max(v)] for k, v in ms.items()}


def unfolded(pages, s, buf, fn):
    """fn(rows, w0) on the pages' windows, unfolded plane by plane into buf, float32 [2^20, 256], whole window rows at a time"""
    n_p, h, w = pages.shape
    oh, ow = window_grid(h, w, s)
    per = max(1, CHUNK // ow)
    for p in range(n_p):
        win = pages[p].unfold(0, 16, s).unfold(1, 16, s)
        for r0 in range(0, oh, per):
            r1 = min(oh, r0 + per)
            k = (r1 - r0) * ow
            buf[:k].view(r1 - r0, ow, 16, 16).copy_(win[r0:r1])
            fn(buf[:k], (p * oh + r0) * ow)


def labels_case(e, pages, s):
    n_p, h, w = pages.shape
    grid = (n_p,) + window_grid(h, w, s)
    la = [torch.empty(grid, dtype=torch.int32, device="cuda") for _ in range(2)]

    def loop():
        for p in range(n_p):
            e.infer_windows_device(pages[p], s, None, la[1][p])
    variants = {"stacked": lambda: e.scan_windows_device(pages, s, None, la[0]), "per-page loop": loop}
    return variants, lambda: bool(torch.equal(la[0], la[1]))


def topk_case(e, pages, s):
    n_p, h, w = pages.shape
    grid = (n_p,) + window_grid(h, w, s)
    cls = torch.empty(grid + (K,), dtype=torch.int32, device="cuda")
    sc = torch.empty(grid + (K,), dtype=torch.int32, device="cuda")
    lo = torch.empty(grid + (e.n_classes,), dtype=torch.int32, device="cuda")
    out = {}

    def logits_topk():
        e.scan_windows_device(pages, s, lo, None)
        out["v"] = torch.topk(lo, K, dim=-1).values

    def same():
        order = torch.sort(lo, dim=-1, descending=True, stable=True).indices[..., :K]
        return bool(torch.equal(sc, out["v"]) and torch.equal(cls.long(), order))
    return {"top-5": lambda: e.scan_windows_topk_device(pages, s, K, cls, sc), "logits + torch.topk": logits_topk}, same


def emulator_case(e, pages, s):
    n_p, h, w = pages.shape
    grid = (n_p,) + window_grid(h, w, s)
    la = [torch.empty(grid, dtype=torch.int32, device="cuda") for _ in range(2)]
    flat = la[1].view(-1)
    buf = torch.empty((CHUNK, 256), dtype=torch.float32, device="cuda")

    def unfold():
        unfolded(pages, s, buf, lambda rows, w0: e.inference_quantized_device(rows, None, flat[w0:w0 + rows.shape[0]]))
    return {"emulator windows": lambda: e.emulate_windows_device(pages, s, None, la[0]), "unfold + emulator": unfold}, \
        lambda: bool(torch.equal(la[0], la[1]))


def run(kind, make, label, e, pages, strides, rounds, steps):
    rows = []
    n_p, h, w = pages.shape
    for s in strides:
        n = n_p * int(np.prod(window_grid(h, w, s)))
        variants, same = make(e, pages, s)
        med, rng = timed(variants, rounds, steps)
        a, b = list(variants)
        row = {"case": kind, "model": label, "pages": f"{n_p} x {h}x{w}", "stride": s, "windows": n, "ms": med, "ms_range": rng,
               "speedup": med[b] / med[a], "outputs_equal": same()}
        print(f"{kind:<8} {label:<22} {n_p:>2} x {h}x{w} stride {s:>2} {n:>10} windows  {a} {med[a]:9.3f} ms "
              f"({n / med[a] * 1e-6:.2f} G win/s)  {b} {med[b]:9.3f} ms ({n / med[b] * 1e-6:.2f} G win/s)  x{row['speedup']:.2f}  "
              f"outputs equal: {row['outputs_equal']}", flush=True)
        rows.append(row)
        torch.cuda.empty_cache()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("window_pages_bench.py measures on a CUDA device; none is available")
    name, clocks = card()
    print(f"card: {name}, power limit, max SM clock, SM clock: {clocks}", flush=True)
    print(f"float32 pages, medians of {args.rounds} alternated rounds of {args.steps} calls", flush=True)
    strides = (1, 4, 16)
    g = torch.Generator(device="cuda").manual_seed(1024)
    small = torch.randn((64, 1024, 1024), generator=g, device="cuda", dtype=torch.float32)
    large = torch.randn((16, 4096, 4096), generator=g, device="cuda", dtype=torch.float32)
    rows = []
    for label, model in (("FC 4bitsym-64", Model.load(os.path.join(ROOT, "tests", "golden", "models", "fc.bnm"))),
                         ("4bitsym-64, 37 classes", pack.random_fc_model(4, (256, 64, 64, 64, 37), seed=37)),
                         ("CNN-48", Model.load(os.path.join(ROOT, "tests", "golden", "models", "cnn_48.bnm")))):
        e = Engine(model)
        rows += run("labels", labels_case, label, e, small, strides, args.rounds, args.steps)
        rows += run("labels", labels_case, label, e, large, strides, args.rounds, args.steps)
        rows += run("top-5", topk_case, label, e, small, strides, args.rounds, args.steps)
        rows += run("emulator", emulator_case, label, e, small, strides, args.rounds, args.steps)
        e.close()
    print(json.dumps({"card": name, "power_limit_max_sm_clock_sm_clock": clocks, "rounds": args.rounds, "steps": args.steps, "rows": rows}))
    if not all(r["outputs_equal"] for r in rows):
        sys.exit(1)


if __name__ == "__main__":
    main()
