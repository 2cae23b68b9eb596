"""Window scan against what a caller does without it, alternated in one process: every 16x16 window of a 4096 x 4096 float page
classified, labels only.

Variants, each per page on one stream, timed with CUDA events over back-to-back pages:
  * windows: bnm_infer_windows_device_f32 (Engine.infer_windows_device): the scaling kernel k_quantize_windows, which loads
             each run of windows' 16-row band into shared memory once with ordinary loads, then the int8 route;
  * unfold:  page.unfold(0, 16, sy).unfold(1, 16, sx) copied into a float buffer of up to 2^20 windows (whole window rows), then
             bnm_infer_batch_device_f32 on it, chunk after chunk -- 1 KB of float rows written and read again per window.
Strides 1, 2, 4 and 16 (non-overlapping).  Models: FC 4bitsym-64, a 64-wide 4bitsym model with 37 classes (random weights: speed
does not depend on them) and CNN-48.  Each round times every variant, the rounds rotate which goes first, the report is the
median over rounds.  The two variants' labels are checked equal.  Prints the card name, its power limit and SM clocks.

    python tools/window_bench.py [--rounds 5] [--steps 3] [--size 4096]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bitnetmcu_b200 import pack  # noqa: E402
from bitnetmcu_b200.engine import Engine, window_grid  # noqa: E402
from bitnetmcu_b200.model import Model  # noqa: E402

CHUNK = 1 << 20


def card():
    name = torch.cuda.get_device_name(0)
    try:
        vis = os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0] or "0"
        out = subprocess.run(["nvidia-smi", "-i", vis, "--query-gpu=power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        out = ""
    return name, out or "unknown"


def events_ms(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / steps


def case(label, model, size, strides, rounds, steps):
    e = Engine(model)
    g = torch.Generator(device="cuda").manual_seed(size)
    page = torch.randn((size, size), generator=g, device="cuda", dtype=torch.float32)
    buf = torch.empty((CHUNK, 256), dtype=torch.float32, device="cuda")
    rows = []
    for s in strides:
        oh, ow = window_grid(size, size, s)
        n = oh * ow
        la = [torch.empty((oh, ow), dtype=torch.int32, device="cuda") for _ in range(2)]
        win = page.unfold(0, 16, s).unfold(1, 16, s)   # a view [oh, ow, 16, 16]
        per = max(1, CHUNK // ow)                      # whole window rows per chunk

        def unfold():
            flat = la[1].view(-1)
            for r0 in range(0, oh, per):
                r1 = min(oh, r0 + per)
                k = (r1 - r0) * ow
                buf[:k].view(r1 - r0, ow, 16, 16).copy_(win[r0:r1])
                e.infer_device_f32(buf[:k], None, flat[r0 * ow:r0 * ow + k])

        variants = {"windows": lambda: e.infer_windows_device(page, s, None, la[0]), "unfold": unfold}
        names = list(variants)
        ms = {k: [] for k in names}
        for r in range(rounds):
            for k in names[r % len(names):] + names[:r % len(names)]:
                ms[k].append(events_ms(variants[k], steps, 1))
        torch.cuda.synchronize()
        same = bool(torch.equal(la[0], la[1]))
        med = {k: float(np.median(v)) for k, v in ms.items()}
        rate = {k: n / (v * 1e-3) / 1e9 for k, v in med.items()}
        row = {"case": label, "stride": s, "windows": n, "ms": med, "gwin_s": rate,
               "ms_range": {k: [min(v), max(v)] for k, v in ms.items()}, "speedup": med["unfold"] / med["windows"], "labels_equal": same}
        print(f"{label:<22} stride {s:>2}  {n:>9} windows  windows {med['windows']:8.2f} ms ({rate['windows']:.2f} G win/s)  "
              f"unfold {med['unfold']:8.2f} ms ({rate['unfold']:.2f} G win/s)  x{row['speedup']:.2f}  labels equal: {same}", flush=True)
        rows.append(row)
    e.close()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--size", type=int, default=4096)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("window_bench.py measures on a CUDA device; none is available")
    name, clocks = card()
    print(f"card: {name}, power limit, max SM clock, SM clock: {clocks}", flush=True)
    print(f"page {args.size} x {args.size} float32, labels only, medians of {args.rounds} rounds of {args.steps} pages", flush=True)
    strides = (1, 2, 4, 16)
    rows = []
    for label, model in (("FC 4bitsym-64", Model.load(os.path.join(ROOT, "tests", "golden", "models", "fc.bnm"))),
                         ("4bitsym-64, 37 classes", pack.random_fc_model(4, (256, 64, 64, 64, 37), seed=37)),
                         ("CNN-48", Model.load(os.path.join(ROOT, "tests", "golden", "models", "cnn_48.bnm")))):
        rows += case(label, model, args.size, strides, args.rounds, args.steps)
    print(json.dumps({"card": name, "power_limit_max_sm_clock_sm_clock": clocks, "rounds": args.rounds, "rows": rows}))
    if not all(r["labels_equal"] for r in rows):
        sys.exit(1)


if __name__ == "__main__":
    main()
