"""Window scan of float16 / bfloat16 page stacks (include/bitnetmcu_b200.h section 12) against what a torch caller does without
the 16-bit window entries, alternated in one process.  Per model, stack, stride and format, three variants on the same
device-resident pages:
  16-bit      the 16-bit stacked entry on the torch.float16 / torch.bfloat16 stack
  .float()    pages.float() followed by the float32 stacked entry (the caller's path before section 12)
  f32         the float32 stacked entry on pages converted beforehand (no conversion in the timed call)
Cases: labels only (bnm_scan_windows_device_f16) on FC 4bitsym-64, a 64-wide 4bitsym model with 37 classes (random weights:
speed does not depend on them) and CNN-48, on 64 pages of 1024 x 1024 and 16 pages of 4096 x 4096, strides 1, 4 and 16 (CNN-48:
float16 only); top-5 with scores and the emulator's labels on FC 4bitsym-64, 64 pages of 1024 x 1024.  Each round times every
variant, the rounds rotate which goes first, the report is the median over rounds of the mean over `steps` calls, timed with CUDA
events.  Every row checks that the variants' outputs are equal.  Per stack and format, the peak of torch's device allocations
(torch.cuda.max_memory_allocated) during one 16-bit call and during one .float() call, both with only the 16-bit pages and the
outputs allocated (the library's own scratch comes from its own pool and is the same for both).  Prints the card's name, power
limit and max SM clock read in the same run.

    python tools/window_pages_f16_bench.py [--rounds 3] [--steps 2] [--out profiles/h100_window_pages_f16.txt]
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

K = 5
MIB = 1 << 20


def timed(variants, rounds, steps):
    """{name: median ms per call} of alternated rounds"""
    names = list(variants)
    ms = {k: [] for k in names}
    for r in range(rounds):
        for k in names[r % len(names):] + names[:r % len(names)]:
            ms[k].append(events_ms(variants[k], steps, 1))
    torch.cuda.synchronize()
    return {k: float(np.median(v)) for k, v in ms.items()}


def outputs(e, kind, grid):
    """the output tensors of one variant: labels; (classes, scores); or emulator labels"""
    if kind == "top-5":
        return (torch.empty(grid + (K,), dtype=torch.int32, device="cuda"), torch.empty(grid + (K,), dtype=torch.int32, device="cuda"))
    return (torch.empty(grid, dtype=torch.int32, device="cuda"),)


def call(e, kind, pages, s, out):
    if kind == "labels":
        e.scan_windows_device(pages, s, None, out[0])
    elif kind == "top-5":
        e.scan_windows_topk_device(pages, s, K, out[0], out[1])
    else:
        e.emulate_windows_device(pages, s, None, out[0])


def peak_mib(fn):
    """torch's peak device allocation during fn, in MiB"""
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() / MIB


def row(e, kind, label, p16, p32, s, rounds, steps, mem):
    n_p, h, w = p16.shape
    grid = (n_p,) + window_grid(h, w, s)
    n = int(np.prod(grid))
    outs = [outputs(e, kind, grid) for _ in range(3)]
    variants = {"16-bit": lambda: call(e, kind, p16, s, outs[0]), ".float()": lambda: call(e, kind, p16.float(), s, outs[1]),
                "f32": lambda: call(e, kind, p32, s, outs[2])}
    med = timed(variants, rounds, steps)
    same = all(torch.equal(a, b) for o in outs[1:] for a, b in zip(outs[0], o))
    fmt = str(p16.dtype).replace("torch.", "")
    r = {"case": kind, "model": label, "format": fmt, "pages": f"{n_p} x {h}x{w}", "stride": s, "windows": n, "ms": med,
         "x_vs_float": med[".float()"] / med["16-bit"], "x_vs_f32": med["f32"] / med["16-bit"], "outputs_equal": same, **mem}
    print(f"{kind:<8} {label:<22} {fmt:<8} {n_p:>2} x {h}x{w} stride {s:>2} {n:>10} windows  "
          + "  ".join(f"{k} {v:9.3f} ms ({n / v * 1e-6:.2f} G win/s)" for k, v in med.items())
          + f"  x{r['x_vs_float']:.2f} vs .float(), x{r['x_vs_f32']:.2f} vs f32  outputs equal: {same}", flush=True)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_window_pages_f16.txt"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("window_pages_f16_bench.py measures on a CUDA device; none is available")
    name, clocks = card()
    lines = [f"card: {name}, power limit, max SM clock, SM clock: {clocks}",
             f"16-bit pages, medians of {args.rounds} alternated rounds of {args.steps} calls"]
    print("\n".join(lines), flush=True)
    models = [("FC 4bitsym-64", Model.load(os.path.join(ROOT, "tests", "golden", "models", "fc.bnm"))),
              ("4bitsym-64, 37 classes", pack.random_fc_model(4, (256, 64, 64, 64, 37), seed=37)),
              ("CNN-48", Model.load(os.path.join(ROOT, "tests", "golden", "models", "cnn_48.bnm")))]
    engines = [(label, Engine(m)) for label, m in models]
    rows = []
    g = torch.Generator(device="cuda").manual_seed(1024)
    for shape in ((64, 1024, 1024), (16, 4096, 4096)):
        for fmt in (torch.float16, torch.bfloat16):
            p16 = torch.randn(shape, generator=g, device="cuda", dtype=torch.float32).to(fmt)
            torch.cuda.empty_cache()
            fc = engines[0][1]
            grid = (shape[0],) + window_grid(shape[1], shape[2], 4)
            out = outputs(fc, "labels", grid)
            call(fc, "labels", p16, 4, out)   # warm the pool and the kernels
            mem = {"peak_mib_16bit": peak_mib(lambda: call(fc, "labels", p16, 4, out)),
                   "peak_mib_float": peak_mib(lambda: call(fc, "labels", p16.float(), 4, out))}
            print(f"peak torch allocation, {fmt} {shape}: 16-bit call {mem['peak_mib_16bit']:.0f} MiB, .float() + float32 call "
                  f"{mem['peak_mib_float']:.0f} MiB", flush=True)
            del out
            p32 = p16.float()
            for label, e in engines:
                if label == "CNN-48" and fmt != torch.float16:
                    continue
                for s in (1, 4, 16):
                    rows.append(row(e, "labels", label, p16, p32, s, args.rounds, args.steps, mem))
                    torch.cuda.empty_cache()
            if shape[0] == 64:
                label, e = engines[0]
                for kind in ("top-5", "emulator"):
                    for s in (1, 4, 16):
                        rows.append(row(e, kind, label, p16, p32, s, args.rounds, args.steps, mem))
                        torch.cuda.empty_cache()
            del p16, p32
            torch.cuda.empty_cache()
    for _, e in engines:
        e.close()
    result = {"card": name, "power_limit_max_sm_clock_sm_clock": clocks, "rounds": args.rounds, "steps": args.steps, "rows": rows}
    print(json.dumps(result), flush=True)
    with open(args.out, "w") as f:
        f.write("\n".join(lines) + "\n")
        for r in rows:
            f.write(f"{r['case']:<8} {r['model']:<22} {r['format']:<8} {r['pages']} stride {r['stride']:>2} {r['windows']:>10} windows  "
                    + "  ".join(f"{k} {v:9.3f} ms" for k, v in r["ms"].items())
                    + f"  x{r['x_vs_float']:.2f} vs .float(), x{r['x_vs_f32']:.2f} vs f32  peak MiB 16-bit {r['peak_mib_16bit']:.0f}, "
                    f".float() {r['peak_mib_float']:.0f}  outputs equal: {r['outputs_equal']}\n")
        f.write(json.dumps(result) + "\n")
    if not all(r["outputs_equal"] for r in rows):
        sys.exit(1)


if __name__ == "__main__":
    main()
