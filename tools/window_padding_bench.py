"""Window scan of padded pages (include/bitnetmcu_b200.h section 13) against what a torch caller does without the padded entries,
alternated in one process.  Per model, stack, stride, format and mode, two variants on the same device-resident pages:
  padded      the padded stacked entry on the pages (padding=(7, 8, 7, 8): one window per pixel at stride 1)
  F.pad       F.pad(pages, (7, 8, 7, 8), mode) in the pages' own dtype, its right side widened so that rows are 16 bytes apart
              (the entries' pitch rule) and viewed at the padded width, then the unpadded stacked entry on that view (the
              cheapest caller-side path: for float32, and for 16-bit pages with a fill value the format holds exactly, as 0.0
              here, it is the section 13 definition F.pad(pages.float(), ...))
Cases: labels only on FC 4bitsym-64, on 16 pages of 4096 x 4096 and 64 pages of 1024 x 1024, strides 1, 4 and 16, float32 and
bfloat16, replicate and constant (0.0); CNN-48, labels only, on 64 pages of 1024 x 1024, float32, replicate, strides 4 and 16.  Each
round times both variants, the rounds alternate which goes first, the report is the median over rounds of the mean over `steps`
calls, timed with CUDA events.  Every row checks that both variants' outputs are equal.  Per stack, format and mode, the peak of
torch's device allocations (torch.cuda.max_memory_allocated) during one call of each variant, with the pages and the outputs
already allocated (the library's own scratch comes from its own pool and is the same for both).  Prints the card's name, power
limit and max SM clock read in the same run.

    python tools/window_padding_bench.py [--rounds 3] [--steps 2] [--out profiles/h100_window_padding.txt]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bitnetmcu_b200.engine import Engine, window_grid  # noqa: E402
from bitnetmcu_b200.model import Model  # noqa: E402
from window_bench import card, events_ms  # noqa: E402

PAD = (7, 8, 7, 8)
MIB = 1 << 20


def timed(variants, rounds, steps):
    """{name: median ms per call}, {name: [min, max]} of alternated rounds"""
    names = list(variants)
    ms = {k: [] for k in names}
    for r in range(rounds):
        for k in names[r % len(names):] + names[:r % len(names)]:
            ms[k].append(events_ms(variants[k], steps, 1))
    torch.cuda.synchronize()
    return {k: float(np.median(v)) for k, v in ms.items()}, {k: [min(v), max(v)] for k, v in ms.items()}


def peak_mib(fn):
    """torch's peak device allocation during fn, in MiB"""
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() / MIB


def row(e, label, pages, s, mode, rounds, steps):
    n_p, h, w = pages.shape
    grid = (n_p,) + window_grid(h, w, s, PAD)
    n = int(np.prod(grid))
    outs = [torch.empty(grid, dtype=torch.int32, device="cuda") for _ in range(2)]

    def padded():
        e.scan_windows_device(pages, s, None, outs[0], padding=PAD, pad_mode=mode)

    left, right, top, bottom = PAD
    extra = -(w + left + right) % (16 // pages.element_size())   # columns past the view, never read

    def fpad():
        copy = F.pad(pages, (left, right + extra, top, bottom), mode=mode)
        e.scan_windows_device(copy[..., :w + left + right], s, None, outs[1])
    variants = {"padded": padded, "F.pad": fpad}
    padded(), fpad()   # warm the pool and the kernels
    mem = {k: peak_mib(v) for k, v in variants.items()}
    med, rng = timed(variants, rounds, steps)
    same = bool(torch.equal(outs[0], outs[1]))
    fmt = str(pages.dtype).replace("torch.", "")
    r = {"model": label, "format": fmt, "mode": mode, "pages": f"{n_p} x {h}x{w}", "stride": s, "windows": n, "ms": med,
         "ms_range": rng, "speedup": med["F.pad"] / med["padded"], "peak_mib": mem, "outputs_equal": same}
    print(format_row(r), flush=True)
    del outs
    torch.cuda.empty_cache()
    return r


def format_row(r):
    return (f"{r['model']:<14} {r['format']:<8} {r['mode']:<9} {r['pages']:>14} stride {r['stride']:>2} {r['windows']:>10} windows  "
            + "  ".join(f"{k} {v:8.3f} ms [{r['ms_range'][k][0]:.3f}, {r['ms_range'][k][1]:.3f}]" for k, v in r["ms"].items())
            + f"  x{r['speedup']:.2f}  peak MiB padded {r['peak_mib']['padded']:.0f}, F.pad {r['peak_mib']['F.pad']:.0f}"
            + f"  outputs equal: {r['outputs_equal']}")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_window_padding.txt"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("window_padding_bench.py measures on a CUDA device; none is available")
    name, clocks = card()
    lines = [f"card: {name}, power limit, max SM clock, SM clock: {clocks}",
             f"padding {PAD} (left, right, top, bottom), labels only; medians [min, max] of {args.rounds} alternated rounds of "
             f"{args.steps} calls"]
    print("\n".join(lines), flush=True)
    fc = Engine(Model.load(os.path.join(ROOT, "tests", "golden", "models", "fc.bnm")))
    cnn = Engine(Model.load(os.path.join(ROOT, "tests", "golden", "models", "cnn_48.bnm")))
    rows = []
    g = torch.Generator(device="cuda").manual_seed(1024)
    for shape in ((16, 4096, 4096), (64, 1024, 1024)):
        for fmt in (torch.float32, torch.bfloat16):
            pages = torch.randn(shape, generator=g, device="cuda", dtype=torch.float32).to(fmt)
            for mode in ("replicate", "constant"):
                for s in (1, 4, 16):
                    rows.append(row(fc, "FC 4bitsym-64", pages, s, mode, args.rounds, args.steps))
            if shape[0] == 64 and fmt == torch.float32:
                for s in (4, 16):
                    rows.append(row(cnn, "CNN-48", pages, s, "replicate", args.rounds, args.steps))
            del pages
            torch.cuda.empty_cache()
    fc.close()
    cnn.close()
    result = {"card": name, "power_limit_max_sm_clock_sm_clock": clocks, "padding": PAD, "rounds": args.rounds, "steps": args.steps,
              "rows": rows}
    print(json.dumps(result), flush=True)
    with open(args.out, "w") as f:
        f.write("\n".join(lines) + "\n")
        for r in rows:
            f.write(format_row(r) + "\n")
        f.write(json.dumps(result) + "\n")
    if not all(r["outputs_equal"] for r in rows):
        sys.exit(1)


if __name__ == "__main__":
    main()
