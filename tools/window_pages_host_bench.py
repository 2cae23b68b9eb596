"""Window scan of page stacks in host memory (include/bitnetmcu_b200.h section 14) against what a caller does without the host
entries, alternated in one process.  Per model, stack, stride, output, format and host memory kind, two variants on the same host
pages (CPU tensors: pinned with pin_memory(), or pageable):
  host          Engine.scan_windows / scan_windows_topk on the host pages: the library streams them to the GPU in bands and
                scans one band while the next is copied, returning NumPy outputs
  upload        what a caller does today: the whole stack to the GPU (pages.cuda(), or pages.to(device, non_blocking=True) from
                pinned memory), the device entry, then .cpu() of the outputs
Cases: FC 4bitsym-64 and CNN-48 on 16 pages of 4096 x 4096 and 64 pages of 1024 x 1024, float32 and bfloat16, pinned and
pageable, labels only at strides 1, 4 and 16 and top-5 with scores at strides 4 and 16 (at stride 1 a top-5 stack's classes and
scores would be 10 GiB).  Each round times both variants with a host clock around the whole call (both end with the results in
host memory), the rounds alternate which goes first, the report is the median over rounds with the range.  Every row checks
that both variants' outputs are equal.  Per stack, format and output, the peak device memory of each variant on a fresh engine:
free device memory (torch.cuda.mem_get_info) before the call minus after it, with torch's cache emptied before and kept after,
so torch's reservations and the library's pools both count.  The PCIe copy rates of the same run (1 GiB host to device and back,
pinned and pageable) are printed beside the link's data-sheet rate.  Prints the card's name, power limit and max SM clock read
in the same run.

    python tools/window_pages_host_bench.py [--rounds 3] [--out profiles/h100_window_pages_host.txt]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bitnetmcu_b200.engine import Engine, window_grid  # noqa: E402
from bitnetmcu_b200.model import Model  # noqa: E402
from window_bench import card  # noqa: E402

MIB, GIB = 1 << 20, 1 << 30
K = 5


def seconds(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def copy_rates():
    """GB/s of 1 GiB host -> device and device -> host, pinned and pageable (median of 5)"""
    d = torch.empty(GIB // 4, dtype=torch.float32, device="cuda")
    out = {}
    for kind in ("pinned", "pageable"):
        h = torch.ones(GIB // 4, dtype=torch.float32)
        h = h.pin_memory() if kind == "pinned" else h
        out[f"h2d {kind}"] = GIB / 1e9 / float(np.median([seconds(lambda: d.copy_(h, non_blocking=True)) for _ in range(5)]))
        out[f"d2h {kind}"] = GIB / 1e9 / float(np.median([seconds(lambda: h.copy_(d, non_blocking=True)) for _ in range(5)]))
    return out


def make_pages(planes, size, fmt, pinned):
    g = torch.Generator().manual_seed(planes * size)
    x = torch.randn((planes, size, size), generator=g, dtype=torch.float32).to(fmt)
    return x.pin_memory() if pinned else x


def variants(e, pages, s, topk, pinned):
    def host():
        if topk:
            return e.scan_windows_topk(pages, s, K)
        return e.scan_windows(pages, s, want_logits=False)

    def upload():
        d = pages.to("cuda", non_blocking=True) if pinned else pages.cuda()
        grid = (d.shape[0],) + window_grid(d.shape[1], d.shape[2], s)
        if topk:
            c = torch.empty(grid + (K,), dtype=torch.int32, device="cuda")
            sc = torch.empty(grid + (K,), dtype=torch.int32, device="cuda")
            e.scan_windows_topk_device(d, s, K, c, sc)
            return c.cpu(), sc.cpu()
        la = torch.empty(grid, dtype=torch.int32, device="cuda")
        e.scan_windows_device(d, s, None, la)
        return None, la.cpu()

    return {"host": host, "upload": upload}


def same(a, b):
    return all(x is None and y is None or np.array_equal(np.asarray(x).view(np.int32), y.numpy()) for x, y in zip(a, b))


def peak_gib(model, fn):
    """device memory fn takes on a fresh engine: free memory before minus after (torch's cache kept, the library's pools held)"""
    e = Engine(model)
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    free0 = torch.cuda.mem_get_info()[0]
    fn(e)
    torch.cuda.synchronize()
    used = (free0 - torch.cuda.mem_get_info()[0]) / GIB
    e.close()
    torch.cuda.empty_cache()
    return used


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_window_pages_host.txt"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("window_pages_host_bench.py measures on a CUDA device; none is available")
    name, clocks = card()
    lines = [f"card: {name}, power limit, max SM clock, SM clock: {clocks}"]
    rates = copy_rates()
    lines.append("PCIe copy rate, 1 GiB, this run: " + ", ".join(f"{k} {v:.1f} GB/s" for k, v in rates.items())
                 + " (data sheet: PCIe Gen5 x16, 64 GB/s per direction)")
    lines.append(f"medians of {args.rounds} alternated rounds [min - max]; host = Engine.scan_windows*, upload = pages to the GPU + "
                 "device entry + .cpu()")
    for l in lines:
        print(l, flush=True)
    models = (("FC 4bitsym-64", Model.load(os.path.join(ROOT, "tests", "golden", "models", "fc.bnm"))),
              ("CNN-48", Model.load(os.path.join(ROOT, "tests", "golden", "models", "cnn_48.bnm"))))
    rows = []
    for planes, size in ((16, 4096), (64, 1024)):
        for fmt in (torch.float32, torch.bfloat16):
            for pinned in (True, False):
                pages = make_pages(planes, size, fmt, pinned)
                for label, model in models:
                    e = Engine(model)
                    for topk in (False, True):
                        for s in ((4, 16) if topk else (1, 4, 16)):
                            v = variants(e, pages, s, topk, pinned)
                            outs = {k: f() for k, f in v.items()}   # warm-up, and the outputs compared
                            eq = same(outs["host"], outs["upload"])
                            del outs
                            t = {k: [] for k in v}
                            for r in range(args.rounds):
                                for k in (list(v) if r % 2 == 0 else list(v)[::-1]):
                                    t[k].append(seconds(v[k]) * 1e3)
                            med = {k: float(np.median(x)) for k, x in t.items()}
                            peak = {}
                            if not pinned:   # the same for pinned pages: the device side does not depend on the host memory kind
                                for k in v:
                                    peak[k] = peak_gib(model, lambda eng, k=k: variants(eng, pages, s, topk, pinned)[k]())
                            row = {"model": label, "stack": f"{planes} x {size}x{size}", "format": str(fmt).split(".")[1],
                                   "memory": "pinned" if pinned else "pageable", "output": "top-5" if topk else "labels",
                                   "stride": s, "ms": med, "ms_range": {k: [min(x), max(x)] for k, x in t.items()},
                                   "speedup": med["upload"] / med["host"], "peak_device_gib": peak, "outputs_equal": eq}
                            text = (f"{row['output']:<6} {label:<14} {row['stack']:<14} {row['format']:<8} {row['memory']:<8} "
                                    f"stride {s:>2}  host {med['host']:8.1f} ms [{min(t['host']):.1f} - {max(t['host']):.1f}]  "
                                    f"upload {med['upload']:8.1f} ms [{min(t['upload']):.1f} - {max(t['upload']):.1f}]  "
                                    f"x{row['speedup']:.2f}")
                            if peak:
                                text += f"  peak device GiB host {peak['host']:.2f} upload {peak['upload']:.2f}"
                            text += f"  outputs equal: {eq}"
                            print(text, flush=True)
                            lines.append(text)
                            rows.append(row)
                    e.close()
                del pages
    print(json.dumps({"card": name, "power_limit_max_sm_clock_sm_clock": clocks, "copy_gb_s": rates, "rounds": args.rounds,
                      "rows": rows}))
    with open(args.out, "w") as f:
        f.write("# tools/window_pages_host_bench.py -- window scan of host page stacks: the host entries against upload + device "
                "entry + .cpu()\n")
        f.write("\n".join(lines) + "\n")
    if not all(r["outputs_equal"] for r in rows):
        sys.exit(1)


if __name__ == "__main__":
    main()
