"""With-logits vs labels-only inference, alternated in one process: what a NULL logits buffer saves on each path.

Device paths (CUDA events around back-to-back launches on one stream, inputs resident and double-buffered): FC 4bitsym-64 at
2^20 and 2^22, Ternary-64, Binary-160, CNN-48 and the fused float-input path.  Host path: bnm_infer_batch at 2^22 from pinned
host buffers (a synchronous call: host clock around it).  Each round times both variants, rounds alternate which goes first;
the labels of the two variants are compared.  Prints the card name and power limit of this run.

    python tools/labels_only_bench.py [--rounds 5] [--steps 20]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bitnetmcu_b200.engine import Engine  # noqa: E402
from bitnetmcu_b200.model import Model  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        vis = os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0] or "0"
        out = subprocess.run(["nvidia-smi", "-i", vis, "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
    except Exception:
        out = ""
    return name, out or "unknown"


def load(name):
    return Model.load(os.path.join(ROOT, "tests", "golden", "models", name + ".bnm"))


def events_ms(fn, steps, warmup):
    for i in range(warmup):
        fn(i)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for i in range(steps):
        fn(i)
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / steps


def device_case(label, model, n, rounds, steps, float_input=False):
    e = Engine(model)
    g = torch.Generator(device="cuda").manual_seed(n)
    if float_input:
        x = [torch.randn((n, e.img_bytes), generator=g, device="cuda") for _ in range(2)]
        run = e.infer_device_f32
    else:
        x = [torch.randint(-128, 128, (n, e.img_bytes), generator=g, device="cuda", dtype=torch.int8) for _ in range(2)]
        run = e.infer_device
    lo = [torch.empty((n, e.n_classes), dtype=torch.int32, device="cuda") for _ in range(2)]
    la = [torch.empty(n, dtype=torch.int32, device="cuda") for _ in range(2)]
    variants = {"logits": lambda i: run(x[i & 1], lo[i & 1], la[i & 1]), "labels_only": lambda i: run(x[i & 1], None, la[i & 1])}
    ms = {k: [] for k in variants}
    for r in range(rounds):
        for k in (list(variants) if r % 2 == 0 else list(variants)[::-1]):
            ms[k].append(events_ms(variants[k], steps, 3))
    run(x[0], lo[0], la[0])
    run(x[0], None, la[1])
    torch.cuda.synchronize()
    same = bool(torch.equal(la[0], la[1]))
    e.close()
    return report(label, n, ms, same)


def host_case(label, model, n, rounds, steps):
    e = Engine(model)
    g = torch.Generator(device="cuda").manual_seed(7)
    imgs = torch.empty((n, e.img_bytes), dtype=torch.int8, pin_memory=True)
    imgs.copy_(torch.randint(-128, 128, (n, e.img_bytes), generator=g, device="cuda", dtype=torch.int8))
    h_in = imgs.numpy()
    h_lo = torch.empty((n, e.n_classes), dtype=torch.int32, pin_memory=True).numpy()
    h_la = [torch.empty(n, dtype=torch.int32, pin_memory=True).numpy().view(np.uint32) for _ in range(2)]
    variants = {"logits": lambda: e.infer(h_in, out_logits=h_lo, out_labels=h_la[0]),
                "labels_only": lambda: e.infer(h_in, want_logits=False, out_labels=h_la[1])}

    def timed(fn):   # bnm_infer_batch returns once its results are in host memory
        fn()
        t = time.perf_counter()
        for _ in range(steps):
            fn()
        return (time.perf_counter() - t) / steps * 1e3
    ms = {k: [] for k in variants}
    for r in range(rounds):
        for k in (list(variants) if r % 2 == 0 else list(variants)[::-1]):
            ms[k].append(timed(variants[k]))
    same = bool(np.array_equal(h_la[0], h_la[1]))
    e.close()
    return report(label, n, ms, same)


def report(label, n, ms, same):
    med = {k: float(np.median(v)) for k, v in ms.items()}
    rate = {k: n / (v * 1e-3) / 1e9 for k, v in med.items()}
    row = {"case": label, "batch": n, "ms_logits": med["logits"], "ms_labels_only": med["labels_only"],
           "gimg_s_logits": rate["logits"], "gimg_s_labels_only": rate["labels_only"],
           "gimg_s_logits_range": [n / (max(ms["logits"]) * 1e-3) / 1e9, n / (min(ms["logits"]) * 1e-3) / 1e9],
           "gimg_s_labels_only_range": [n / (max(ms["labels_only"]) * 1e-3) / 1e9, n / (min(ms["labels_only"]) * 1e-3) / 1e9],
           "speedup": med["logits"] / med["labels_only"], "labels_identical": same}
    print(f"{label:<22} n={n:>8}  with logits {rate['logits']:7.3f} G img/s  labels only {rate['labels_only']:7.3f} G img/s  "
          f"x{row['speedup']:.3f}  labels identical: {same}", flush=True)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    args = ap.parse_args()
    name, power = card()
    print(f"card: {name}, power limit {power}", flush=True)
    R, S = args.rounds, args.steps
    rows = [
        device_case("FC 4bitsym-64", load("fc"), 1 << 20, R, S),
        device_case("FC 4bitsym-64", load("fc"), 1 << 22, R, S),
        device_case("Ternary-64", load("ternary64"), 1 << 20, R, S),
        device_case("Binary-160", load("binary160"), 1 << 20, R, S),
        device_case("CNN-48", load("cnn_48"), 1 << 20, R, max(2, S // 4)),
        device_case("FC float input", load("fc"), 1 << 20, R, S, float_input=True),
        host_case("FC host bnm_infer_batch", load("fc"), 1 << 22, R, max(2, S // 4)),
    ]
    print(json.dumps({"card": name, "power_limit": power, "rounds": R, "rows": rows}))
    if not all(r["labels_identical"] for r in rows):
        sys.exit(1)


if __name__ == "__main__":
    main()
