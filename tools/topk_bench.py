"""Top-k against the entries it stands between, alternated in one process: what returning each image's k best classes costs next
to labels only, logits, and logits followed by torch.topk.

Device paths, 2^20 device-resident images, double-buffered, back-to-back launches on one stream timed with CUDA events; each round
times every variant, the rounds rotate which goes first, the report is the median over rounds.  Models: FC 4bitsym-64 (10
classes), 64-wide 4bitsym models with 37 and 47 classes (random weights: speed does not depend on them), Binary-160 and CNN-48.
Variants: bnm_infer_topk_device at k = 1 and 5 with and without scores; bnm_infer_batch_device labels-only and with logits; with
logits, then torch.topk(k = 5) of them.  The top-k classes are checked against a stable descending sort of the logits, and rank 0
against the labels.  Prints the card name, its power limit and its maximum SM clock (the clock this run was allowed).

    python tools/topk_bench.py [--rounds 7] [--steps 20] [--batch 1048576]
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
from bitnetmcu_b200.engine import Engine  # noqa: E402
from bitnetmcu_b200.model import Model  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        vis = os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0] or "0"
        out = subprocess.run(["nvidia-smi", "-i", vis, "--query-gpu=power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        out = ""
    return name, out or "unknown"


def fixture(name):
    return Model.load(os.path.join(ROOT, "tests", "golden", "models", name + ".bnm"))


def wide_head(n_classes):
    return pack.random_fc_model(4, (256, 64, 64, 64, n_classes), seed=n_classes)


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


def case(label, model, n, rounds, steps):
    e = Engine(model)
    c = e.n_classes
    g = torch.Generator(device="cuda").manual_seed(n + c)
    x = [torch.randint(-128, 128, (n, e.img_bytes), generator=g, device="cuda", dtype=torch.int8) for _ in range(2)]
    lo = [torch.empty((n, c), dtype=torch.int32, device="cuda") for _ in range(2)]
    la = [torch.empty(n, dtype=torch.int32, device="cuda") for _ in range(2)]
    cls = {k: [torch.empty((n, k), dtype=torch.int32, device="cuda") for _ in range(2)] for k in (1, 5)}
    sc = {k: [torch.empty((n, k), dtype=torch.int32, device="cuda") for _ in range(2)] for k in (1, 5)}
    variants = {
        "labels_only": lambda i: e.infer_device(x[i & 1], None, la[i & 1]),
        "logits": lambda i: e.infer_device(x[i & 1], lo[i & 1], la[i & 1]),
        "logits+torch.topk5": lambda i: (e.infer_device(x[i & 1], lo[i & 1], None), torch.topk(lo[i & 1], 5, dim=1)),
    }
    for k in (1, 5):
        variants[f"topk{k}+scores"] = lambda i, k=k: e.topk_device(x[i & 1], k, cls[k][i & 1], sc[k][i & 1])
        variants[f"topk{k}"] = lambda i, k=k: e.topk_device(x[i & 1], k, cls[k][i & 1], None)
    names = list(variants)
    ms = {k: [] for k in names}
    for r in range(rounds):
        order = names[r % len(names):] + names[:r % len(names)]
        for k in order:
            ms[k].append(events_ms(variants[k], steps, 3))
    # outputs: top-5 classes = a stable descending sort of the logits, scores = the logits there, rank 0 = the label
    e.infer_device(x[0], lo[0], la[0])
    e.topk_device(x[0], 5, cls[5][0], sc[5][0])
    torch.cuda.synchronize()
    order = torch.sort(lo[0], dim=1, descending=True, stable=True).indices[:, :5].to(torch.int32)
    same = bool(torch.equal(cls[5][0], order) and torch.equal(sc[5][0], torch.gather(lo[0], 1, order.long()))
                and torch.equal(cls[5][0][:, 0], la[0]))
    e.close()
    med = {k: float(np.median(v)) for k, v in ms.items()}
    rate = {k: n / (v * 1e-3) / 1e9 for k, v in med.items()}
    spread = {k: [n / (max(v) * 1e-3) / 1e9, n / (min(v) * 1e-3) / 1e9] for k, v in ms.items()}
    print(f"{label:<22} n={n} classes={c}  " + "  ".join(f"{k} {rate[k]:.2f}" for k in names) + f"  G img/s; outputs agree: {same}",
          flush=True)
    return {"case": label, "batch": n, "classes": c, "ms": med, "gimg_s": rate, "gimg_s_range": spread, "outputs_agree": same}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--batch", type=int, default=1 << 20)
    args = ap.parse_args()
    name, clocks = card()
    print(f"card: {name}, power limit, max SM clock, SM clock: {clocks}", flush=True)
    R, S, n = args.rounds, args.steps, args.batch
    rows = [case("FC 4bitsym-64", fixture("fc"), n, R, S),
            case("4bitsym-64, 37 classes", wide_head(37), n, R, S),
            case("4bitsym-64, 47 classes", wide_head(47), n, R, S),
            case("Binary-160", fixture("binary160"), n, R, S),
            case("CNN-48", fixture("cnn_48"), n, R, max(2, S // 4))]
    print(json.dumps({"card": name, "power_limit_max_sm_clock_sm_clock": clocks, "rounds": R, "rows": rows}))
    if not all(r["outputs_agree"] for r in rows):
        sys.exit(1)


if __name__ == "__main__":
    main()
