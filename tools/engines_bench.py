"""Both engines scored in one call (bnm_compare_engines_device) next to the two calls and torch comparisons it replaces, alternated
in one process.

At 2^20 float32 images resident on the GPU (CUDA events around back-to-back calls on one stream, inputs double-buffered), per
model:
  * one pass: compare_engines_device with both labels, truth and counts;
  * two calls: infer_device_f32 labels only, inference_quantized_device labels only, then the torch comparisons that add images,
    correct_c, correct_py and mismatches to a device counts tensor.
Models: FC 4bitsym-64 (fc: fc_engines_kernel), Binary-160 and CNN-48 (the two routes and k_engine_counts).  Each round times every
case, rounds alternate the order; medians over the rounds.  Checks that both variants give identical labels and counts.  Prints
the card name and power limit of this run.

    python tools/engines_bench.py [--rounds 5] [--steps 20]
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
from bitnetmcu_b200.engine import Engine  # noqa: E402
from labels_only_bench import card, events_ms, load  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    args = ap.parse_args()
    name, power = card()
    print(f"card: {name}, power limit {power}", flush=True)
    n, S = 1 << 20, args.steps
    g = torch.Generator(device="cuda").manual_seed(1)
    x = [torch.randn((n, 256), generator=g, device="cuda") for _ in range(2)]
    truth = torch.randint(0, 10, (n,), generator=g, device="cuda", dtype=torch.int32)
    n_t = torch.tensor(n, dtype=torch.int64, device="cuda")
    cases, engines, outs = {}, {}, {}
    for tag in ("fc", "binary160", "cnn_48"):
        e = Engine(load(tag))
        engines[tag] = e
        # [one pass: labels_c, labels_py, counts], [two calls: the same]
        o = [[torch.empty(n, dtype=torch.int32, device="cuda") for _ in range(2)] + [torch.zeros(4, dtype=torch.int64, device="cuda")]
             for _ in range(2)]
        outs[tag] = o

        def one_pass(i, e=e, o=o[0]):
            e.compare_engines_device(x[i & 1], truth=truth, labels_c=o[0], labels_py=o[1], counts=o[2])

        def two_calls(i, e=e, o=o[1]):
            e.infer_device_f32(x[i & 1], None, o[0])
            e.inference_quantized_device(x[i & 1], None, o[1])
            o[2] += torch.stack([n_t, (o[0] == truth).sum(), (o[1] == truth).sum(), (o[0] != o[1]).sum()])
        steps = S if tag == "fc" else max(2, S // 4)
        cases[f"one pass ({tag})"] = (one_pass, steps)
        cases[f"two calls + torch ({tag})"] = (two_calls, steps)
    ms = {k: [] for k in cases}
    for r in range(args.rounds):
        for k in (list(cases) if r % 2 == 0 else list(cases)[::-1]):
            fn, steps = cases[k]
            ms[k].append(events_ms(fn, steps, 2))
    same = {}
    for tag, (fn1, _), (fn2, _) in [(t, cases[f"one pass ({t})"], cases[f"two calls + torch ({t})"]) for t in engines]:
        for o in outs[tag]:
            o[2].zero_()
        fn1(0)
        fn2(0)
        torch.cuda.synchronize()
        a, b = outs[tag]
        same[tag] = bool(torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and torch.equal(a[2], b[2]))
        print(f"{tag:<10} counts {a[2].tolist()} (images, correct_c, correct_py, mismatches); identical labels and counts: {same[tag]}")
    rows = []
    for k, (_, _) in cases.items():
        med = float(np.median(ms[k]))
        row = {"case": k, "batch": n, "ms": med, "gimg_s": n / (med * 1e-3) / 1e9,
               "gimg_s_range": [n / (max(ms[k]) * 1e-3) / 1e9, n / (min(ms[k]) * 1e-3) / 1e9]}
        rows.append(row)
        print(f"{k:<28} n={n:>8}  {med:9.3f} ms  {row['gimg_s']:8.4f} G img/s  (range {row['gimg_s_range'][0]:.4f} .. "
              f"{row['gimg_s_range'][1]:.4f})", flush=True)
    for tag in engines:
        one, two = float(np.median(ms[f"one pass ({tag})"])), float(np.median(ms[f"two calls + torch ({tag})"]))
        print(f"{tag:<10} one pass / two calls speed-up x{two / one:6.2f}")
    print(json.dumps({"card": name, "power_limit": power, "rounds": args.rounds, "rows": rows, "identical": same}))
    for e in engines.values():
        e.close()
    if not all(same.values()):
        sys.exit(1)


if __name__ == "__main__":
    main()
