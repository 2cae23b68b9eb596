"""The Python emulator on the GPU (QuantizedModel.inference_quantized) next to the C-rule float path, alternated in one process.

Device cases at 2^20 float32 images resident on the GPU (CUDA events around back-to-back calls on one stream, inputs
double-buffered): on FC 4bitsym-64 the C-rule float path (bnm_infer_batch_device_f32), the fused emulator (bnm_emulate_batch_device:
fc_emul_kernel) with float64 logits + labels and labels only, and the layer-by-layer emulator (BNM_PATH_LAYERS).  Then, for each
model the float-input row does not take -- CNN-48, CNN-64 (cnn), Binary-160, 2bitsym-96 and a random 64-wide FC model with 37
classes -- its default route (the int8 emulator row behind k_cnn_emul_frontend or k_quantize_images) next to its layer-by-layer
emulator, float64 logits + labels.  Host case: bnm_emulate_inference_quantized from a pageable NumPy array (a synchronous call:
host clock around it).  Each round times every case, rounds alternate the order.  Checks that the default route and the
layer-by-layer emulator of every model give identical logits and labels at the timed size.  Prints the card name and power limit
of this run.

    python tools/emulator_bench.py [--rounds 5] [--steps 20]
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
from bitnetmcu_b200 import _lib, model as M, pack as P  # noqa: E402
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
    fc, fc_layers = Engine(load("fc")), Engine(load("fc"), path=_lib.PATH_LAYERS)
    g = torch.Generator(device="cuda").manual_seed(1)
    x = [torch.randn((n, 256), generator=g, device="cuda") for _ in range(2)]
    lo32 = torch.empty((n, 10), dtype=torch.int32, device="cuda")
    lo = [torch.empty((n, 10), dtype=torch.float64, device="cuda") for _ in range(2)]
    la = [torch.empty(n, dtype=torch.int32, device="cuda") for _ in range(2)]
    h_x = x[0].cpu().numpy()

    def host(i):   # 1 GB of images in, 80 MB of logits out per call
        fc.inference_quantized(h_x)
    cases = {   # label -> (call, images per call, steps)
        "C-rule float path (fc)": (lambda i: fc.infer_device_f32(x[i & 1], lo32, la[0]), n, S),
        "fused emulator (fc)": (lambda i: fc.inference_quantized_device(x[i & 1], lo[0], la[0]), n, S),
        "fused emulator labels only (fc)": (lambda i: fc.inference_quantized_device(x[i & 1], None, la[0]), n, S),
        "layered emulator (fc)": (lambda i: fc_layers.inference_quantized_device(x[i & 1], lo[1], la[1]), n, max(2, S // 4)),
        "host entry (fc)": (None, n, 2),
    }
    # the routes behind the int8 emulator row: (fused engine, layered engine, logits / labels of each)
    models = {"cnn_48": load("cnn_48"), "cnn": load("cnn"), "binary160": load("binary160"), "2bitsym96": load("2bitsym96"),
              "fc64_37cls": P.random_fc_model(M.ENC_4BITSYM, (256, 64, 64, 64, 37), seed=37)}
    pairs = {}
    for tag, m in models.items():
        ef, el = Engine(m), Engine(m, path=_lib.PATH_LAYERS)
        out = [(torch.empty((n, m.n_classes), dtype=torch.float64, device="cuda"), torch.empty(n, dtype=torch.int32, device="cuda"))
               for _ in range(2)]
        pairs[tag] = (ef, el, out)
        cases[f"fused emulator ({tag})"] = (lambda i, e=ef, o=out[0]: e.inference_quantized_device(x[i & 1], o[0], o[1]), n, S)
        cases[f"layered emulator ({tag})"] = (lambda i, e=el, o=out[1]: e.inference_quantized_device(x[i & 1], o[0], o[1]), n,
                                              max(2, S // 8))

    def timed_host(steps):
        host(0)
        t = time.perf_counter()
        for i in range(steps):
            host(i)
        return (time.perf_counter() - t) / steps * 1e3
    ms = {k: [] for k in cases}
    for r in range(args.rounds):
        for k in (list(cases) if r % 2 == 0 else list(cases)[::-1]):
            fn, _, steps = cases[k]
            ms[k].append(timed_host(steps) if fn is None else events_ms(fn, steps, 2))
    same = {}
    fc.inference_quantized_device(x[0], lo[0], la[0])
    fc_layers.inference_quantized_device(x[0], lo[1], la[1])
    torch.cuda.synchronize()
    same["fc"] = bool(torch.equal(lo[0], lo[1]) and torch.equal(la[0], la[1]))
    for tag, (ef, el, out) in pairs.items():
        ef.inference_quantized_device(x[0], *out[0])
        el.inference_quantized_device(x[0], *out[1])
        torch.cuda.synchronize()
        same[tag] = bool(torch.equal(out[0][0], out[1][0]) and torch.equal(out[0][1], out[1][1]))
    rows = []
    for k, (_, m, _) in cases.items():
        med = float(np.median(ms[k]))
        row = {"case": k, "batch": m, "ms": med, "gimg_s": m / (med * 1e-3) / 1e9,
               "gimg_s_range": [m / (max(ms[k]) * 1e-3) / 1e9, m / (min(ms[k]) * 1e-3) / 1e9]}
        rows.append(row)
        print(f"{k:<34} n={m:>8}  {med:9.3f} ms  {row['gimg_s']:8.4f} G img/s  (range {row['gimg_s_range'][0]:.4f} .. "
              f"{row['gimg_s_range'][1]:.4f})", flush=True)
    for tag in same:
        f, l = float(np.median(ms[f"fused emulator ({tag})"])), float(np.median(ms[f"layered emulator ({tag})"]))
        print(f"{tag:<12} fused / layered speed-up x{l / f:8.2f}; logits / labels identical at n={n}: {same[tag]}")
    print(json.dumps({"card": name, "power_limit": power, "rounds": args.rounds, "rows": rows, "fused_equals_layered": same}))
    for e in [fc, fc_layers] + [e for p in pairs.values() for e in p[:2]]:
        e.close()
    if not all(same.values()):
        sys.exit(1)


if __name__ == "__main__":
    main()
