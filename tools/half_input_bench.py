"""float16 / bfloat16 images on the float entries (include/bitnetmcu_b200.h section 11) against what a torch caller does without
them.  Per model, batch size and entry, three variants on the same device-resident images:
  f16 / bf16   the 16-bit entry on the torch.float16 / torch.bfloat16 tensor
  .float()     images.float() followed by the float32 entry (the caller's path before section 11)
  f32          the float32 entry on images already converted (no conversion in the timed call)
and, on the FC 4bitsym-64 model, the route the one-kernel 16-bit forms replace: the 16-bit scaling kernel
(bnm_quantize_images_device_f16) followed by the int8 entry.
Rounds alternate the variants; each number is the median over rounds of the mean over `steps` calls, timed with CUDA events.
Every variant's outputs are checked equal to the f32 variant's.  The card's name and power limit are read in the same run.

  python tools/half_input_bench.py [--rounds 5] [--steps 10] [--out FILE]
"""
import argparse
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bitnetmcu_b200 import engine as E          # noqa: E402
from bitnetmcu_b200 import pack as P            # noqa: E402
from bitnetmcu_b200.engine import Engine        # noqa: E402
from bitnetmcu_b200.model import Model          # noqa: E402


def models():
    load = lambda n: Model.load(os.path.join(ROOT, "tests", "golden", "models", n + ".bnm"))
    fc37 = P.random_fc_model(4, (256, 64, 64, 37), seed=2)
    fc37.img_bytes = 256
    return [("FC 4bitsym-64", load("fc")), ("FC 64 wide, 37 classes", fc37), ("Binary-160", load("binary160")), ("CNN-48", load("cnn_48"))]


def timed(fn, steps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps * 1e3   # us per call


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--sizes", default="20,22", help="log2 of the batch sizes")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "half_input_bench needs a CUDA device"
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    lines = [f"# {torch.cuda.get_device_name(0)} | nvidia-smi: {smi} | rounds {a.rounds}, steps {a.steps}",
             "# G images/s (median of rounds); x = 16-bit entry over .float() + float32 entry",
             f"{'model':24s} {'n':>8s} {'entry':22s} {'f16':>7s} {'bf16':>7s} {'.float()':>9s} {'f32':>7s} {'x f16':>6s} {'x bf16':>6s}  equal"]
    print("\n".join(lines), flush=True)
    for mname, m in models():
        e = Engine(m, device=0)
        C = e.n_classes
        for lg in (int(s) for s in a.sizes.split(",")):
            n = 1 << lg
            torch.manual_seed(lg)
            x32 = torch.randn((n, 256), device="cuda") * torch.exp(torch.randn((n, 1), device="cuda"))
            xs = {"f16": x32.half(), "bf16": x32.bfloat16()}
            zi = lambda *s: torch.empty(s, dtype=torch.int32, device="cuda")
            entries = {
                "C labels+logits": (lambda x, o: e.infer_device_f32(x, o[0], o[1]), lambda: (zi(n, C), zi(n))),
                "C labels only": (lambda x, o: e.infer_device_f32(x, None, o[0]), lambda: (zi(n),)),
                "emulator": (lambda x, o: e.inference_quantized_device(x, o[0], o[1]),
                             lambda: (torch.empty((n, C), dtype=torch.float64, device="cuda"), zi(n))),
                "two engines": (lambda x, o: e.compare_engines_device(x, None, o[0], o[1], o[2]),
                                lambda: (zi(n), zi(n), torch.zeros(4, dtype=torch.int64, device="cuda"))),
                "top-5": (lambda x, o: e.topk_device_f32(x, 5, o[0], o[1]), lambda: (zi(n, 5), zi(n, 5))),
            }
            for ename, (call, alloc) in entries.items():
                outs = {k: alloc() for k in ("f16", "bf16", ".float()", "f32", "scale+int8")}
                xf = {k: v.float() for k, v in xs.items()}   # the f32 variant's images, converted once
                q = torch.empty((n, 256), dtype=torch.int8, device="cuda")
                variants = {
                    "f16": lambda: call(xs["f16"], outs["f16"]),
                    "bf16": lambda: call(xs["bf16"], outs["bf16"]),
                    ".float()": lambda: call(xs["f16"].float(), outs[".float()"]),
                    "f32": lambda: call(xf["f16"], outs["f32"]),
                }
                if mname == "FC 4bitsym-64" and ename.startswith("C "):
                    lab_only = ename == "C labels only"
                    variants["scale+int8"] = lambda: (E.quantize_images_device(xs["f16"], q),
                                                      e.infer_device(q, None if lab_only else outs["scale+int8"][0], outs["scale+int8"][-1]))
                for v in variants.values():   # warm-up: every shape and module
                    v()
                torch.cuda.synchronize()
                times = {k: [] for k in variants}
                for r in range(a.rounds):
                    order = list(variants) if r % 2 == 0 else list(reversed(variants))
                    for k in order:
                        times[k].append(timed(variants[k], a.steps))
                rate = {k: n / statistics.median(t) / 1e3 for k, t in times.items()}   # G images/s
                # outputs: every variant on the f16 images equals the f32 entry on them widened (counts accumulate: not compared)
                for k in variants:
                    for t in outs[k]:
                        if t.dtype != torch.int64:
                            t.zero_()
                    variants[k]()
                torch.cuda.synchronize()
                same = all(torch.equal(outs[k][i], outs["f32"][i]) for k in ("f16", ".float()") for i in range(len(outs["f32"]))
                           if outs["f32"][i].dtype != torch.int64)
                row = (f"{mname:24s} {n:8d} {ename:22s} {rate['f16']:7.2f} {rate['bf16']:7.2f} {rate['.float()']:9.2f} {rate['f32']:7.2f} "
                       f"{rate['f16'] / rate['.float()']:6.2f} {rate['bf16'] / rate['.float()']:6.2f}  {same}")
                if "scale+int8" in rate:
                    row += f"  | 16-bit scaling kernel + int8 entry {rate['scale+int8']:.2f} (one kernel x{rate['f16'] / rate['scale+int8']:.2f})"
                print(row, flush=True)
                lines.append(row)
                del outs, xf, q
            del x32, xs
            torch.cuda.empty_cache()
        e.close()
    if a.out:
        with open(a.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
