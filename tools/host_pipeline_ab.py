"""The host pipeline's batch entries (bnm_infer_batch, bnm_infer_topk, bnm_emulate_inference_quantized) on two builds of the
library in one process, alternated: what a change to the pipeline (its copy order, its staging) costs or gains on the existing
host entries.  Each --lib is loaded with ctypes on its own; both serve the same model on the same GPU.

Cases, FC 4bitsym-64 at the default chunk (65 536 images): bnm_infer_batch at 2^22 int8 images with logits and labels and labels
only, bnm_infer_topk at 2^22 (k = 5, scores), bnm_emulate_inference_quantized at 2^20 float images; inputs and outputs in pinned
memory (torch's pin_memory) and in pageable memory.  Each round times every build with a host clock around the call (the call
returns with the results in host memory), the rounds alternate which build goes first, the report is the median over rounds with
the range.  Every row checks that both builds' outputs are equal.  Prints the card's name, power limit and max SM clock.

    python tools/host_pipeline_ab.py --lib NAME=PATH --lib NAME=PATH [--rounds 7] [--out FILE]
"""
import argparse
import ctypes as C
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bitnetmcu_b200.model import Model  # noqa: E402
from window_bench import card  # noqa: E402

vp, sz, u32 = C.c_void_p, C.c_size_t, C.c_uint32


def load(path, blob):
    lib = C.CDLL(path)
    lib.bnm_model_load_blob.argtypes = [vp, sz, C.c_int, C.POINTER(vp)]
    lib.bnm_infer_batch.argtypes = [vp, vp, sz, vp, vp]
    lib.bnm_infer_topk.argtypes = [vp, vp, sz, u32, vp, vp]
    lib.bnm_emulate_inference_quantized.argtypes = [vp, vp, sz, vp]
    lib.bnm_last_error.restype = C.c_char_p
    h = vp()
    buf = (C.c_char * len(blob)).from_buffer_copy(blob)
    assert lib.bnm_model_load_blob(buf, len(blob), 0, C.byref(h)) == 0, lib.bnm_last_error()
    return lib, h, buf


def array(shape, dtype, pinned):
    if pinned:
        return torch.empty(shape, dtype=dtype, pin_memory=True).numpy()
    return np.empty(shape, dtype=torch.empty((), dtype=dtype).numpy().dtype)


def ptr(a):
    return None if a is None else vp(a.ctypes.data)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", required=True, help="NAME=PATH of a libbitnetmcu_b200.so build")
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("host_pipeline_ab.py measures on a CUDA device; none is available")
    torch.cuda.init()
    blob = Model.load(os.path.join(ROOT, "tests", "golden", "models", "fc.bnm")).to_blob()
    libs = {n: load(p, blob) for n, p in (l.split("=", 1) for l in args.lib)}
    name, clocks = card()
    lines = [f"card: {name}, power limit, max SM clock, SM clock: {clocks}",
             f"FC 4bitsym-64, default chunk; medians of {args.rounds} alternated rounds [min - max], ms per call"]
    print("\n".join(lines), flush=True)
    rng = np.random.default_rng(0)
    n8, nf = 1 << 22, 1 << 20
    ok = True
    for pinned in (True, False):
        mem = "pinned" if pinned else "pageable"
        x8 = array((n8, 256), torch.int8, pinned)
        x8[:] = rng.integers(-128, 128, size=(n8, 256), dtype=np.int8)
        xf = array((nf, 256), torch.float32, pinned)
        xf[:] = rng.standard_normal((nf, 256), dtype=np.float32)
        outs = {n: {"logits": array((n8, 10), torch.int32, pinned), "labels": array((n8,), torch.int32, pinned),
                    "classes": array((n8, 5), torch.int32, pinned), "scores": array((n8, 5), torch.int32, pinned),
                    "emul": array((nf, 10), torch.float64, pinned)} for n in libs}
        cases = {
            "bnm_infer_batch logits+labels 2^22": (lambda l, h, o: l.bnm_infer_batch(h, ptr(x8), n8, ptr(o["logits"]), ptr(o["labels"])),
                                                   ("logits", "labels")),
            "bnm_infer_batch labels 2^22": (lambda l, h, o: l.bnm_infer_batch(h, ptr(x8), n8, None, ptr(o["labels"])), ("labels",)),
            "bnm_infer_topk k=5 2^22": (lambda l, h, o: l.bnm_infer_topk(h, ptr(x8), n8, 5, ptr(o["classes"]), ptr(o["scores"])),
                                        ("classes", "scores")),
            "bnm_emulate_inference_quantized 2^20": (lambda l, h, o: l.bnm_emulate_inference_quantized(h, ptr(xf), nf, ptr(o["emul"])),
                                                     ("emul",)),
        }
        for case, (fn, keys) in cases.items():
            t = {n: [] for n in libs}
            order = list(libs)
            for n in order:   # warm-up
                assert fn(libs[n][0], libs[n][1], outs[n]) == 0
            for r in range(args.rounds):
                for n in (order if r % 2 == 0 else order[::-1]):
                    lib, h, _ = libs[n]
                    t0 = time.perf_counter()
                    rc = fn(lib, h, outs[n])
                    t[n].append((time.perf_counter() - t0) * 1e3)
                    assert rc == 0, lib.bnm_last_error()
            first = order[0]
            equal = all(np.array_equal(outs[first][k], outs[n][k]) for n in order[1:] for k in keys)
            ok &= equal
            text = f"{case:<38} {mem:<8}" + "".join(
                f"  {n} {np.median(v):8.2f} [{min(v):.2f} - {max(v):.2f}]" for n, v in t.items())
            if len(order) == 2:
                text += f"  {order[1]}/{order[0]} {np.median(t[order[1]]) / np.median(t[order[0]]):.3f}"
            text += f"  outputs equal: {equal}"
            print(text, flush=True)
            lines.append(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write("# tools/host_pipeline_ab.py -- the host pipeline's batch entries on two builds, alternated in one process\n")
            f.write("\n".join(lines) + "\n")
    if not ok:
        sys.exit(1)


if __name__ == "__main__":
    main()
