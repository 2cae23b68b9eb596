"""Inference() from T threads at once: calls per second and per-call latency of the drop-in shim next to the reference's DLL.

Builds host/bitnetmcu_b200_concurrency.c (gcc -pthread) and the gcc-built shim of this library (host/bitnetmcu_b200_dll.c with
a header written from the fixture model), then runs the harness for each model (fc, cnn) and T = 1, 2, 4, 8, 16, 32, 64 against
the shim and, when they were built next to the oracle, against the reference's own DLLs (oracle/_ref/Bitnet_inf_<model>.so),
which run each thread's calls on its own host core.  Every row is one harness run: `--calls` calls in all, split over the T
threads, one 16x16 image per call over the ten reference digits.  A row reports calls per second over the run, the median and
99th percentile microseconds per call, whether the first ten labels are the reference KAT and how many calls returned a label
other than the one-thread label of their image.  Prints the card name and its power limit first.

    python tools/concurrency_bench.py [--calls 40000] [--threads 1,2,4,8,16,32,64] [--models fc,cnn]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bitnetmcu_b200 import _lib  # noqa: E402
from bitnetmcu_b200.model import Model  # noqa: E402
from bitnetmcu_b200.pack import write_header  # noqa: E402


def card():
    try:
        vis = os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0] or "0"
        return subprocess.run(["nvidia-smi", "-i", vis, "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip() or "unknown"
    except Exception:
        return "unknown"


def build(tmp, models):
    """the harness and one shim per model in tmp -> (harness, {model: shim}, digits.bin, the KAT labels)"""
    exe = os.path.join(tmp, "concurrency")
    subprocess.run(["gcc", "-O2", "-pthread", "-o", exe, os.path.join(ROOT, "host", "bitnetmcu_b200_concurrency.c"), "-ldl"], check=True)
    libdir = os.path.dirname(_lib.LIB_PATH)
    shims = {}
    for name in models:
        d = os.path.join(tmp, name)
        os.makedirs(d)
        write_header(Model.load(os.path.join(ROOT, "tests", "golden", "models", name + ".bnm")), os.path.join(d, "BitNetMCU_model.h"))
        shims[name] = os.path.join(d, "Bitnet_inf.dll")
        subprocess.run(["gcc", "-O2", "-fPIC", "-shared", "-D_DLL", "-o", shims[name], os.path.join(ROOT, "host", "bitnetmcu_b200_dll.c"),
                        "-I" + d, "-I" + os.path.join(ROOT, "include"), "-L" + libdir, "-lbitnetmcu_b200", "-Wl,-rpath," + libdir], check=True)
    digits = np.load(os.path.join(ROOT, "tests", "golden", "digits.npz"))
    path = os.path.join(tmp, "digits.bin")
    digits["images"].astype(np.int8).tofile(path)
    return exe, shims, path, ",".join(str(int(v)) for v in digits["labels"])


def run(exe, dll, digits, threads, calls):
    r = subprocess.run([exe, dll, digits, str(threads), str(max(1, calls // threads))], capture_output=True, text=True, timeout=900)
    if r.returncode != 0:
        raise RuntimeError(f"{dll} with {threads} threads: exit {r.returncode}: {r.stderr[-500:]}")
    return json.loads(r.stdout.strip().splitlines()[-1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=40000, help="calls per row, split over its threads")
    ap.add_argument("--threads", default="1,2,4,8,16,32,64")
    ap.add_argument("--models", default="fc,cnn")
    args = ap.parse_args()
    models = args.models.split(",")
    print("card, power limit:", card())
    print(f"host cores: {os.cpu_count()}; {args.calls} calls per row, one image per call")
    print(f"{'model':5} {'library':9} {'T':>3} {'calls/s':>10} {'p50 us':>9} {'p99 us':>9}  KAT  mismatches")
    with tempfile.TemporaryDirectory(prefix="bnm_conc_") as tmp:
        exe, shims, digits, kat = build(tmp, models)
        for name in models:
            ref = os.path.join(ROOT, "oracle", "_ref", f"Bitnet_inf_{name}.so")
            libs = [("this", shims[name])] + ([("reference", ref)] if os.path.exists(ref) else [])
            for t in (int(x) for x in args.threads.split(",")):
                for what, dll in libs:
                    r = run(exe, dll, digits, t, args.calls)
                    print(f"{name:5} {what:9} {t:>3} {r['calls_per_s']:>10.0f} {r['p50_us']:>9.2f} {r['p99_us']:>9.2f}  "
                          f"{'ok ' if r['labels'] == kat else 'BAD'}  {r['mismatches']}", flush=True)


if __name__ == "__main__":
    main()
