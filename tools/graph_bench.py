"""Per-call time of eager device calls next to the replay of a CUDA graph that holds the same call, alternated in one process.

A measurement is K back-to-back calls (or K replays) on one stream ended by one synchronise, host clock around it, divided by
K; rounds alternate which variant goes first, and the table gives each variant's median over the rounds.  Inputs are resident
on the device.  Configurations: FC 4bitsym-64 labels-only at n = 1, 1 024, 16 384 and 2^20; FC 4bitsym-64 float top-5; CNN-48;
and the chain quantize_images_device -> infer_device -> topk_device.  After the timing the outputs of one eager call and one
replay on the same inputs are compared.  Prints the card name, power limit, max SM clock and driver version of this run.

    python tools/graph_bench.py [--rounds 7]
"""
import argparse
import ctypes
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bitnetmcu_b200.engine import Engine, quantize_images_device  # noqa: E402
from bitnetmcu_b200.model import Model  # noqa: E402


def card():
    vis = os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0] or "0"
    try:
        out = subprocess.run(["nvidia-smi", "-i", vis, "--query-gpu=power.limit,clocks.max.sm,driver_version", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        out = ""
    v = ctypes.c_int(0)
    ctypes.CDLL("libcuda.so.1").cuDriverGetVersion(ctypes.byref(v))
    return torch.cuda.get_device_name(0), out or "unknown", v.value


def load(name):
    return Model.load(os.path.join(ROOT, "tests", "golden", "models", name + ".bnm"))


def per_call_us(fn, k):
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(k):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) / k * 1e6


def case(label, n, call, outs, rounds):
    """call() issues the configuration on torch's current stream; outs: its output tensors"""
    k = 2000 if n <= 16384 else 200
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        for _ in range(3):
            call()
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            call()
        g.replay()
        variants = {"eager": call, "graph": g.replay}
        t = {v: [] for v in variants}
        for r in range(rounds):
            for v in (list(variants) if r % 2 == 0 else list(variants)[::-1]):
                per_call_us(variants[v], 20)
                t[v].append(per_call_us(variants[v], k))
        for o in outs:
            o.fill_(-7)
        call()
        torch.cuda.synchronize()
        eager = [o.clone() for o in outs]
        for o in outs:
            o.fill_(-7)
        g.replay()
        torch.cuda.synchronize()
    same = all(torch.equal(a, b) for a, b in zip(eager, outs))
    e_us, g_us = statistics.median(t["eager"]), statistics.median(t["graph"])
    print(f"{label:<44} {n:>8} {k:>6} {e_us:>10.2f} {g_us:>10.2f} {e_us / g_us:>8.2f}x  {'identical' if same else 'DIFFERENT'}", flush=True)
    del g
    return same


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    a = ap.parse_args()
    name, limits, drv = card()
    print(f"card: {name}; power.limit, clocks.max.sm, driver: {limits}; cuDriverGetVersion {drv}")
    print(f"{'configuration':<44} {'n':>8} {'calls':>6} {'eager us':>10} {'graph us':>10} {'speed-up':>9}  outputs")
    gen = torch.Generator(device="cuda").manual_seed(0)
    i8 = lambda n, w: torch.randint(-128, 128, (n, w), generator=gen, device="cuda", dtype=torch.int8)
    f32 = lambda n, w: torch.randn((n, w), generator=gen, device="cuda")
    i32 = lambda *s: torch.empty(s, dtype=torch.int32, device="cuda")
    ok = True
    fc, cnn = Engine(load("fc")), Engine(load("cnn_48"))
    for n in (1, 1024, 16384, 1 << 20):
        x, la = i8(n, 256), i32(n)
        ok &= case("FC 4bitsym-64 labels only (infer_device)", n, lambda: fc.infer_device(x, None, la), [la], a.rounds)
    for n in (1024, 1 << 20):
        x, cls, sc = f32(n, 256), i32(n, 5), i32(n, 5)
        ok &= case("FC 4bitsym-64 float top-5 (topk_device_f32)", n, lambda: fc.topk_device_f32(x, 5, cls, sc), [cls, sc], a.rounds)
    for n in (1024, 1 << 20):
        x, lo, la = i8(n, 256), i32(n, cnn.n_classes), i32(n)
        ok &= case("CNN-48 logits + labels (infer_device)", n, lambda: cnn.infer_device(x, lo, la), [lo, la], a.rounds)
    for n in (1024, 16384):
        x, q, la, cls = f32(n, 256), torch.empty((n, 256), dtype=torch.int8, device="cuda"), i32(n), i32(n, 5)

        def chain():
            quantize_images_device(x, q)
            fc.infer_device(q, None, la)
            fc.topk_device(q, 5, cls)
        ok &= case("FC chain: quantize -> infer labels -> top-5", n, chain, [q, la, cls], a.rounds)
    fc.close()
    cnn.close()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
