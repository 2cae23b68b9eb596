"""Fused float-input path vs the chain of the scaling kernel and the int8 kernel: us per step at batch 2^20."""
import os, sys, numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench import measured_peaks
from bitnetmcu_b200 import engine as E
from bitnetmcu_b200.engine import Engine
from bitnetmcu_b200.model import Model
root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
e = Engine(Model.load(os.path.join(root, "tests", "golden", "models", "fc.bnm")))
n = 1 << 20
x = [torch.randn((n, 256), dtype=torch.float32, device="cuda") for _ in range(2)]
q = torch.empty((n, 256), dtype=torch.int8, device="cuda")
lo = torch.empty((n, 10), dtype=torch.int32, device="cuda"); la = torch.empty(n, dtype=torch.int32, device="cuda")
lo2 = torch.empty_like(lo); la2 = torch.empty_like(la)
def t(fn):
    for i in range(3): fn(i)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for i in range(20): fn(i)
    b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b) / 20 * 1e3
fused = t(lambda i: e.infer_device_f32(x[i & 1], lo, la))
def chained(i):
    E.quantize_images_device(x[i & 1], q); e.infer_device(q, lo2, la2)
ch = t(chained)
e.infer_device_f32(x[0], lo, la); chained(0); torch.cuda.synchronize()
print(f"fused {fused:.1f} us = {n / fused / 1e3:.2f} G img/s ({1064 * n / fused / 1e3 / measured_peaks()[0]:.3f} of HBM peak at 1064 B/img) | chained {ch:.1f} us = {n / ch / 1e3:.2f} G img/s | equal {bool(torch.equal(lo, lo2) and torch.equal(la, la2))}")
