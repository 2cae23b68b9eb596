#!/usr/bin/env python
"""BASELINE.json config 5: encoding sweep x batch sweep at 1 / 2 / 4 / 8 GPUs (device-timed, CUDA events, inputs resident in HBM).

    python tools/sweep.py                                         # one GPU
    python -m torch.distributed.run --nproc-per-node N ... tools/sweep.py   # N ranks, weak scaling: every rank runs `batch` images

Every point: 3 warm-up + 10 timed plain launches between two events, barrier + synchronise on both sides, max over ranks;
parity of a 4096-image sample of every rank's result against the oracle (checker only).  Rank 0 prints a markdown table and
writes sweep_out/sweep_<N>gpu.json.
"""
import json, os, sys, statistics
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
import torch.distributed as dist
from bitnetmcu_b200 import dist as bdist
from bitnetmcu_b200.engine import Engine
from bitnetmcu_b200.model import Model
from oracle.oracle import Oracle

rank, local_rank, world = bdist.env_rank_world()
if world > 1:
    os.environ.setdefault("NCCL_DEBUG_FILE", "/dev/stderr")
    bdist.init_process_group("nccl")
torch.cuda.set_device(local_rank)
dev = torch.device("cuda", local_rank)
orc = Oracle()
from bench import measured_peaks  # noqa: E402
PEAK = measured_peaks()[0]   # GB/s: MEASURED_PEAKS.json when present, else the H100 data-sheet figure


def barrier():
    if world > 1:
        dist.barrier()
    torch.cuda.synchronize()


def run(name, n, steps=10, nf4=False):
    m = Model.load(os.path.join(ROOT, "tests", "golden", "models", name + ".bnm"))
    e = Engine(m, device=local_rank, nf4_extension=nf4)
    rng = np.random.default_rng(1 + rank)
    h = rng.integers(-128, 128, size=(min(n, 1 << 20), 256), dtype=np.int8)
    x = torch.from_numpy(h).to(dev)
    if n > x.shape[0]:
        x = x.repeat(n // x.shape[0], 1)
    lo = torch.empty((n, e.n_classes), dtype=torch.int32, device=dev)
    la = torch.empty(n, dtype=torch.int32, device=dev)
    for _ in range(3):
        e.infer_device(x, lo, la)
    barrier()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        e.infer_device(x, lo, la)
    b.record()
    barrier()
    ms = a.elapsed_time(b) / steps
    ns = min(n, 4096)
    want, wl = orc.infer(m, h[:ns], nf4_extension=nf4)
    ok = bool(np.array_equal(lo[:ns].cpu().numpy(), want) and np.array_equal(la[:ns].cpu().numpy().astype(np.uint32), wl))
    if world > 1:
        t = torch.tensor([ms, 0.0 if ok else 1.0], dtype=torch.float64, device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        ms, ok = float(t[0]), float(t[1]) == 0.0
    e.close()
    del x, lo, la
    torch.cuda.empty_cache()
    return {"model": name + (" (NF4 LUT extension)" if nf4 else ""), "batch_per_gpu": n, "n_gpus": world, "g_images_per_s": world * n / ms / 1e6,
            "hbm_frac_per_gpu": (256 + 4 * m.n_classes) * n / ms / 1e6 / PEAK, "ms_per_launch": ms, "parity": ok}


ENCODINGS = [("rand_binary64", False), ("ternary64", False), ("1k", False), ("2bitsym96", False), ("fc", False), ("4bit64", False),
             ("12k_FP130", False), ("rand_nf4_64", True), ("8bit64", False), ("binary160", False)]
BATCHES = [1 << 10, 1 << 14, 1 << 17, 1 << 20, 1 << 22, 1 << 24]
rows = []
if rank == 0:
    print(f"| model | batch per GPU | GPUs | G images/s (all GPUs) | of measured HBM roofline (per GPU) | ms/launch | parity |\n|---|---|---|---|---|---|---|")
quick = os.environ.get("SWEEP_QUICK") == "1"
for name, nf4 in ENCODINGS:
    for n in BATCHES:
        if quick and n not in (1 << 10, 1 << 20, 1 << 24):
            continue
        r = run(name, n, nf4=nf4)
        rows.append(r)
        if rank == 0:
            print(f"| {r['model']} | 2^{n.bit_length() - 1} | {world} | {r['g_images_per_s']:.3f} | {r['hbm_frac_per_gpu']:.3f} | {r['ms_per_launch']:.4f} | "
                  f"{'bit-exact' if r['parity'] else 'MISMATCH'} |", flush=True)
for name in ("cnn", "cnn_48"):
    r = run(name, 1 << 20)
    rows.append(r)
    if rank == 0:
        print(f"| {r['model']} | 2^20 | {world} | {r['g_images_per_s']:.3f} | {r['hbm_frac_per_gpu']:.3f} | {r['ms_per_launch']:.4f} | {'bit-exact' if r['parity'] else 'MISMATCH'} |", flush=True)
if rank == 0:
    os.makedirs(os.path.join(ROOT, "sweep_out"), exist_ok=True)
    json.dump(rows, open(os.path.join(ROOT, "sweep_out", f"sweep_{world}gpu.json"), "w"), indent=0)
if world > 1:
    dist.destroy_process_group()
