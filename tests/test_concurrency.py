"""One model served from many host threads and streams: every entry point called concurrently returns exactly what the same call
returns alone.  The reference's Inference() keeps no state, so its callers spread calls over threads; these tests hold the
library to the same.  Results are compared with the same library called from one thread (the parity suite ties that to the
oracle) and, where they apply, with the reference's digit labels.  Threads always join within a deadline."""
import json
import os
import re
import subprocess
import sys
import threading
import time

import numpy as np
import pytest

from conftest import GOLDEN, ROOT, load_model
from support import build_c_shim, engine

JOIN_S = 600


def run_threads(targets, timeout=JOIN_S):
    """run every callable on its own thread, join all within `timeout` seconds, re-raise the first failure"""
    errors = []

    def guarded(fn):
        def run():
            try:
                fn()
            except BaseException as ex:   # noqa: B902 -- carried to the main thread
                errors.append(ex)
        return run
    threads = [threading.Thread(target=guarded(f), daemon=True) for f in targets]
    for t in threads:
        t.start()
    deadline = time.monotonic() + timeout
    for t in threads:
        t.join(max(0.0, deadline - time.monotonic()))
    stuck = [t for t in threads if t.is_alive()]
    assert not stuck, f"{len(stuck)} of {len(threads)} threads did not finish within {timeout} s"
    if errors:
        raise errors[0]


def digits():
    d = np.load(os.path.join(GOLDEN, "digits.npz"))
    return d["images"].astype(np.int8), d["labels"].astype(np.uint32)


def harness(tmp):
    exe = os.path.join(tmp, "concurrency")
    subprocess.run(["gcc", "-O2", "-Wall", "-Werror", "-pthread", "-I" + os.path.join(ROOT, "include"), "-o", exe,
                    os.path.join(ROOT, "host", "bitnetmcu_b200_concurrency.c"), "-ldl"], check=True)
    return exe


# ---- CPU: the measurement harness and the shim it loads -----------------------------------------------------------------------

@pytest.mark.parametrize("name", ["fc", "cnn"])
def test_concurrency_harness_and_shim_compile(built, tmp_path, name):
    dll, _, _ = build_c_shim(str(tmp_path), name)
    exe = harness(str(tmp_path))
    assert os.access(exe, os.X_OK) and os.path.exists(dll)
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 2 and "usage" in out.stderr


# ---- 1. small bnm_infer_batch calls batched together -----------------------------------------------------------------------

SIZES = (1, 7, 1024)
OUTPUTS = ((False, True), (True, False), (True, True))   # (logits, labels): labels only, logits only, both


def small_case(i, rng, d_img):
    """thread i's batch size, outputs and images: the digits first, then random rows"""
    n = SIZES[i % 3]
    x = rng.integers(-128, 128, size=(n, 256)).astype(np.int8)
    k = min(n, 10)
    x[:k] = np.roll(d_img, -i, axis=0)[:k]
    return n, OUTPUTS[(i // 3) % 3], x


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["fc", "cnn_48"])
@pytest.mark.parametrize("path", ["fused", "layers"])
def test_small_calls_from_16_threads(built, name, path):
    from bitnetmcu_b200 import _lib
    e = engine(load_model(name), path=_lib.PATH_LAYERS if path == "layers" else _lib.PATH_AUTO)
    d_img, d_lab = digits()
    rng = np.random.default_rng(7)
    cases = [small_case(i, rng, d_img) for i in range(16)]
    want = [e.infer(x) for _, _, x in cases]   # one thread
    if name == "fc":   # the reference's KAT on this model
        for i, (n, _, _) in enumerate(cases):
            k = min(n, 10)
            assert want[i][1][:k].tolist() == np.roll(d_lab, -i)[:k].tolist()
    start = threading.Barrier(16)

    def caller(i):
        n, (lo, la), x = cases[i]

        def run():
            start.wait(timeout=60)
            for rep in range(25):
                logits, labels = e.infer(x, want_logits=lo, want_labels=la)
                if lo:
                    assert np.array_equal(logits, want[i][0]), (name, path, i, rep, "logits")
                else:
                    assert logits is None
                if la:
                    assert np.array_equal(labels, want[i][1]), (name, path, i, rep, "labels")
        return run
    run_threads([caller(i) for i in range(16)])
    e.close()


BATCH_SCRIPT = r'''
import os, sys, threading
import numpy as np
sys.path.insert(0, os.environ["BNM_ROOT"])
from bitnetmcu_b200.engine import Engine
from bitnetmcu_b200.model import Model
root = os.environ["BNM_ROOT"]
e = Engine(Model.load(os.path.join(root, "tests", "golden", "models", "fc.bnm")))
d = np.load(os.path.join(root, "tests", "golden", "digits.npz"))
imgs, labs = d["images"].astype(np.int8), d["labels"].astype(np.int64)   # read once: an npz archive is not for threads
T = int(sys.argv[1])
start = threading.Barrier(T)
bad, done = [], []
def work(i):
    start.wait()
    for r in range(300):
        k = (i + r) % 10
        _, la = e.infer(imgs[k][None], want_logits=False)
        if int(la[0]) != int(labs[k]):
            bad.append((i, r))
    done.append(i)
ts = [threading.Thread(target=work, args=(i,), daemon=True) for i in range(T)]
for t in ts: t.start()
for t in ts: t.join(300)
if any(t.is_alive() for t in ts): print("TIMEOUT", flush=True); os._exit(4)
print("OK" if not bad and len(done) == T else "BAD", len(bad), len(done), flush=True)
e.close()
'''


@pytest.mark.gpu
def test_small_batch_lines_under_verbose(built, tmp_path):
    script = tmp_path / "batch.py"
    script.write_text(BATCH_SCRIPT)
    env = dict(os.environ, BNM_VERBOSE="1", BNM_ROOT=ROOT)
    pat = re.compile(r"bitnetmcu_b200: small batch: (\d+) images from (\d+) calls$")
    calls = {}
    for t in (16, 1):
        r = subprocess.run([sys.executable, str(script), str(t)], env=env, capture_output=True, text=True, timeout=600)
        assert r.returncode == 0 and r.stdout.startswith("OK"), (t, r.stdout[-500:], r.stderr[-2000:])
        lines = [pat.search(l) for l in r.stderr.splitlines()]
        calls[t] = [(int(m.group(1)), int(m.group(2))) for m in lines if m]
    assert any(c >= 2 for _, c in calls[16]), calls[16][:20]
    assert all(n == c for n, c in calls[16]), "one image per call"
    assert calls[1] == []


# ---- 2. the plan's tensor-map cache under contention -------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("overlap", [0, 2])
def test_tensor_map_cache_8_threads_3_buffers_each(built, overlap):
    import torch
    from bitnetmcu_b200 import _lib
    e = engine(load_model("fc"))
    assert e.active_path == _lib.PATH_TCGEN05
    e.set_option(_lib.OPT_LAUNCH_OVERLAP, overlap)
    d_img, d_lab = digits()
    T, CALLS, C = 8, 50, e.n_classes
    rng = np.random.default_rng(11)
    bufs, want, outs, streams = [], [], [], []
    for t in range(T):
        n = 1000 + 37 * t   # the threads' pointers and sizes all differ: more (pointer, n) pairs than the cache holds
        xs = [rng.integers(-128, 128, size=(n, 256)).astype(np.int8) for _ in range(3)]
        xs[0][:10] = d_img
        bufs.append([torch.from_numpy(x).cuda() for x in xs])
        want.append([e.infer(x) for x in xs])
        outs.append((torch.full((CALLS, n, C), -7, dtype=torch.int32, device="cuda"),
                     torch.full((CALLS, n), -7, dtype=torch.int32, device="cuda")))
        streams.append(torch.cuda.Stream())
    assert want[0][0][1][:10].tolist() == d_lab.tolist()
    torch.cuda.synchronize()

    def caller(t):
        def run():
            st = streams[t].cuda_stream
            for c in range(CALLS):
                e.infer_device(bufs[t][c % 3], outs[t][0][c], outs[t][1][c], stream=st)
        return run
    run_threads([caller(t) for t in range(T)])
    torch.cuda.synchronize()
    for t in range(T):
        lo, la = outs[t][0].cpu().numpy(), outs[t][1].cpu().numpy().astype(np.uint32)
        for c in range(CALLS):
            assert np.array_equal(lo[c], want[t][c % 3][0]), (overlap, t, c, "logits")
            assert np.array_equal(la[c], want[t][c % 3][1]), (overlap, t, c, "labels")
    e.close()


# ---- 3. device entries that run through scratch, on concurrent streams --------------------------------------------------------

CNN_CHUNK, EMUL_FC_CHUNK = 1 << 20, 65536   # images per chunk of the routes below (capi.cu)


def _i32(*shape):
    import torch
    return torch.full(shape, -7, dtype=torch.int32, device="cuda")


def _f64(*shape):
    import torch
    return torch.full(shape, np.nan, dtype=torch.float64, device="cuda")


# name -> (model, path, input dtype, images, outputs(e, n), call(e, x, outs, stream))
DEVICE_CASES = {
    "infer_device cnn": ("cnn", "fused", "i8", CNN_CHUNK + 77, lambda e, n: [_i32(n, e.n_classes), _i32(n)],
                         lambda e, x, o, st: e.infer_device(x, o[0], o[1], stream=st)),
    "infer_device cnn_48 layers": ("cnn_48", "layers", "i8", 2 * (1 << 17) + 5, lambda e, n: [_i32(n, e.n_classes), _i32(n)],
                                   lambda e, x, o, st: e.infer_device(x, o[0], o[1], stream=st)),
    "infer_device_f32 binary160": ("binary160", "fused", "f32", 70001, lambda e, n: [_i32(n, e.n_classes), _i32(n)],
                                   lambda e, x, o, st: e.infer_device_f32(x, o[0], o[1], stream=st)),
    "emulator int8 rows cnn_48": ("cnn_48", "fused", "f32", CNN_CHUNK + 33, lambda e, n: [_f64(n, e.n_classes), _i32(n)],
                                  lambda e, x, o, st: e.inference_quantized_device(x, o[0], o[1], stream=st)),
    "emulator int8 rows 37 classes": ("wide37", "fused", "f32", CNN_CHUNK + 21, lambda e, n: [_f64(n, e.n_classes), _i32(n)],
                                      lambda e, x, o, st: e.inference_quantized_device(x, o[0], o[1], stream=st)),
    "emulator layers fc": ("fc", "layers", "f32", 2 * EMUL_FC_CHUNK + 9, lambda e, n: [_f64(n, e.n_classes), _i32(n)],
                           lambda e, x, o, st: e.inference_quantized_device(x, o[0], o[1], stream=st)),
    "compare_engines counts only binary160": ("binary160", "fused", "f32", CNN_CHUNK + 3, lambda e, n: [_zero_counts()],
                                              lambda e, x, o, st: e.compare_engines_device(x, counts=o[0], stream=st)),
    "topk_device_f32 fc": ("fc", "fused", "f32", CNN_CHUNK + 9, lambda e, n: [_i32(n, 3), _i32(n, 3)],
                           lambda e, x, o, st: e.topk_device_f32(x, 3, o[0], o[1], stream=st)),
    "emulate_topk_device cnn_48": ("cnn_48", "fused", "f32", CNN_CHUNK + 5, lambda e, n: [_i32(n, 4), _f64(n, 4)],
                                   lambda e, x, o, st: e.emulate_topk_device(x, 4, o[0], o[1], stream=st)),
    "emulate_topk_device fc layers": ("fc", "layers", "f32", 2 * EMUL_FC_CHUNK + 9, lambda e, n: [_i32(n, 4), _f64(n, 4)],
                                      lambda e, x, o, st: e.emulate_topk_device(x, 4, o[0], o[1], stream=st)),
}


def _zero_counts():
    import torch
    return torch.zeros(4, dtype=torch.int64, device="cuda")


def _model(name):
    if name == "wide37":
        from support import random_fc
        return random_fc(4, (256, 64, 64, 37), 2)
    return load_model(name)


@pytest.mark.gpu
@pytest.mark.parametrize("streams", ["own", "shared"])
@pytest.mark.parametrize("case", list(DEVICE_CASES))
def test_device_scratch_routes_concurrently(built, case, streams):
    import torch
    from bitnetmcu_b200 import _lib
    name, path, dtype, n, outputs, call = DEVICE_CASES[case]
    e = engine(_model(name), path=_lib.PATH_LAYERS if path == "layers" else _lib.PATH_AUTO)
    T = 3
    g = torch.Generator(device="cuda").manual_seed(5)
    if dtype == "i8":
        base = torch.randint(-128, 128, (n, e.img_bytes), dtype=torch.int8, device="cuda", generator=g)
    else:
        base = torch.randn((n, e.img_bytes), dtype=torch.float32, device="cuda", generator=g)
    base[:10] = torch.from_numpy(digits()[0][:, :e.img_bytes].astype(np.float32 if dtype == "f32" else np.int8)).cuda()
    want = outputs(e, n)
    call(e, base, want, torch.cuda.current_stream().cuda_stream)   # serial
    torch.cuda.synchronize()
    want = [w.cpu() for w in want]
    shift = lambda t: 131 * t   # thread t's images: the base rows rotated, so every thread's results differ
    xs = [torch.roll(base, shift(t), 0).contiguous() for t in range(T)]
    del base
    outs = [outputs(e, n) for _ in range(T)]
    own = [torch.cuda.Stream() for _ in range(T)]
    shared = torch.cuda.Stream()
    torch.cuda.synchronize()

    def caller(t):
        def run():
            call(e, xs[t], outs[t], (own[t] if streams == "own" else shared).cuda_stream)   # enqueue only
        return run
    run_threads([caller(t) for t in range(T)])
    torch.cuda.synchronize()
    for t in range(T):
        for i, (got, w) in enumerate(zip(outs[t], want)):
            exp = w if w.dim() == 1 and w.numel() == 4 and w.dtype == torch.int64 else torch.roll(w, shift(t), 0)
            assert torch.equal(got.cpu(), exp), (case, streams, t, i)
    e.close()


# ---- 4. large host calls concurrently -----------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("name", ["fc", "cnn_48"])
def test_large_host_calls_take_turns(built, name):
    from bitnetmcu_b200 import _lib
    e = engine(load_model(name))
    chunk = 4096
    e.set_option(_lib.OPT_CHUNK_IMAGES, chunk)
    n = 3 * chunk + 17
    rng = np.random.default_rng(3)
    xa, xb = (rng.integers(-128, 128, size=(n, 256)).astype(np.int8) for _ in range(2))
    xf = rng.normal(size=(3000, 256)).astype(np.float32)
    want_a, want_b = e.infer(xa), e.infer(xb)
    want_k = e.topk(xa, 3)
    want_q = e.inference_quantized(xf)

    def batch(x, want):
        def run():
            for _ in range(3):
                lo, la = e.infer(x)
                assert np.array_equal(lo, want[0]) and np.array_equal(la, want[1])
        return run

    def topk():
        for _ in range(3):
            c, s = e.topk(xa, 3)
            assert np.array_equal(c, want_k[0]) and np.array_equal(s, want_k[1])

    def emulate():
        for _ in range(3):
            assert np.array_equal(e.inference_quantized(xf), want_q)
    run_threads([batch(xa, want_a), batch(xb, want_b), topk, emulate])
    e.close()


# ---- 5. the drop-in shim from 8 threads ---------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("name", ["fc", "cnn"])
def test_shim_inference_from_8_threads(built, tmp_path, name):
    dll, _, d = build_c_shim(str(tmp_path), name)
    exe = harness(str(tmp_path))
    path = os.path.join(str(tmp_path), "digits.bin")
    d["images"].astype(np.int8).tofile(path)
    r = subprocess.run([exe, dll, path, "8", "300"], capture_output=True, text=True, timeout=JOIN_S)
    assert r.returncode == 0, r.stderr[-2000:]
    out = json.loads(r.stdout.strip().splitlines()[-1])
    assert out["labels"] == ",".join(str(int(v)) for v in d["labels"])   # the reference's KAT
    assert out["mismatches"] == 0 and out["calls"] == 8 * 300


# ---- 6. two models, each from its own threads ---------------------------------------------------------------------------------

@pytest.mark.gpu
def test_two_models_created_and_used_concurrently(built):
    import torch
    d_img, d_lab = digits()
    rng = np.random.default_rng(9)
    x = rng.integers(-128, 128, size=(5000, 256)).astype(np.int8)
    x[:10] = d_img
    want = {}
    for name in ("fc", "cnn"):
        e = engine(load_model(name))
        want[name] = e.infer(x)
        assert want[name][1][:10].tolist() == d_lab.tolist()
        e.close()
    d_x = torch.from_numpy(x).cuda()

    def user(name):
        def run():
            e = engine(load_model(name))
            st = torch.cuda.Stream()
            lo, la = _i32(x.shape[0], e.n_classes), _i32(x.shape[0])
            for _ in range(3):
                got = e.infer(x)   # host pipeline
                assert np.array_equal(got[0], want[name][0]) and np.array_equal(got[1], want[name][1]), name
                for i in range(0, 40, 7):   # small calls
                    assert np.array_equal(e.infer(x[i:i + 7])[1], want[name][1][i:i + 7]), name
                e.infer_device(d_x, lo, la, stream=st.cuda_stream)
                st.synchronize()
                assert np.array_equal(lo.cpu().numpy(), want[name][0]), name
                assert np.array_equal(la.cpu().numpy().astype(np.uint32), want[name][1]), name
            e.close()
        return run
    run_threads([user("fc"), user("cnn"), user("fc"), user("cnn")])
