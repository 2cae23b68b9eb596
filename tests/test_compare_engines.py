"""Both engines in one call: bnm_compare_engines_device / Engine.compare_engines_device (the reference's verification loop,
test_inference.py:130-175).  The C engine's labels, the Python emulator's labels, and counts {images, correct_c, correct_py,
mismatches} that every call adds to.  FC models of the float-input row run fc_engines_kernel (one input scaling, one layer 1, the
two hidden-layer chains, the counts in its epilogue); every other model runs the two existing routes, then k_engine_counts.

CPU tests: the new kernels' SASS, the entry's failure without a device, and the expectations the GPU tests use (the oracle on the
scaled images for the C engine, the NumPy restatement of the emulator for the other).  GPU tests: tolerance 0."""
import ctypes as C
import os
import re
import zlib

import numpy as np
import pytest

from conftest import GOLDEN, load_model
from restate import TILE, cnn_features, emulate, scale_images
from support import N_MANY, Sweep, crafted_cnn_case, cnn_model, engine, instructions, lib, local_memory, normal_images, \
    plan_line, route, sass_functions, scattered_edge_images, verbose_engine

GOLDEN_NAMES = ["fc", "1k", "12k_FP130", "8bit64", "ternary64", "binary160", "2bitsym96", "cnn", "cnn_48", "cnn_16small"]
FUSED = {"fc", "1k", "12k_FP130", "8bit64", "ternary64"}          # the float-input row's models
ENGINES_ROW = "fc_engines_kernel<64,1,float,engines>"
FALLBACK = "bnm_infer_batch_device_f32 + bnm_emulate_batch_device + k_engine_counts"


def expected_counts(lc, lp, truth=None, n_classes=10):
    """the NumPy counts: [images, correct_c, correct_py, mismatches]"""
    lc, lp = np.asarray(lc, dtype=np.int64), np.asarray(lp, dtype=np.int64)
    out = [lc.size, 0, 0, int((lc != lp).sum())]
    if truth is not None:
        t = np.asarray(truth, dtype=np.int64)
        ok = t < n_classes
        out[1], out[2] = int((ok & (lc == t)).sum()), int((ok & (lp == t)).sum())
    return out


# ---- CPU -------------------------------------------------------------------------------------------------------------------

def test_engines_kernels_sass(built):
    """exactly one fc_engines_kernel (IGMMA, no local memory) and k_engine_counts (no local memory)"""
    kernels = sass_functions()
    fused = [k for k in kernels if k.startswith("_ZN3bnm17fc_engines_kernel")]
    counts = [k for k in kernels if k.startswith("_ZN3bnm15k_engine_counts")]
    assert len(fused) == 1 and len(counts) == 1, (fused, counts)
    for k in fused + counts:
        ins = instructions(kernels[k])
        assert len(ins) > 20, k
        assert not local_memory(ins), f"local memory in {k}"
        assert (k in fused) == any(i.startswith("IGMMA") for i in ins), k
    assert "VOTE.ANY" in kernels[counts[0]] and "POPC" in kernels[counts[0]]


def test_no_fallback_without_gpu(built):
    from bitnetmcu_b200 import _lib
    lib = _lib.load()
    if lib.bnm_device_count() > 0:
        pytest.skip("a CUDA device is present")
    x = np.zeros((4, 256), dtype=np.float32)
    lab = np.zeros(4, dtype=np.uint32)
    assert lib.bnm_compare_engines_device(None, C.c_void_p(x.ctypes.data), 4, None, C.c_void_p(lab.ctypes.data), None, None, None) != 0
    from bitnetmcu_b200.engine import Engine
    with pytest.raises(_lib.BnmError):
        Engine(load_model("fc"))


def test_expectations(oracle):
    """the GPU tests' expectations: the oracle on the scaled golden images (C engine) and the restatement's np.argmax (emulator,
    == the reference emulator's own logits) disagree on some images of some models, so the counts have mismatches to find"""
    g = np.load(os.path.join(GOLDEN, "emulator.npz"))
    total = 0
    for name in GOLDEN_NAMES:
        m = load_model(name)
        _, lc = oracle.infer(m, scale_images(g["images"]))
        lp = np.argmax(emulate(m, g["images"]), axis=1)
        assert np.array_equal(lp, np.argmax(g[name], axis=1)), name
        c = expected_counts(lc, lp, np.arange(64) % 12)
        assert c[0] == 64 and 0 <= c[3] <= 64 and c[1] <= 64 - (np.arange(64) % 12 >= 10).sum()
        total += c[3]
    assert total > 0


# ---- GPU ------------------------------------------------------------------------------------------------------------------

def _compare(e, d_x, truth=None, want=("c", "py", "counts"), counts=None, stream=None, sentinel=-7):
    """one call -> (labels_c, labels_py, counts) as NumPy (None for what was not asked for)"""
    import torch
    n = d_x.shape[0]
    lc = torch.full((n,), sentinel, dtype=torch.int32, device="cuda") if "c" in want else None
    lp = torch.full((n,), sentinel, dtype=torch.int32, device="cuda") if "py" in want else None
    if counts is None and "counts" in want:
        counts = torch.zeros(4, dtype=torch.int64, device="cuda")
    d_t = None if truth is None else (truth if isinstance(truth, torch.Tensor) else torch.from_numpy(np.asarray(truth, dtype=np.int32)).cuda())
    e.compare_engines_device(d_x, truth=d_t, labels_c=lc, labels_py=lp, counts=counts, stream=stream)
    torch.cuda.synchronize()
    as_np = lambda t: None if t is None else t.cpu().numpy().astype(np.int64)
    return as_np(lc), as_np(lp), (None if counts is None else counts.cpu().numpy().tolist())


def _two_entries(e, d_x):
    """the labels of bnm_infer_batch_device_f32 and bnm_emulate_batch_device"""
    import torch
    n = d_x.shape[0]
    lc = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    lp = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    e.infer_device_f32(d_x, None, lc)
    e.inference_quantized_device(d_x, None, lp)
    torch.cuda.synchronize()
    return lc.cpu().numpy().astype(np.int64), lp.cpu().numpy().astype(np.int64)


def _truth(n, n_classes, seed):
    """random classes, with values of n_classes and above (never a match) mixed in"""
    return np.random.default_rng(seed).integers(0, n_classes + 3, size=n).astype(np.int32)


def _cuda(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).cuda()


@pytest.mark.gpu
@pytest.mark.parametrize("name", GOLDEN_NAMES)
def test_golden_models(lib, oracle, capfd, monkeypatch, name):
    """labels_c == the oracle on the scaled images, labels_py == np.argmax of the reference emulator's logits, counts == NumPy's
    against a seeded truth; the route names the fused kernel exactly for the float-row models"""
    g = np.load(os.path.join(GOLDEN, "emulator.npz"))
    x = np.concatenate([g["images"], normal_images(4000, seed=21)])
    m = load_model(name)
    e, err = verbose_engine(capfd, monkeypatch, lambda: engine(m))
    assert route(err, "engines") == (ENGINES_ROW if name in FUSED else FALLBACK), (name, err)
    _, want_c = oracle.infer(m, scale_images(x))
    want_py = np.argmax(emulate(m, x), axis=1)
    assert np.array_equal(want_py[:64], np.argmax(g[name], axis=1))
    truth = _truth(len(x), m.n_classes, seed=len(name))
    lc, lp, cnt = _compare(e, _cuda(x), truth)
    assert np.array_equal(lc, want_c.astype(np.int64)), (name, np.flatnonzero(lc != want_c)[:5])
    assert np.array_equal(lp, want_py), (name, np.flatnonzero(lp != want_py)[:5])
    assert cnt == expected_counts(want_c, want_py, truth, m.n_classes), name
    e.close()


def _fc_models():
    """float-row FC models of depth 1, 2, 4 and 8 (every layer <= 64 wide, <= 16 classes)"""
    from bitnetmcu_b200 import model as M, pack as P
    return [("4bitsym-d1", P.random_fc_model(M.ENC_4BITSYM, (256, 10), seed=1)),
            ("2bitsym-d2", P.random_fc_model(M.ENC_2BITSYM, (256, 48, 16), seed=2)),
            ("fp130-d4", P.random_fc_model(M.ENC_FP130, (256, 64, 64, 64, 10), seed=4)),
            ("ternary-d8", P.random_fc_model(M.ENC_TERNARY, (256,) + (64,) * 7 + (12,), seed=8))]


@pytest.mark.gpu
@pytest.mark.parametrize("idx", range(4))
def test_random_fc_models(lib, capfd, monkeypatch, idx):
    """one call == the two entries, at 1, 127, 128, 129 and N_MANY images; normal-distributed images make the engines disagree"""
    tag, m = _fc_models()[idx]
    e, err = verbose_engine(capfd, monkeypatch, lambda: engine(m))
    assert route(err, "engines") == ENGINES_ROW, (tag, err)
    d_all = _cuda(normal_images(N_MANY, seed=idx + 40))
    truth = _truth(N_MANY, m.n_classes, seed=idx)
    for n in (1, 127, 128, 129, N_MANY):
        d_x = d_all[:n]
        want_c, want_py = _two_entries(e, d_x)
        lc, lp, cnt = _compare(e, d_x, truth[:n])
        assert np.array_equal(lc, want_c) and np.array_equal(lp, want_py), (tag, n)
        assert cnt == expected_counts(want_c, want_py, truth[:n], m.n_classes), (tag, n)
    if idx > 0:
        assert cnt[3] > 0, (tag, "no disagreement to count")
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("channels,n_classes", [(16, 10), (48, 37), (128, 10)])
def test_random_cnn_models(lib, capfd, monkeypatch, channels, n_classes):
    m = cnn_model(channels, n_classes, seed=channels + n_classes)
    e, err = verbose_engine(capfd, monkeypatch, lambda: engine(m))
    assert route(err, "engines") == FALLBACK, err
    d_all = _cuda(normal_images(4000, seed=channels))
    truth = _truth(4000, n_classes, seed=channels)
    for n in (1, 129, 4000):
        want_c, want_py = _two_entries(e, d_all[:n])
        lc, lp, cnt = _compare(e, d_all[:n], truth[:n])
        assert np.array_equal(lc, want_c) and np.array_equal(lp, want_py), (channels, n)
        assert cnt == expected_counts(want_c, want_py, truth[:n], n_classes), (channels, n)
    assert cnt[3] > 0
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["fc", "8bit64"])
def test_engines_row_past_two_ring_rounds(lib, oracle, capfd, monkeypatch, name):
    """fc_engines_kernel has the float row's layout: over the sweep of the plan's float stage count, every label against the
    oracle and the restatement, nothing written past row n, and the counts"""
    import torch
    m = load_model(name)
    e, err = verbose_engine(capfd, monkeypatch, lambda: engine(m))
    line = plan_line(err)
    assert route(err, "engines") == ENGINES_ROW and line, err
    stages = int(re.search(r"float input stages (\d+)", line).group(1))
    sw = Sweep(f"<64,1,float,engines> ({name})", (1, stages, 1))
    x = scattered_edge_images(sw.sizes[-1], m.img_bytes, zlib.crc32(name.encode()) + 2)
    _, want_c = oracle.infer(m, scale_images(x))
    want_c = want_c.astype(np.int64)
    want_py = np.argmax(emulate(m, x), axis=1)
    truth = _truth(len(x), m.n_classes, seed=3)
    d_x, d_t = _cuda(x), torch.from_numpy(truth).cuda()
    for n in sw.sizes:
        d_lc = torch.full((n + TILE,), -7, dtype=torch.int32, device="cuda")
        d_lp = torch.full((n + TILE,), -7, dtype=torch.int32, device="cuda")
        counts = torch.zeros(4, dtype=torch.int64, device="cuda")
        e.compare_engines_device(d_x[:n], truth=d_t[:n], labels_c=d_lc[:n], labels_py=d_lp[:n], counts=counts)
        torch.cuda.synchronize()
        sw.check(n, d_lc, want_c, -7, "labels")
        sw.check(n, d_lp, want_py, -7, "labels")
        assert counts.cpu().numpy().tolist() == expected_counts(want_c[:n], want_py[:n], truth[:n], m.n_classes), (sw.tag, n)
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["fc", "cnn_48"])
def test_output_combinations(lib, name):
    """each output NULL in turn leaves the others unchanged; all three NULL, truth without counts and misaligned images are
    BNM_E_ARG; n == 0 leaves the counts alone"""
    import torch
    m = load_model(name)
    e = engine(m)
    n = 3001
    d_x = _cuda(normal_images(n, seed=9))
    truth = _truth(n, m.n_classes, seed=9)
    full = _compare(e, d_x, truth)
    no_truth = full[2][:1] + [0, 0] + full[2][3:]

    def same(got, want):
        return all((g is None and w is None) or (g is not None and w is not None and np.array_equal(g, w)) for g, w in zip(got, want))
    assert same(_compare(e, d_x, truth, want=("py", "counts")), (None, full[1], full[2]))
    assert same(_compare(e, d_x, truth, want=("c", "counts")), (full[0], None, full[2]))
    assert same(_compare(e, d_x, None, want=("c", "py")), (full[0], full[1], None))
    assert same(_compare(e, d_x, None, want=("c",)), (full[0], None, None))
    assert same(_compare(e, d_x, None, want=("py",)), (None, full[1], None))
    assert same(_compare(e, d_x, None, want=("counts",)), (None, None, no_truth))
    assert full[2][0] == n and full[2][3] > 0

    h = e.handle
    xp = C.c_void_p(d_x.data_ptr())
    lab = torch.zeros(n, dtype=torch.int32, device="cuda")
    d_t = torch.from_numpy(truth).cuda()
    counts = torch.full((4,), 5, dtype=torch.int64, device="cuda")
    lp_, tp, cp = C.c_void_p(lab.data_ptr()), C.c_void_p(d_t.data_ptr()), C.c_void_p(counts.data_ptr())
    assert lib.bnm_compare_engines_device(h, xp, n, None, None, None, None, None) == -1
    assert b"no output" in lib.bnm_last_error()
    assert lib.bnm_compare_engines_device(h, xp, n, tp, lp_, None, None, None) == -1
    assert b"truth without counts" in lib.bnm_last_error()
    assert lib.bnm_compare_engines_device(h, C.c_void_p(d_x.data_ptr() + 4), n - 1, None, lp_, None, cp, None) == -1
    assert lib.bnm_compare_engines_device(h, xp, n, None, lp_, None, C.c_void_p(counts.data_ptr() + 4), None) == -1
    assert lib.bnm_compare_engines_device(h, xp, 0, tp, lp_, lp_, cp, None) == 0
    assert lib.bnm_compare_engines_device(h, None, 0, None, None, None, cp, None) == 0
    torch.cuda.synchronize()
    assert counts.cpu().numpy().tolist() == [5, 5, 5, 5] and not lab.any()
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["fc", "binary160", "cnn_48"])
def test_counts_accumulate(lib, name):
    """two calls on the halves of a batch add up to one call on the whole, into the same counts"""
    import torch
    m = load_model(name)
    e = engine(m)
    n = 148 * 128 + 1001
    d_x = _cuda(normal_images(n, seed=12))
    d_t = torch.from_numpy(_truth(n, m.n_classes, seed=12)).cuda()
    whole = torch.zeros(4, dtype=torch.int64, device="cuda")
    halves = torch.zeros(4, dtype=torch.int64, device="cuda")
    e.compare_engines_device(d_x, truth=d_t, counts=whole)
    h = 148 * 64 + 13
    e.compare_engines_device(d_x[:h], truth=d_t[:h], counts=halves)
    e.compare_engines_device(d_x[h:], truth=d_t[h:], counts=halves)
    torch.cuda.synchronize()
    assert whole.cpu().tolist() == halves.cpu().tolist() and whole[0].item() == n and whole[3].item() > 0
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["fc", "cnn_48"])
def test_layered_path(lib, name):
    """BNM_PATH_LAYERS gives the labels and counts of the default path"""
    from bitnetmcu_b200 import _lib
    m = load_model(name)
    e = engine(m)
    x = normal_images(5000, seed=13)
    truth = _truth(5000, m.n_classes, seed=13)
    d_x = _cuda(x)
    default = _compare(e, d_x, truth)
    e.set_option(_lib.OPT_PATH, _lib.PATH_LAYERS)
    layered = _compare(e, d_x, truth)
    assert np.array_equal(default[0], layered[0]) and np.array_equal(default[1], layered[1]) and default[2] == layered[2]
    assert default[2][3] > 0
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["fc", "cnn_48"])
def test_non_default_stream(lib, name):
    """images copied from pinned memory on a side stream and the call on that stream, ordered by it alone"""
    import torch
    m = load_model(name)
    n = 148 * 128 * 3 + 5
    x = normal_images(n, seed=3)
    truth = _truth(n, m.n_classes, seed=3)
    e = engine(m)
    h_x = torch.from_numpy(x).pin_memory()
    d_t = torch.from_numpy(truth).cuda()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        d_x = torch.empty((n, 256), dtype=torch.float32, device="cuda")
        d_x.copy_(h_x, non_blocking=True)
        lc = torch.empty(n, dtype=torch.int32, device="cuda")
        lp = torch.empty(n, dtype=torch.int32, device="cuda")
        counts = torch.zeros(4, dtype=torch.int64, device="cuda")
        e.compare_engines_device(d_x, truth=d_t, labels_c=lc, labels_py=lp, counts=counts)
    s.synchronize()
    got = (lc.cpu().numpy().astype(np.int64), lp.cpu().numpy().astype(np.int64), counts.cpu().numpy().tolist())
    want = _compare(e, _cuda(x), truth)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]) and got[2] == want[2]
    assert np.array_equal(got[1][:1000], np.argmax(emulate(m, x[:1000]), axis=1))
    e.close()


@pytest.mark.gpu
def test_crafted_inputs(lib, oracle):
    """all-zero images, one negative pixel, and CNN models whose conv2 or conv3 outputs are never positive (the inputs of
    test_emulator_routes.test_crafted_inputs); and the fused row on the same images"""
    x, models = crafted_cnn_case()
    truth = _truth(700, 10, seed=5)
    models.append((load_model("fc"), "fc"))
    for m, what in models:
        if what.startswith("conv"):
            assert not cnn_features(m, x).any(), what
        e = engine(m)
        _, want_c = oracle.infer(m, scale_images(x))
        want_py = np.argmax(emulate(m, x), axis=1)
        lc, lp, cnt = _compare(e, _cuda(x), truth)
        assert np.array_equal(lc, want_c.astype(np.int64)) and np.array_equal(lp, want_py), what
        assert cnt == expected_counts(want_c, want_py, truth, 10), what
        e.close()
