"""The reference's Python emulator (QuantizedModel.inference_quantized, BitNetMCU.py:420-535) on device buffers:
bnm_emulate_batch_device / Engine.inference_quantized_device.  FC models up to 64 wide run one kernel (fc_emul_kernel, the
float-input kernel with the emulator's hidden-layer rule); everything else the emulation kernels layer by layer.

CPU tests: the integer form of the emulator's hidden-layer rule, a NumPy float64 restatement of the emulator's FC path (the
expectation of the GPU tests) against the reference's own logits, and the emulator kernel's SASS.  GPU tests: tolerance 0."""
import ctypes as C
import importlib.util
import os

import numpy as np
import pytest

from conftest import GOLDEN, ROOT, load_model
from restate import emulate_fc, scale_images
from support import N_MANY, engine, instructions, lib, local_memory, normal_images, plan_line, random_fc, run_emulator, \
    sass_functions, verbose_engine

FC_GOLDEN = ["fc", "1k", "12k_FP130", "2bitsym96", "8bit64", "binary160", "ternary64"]
ALL_GOLDEN = FC_GOLDEN + ["cnn", "cnn_48", "cnn_16small"]


def emul_exponent(m):
    """e = floor(log2(127 / m)) of row maxima m >= 1 (int64 array) by a bit length and one compare, as emul_coef computes it"""
    m = np.asarray(m, dtype=np.int64)
    z = 32 - np.frexp(m.astype(np.float64))[1].astype(np.int64)    # 32 - bit length (exact below 2^53)
    return z - 25 - ((m << z) > (127 << 25)).astype(np.int64)


def int_rule(v, m):
    """The integer form of the hidden-layer rule that fc_emul_kernel runs (fc_wgmma.cu emul_coef / emul_q), elementwise over int64
    arrays: m = relu'd row maximum, v = accumulator."""
    v = np.asarray(v, dtype=np.int64)
    e = emul_exponent(np.maximum(np.asarray(m, dtype=np.int64), 1))
    mult = np.where(e > 0, np.int64(1) << np.maximum(e, 0), 1)
    s = np.maximum(-e, 0)
    bias = np.where(s > 0, (np.int64(1) << np.maximum(s - 1, 0)) - 1, 0)
    t = np.maximum(v, 0) * mult
    return (t + bias + ((t >> s) & (s > 0))) >> s


def float_rule(v, m, ls):
    """BitNetMCU.py:452-457 on conv = acc / 2^ls"""
    conv, top = np.asarray(v, dtype=np.float64) / 2.0 ** ls, np.maximum(np.asarray(m, dtype=np.float64) / 2.0 ** ls, 1e-5)
    return np.round(conv * np.exp2(np.floor(np.log2(127.0 / top)))).clip(0, 127)


def _check_rule(m):
    rng = np.random.default_rng(int(m.size))
    half = [np.zeros_like(m)]
    for s in range(1, 25):                                            # exact .5 ties at every shift that can round
        half.append(np.minimum(m, (2 * rng.integers(0, 1 << 8, size=m.shape) + 1) << (s - 1)))
    vs = [np.zeros_like(m), np.ones_like(m), m, m - 1, rng.integers(0, m + 1), rng.integers(-m, 1)] + half
    for v in vs:
        got = int_rule(v, m)
        assert got.min() >= 0 and got.max() <= 127
        for ls in (0, 1):
            want = float_rule(v, m, ls)
            bad = np.flatnonzero(got != want)
            assert bad.size == 0, (ls, m[bad[:5]], v[bad[:5]], got[bad[:5]], want[bad[:5]])


def test_integer_rule_every_small_maximum():
    _check_rule(np.arange(1, (1 << 16) + 1, dtype=np.int64))


def test_integer_rule_sampled_large_maxima():
    rng = np.random.default_rng(7)
    m = np.concatenate([rng.integers(1 << 16, 1 << 23, size=200000), (np.int64(127) << np.arange(0, 17)),
                        (np.int64(127) << np.arange(0, 17)) + 1, np.int64(1) << np.arange(16, 24)])
    _check_rule(m.astype(np.int64))


def test_integer_rule_non_positive_maximum():
    """m <= 0: every value is <= 0 and the whole row is zero (the emulator's 1e-5 floor)"""
    v = np.array([0, -1, -5, -(1 << 30)], dtype=np.int64)
    for m in (0, -1, -7):
        assert not int_rule(v, np.full_like(v, max(m, 0))).any()
        assert not float_rule(v, np.full_like(v, m), 1).any() and not float_rule(v, np.full_like(v, m), 0).any()


@pytest.mark.parametrize("name", FC_GOLDEN)
def test_restatement_reproduces_reference_emulator(name):
    """tests/golden/emulator.npz holds the reference emulator's own logits"""
    g = np.load(os.path.join(GOLDEN, "emulator.npz"))
    got = emulate_fc(load_model(name), g["images"])
    assert got.dtype == np.float64 and np.array_equal(got, g[name]), (name, np.argwhere(got != g[name])[:5])


def test_emulator_kernel_sass(built):
    """fc_emul_kernel is its own function (not a ninth fc_chain_kernel instantiation) and keeps everything in registers"""
    kernels = sass_functions()
    emul = [k for k in kernels if k.startswith("_ZN3bnm14fc_emul_kernel")]
    assert len(emul) == 1, sorted(kernels)
    ins = instructions(kernels[emul[0]])
    assert len(ins) > 100 and any(i.startswith("IGMMA") for i in ins)
    assert not local_memory(ins), "local memory in fc_emul_kernel"


# ---- GPU ------------------------------------------------------------------------------------------------------------------

def _fused_engine(capfd, monkeypatch, model):
    """an engine, and whether its plan runs the fused emulator kernel"""
    e, err = verbose_engine(capfd, monkeypatch, lambda: engine(model))
    return e, "emulator <64,1,float,emul>" in (plan_line(err) or "")


@pytest.mark.gpu
@pytest.mark.parametrize("name", ALL_GOLDEN)
def test_device_entry_matches_reference_emulator(lib, capfd, monkeypatch, name):
    """every golden model on the default path (fused where the plan has the emulator kernel, else the fallback) and on the
    layer-by-layer path: the reference emulator's logits bit for bit, labels = np.argmax"""
    from bitnetmcu_b200 import _lib
    g = np.load(os.path.join(GOLDEN, "emulator.npz"))
    want = g[name]
    m = load_model(name)
    e, fused = _fused_engine(capfd, monkeypatch, m)
    # FC models up to 64 wide; a CNN model's plan has the kernel too (its FC part fits), but CNN models always take the fallback
    assert fused == (name in ("fc", "1k", "12k_FP130", "8bit64", "ternary64", "cnn_16small")), name
    for path in (None, _lib.PATH_LAYERS):
        if path is not None:
            e.set_option(_lib.OPT_PATH, path)
        lo, la = run_emulator(e, g["images"])
        assert np.array_equal(lo, want), (name, path, np.argwhere(lo != want)[:5])
        assert np.array_equal(la, np.argmax(want, axis=1)), (name, path)
    e.close()


def _random_models():
    from bitnetmcu_b200 import model as M, pack as P
    out = []
    for enc in (M.ENC_BINARY, M.ENC_2BITSYM, M.ENC_4BITSYM, M.ENC_4BIT, M.ENC_8BIT, M.ENC_FP130, M.ENC_TERNARY):
        out.append((M.ENC_NAMES[enc], P.random_fc_model(enc, (256, 64, 64, 64, 10), seed=enc)))
    out.append(("2bitsym-16cls", P.random_fc_model(M.ENC_2BITSYM, (256, 48, 16), seed=3)))
    out.append(("4bitsym-160in", random_fc(M.ENC_4BITSYM, (160, 64, 32, 7), 5)))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("idx", range(9))
def test_fused_equals_layered_and_restatement(lib, capfd, monkeypatch, idx):
    """random FC models of every encoding (2bitsym / 4bitsym hidden and last layers, FP130's residual plane, Ternary's padded
    inputs): the fused emulator, the layer-by-layer emulator and the NumPy restatement agree exactly"""
    from bitnetmcu_b200 import _lib
    tag, m = _random_models()[idx]
    x = normal_images(3001, seed=idx, elems=m.img_bytes)
    want = emulate_fc(m, x)
    e, fused = _fused_engine(capfd, monkeypatch, m)
    assert fused, tag
    lo, la = run_emulator(e, x)
    assert np.array_equal(lo, want), (tag, np.argwhere(lo != want)[:5])
    assert np.array_equal(la, np.argmax(want, axis=1)), tag
    e.set_option(_lib.OPT_PATH, _lib.PATH_LAYERS)
    lo2, la2 = run_emulator(e, x)
    assert np.array_equal(lo2, lo) and np.array_equal(la2, la), tag
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 127, 128, 129, N_MANY])
def test_batch_sizes(lib, n):
    """ragged tiles, one tile, several tiles per CTA; twice in a row (the launch is repeatable: each one starts its ring at stage
    0, phase 0; tests/test_fc_ring_rounds.py runs the ring past its first rounds)"""
    m = load_model("fc")
    x = normal_images(n, seed=n)
    want = emulate_fc(m, x)
    e = engine(m)
    for _ in range(2):
        lo, la = run_emulator(e, x)
        assert np.array_equal(lo, want) and np.array_equal(la, np.argmax(want, axis=1)), n
    e.close()


def _crafted_images(n_rows=512, elems=256):
    """all-zero images; images below the 1e-5 floor (tiny integers after scaling: small first-layer maxima, e >= 0); one-pixel
    images; and random rows"""
    rng = np.random.default_rng(11)
    x = rng.normal(size=(n_rows, elems)).astype(np.float32)
    x[0:8] = 0.0
    x[8:64] = (rng.integers(-4, 5, size=(56, elems)) * 1e-7).astype(np.float32)
    x[64:128] = 0.0
    for k in range(32):
        x[64 + k, (7 * k) % elems] = np.float32(1e-7)               # one pixel of 1 after scaling: row maxima of one weight
    x[80:96, 3] = np.float32(-1e-7)
    for k in range(32):
        x[96 + k, k] = np.float32(3.0)
    return x


def _first_layer_stats(model, x):
    """layer-1 row maxima and whether round-half-even met an exact tie there, per the restatement"""
    from bitnetmcu_b200 import model as M, pack as P
    l = [l for l in model.layers if l.kind == M.LAYER_FC][0]
    acc = scale_images(x).astype(np.int64) @ P.decode_int_weights(l).astype(np.int64)[:, :x.shape[1]].T
    mx = acc.max(axis=1)
    e = emul_exponent(np.maximum(mx, 1))
    s = np.maximum(-e, 0)[:, None]
    ties = ((s > 0) & (acc > 0) & ((acc & ((np.int64(1) << s) - 1)) == (np.int64(1) << np.maximum(s - 1, 0)))).any()
    return mx, e, bool(ties)


@pytest.mark.gpu
def test_crafted_rows(lib):
    """all-zero images, a hidden layer whose maximum is <= 0, small maxima (e >= 0) and exact .5 ties, fused and layered"""
    from bitnetmcu_b200 import _lib, model as M, pack as P
    x = _crafted_images()
    # layer 1 of all -1 binary weights: a non-negative image gives a row maximum <= 0, so the next layer sees zeros
    neg = P.random_fc_model(M.ENC_4BITSYM, (256, 64, 64, 10), seed=9)
    neg.layers[0] = P.fc_layer_from_codes("L1", M.ENC_BINARY, np.zeros((64, 256), dtype=np.uint32))
    xn = np.abs(x)
    for m, xs in ((load_model("fc"), x), (P.random_fc_model(M.ENC_2BITSYM, (256, 64, 64, 10), seed=1), x), (neg, xn)):
        mx, ex, ties = _first_layer_stats(m, xs)
        if m is neg:
            assert (mx <= 0).all()
        else:
            assert (ex[mx > 0] >= 0).any() and (ex < 0).any() and ties and (mx <= 0).any()
        want = emulate_fc(m, xs)
        e = engine(m)
        for path in (None, _lib.PATH_LAYERS):
            if path is not None:
                e.set_option(_lib.OPT_PATH, path)
            lo, la = run_emulator(e, xs)
            assert np.array_equal(lo, want) and np.array_equal(la, np.argmax(want, axis=1)), (m.source, path)
        e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["fc", "binary160", "cnn_48"])
def test_labels_only_and_logits_only(lib, name):
    m = load_model(name)
    g = np.load(os.path.join(GOLDEN, "emulator.npz"))
    x = np.concatenate([g["images"]] * 20)
    e = engine(m)
    full, lab = run_emulator(e, x)
    lo, la = run_emulator(e, x, want_logits=False)
    assert lo is None and np.array_equal(la, lab)
    lo, la = run_emulator(e, x, want_labels=False)
    assert la is None and np.array_equal(lo, full)
    assert np.array_equal(full[:64], g[name])
    e.close()


@pytest.mark.gpu
def test_argument_errors(lib):
    import torch
    e = engine(load_model("fc"))
    h, n = e.handle, 300
    d_x = torch.zeros((n + 1, 256), dtype=torch.float32, device="cuda")
    d_lo = torch.zeros((n + 1, 10), dtype=torch.float64, device="cuda")
    d_la = torch.zeros(n, dtype=torch.int32, device="cuda")
    xp, lop, lap = C.c_void_p(d_x.data_ptr()), C.c_void_p(d_lo.data_ptr()), C.c_void_p(d_la.data_ptr())
    assert lib.bnm_emulate_batch_device(h, xp, n, None, None, None) == -1
    assert b"no output" in lib.bnm_last_error()
    assert lib.bnm_emulate_batch_device(h, C.c_void_p(d_x.data_ptr() + 4), n, lop, lap, None) == -1     # images not 16-byte aligned
    assert lib.bnm_emulate_batch_device(h, xp, n, C.c_void_p(d_lo.data_ptr() + 4), lap, None) == -1    # logits not 8-byte aligned
    assert lib.bnm_emulate_batch_device(h, None, n, lop, lap, None) == -1
    assert lib.bnm_emulate_batch_device(h, None, 0, None, None, None) == 0                              # n = 0: nothing to do
    assert lib.bnm_emulate_batch_device(h, xp, 0, lop, lap, None) == 0
    torch.cuda.synchronize()
    assert not d_lo.any() and not d_la.any()
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["fc", "cnn_48"])
def test_non_default_stream(lib, name):
    """images made on a side stream and the call on that stream: ordered by it alone"""
    import torch
    m = load_model(name)
    n = 148 * 128 * 3 + 5
    x = normal_images(n, seed=3)
    want = emulate_fc(m, x) if m.model_class == 0 else None
    e = engine(m)
    h_x = torch.from_numpy(x).pin_memory()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        d_x = torch.empty((n, 256), dtype=torch.float32, device="cuda")
        d_x.copy_(h_x, non_blocking=True)
        d_x.mul_(1.0)
        lo = torch.empty((n, m.n_classes), dtype=torch.float64, device="cuda")
        la = torch.empty(n, dtype=torch.int32, device="cuda")
        e.inference_quantized_device(d_x, lo, la)
    s.synchronize()
    got = lo.cpu().numpy()
    if want is None:
        want = e.inference_quantized(x)
    assert np.array_equal(got, want) and np.array_equal(la.cpu().numpy(), np.argmax(want, axis=1))
    e.close()


@pytest.mark.gpu
def test_verbose_names_emulator_kernel(lib, capfd, monkeypatch):
    e, fused = _fused_engine(capfd, monkeypatch, load_model("fc"))
    assert fused
    e.close()
    e, fused = _fused_engine(capfd, monkeypatch, load_model("binary160"))
    assert not fused
    e.close()


def _host_module(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, "host", name + ".py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["fc", "ternary64"])
def test_driver_emulator_lines(lib, oracle, which):
    """host/evaluate_engines.py: the three lines of the C-engine driver unchanged, then the emulator's counters"""
    m = load_model(which)
    x = normal_images(4000, seed=21)
    labels = np.random.default_rng(5).integers(0, 10, size=4000)
    lines, c_lines = [], []
    res = _host_module("evaluate_engines").evaluate(m, x, labels, out=lines.append)
    _host_module("test_inference_batched").evaluate(m, x, labels, out=c_lines.append)
    py = np.argmax(emulate_fc(m, x), axis=1)
    _, c = oracle.infer(m, res["quantized"])
    wrong_py, mism = int((py != labels).sum()), int((py != c.astype(np.int64)).sum())
    assert lines[:3] == c_lines and lines[0] == "size of test data: 4000"
    assert lines[3] == f"Mispredictions Py: {wrong_py}"
    assert lines[4] == f"Overall accuracy Python: {(4000 - wrong_py) / 4000 * 100} %"
    assert lines[5] == f"Mismatches between engines: {mism} ({mism / 4000 * 100}%)"
    assert np.array_equal(res["predicted_py"], py)
