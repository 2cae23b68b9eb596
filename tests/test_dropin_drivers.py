"""The library as a link-time drop-in for the reference (INTEGRATION.md sections 1 and 2), against the unmodified reference.

oracle/Makefile builds the reference's own drivers twice, once on the reference kernels and once on the library's
reference-named symbols (processfclayer, ReLUNorm, processconv33ReLU, processmaxpool22), which run one item per call on the
GPU from host pointers:
  _ref/libbitnetmcu_ref.so / libbitnetmcu_dropin.so   oracle/ref_driver.c, int32 logits for any layer table
  _ref/dll_<model>/ref.so / dropin.so                 BitNetMCU_MNIST_dll.c itself, for every model dropin_headers.py lists
  _ref/mnist_test_{fc,cnn}_dropin                     BitNetMCU_MNIST_test.c on the library
The tests compare the two builds of each driver at tolerance 0, run the C shim of host/ (bnm_model_create from a header) on
the same headers, and call the four symbols, single-item and batched, at the parameters the drivers never use, against the
reference's own symbols in libbitnetmcu_ref.so.  They skip only where oracle/_ref lacks the builds, as the `reference`
fixture does."""
import ctypes as C
import os
import re
import subprocess
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from conftest import GOLDEN, ROOT, load_model, model_names, xorshift_images
from oracle import dropin_headers as DH
from support import build_c_shim, cnn_model, lib

REF_DIR = os.path.join(ROOT, "oracle", "_ref")
FC_KERNELS = {"processfclayer", "ReLUNorm"}
KERNELS = FC_KERNELS | {"processconv33ReLU", "processmaxpool22"}
DLL_MODELS = DH.dll_models()
ENCODINGS = [1, 2, 4, 12, 16, 20, 36, 64]
UNKNOWN_ENC = 3          # no branch of inference.c:96-202 takes it: zeros
INT32_MIN = np.iinfo(np.int32).min
INT32_MAX = np.iinfo(np.int32).max


def _ref_path(*parts):
    p = os.path.join(REF_DIR, *parts)
    if not os.path.exists(p):
        pytest.skip(f"oracle/_ref/{'/'.join(parts)} not built (the reference sources were absent at build time)")
    return p


def _symbols(path, flag):
    out = subprocess.run(["nm", "-D", flag, path], capture_output=True, text=True, check=True).stdout
    return {l.split()[-1].split("@")[0] for l in out.splitlines() if l.strip()}


def _kernels_of(name):
    return KERNELS if load_model(name).model_class == 1 else FC_KERNELS


def _set_kernel_types(dll):
    vp, u32 = C.c_void_p, C.c_uint32
    for fn, res, args in (("ReLUNorm", u32, [vp, vp, u32]), ("processfclayer", None, [vp, vp, C.c_int32, u32, u32, vp]),
                          ("processconv33ReLU", vp, [vp, vp, u32, u32, vp]), ("processmaxpool22", vp, [vp, u32, vp])):
        f = getattr(dll, fn)
        f.restype, f.argtypes = res, args
    return dll


def _ptr(a):
    return C.c_void_p(a.ctypes.data)


# ---- models and images --------------------------------------------------------------------------------------------------

def _random_model(enc, widths, seed):
    """pack.random_fc_model for an encoding id; the unknown id keeps 4bitsym-sized weight arrays"""
    from bitnetmcu_b200 import pack as P
    m = P.random_fc_model(4 if enc == UNKNOWN_ENC else enc, widths, seed=seed)
    if enc == UNKNOWN_ENC:
        for l in m.layers:
            l.bitperweight = UNKNOWN_ENC
    return m


CHAIN8 = (256, 96, 64, 32, 160, 64, 128, 32, 10)   # eight layers, every width a whole number of words in every encoding


def _random_widths(enc):
    # the layer kernel's shared-memory bound; Ternary rows pad to tens, Binary rows to 32 weights
    wide = {64: (1790, 16, 10), 1: (1792, 32, 10)}.get(enc, (1792, 16, 10))
    return [(256, 64, 10), (256, 320, 257), wide, CHAIN8]


SHARED_MODELS = ([(f"fixture-{n}", (lambda n=n: load_model(n))) for n in model_names()]
                 + [(f"enc{e}-{'x'.join(map(str, w))}", (lambda e=e, w=w, i=i: _random_model(e, w, seed=100 * e + i)))
                    for e in ENCODINGS + [UNKNOWN_ENC] for i, w in enumerate(_random_widths(e))]
                 + [(f"cnn{c}", (lambda c=c: cnn_model(c, 10, seed=c))) for c in (8, 24, 144, 256)])


def _images(img_bytes, n, seed):
    """the ten digits (256-byte rows), the xorshift stream, the rails -128, 127 and alternating, then uniform noise"""
    rows = [np.load(os.path.join(GOLDEN, "digits.npz"))["images"]] if img_bytes == 256 else []
    rows += [xorshift_images(max(n // 2, 1), img_bytes),
             np.full((1, img_bytes), -128), np.full((1, img_bytes), 127), np.where(np.arange(img_bytes) % 2, -128, 127)[None]]
    have = sum(r.shape[0] for r in rows)
    rows.append(np.random.default_rng(seed).integers(-128, 128, size=(max(n - have, 1), img_bytes)))
    return np.ascontiguousarray(np.concatenate(rows).astype(np.int8))


# ---- CPU: the builds and the headers --------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", DLL_MODELS)
def test_dll_builds_leave_the_kernels_to_the_library(built, name):
    """dll.c on the stub leaves exactly the kernels it calls undefined, resolved in libbitnetmcu_b200.so; on the reference
    kernels it defines them (FC models: processfclayer and ReLUNorm, inference.c:210 keeps conv and pool out)"""
    from bitnetmcu_b200 import _lib
    exported = _symbols(_lib.LIB_PATH, "--defined-only")
    assert KERNELS <= exported
    dropin, ref = _ref_path(f"dll_{name}", "dropin.so"), _ref_path(f"dll_{name}", "ref.so")
    assert _symbols(dropin, "--undefined-only") & exported == _kernels_of(name)
    assert not _symbols(dropin, "--defined-only") & KERNELS
    assert _kernels_of(name) <= _symbols(ref, "--defined-only")
    assert "Inference" in _symbols(dropin, "--defined-only") and "Inference" in _symbols(ref, "--defined-only")
    libs = subprocess.run(["ldd", dropin], capture_output=True, text=True).stdout
    assert "libbitnetmcu_b200.so" in libs and "not found" not in libs, libs


def test_shared_driver_and_test_programs_leave_the_kernels_to_the_library(built):
    from bitnetmcu_b200 import _lib
    exported = _symbols(_lib.LIB_PATH, "--defined-only")
    shared = os.path.join(REF_DIR, "libbitnetmcu_dropin.so")
    assert os.path.exists(shared), "build() makes the shared driver on the library, with or without the reference"
    assert _symbols(shared, "--undefined-only") & exported == KERNELS
    assert not _symbols(shared, "--defined-only") & KERNELS
    assert KERNELS <= _symbols(_ref_path("libbitnetmcu_ref.so"), "--defined-only")
    for name in ("fc", "cnn"):
        assert _symbols(_ref_path(f"mnist_test_{name}_dropin"), "--undefined-only") & exported == _kernels_of(name)


@pytest.mark.parametrize("name", DH.FC_MODELS + DH.CNN_MODELS)
def test_generated_headers_parse_back(tmp_path, name):
    """write_header's header of each model parses back to its layers and weights, and sizes dll.c's stack buffers for every
    layer (MAX_N_ACTIVATIONS: 16x16 int32 scratch, the CNN features, every layer's inputs and outputs)"""
    from bitnetmcu_b200.model import parse_header
    from bitnetmcu_b200.pack import write_header
    m = load_model(name)
    path = str(tmp_path / "BitNetMCU_model.h")
    write_header(m, path)
    built_hdr = os.path.join(REF_DIR, f"hdr_{name}", "BitNetMCU_model.h")
    if name in DLL_MODELS and os.path.exists(built_hdr):
        assert open(built_hdr).read() == open(path).read()
    got = parse_header(path)
    assert got.model_class == m.model_class and len(got.layers) == len(m.layers)
    for a, b in zip(got.layers, m.layers):
        assert (a.kind, a.name, a.bitperweight, a.n_in, a.n_out) == (b.kind, b.name, b.bitperweight, b.n_in, b.n_out)
        assert (a.weights is None) == (b.weights is None)
        if b.weights is not None:
            assert a.weights.dtype == b.weights.dtype and np.array_equal(a.weights, b.weights), a.name
    if m.model_class == 1:
        assert (got.layers[0].in_channels, got.layers[1].groups) == (m.layers[0].in_channels, m.layers[1].groups)
    text = open(path).read()
    if any(l.bitperweight == 64 for l in m.fc_layers):
        assert re.search(r"const uint16_t L\d+_weights\[\]", text)
    if m.model_class == 0:   # dll.c:111 runs the fourth layer behind L4_active
        assert ("#define L4_active" in text) == (len(m.layers) == 4)
    max_act = int(re.search(r"#define MAX_N_ACTIVATIONS (\d+)", text).group(1))
    assert max_act >= max([256, 4 * m.channels] + [l.n_in for l in m.fc_layers] + [l.n_out for l in m.fc_layers])


def _reads_undefined(m):
    """restated: a Ternary layer's non-zero trit at a column past the bytes dll.c defines for that layer (the 256-byte
    image, then the previous layer's n_out)"""
    from bitnetmcu_b200 import pack as P
    width = 256 if m.model_class == 0 else 1 << 30
    for l in m.fc_layers:
        if l.bitperweight == 64:
            t = P.decode_int_weights(l)
            if np.any(t[:, width:] != 0):
                return True
        width = l.n_out
    return False


def test_ternary_pad_trit_exclusion_rule():
    """rand_ternary64 (and any other fixture) goes through dll.c exactly when no Ternary layer has a non-zero trit past its
    defined input; a trit set there excludes the model"""
    from bitnetmcu_b200 import pack as P
    cands = DH.FC_MODELS + DH.CNN_MODELS
    assert set(cands) <= set(model_names())
    for name in cands:
        assert DH.reads_past_its_input(load_model(name)) == _reads_undefined(load_model(name)), name
    assert DLL_MODELS == [n for n in cands if not _reads_undefined(load_model(n))]
    assert "rand_ternary64" in DLL_MODELS and "ternary64" in DLL_MODELS   # their pad trits (64..69, 256..259) are zero
    for layer, col in ((0, 257), (1, 64), (3, 69)):
        m = load_model("rand_ternary64")
        l = m.layers[layer]
        t = P.decode_int_weights(l)
        t[3, col] = -1
        m.layers[layer] = P.fc_layer_from_trits(l.name, t)
        assert DH.reads_past_its_input(m) and _reads_undefined(m), (layer, col)


@pytest.mark.parametrize("name", DLL_MODELS)
def test_c_shim_compiles_on_every_header(built, tmp_path, name):
    dll, _, _ = build_c_shim(str(tmp_path), name)
    assert {"Inference", "InferenceBatch", "InferenceNumClasses"} <= _symbols(dll, "--defined-only")


# ---- GPU 1: the shared driver, logits ------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def drivers(built):
    from oracle.oracle import Reference
    return Reference(_ref_path("libbitnetmcu_ref.so")), Reference(_ref_path("libbitnetmcu_dropin.so"))


@pytest.mark.gpu
@pytest.mark.parametrize("name,make", SHARED_MODELS, ids=[n for n, _ in SHARED_MODELS])
def test_shared_driver_logits(lib, drivers, name, make):
    """ref_driver.c on the library equals it on the reference kernels: int32 logits and labels, one thread (and eight on
    fc and cnn: concurrent single-item calls)"""
    ref, dropin = drivers
    m = make()
    imgs = _images(m.img_bytes, 40 if m.model_class == 1 else 300, seed=len(name))
    want_lo, want_la = ref.infer(m, imgs, threads=1)
    for threads in ((1, 8) if name in ("fixture-fc", "fixture-cnn") else (1,)):
        t0 = time.perf_counter()
        lo, la = dropin.infer(m, imgs, threads=threads)
        dt = time.perf_counter() - t0
        print(f"{name}: {imgs.shape[0]} images, {threads} threads: {1e3 * dt / imgs.shape[0]:.2f} ms per image")
        bad = np.flatnonzero((lo != want_lo).any(axis=1))
        assert bad.size == 0, (name, threads, f"{bad.size} rows differ, first {bad[:5].tolist()}")
        assert np.array_equal(la, want_la), (name, threads)


# ---- GPU 2: the reference's own dll.c ----------------------------------------------------------------------------------------

def _inference(path):
    dll = C.CDLL(path)
    dll.Inference.restype, dll.Inference.argtypes = C.c_uint32, [C.c_void_p]
    return dll


def _labels(dll, imgs, threads=1):
    one = lambda i: dll.Inference(_ptr(imgs[i]))
    if threads == 1:
        return np.array([one(i) for i in range(imgs.shape[0])], dtype=np.uint32)
    with ThreadPoolExecutor(threads) as ex:   # ctypes drops the GIL: the calls overlap
        return np.array(list(ex.map(one, range(imgs.shape[0]))), dtype=np.uint32)


@pytest.mark.gpu
@pytest.mark.parametrize("name", DLL_MODELS)
def test_reference_dll_on_the_library(lib, golden, name):
    """Inference() of dll.c on the library equals Inference() of dll.c on the reference kernels and golden.npz's labels"""
    ref = _inference(_ref_path(f"dll_{name}", "ref.so"))
    dropin = _inference(_ref_path(f"dll_{name}", "dropin.so"))
    cnn = load_model(name).model_class == 1
    n_xs = 24 if cnn else 256
    imgs = _images(256, n_xs * 2, seed=7)
    want = _labels(ref, imgs)
    assert np.array_equal(want[:10], golden[name + "/digits_labels"])
    assert np.array_equal(want[10:10 + n_xs], golden[name + "/xs_labels"][:n_xs])
    for threads in ((1, 8) if name in ("fc", "cnn") else (1,)):
        t0 = time.perf_counter()
        got = _labels(dropin, imgs, threads)
        dt = time.perf_counter() - t0
        print(f"dll.c {name}: {imgs.shape[0]} Inference() calls, {threads} threads: {1e3 * dt / imgs.shape[0]:.2f} ms per call")
        assert np.array_equal(got, want), (name, threads, np.flatnonzero(got != want)[:8].tolist())


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["fc", "cnn"])
def test_reference_test_program_on_the_library(lib, digits, name):
    exe = _ref_path(f"mnist_test_{name}_dropin")
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300).stdout
    _, labels = digits
    assert out == "".join(f"label: {int(l)} predicted: {int(l)}\n" for l in labels)


# ---- GPU 3: the C shim of host/ on every header ------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("name", DLL_MODELS)
def test_c_shim_on_every_header(lib, reference, golden, digits, tmp_path, name):
    """host/bitnetmcu_b200_dll.c built on each header: InferenceBatch logits and labels equal golden.npz and the Reference,
    Inference() labels, InferenceNumClasses"""
    m = load_model(name)
    path, _, _ = build_c_shim(str(tmp_path), name)
    dll = C.CDLL(path)
    dll.Inference.restype, dll.Inference.argtypes = C.c_uint32, [C.c_void_p]
    dll.InferenceBatch.restype, dll.InferenceBatch.argtypes = C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
    dll.InferenceNumClasses.restype = C.c_uint32
    assert dll.InferenceNumClasses() == m.n_classes

    def batch(imgs):
        lo = np.full((imgs.shape[0], m.n_classes), -7, dtype=np.int32)
        la = np.full(imgs.shape[0], 999, dtype=np.uint32)
        assert dll.InferenceBatch(_ptr(imgs), imgs.shape[0], _ptr(lo), _ptr(la)) == 0
        return lo, la
    imgs, _ = digits
    lo, la = batch(np.ascontiguousarray(imgs))
    assert np.array_equal(lo, golden[name + "/digits_logits"]) and np.array_equal(la, golden[name + "/digits_labels"])
    xs = xorshift_images(256)
    lo, la = batch(xs)
    assert np.array_equal(lo, golden[name + "/xs_logits"]) and np.array_equal(la, golden[name + "/xs_labels"])
    r = _images(256, 700, seed=11)
    want_lo, want_la = reference.infer(m, r)
    lo, la = batch(r)
    assert np.array_equal(lo, want_lo) and np.array_equal(la, want_la)
    assert np.array_equal(_labels(dll, r[:40]), want_la[:40])


# ---- GPU 4: the four symbols at the parameters the drivers skip -------------------------------------------------------------

@pytest.fixture(scope="module")
def ref_kernels(built):
    return _set_kernel_types(C.CDLL(_ref_path("libbitnetmcu_ref.so")))


@pytest.mark.gpu
def test_conv33relu_every_shift_and_size(lib, ref_kernels):
    """processconv33ReLU in place with its end pointer, and bnm_conv33relu_batch, at every n_shift 0..15 and 31 and odd and
    even sizes, on activations up to +-2^20 (no int32 sum overflows)"""
    from bitnetmcu_b200 import engine as E
    rng = np.random.default_rng(5)
    for xy in (3, 4, 5, 7, 16, 17, 32):
        o = (xy - 2) ** 2
        for n_shift in list(range(16)) + [31]:
            act = rng.integers(-(1 << 20), (1 << 20) + 1, size=(6, xy * xy)).astype(np.int32)
            act[1] = np.abs(act[1])                       # positive sums: the shift decides every output
            act[2] = rng.integers(-128, 128, size=xy * xy)
            w = rng.integers(-128, 128, size=(3, 9)).astype(np.int8)
            w[0] = np.where(w[0] < 0, -128, 127)
            want = []
            for i in range(act.shape[0]):
                ref_buf, buf = act[i].copy(), act[i].copy()
                ref_kernels.processconv33ReLU(_ptr(ref_buf), _ptr(w[i % 3]), xy, n_shift, _ptr(ref_buf))
                end = lib.processconv33ReLU(_ptr(buf), _ptr(w[i % 3]), xy, n_shift, _ptr(buf))
                assert end == buf.ctypes.data + 4 * o, (xy, n_shift)
                assert np.array_equal(buf, ref_buf), (xy, n_shift, i)   # the tail past the output stays as it was
                want.append(ref_buf[:o])
            got = E.conv33relu(act, w, xy, n_shift)
            assert np.array_equal(got, np.stack(want)), (xy, n_shift)


@pytest.mark.gpu
def test_maxpool22_every_size(lib, ref_kernels):
    """processmaxpool22 in place with its end pointer, and bnm_maxpool22_batch, at odd (floored) and even sizes 2..33 on
    negative and full-range inputs"""
    from bitnetmcu_b200 import engine as E
    rng = np.random.default_rng(6)
    for xy in range(2, 34):
        o = (xy // 2) ** 2
        act = rng.integers(INT32_MIN, 1 << 31, size=(5, xy * xy), dtype=np.int64).astype(np.int32)
        act[1] = -np.abs(rng.integers(1, 1 << 20, size=xy * xy))
        act[2, ::3] = INT32_MIN
        act[3] = INT32_MIN
        act[3, -1] = 5                                   # the last row and column: read by no window of an odd size
        want = []
        for i in range(act.shape[0]):
            ref_buf, buf = act[i].copy(), act[i].copy()
            ref_kernels.processmaxpool22(_ptr(ref_buf), xy, _ptr(ref_buf))
            end = lib.processmaxpool22(_ptr(buf), xy, _ptr(buf))
            assert end == buf.ctypes.data + 4 * o, xy
            assert np.array_equal(buf, ref_buf), (xy, i)
            want.append(ref_buf[:o])
        assert np.array_equal(E.maxpool22(act, xy), np.stack(want)), xy


def _relunorm_rows(n, rng):
    """rows of n int32: random, maxima at 2^k*128 - 1 and 2^k*128 for every k, first-max ties either side of position 255,
    all zero, all negative, then three rows no element of which beats the search's start, -INT32_MAX (position 255): all
    INT32_MIN, all -INT32_MAX, and the two mixed"""
    rows = [rng.integers(-(1 << 20), 1 << 20, size=n)]
    for k in range(24):
        for top in ((128 << k) - 1, 128 << k):
            r = rng.integers(-top, top, size=n)
            r[rng.integers(0, n)] = top
            rows.append(r)
    for a, b in ((254, 256), (255, 256), (10, 255), (256, 300), (0, n - 1), (255, n - 1)):
        if a < b < n:
            r = rng.integers(-1000, 1000, size=n)
            r[a] = r[b] = 5000
            rows.append(r)
    rows += [np.zeros(n), -np.abs(rng.integers(1, 1 << 30, size=n)), np.where(np.arange(n) % 2, INT32_MIN, -1)]
    rows += [np.full(n, INT32_MIN), np.full(n, -INT32_MAX), np.where(np.arange(n) % 3 == 1, -INT32_MAX, INT32_MIN)]
    return np.stack(rows).astype(np.int32)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [0, 1, 255, 256, 257, 1024])
def test_relunorm_edges(lib, ref_kernels, n):
    """ReLUNorm and bnm_relunorm_batch against the reference: argmax (first maximum, 255 when nothing beats -INT32_MAX) and the
    int8 outputs, and dll.c:80's call with an int32 buffer as its own int8 output"""
    from bitnetmcu_b200 import engine as E
    rng = np.random.default_rng(n)
    x = _relunorm_rows(max(n, 1), rng)[:, :n]
    want_out = np.zeros(x.shape, dtype=np.int8)
    want_pos = np.zeros(x.shape[0], dtype=np.uint32)
    for i in range(x.shape[0]):
        row = x[i].copy()
        want_pos[i] = ref_kernels.ReLUNorm(_ptr(row), _ptr(want_out[i]), n)
        out = np.full(n, 99, dtype=np.int8)
        assert lib.ReLUNorm(_ptr(row), _ptr(out), n) == want_pos[i], (n, i)
        assert np.array_equal(out, want_out[i]), (n, i)
        alias, ref_alias = x[i].copy(), x[i].copy()   # int32 input, int8 output over its first n bytes
        assert ref_kernels.ReLUNorm(_ptr(ref_alias), _ptr(ref_alias), n) == want_pos[i]
        assert lib.ReLUNorm(_ptr(alias), _ptr(alias), n) == want_pos[i], (n, i, "aliased")
        assert np.array_equal(alias, ref_alias), (n, i, "aliased")
    if n:
        assert (want_pos[-3:] == 255).all(), "nothing beats -INT32_MAX: position 255"
        out, pos = E.relunorm(x)
        assert np.array_equal(pos, want_pos) and np.array_equal(out, want_out), n


def _fc_weights(enc, n_in, n_out, rng):
    if enc == 64:
        return rng.integers(0, 1 << 16, size=n_out * (n_in // 10), dtype=np.uint32).astype(np.uint16)
    per = {1: 32, 2: 16, 16: 4}.get(enc, 8)
    return rng.integers(0, 1 << 32, size=n_out * (n_in // per), dtype=np.uint64).astype(np.uint32)


@pytest.mark.gpu
@pytest.mark.parametrize("enc", ENCODINGS + [UNKNOWN_ENC])
def test_processfclayer_every_width(lib, ref_kernels, enc):
    """processfclayer and bnm_processfclayer_batch at n_input 32..1792 (Ternary 40..1790) and n_output 1, 64 and 300, on
    random words (every bit pattern is a weight)"""
    from bitnetmcu_b200 import engine as E
    rng = np.random.default_rng(enc)
    widths = (40, 70, 260, 320, 1000, 1790) if enc == 64 else (32, 64, 96, 160, 256, 320, 512, 1024, 1792)
    for n_in in widths:
        for n_out in (1, 64, 300):
            w = _fc_weights(enc, n_in, n_out, rng)
            act = rng.integers(-128, 128, size=(4, n_in)).astype(np.int8)
            act[1] = 127
            act[2] = -128
            want = np.zeros((act.shape[0], n_out), dtype=np.int32)
            for i in range(act.shape[0]):
                ref_kernels.processfclayer(_ptr(act[i]), _ptr(w), enc, n_in, n_out, _ptr(want[i]))
            got = np.full(n_out, -7, dtype=np.int32)
            lib.processfclayer(_ptr(act[0]), _ptr(w), enc, n_in, n_out, _ptr(got))
            assert np.array_equal(got, want[0]), (enc, n_in, n_out)
            assert np.array_equal(E.processfclayer(act, w, enc, n_in, n_out), want), (enc, n_in, n_out)
            if enc in (36, UNKNOWN_ENC):
                assert not want.any()


@pytest.mark.gpu
def test_processfclayer_ternary_pad_bytes_are_never_read(lib, ref_kernels):
    """a Ternary first layer declares 260 inputs with zero pad trits; dll.c hands it a 256-byte image.  Bytes 256..259 of the
    row, 127 here, must not change the result, single-item or batched"""
    from bitnetmcu_b200 import engine as E
    from bitnetmcu_b200 import pack as P
    rng = np.random.default_rng(260)
    for n_out in (1, 64, 300):
        w, n_in = P.pack_ternary(rng.integers(-1, 2, size=(n_out, 256)))
        assert n_in == 260
        act = np.zeros((3, 260), dtype=np.int8)
        act[:, :256] = rng.integers(-128, 128, size=(3, 256))
        want = np.zeros((3, n_out), dtype=np.int32)
        for i in range(3):
            ref_kernels.processfclayer(_ptr(act[i]), _ptr(w), 64, 260, n_out, _ptr(want[i]))
        act[:, 256:] = 127
        got = np.zeros(n_out, dtype=np.int32)
        lib.processfclayer(_ptr(act[0]), _ptr(w), 64, 260, n_out, _ptr(got))
        assert np.array_equal(got, want[0]), n_out
        assert np.array_equal(E.processfclayer(act, w, 64, 260, n_out), want), n_out
