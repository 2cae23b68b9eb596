"""Top-k (include/bitnetmcu_b200.h section 8): each image's k best classes and their scores, from the C engine and the emulator,
on every route -- fc_topk_kernel's epilogue (fc_wgmma.cu), k_topk_rows behind BNM_PATH_LAYERS and models without a fused plan
(generic_kernels.cu), and the host pipeline.

The contract: the classes of a row ranked by logit, highest first, ties to the lower class (np.argsort(-x, kind="stable")); rank 0
is the label of the matching entry; the scores are the logits at those classes (int32 for the C engine, the emulator's float64
logits for the emulator); nothing is written for n == 0; bad k, a NULL classes buffer and misaligned buffers are BNM_E_ARG.

CPU: the restatement (topk_order below) against argsort, the oracle's ReLUNorm argmax and np.argmax on the golden logits, crafted
tie rows, the exported symbols.  GPU (tolerance 0): every fixture model, crafted integer-weight models at every width whose rows
tie across quad lanes, 16-column blocks and 64-column pieces, are all negative or lie on both sides of +-2^23, batches that take
every stage of every top-k form through three ring rounds, every route read from its `topk route:` line, and the argument
checks; the top-k line of host/evaluate_topk.py."""
import ctypes as C
import importlib.util
import os
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, load_model, model_names, xorshift_images
from restate import TILE, emulate, emulate_fc, scale_images
from support import Sweep, engine, frontends, lib, random_fc, verbose_engine

ENC_8BIT = 16
MAX_TOPK = 16
BNM_E_ARG = -1
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def topk_order(x, k):
    """the order of the top-k entries (include/bitnetmcu_b200.h section 8) on rows x [n, C] -> (classes int64 [n, k], their
    values [n, k]), restated as the kernels run it: k rounds of a first-maximum scan, round t over the columns ranked after round
    t - 1's pick (v, p) -- x < v, or x == v at a column > p"""
    x = np.asarray(x)
    n, c = x.shape
    xf = x.astype(np.float64)           # int32 logits are exact in float64
    cols = np.arange(c)
    v = np.full(n, np.inf)
    p = np.full(n, -1)
    classes = np.empty((n, k), dtype=np.int64)
    for t in range(k):
        cand = (xf < v[:, None]) | ((xf == v[:, None]) & (cols > p[:, None]))
        p = np.argmax(np.where(cand, xf, -np.inf), axis=1)     # first maximum among the candidates
        v = xf[np.arange(n), p]
        classes[:, t] = p
    return classes, np.take_along_axis(x, classes, axis=1)


def ks(c):
    return sorted({1, 2, 3, min(c, MAX_TOPK)} & set(range(1, min(c, MAX_TOPK) + 1)))


# ---- CPU -------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("c", [1, 2, 3, 10, 16, 17, 37, 64, 65, 256])
def test_restated_order_is_stable_argsort(c):
    rng = np.random.default_rng(c)
    for x in (rng.integers(-3, 4, size=(400, c)), rng.integers(-2 ** 25, 2 ** 25, size=(400, c)),
              rng.integers(-3, 4, size=(400, c)) * 0.5):
        want = np.argsort(-x, kind="stable", axis=1)
        for k in (range(1, c + 1) if c <= 17 else sorted({1, 2, 3, MAX_TOPK, c // 2, c})):
            cls, val = topk_order(x, k)
            assert np.array_equal(cls, want[:, :k]), (c, k)
            assert np.array_equal(val, np.take_along_axis(x, want[:, :k], axis=1))


def test_rank0_is_the_oracle_argmax_on_golden_logits(oracle, golden):
    """rank 0 of every fixture's golden logits is the oracle's ReLUNorm argmax (inference.c:32-37), i.e. the stored label"""
    names = [k[: -len("_logits")] for k in golden if k.endswith("_logits")]
    assert len(names) >= 2 * len(model_names())
    for name in names:
        x = golden[name + "_logits"]
        cls, _ = topk_order(x, min(x.shape[1], MAX_TOPK))
        assert np.array_equal(cls[:, 0], [oracle.relunorm(r)[1] for r in x]), name
        assert np.array_equal(cls[:, 0], golden[name + "_labels"]), name


def test_rank0_is_np_argmax_on_emulator_golden():
    z = np.load(os.path.join(GOLDEN, "emulator.npz"))
    for name in (k for k in z.files if k != "images"):
        cls, val = topk_order(z[name], min(z[name].shape[1], MAX_TOPK))
        assert np.array_equal(cls[:, 0], np.argmax(z[name], axis=1)), name
        assert np.array_equal(val[:, 0], z[name].max(axis=1))


def test_crafted_tie_rows():
    rows = np.array([[5, 5, 5, 5, 5],          # all equal: class order
                     [1, 7, 3, 7, 0],          # a pair at the top
                     [9, 2, 9, 4, 9],          # three-way with the last class
                     [-4, -1, -9, -1, -2],     # all negative, a tied pair
                     [0, -1, 0, -1, 0]])
    cls, val = topk_order(rows, 5)
    assert cls.tolist() == [[0, 1, 2, 3, 4], [1, 3, 2, 0, 4], [0, 2, 4, 3, 1], [1, 3, 4, 0, 2], [0, 2, 4, 1, 3]]
    assert np.array_equal(val, np.take_along_axis(rows, cls, axis=1))


def test_library_exports_the_topk_entries():
    from bitnetmcu_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("library not built")
    out = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    exported = {l.split()[-1] for l in out.splitlines() if " T " in l}
    for name in ("bnm_infer_topk", "bnm_infer_topk_device", "bnm_infer_topk_device_f32", "bnm_emulate_topk_device"):
        assert name in exported, name


# ---- GPU helpers -------------------------------------------------------------------------------------------------------------

def _topk(e, fn, x, k, scores=True, stream=None):
    """one device top-k call of the engine (fn: "int8", "f32" or "emul") on x (NumPy or CUDA tensor) -> (classes, scores) as NumPy"""
    import torch
    d_x = x if isinstance(x, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(x)).cuda()
    n = d_x.shape[0]
    cls = torch.full((n, k), -1, dtype=torch.int32, device="cuda")
    sc = None
    if scores:
        sc = torch.full((n, k), np.nan, dtype=torch.float64, device="cuda") if fn == "emul" else \
            torch.full((n, k), -7, dtype=torch.int32, device="cuda")
    {"int8": e.topk_device, "f32": e.topk_device_f32, "emul": e.emulate_topk_device}[fn](d_x, k, cls, sc, stream=stream)
    torch.cuda.synchronize()
    return cls.cpu().numpy().astype(np.int64), (sc.cpu().numpy() if scores else None)


def _check(got, logits, k, what, labels=None):
    """(classes, scores) equal the logits ranked by the restatement; rank 0 equals the labels of the matching entry"""
    cls, sc = got
    want_c, want_s = topk_order(logits, k)
    bad = np.flatnonzero((cls != want_c).any(axis=1))
    assert bad.size == 0, (what, k, f"{bad.size} rows wrong, first {bad[:4].tolist()}", cls[bad[:2]], want_c[bad[:2]], logits[bad[:1]])
    if sc is not None:
        assert np.array_equal(sc, want_s), (what, k, "scores")
        assert np.array_equal(sc, np.take_along_axis(logits, cls, axis=1)), (what, k, "scores gathered")
    if labels is not None:
        assert np.array_equal(cls[:, 0], labels), (what, k, "rank 0 vs label")


def _device_logits(e, x, fn):
    """the existing entry's logits and labels: bnm_infer_batch_device (int8), _f32, or bnm_emulate_batch_device (emul)"""
    import torch
    d_x = torch.from_numpy(np.ascontiguousarray(x)).cuda()
    n = d_x.shape[0]
    la = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    if fn == "emul":
        lo = torch.full((n, e.n_classes), np.nan, dtype=torch.float64, device="cuda")
        e.inference_quantized_device(d_x, lo, la)
    else:
        lo = torch.full((n, e.n_classes), -7, dtype=torch.int32, device="cuda")
        (e.infer_device if fn == "int8" else e.infer_device_f32)(d_x, lo, la)
    torch.cuda.synchronize()
    return lo.cpu().numpy(), la.cpu().numpy().astype(np.int64)


def _route_lines(capfd):
    return [l.split("topk route: ")[1] for l in capfd.readouterr().err.splitlines() if "topk route: " in l]


# ---- GPU: fixtures -------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("path", ["fused", "layers"])
@pytest.mark.parametrize("name", model_names())
def test_golden_models_topk(lib, oracle, digits, name, path):
    """the 10 digits, the xorshift images and a ragged random batch against the oracle's logits; a 2^20 batch (fused path)
    against the logits and labels of bnm_infer_batch_device on the same images"""
    from bitnetmcu_b200 import _lib
    m = load_model(name)
    rng = np.random.default_rng(len(name))
    imgs = np.concatenate([digits[0], xorshift_images(256, m.img_bytes),
                           rng.integers(-128, 128, size=(3001, m.img_bytes)).astype(np.int8)]) if m.img_bytes == 256 else \
        rng.integers(-128, 128, size=(3001, m.img_bytes)).astype(np.int8)
    want_lo, want_la = oracle.infer(m, imgs)
    big = rng.integers(-128, 128, size=((1 << 20) + 77 if path == "fused" else 0, m.img_bytes)).astype(np.int8)
    for fe in frontends(m):
        e = engine(m, _lib.PATH_LAYERS if path == "layers" else 0, fe)
        for k in ks(e.n_classes):
            for scores in (True, False):
                _check(_topk(e, "int8", imgs, k, scores), want_lo, k, (name, path, fe, scores), want_la.astype(np.int64))
        if big.shape[0]:
            lo, la = _device_logits(e, big, "int8")
            for k in (1, min(e.n_classes, MAX_TOPK)):
                _check(_topk(e, "int8", big, k), lo, k, (name, "2^20", fe), la)
        e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", model_names())
def test_golden_models_emulator_and_float_topk(lib, oracle, name):
    """the emulator's top-k against the logits and labels of bnm_emulate_batch_device (and those against the golden logits of the
    emulator where emulator.npz has them), and the float entry against the oracle on the scaled images"""
    m = load_model(name)
    e = engine(m)
    gold = np.load(os.path.join(GOLDEN, "emulator.npz"))
    x = np.concatenate([gold["images"], np.random.default_rng(3).normal(size=(1500, 256)).astype(np.float32)])
    want_py, py_la = _device_logits(e, x, "emul")
    if name in gold.files:
        assert np.array_equal(want_py[:64], gold[name]), name
    c_lo, c_la = oracle.infer(m, scale_images(x))
    for k in ks(e.n_classes):
        for scores in (True, False):
            _check(_topk(e, "emul", x, k, scores), want_py, k, (name, "emul", scores), py_la)
            _check(_topk(e, "f32", x, k, scores), c_lo, k, (name, "f32", scores), c_la.astype(np.int64))
    e.close()


# ---- GPU: crafted integer-weight models ----------------------------------------------------------------------------------------

def _fc(name, w):
    from bitnetmcu_b200 import pack as P
    return P.fc_layer_from_codes(name, ENC_8BIT, P.codes_from_int_weights(ENC_8BIT, np.asarray(w, dtype=np.int64)))


def _model(weights, img_bytes):
    from bitnetmcu_b200 import model as M
    m = M.Model(model_class=M.MODEL_FCMNIST, layers=[_fc(f"L{i + 1}", w) for i, w in enumerate(weights)], img_bytes=img_bytes)
    m.validate()
    return m


def identity_model(c, hidden=(), sign=1, img_bytes=256):
    """8bit layers: layer 1 routes pixel j to unit j, the hidden layers pass units on, the head is sign x identity on c units.
    One layer: logits = x[:c]; deeper: sign x relu(x[:c]) (ties at zero)"""
    outs, ws, n_in = list(hidden) + [c], [], img_bytes
    for l, n_out in enumerate(outs):
        w = np.zeros((n_out, n_in), dtype=np.int64)
        j = np.arange(min(n_out, n_in, c if l + 1 == len(outs) else n_out))
        w[j, j] = sign if l + 1 == len(outs) else 1
        ws.append(w)
        n_in = n_out
    return _model(ws, img_bytes)


def _pieces(c):
    """column pairs in one thread (2q / 2q+1, c / c+8), across quad lanes, 16-column blocks and 64-column pieces, the last columns"""
    cand = [(0, 1), (6, 7), (0, 8), (3, 11), (0, 2), (1, 6), (5, 10), (7, 15), (15, 16), (7, 16), (16, 32), (31, 32), (17, 49),
            (63, 64), (0, 64), (62, 65), (64, 128), (127, 128), (100, 130), (128, 192), (191, 192), (0, 192), (200, 255),
            (0, c - 1), (c - 2, c - 1), (c // 2, c - 1)]
    return sorted({(i, j) for i, j in cand if 0 <= i < j < c})


def tie_rows(c, seed):
    """crafted logit rows in [-127, 127] for c classes: all equal (positive, zero, negative); pairs and three-way ties (with the last
    class) at the top and one below it, at the place of every pair of _pieces; all negative; few distinct values.  An odd count,
    so that a batch of repeats puts every pattern on every row of a tile."""
    rng = np.random.default_rng(seed)
    rows = [np.full(c, v) for v in (100, 0, -5, -127)]
    for i, j in _pieces(c):
        for top in (127, 3, -2):
            r = rng.integers(-127, top, size=c)
            r[[i, j]] = top
            rows.append(r)
            r = r.copy()
            r[c - 1] = top
            rows.append(r)
            r = r.copy()
            r[i] = top - 1
            rows.append(r)
    rows += [-rng.integers(1, 128, size=c), -rng.integers(1, 4, size=c), rng.integers(-2, 3, size=c), rng.integers(-127, 128, size=c)]
    if len(rows) % 2 == 0:
        rows.append(rows[0])
    return np.stack(rows)


def tie_images(rows, img_bytes, n):
    """n images repeating the rows on their first pixels (random elsewhere)"""
    rng = np.random.default_rng(n)
    q = rng.integers(-127, 128, size=(n, img_bytes))
    q[:, : rows.shape[1]] = rows[np.arange(n) % rows.shape[0]]
    return q.astype(np.int8)


# (model, what): every top-k row of the fused path, class counts from 2 to 256
CRAFTED = [(c, ()) for c in (2, 3, 7, 10, 16, 17, 33, 64, 65, 100, 128, 129, 191, 192, 193, 255, 256)] + \
          [(c, (w,)) for w in (64, 128, 192, 256) for c in (2, 10, w)]


@pytest.mark.gpu
@pytest.mark.parametrize("c,hidden", CRAFTED)
def test_crafted_ties_every_row(lib, oracle, capfd, monkeypatch, c, hidden):
    """both rules, one launch of fc_topk_kernel each: the C engine against the oracle, the emulator against restate.emulate_fc"""
    for sign in ([1] if not hidden else [1, -1]):
        m = identity_model(c, hidden, sign)
        e, err = verbose_engine(capfd, monkeypatch, lambda: engine(m))
        width = -(-max((c,) + tuple(hidden)) // 64) * 64
        assert any(f"fc_topk_kernel<{width},1,topk>" in l and f"fc_topk_kernel<{width},1,emul,topk>" in l for l in err), err
        rows = tie_rows(c, seed=c + len(hidden))
        imgs = tie_images(rows * sign if hidden else rows, 256, 3 * TILE * rows.shape[0] // 2 + 5)
        want_lo, want_la = oracle.infer(m, imgs)
        x = imgs.astype(np.float32)
        want_py = emulate_fc(m, x)
        for k in ks(c):
            _check(_topk(e, "int8", imgs, k), want_lo, k, (c, hidden, sign, "C"), want_la.astype(np.int64))
            _check(_topk(e, "emul", x, k), want_py, k, (c, hidden, sign, "emul"), np.argmax(want_py, axis=1))
        e.close()


def magnitude_model(c, img_bytes=768):
    """one 8bit layer on 768-byte rows: weights -128 for the first half of the classes and -64 for the second, so that rails of
    -128 / 127 put the logits on both sides of +2^23 / -2^23; pixels 0 and 1 step by one per class (-128 + j, -128 + j // 2),
    where values one apart and ties meet at the top"""
    j = np.arange(c)
    w = -np.repeat(np.where(j < (c + 1) // 2, 128, 64)[:, None], img_bytes, axis=1).astype(np.int64)
    w[:, 0], w[:, 1] = -128 + j, -128 + j // 2
    return _model([w], img_bytes)


def magnitude_images(img_bytes, n):
    rows = []
    for base in (-128, 127):
        for x0 in (-128, -1, 0, 1, 127):
            for x1 in (-128, -1, 0, 1, 127):
                r = np.full(img_bytes, base)
                r[0], r[1] = x0, x1
                rows.append(r)
    rows.append(rows[0])
    rows = np.stack(rows)
    return rows[np.arange(n) % rows.shape[0]].astype(np.int8)


@pytest.mark.gpu
@pytest.mark.parametrize("c", [17, 32, 64])
def test_logits_past_2_23(lib, oracle, capfd, monkeypatch, c):
    """17 and 32 classes: the fused <64,1,topk> rows; 64 classes: no fused plan, k_topk_rows"""
    m = magnitude_model(c)
    e, err = verbose_engine(capfd, monkeypatch, lambda: engine(m))
    imgs = magnitude_images(768, 2 * TILE + 51)
    want_lo, want_la = oracle.infer(m, imgs)
    assert np.abs(want_lo).max() > 2 ** 23 and (np.abs(want_lo) < 2 ** 23).any()
    x = imgs.astype(np.float32)
    want_py = emulate_fc(m, x)
    for k in ks(c):
        _check(_topk(e, "int8", imgs, k), want_lo, k, (c, "C"), want_la.astype(np.int64))
        _check(_topk(e, "emul", x, k), want_py, k, (c, "emul"))
    routes = _route_lines(capfd)
    want = "fc_topk_kernel<64,1," if c <= 32 else "layer by layer + k_topk_rows"
    assert routes and all(want in r for r in routes), routes
    e.close()


# ---- GPU: ring rounds ------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("width", [64, 128, 192, 256])
def test_every_stage_three_ring_rounds(lib, oracle, capfd, monkeypatch, width):
    """batch sizes that take every stage of both top-k forms of the plan through rounds 0, 1 and 2, with a ragged last tile"""
    import re
    m = identity_model(10, (width,))
    e, err = verbose_engine(capfd, monkeypatch, lambda: engine(m))
    line = [l for l in err if "top-k forms" in l]
    assert len(line) == 1, err
    (row, st), (row_py, st_py) = re.findall(r"fc_topk_kernel(<[^>]*>) x (\d+) stages", line[0])
    rows = tie_rows(10, seed=width)
    for r, stages, fn in ((row, int(st), "int8"), (row_py, int(st_py), "emul")):
        sw = Sweep(r, (1, stages, 1))
        imgs = tie_images(rows, 256, max(sw.sizes))
        want_lo, want_la = oracle.infer(m, imgs) if fn == "int8" else (emulate_fc(m, imgs.astype(np.float32)), None)
        x = imgs if fn == "int8" else imgs.astype(np.float32)
        for n in sw.sizes:
            _check(_topk(e, fn, x[:n], 3), want_lo[:n], 3, (sw.tag, n, fn))
    e.close()


# ---- GPU: routes ---------------------------------------------------------------------------------------------------------------

def _images(n, img_bytes=256, seed=0):
    return np.random.default_rng(seed).integers(-128, 128, size=(n, img_bytes)).astype(np.int8)


@pytest.mark.gpu
@pytest.mark.parametrize("width", [64, 128, 192, 256])
def test_route_fused_fc(lib, oracle, capfd, monkeypatch, width):
    m = random_fc(4, (256, width, 37), width)
    e, _ = verbose_engine(capfd, monkeypatch, lambda: engine(m))
    imgs = _images(5000, seed=width)
    want_lo, want_la = oracle.infer(m, imgs)
    _check(_topk(e, "int8", imgs, 5), want_lo, 5, width, want_la.astype(np.int64))
    assert _route_lines(capfd) == [f"bnm_infer_topk_device: fc_topk_kernel<{width},1,topk>"]
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("frontend", [0, 1])
def test_route_cnn(lib, oracle, capfd, monkeypatch, frontend):
    m = load_model("cnn_letters")
    e, _ = verbose_engine(capfd, monkeypatch, lambda: engine(m, cnn_frontend=frontend))
    imgs = _images(3000, seed=frontend)
    want_lo, want_la = oracle.infer(m, imgs)
    _check(_topk(e, "int8", imgs, 5), want_lo, 5, frontend, want_la.astype(np.int64))
    fe = "k_cnn_frontend16_tc" if frontend == 0 and m.channels % 16 == 0 else "k_cnn_frontend16"
    assert _route_lines(capfd) == [f"bnm_infer_topk_device: {fe} + fc_topk_kernel<128,1,topk>"]   # 96-wide layer 1
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["fc", "cnn_letters"])
def test_route_layers(lib, oracle, capfd, monkeypatch, name):
    from bitnetmcu_b200 import _lib
    m = load_model(name)
    e, _ = verbose_engine(capfd, monkeypatch, lambda: engine(m, _lib.PATH_LAYERS))
    imgs = _images(3000, seed=1)
    want_lo, want_la = oracle.infer(m, imgs)
    _check(_topk(e, "int8", imgs, 4), want_lo, 4, name, want_la.astype(np.int64))
    x = np.random.default_rng(2).normal(size=(700, 256)).astype(np.float32)
    _check(_topk(e, "emul", x, 4), emulate(m, x), 4, (name, "emul"))
    routes = _route_lines(capfd)
    assert len(routes) == 2 and routes[0].endswith("layer by layer + k_topk_rows<int32>"), routes
    assert routes[1] == "bnm_emulate_topk_device: layer by layer + k_topk_rows<double>", routes
    e.close()


@pytest.mark.gpu
def test_route_float_and_emulator(lib, oracle, capfd, monkeypatch):
    for name, c_route, py_route in (("fc", "k_quantize_images + fc_topk_kernel<64,1,topk>", "k_quantize_images + fc_topk_kernel<64,1,emul,topk>"),
                                    ("cnn_48", None, "k_cnn_emul_frontend + fc_topk_kernel<128,1,emul,topk>")):
        m = load_model(name)
        e, _ = verbose_engine(capfd, monkeypatch, lambda: engine(m))
        x = np.random.default_rng(5).normal(size=(3001, 256)).astype(np.float32)
        want_lo, want_la = oracle.infer(m, scale_images(x))
        _check(_topk(e, "f32", x, 3), want_lo, 3, (name, "f32"), want_la.astype(np.int64))
        _check(_topk(e, "emul", x, 3), emulate(m, x), 3, (name, "emul"))
        routes = _route_lines(capfd)
        assert routes[0].startswith("bnm_infer_topk_device_f32: k_quantize_images + "), routes
        if c_route:
            assert routes[0] == "bnm_infer_topk_device_f32: " + c_route, routes
        assert routes[1] == "bnm_emulate_topk_device: " + py_route, routes
        e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("pinned", [False, True])
@pytest.mark.parametrize("name", ["fc", "cnn_letters", "binary160"])
def test_route_host(lib, oracle, capfd, monkeypatch, name, pinned):
    """the host entry over several chunks of the three-stream pipeline, from pageable and from pinned memory"""
    from bitnetmcu_b200 import _lib
    m = load_model(name)
    e, _ = verbose_engine(capfd, monkeypatch, lambda: engine(m))
    e.set_option(_lib.OPT_CHUNK_IMAGES, 1000)
    n = 4321
    src = _images(n, seed=int(pinned))
    want_lo, want_la = oracle.infer(m, src)
    if pinned:
        p = lib.bnm_host_alloc(src.nbytes)
        imgs = np.ctypeslib.as_array((C.c_int8 * src.size).from_address(p)).reshape(src.shape)
        imgs[:] = src
    else:
        imgs = src
    for k in (1, min(e.n_classes, MAX_TOPK)):
        cls, sc = e.topk(imgs, k)
        _check((cls.astype(np.int64), sc), want_lo, k, (name, pinned), want_la.astype(np.int64))
        cls2, none = e.topk(imgs, k, want_scores=False)
        assert none is None and np.array_equal(cls2, cls)
    routes = _route_lines(capfd)
    assert routes and all(r.startswith("bnm_infer_topk: ") for r in routes), routes
    if pinned:
        del imgs
        lib.bnm_host_free(p)
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["fc", "binary160", "cnn_letters"])
def test_side_stream(lib, oracle, name):
    import torch
    m = load_model(name)
    e = engine(m)
    imgs = _images(3000, seed=9)
    want_lo, want_la = oracle.infer(m, imgs)
    s = torch.cuda.Stream()
    d_img = torch.from_numpy(imgs).cuda()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        got = _topk(e, "int8", d_img, 3)
    _check(got, want_lo, 3, name, want_la.astype(np.int64))
    got = _topk(e, "int8", d_img, 3, stream=s.cuda_stream)
    s.synchronize()
    _check(got, want_lo, 3, (name, "stream argument"), want_la.astype(np.int64))
    e.close()


# ---- GPU: arguments ------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_argument_errors_and_empty_batches(lib):
    import torch
    e = engine(load_model("cnn_letters"))     # 37 classes
    h, n = e.handle, 256
    d_i8 = torch.zeros((n + 1, 256), dtype=torch.int8, device="cuda")
    d_f = torch.zeros((n + 1, 256), dtype=torch.float32, device="cuda")
    cls = torch.full((n * MAX_TOPK + 4,), 0x5A5A5A5A, dtype=torch.int32, device="cuda")
    sc = torch.full((n * MAX_TOPK + 4,), 0x5A5A5A5A, dtype=torch.int32, device="cuda")
    sd = torch.full((n * MAX_TOPK + 4,), 3.5, dtype=torch.float64, device="cuda")
    p = lambda t, off=0: C.c_void_p(t.data_ptr() + off)
    calls = [(lib.bnm_infer_topk_device, d_i8, sc), (lib.bnm_infer_topk_device_f32, d_f, sc), (lib.bnm_emulate_topk_device, d_f, sd)]
    for fn, img, s in calls:
        for k in (0, MAX_TOPK + 1, 1000):
            assert fn(h, p(img), n, k, p(cls), p(s), None) == BNM_E_ARG, (fn, k)
        assert fn(h, p(img), n, 3, None, p(s), None) == BNM_E_ARG
        assert fn(h, p(img, 4), n, 3, p(cls), p(s), None) == BNM_E_ARG               # images not 16-byte aligned
        assert fn(h, p(img), n, 3, p(cls, 2), p(s), None) == BNM_E_ARG              # classes not 4-byte aligned
        assert fn(h, p(img), n, 3, p(cls), p(s, 2 if s is sc else 4), None) == BNM_E_ARG
        assert fn(h, p(img), 0, 3, p(cls), p(s), None) == 0                         # n == 0: nothing written
    small = engine(load_model("fc"))                                                 # 10 classes
    assert lib.bnm_infer_topk_device(small.handle, p(d_i8), n, 11, p(cls), None, None) == BNM_E_ARG
    ok = torch.zeros((n, 10), dtype=torch.int32, device="cuda")
    assert lib.bnm_infer_topk_device(small.handle, p(d_i8), n, 10, p(ok), None, None) == 0      # k == n_classes
    torch.cuda.synchronize()
    assert (ok.cpu().numpy()[0] == np.arange(10)).all()                                       # all-zero images: all tied
    small.close()
    assert (cls.cpu().numpy() == 0x5A5A5A5A).all() and (sc.cpu().numpy() == 0x5A5A5A5A).all() and (sd.cpu().numpy() == 3.5).all()
    host_cls = np.full((4, 4), 7, dtype=np.uint32)
    for k in (0, 17, 38):
        assert lib.bnm_infer_topk(h, C.c_void_p(np.zeros((4, 256), np.int8).ctypes.data), 4, k, C.c_void_p(host_cls.ctypes.data), None) == BNM_E_ARG
    assert lib.bnm_infer_topk(h, C.c_void_p(np.zeros((4, 256), np.int8).ctypes.data), 4, 3, None, None) == BNM_E_ARG
    assert lib.bnm_infer_topk(h, None, 0, 3, C.c_void_p(host_cls.ctypes.data), None) == 0
    assert (host_cls == 7).all()
    e.close()


# ---- GPU: the batched top-k accuracy driver ------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("which", ["fc", "cnn_letters"])
def test_topk_accuracy_driver(lib, oracle, which):
    """host/evaluate_topk.py: the C-engine report of host/test_inference_batched.py, then "Top-K accuracy C" from the oracle's
    logits ranked by the restatement"""
    spec = importlib.util.spec_from_file_location("evaluate_topk", os.path.join(ROOT, "host", "evaluate_topk.py"))
    drv = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(drv)
    m = load_model(which)
    rng = np.random.default_rng(11)
    x = rng.normal(size=(2001, 256)).astype(np.float32)
    labels = rng.integers(0, m.layers[-1].n_out, size=2001)
    lines = []
    res = drv.evaluate(m, x, labels, 5, out=lines.append)
    want_lo, _ = oracle.infer(m, scale_images(x))
    want_c, _ = topk_order(want_lo, 5)
    assert np.array_equal(res["classes"].astype(np.int64), want_c)
    hits = int((want_c == labels[:, None]).any(axis=1).sum())
    assert len(lines) == 4 and lines[0] == "size of test data: 2001" and res["correct_topk_c"] == hits
    assert lines[3] == f"Top-5 accuracy C: {hits / 2001 * 100} %"
