"""The layer-by-layer FC path on the model shapes only it runs.  The fused plan (fc_chain_plan_create) refuses a layer wider than
256 outputs and an input row that is not a multiple of 16 bytes or is longer than 1024 bytes, so for every model below
k_fc_dp4a, k_relunorm, k_relunorm_emul, k_emul_logits and k_topk_rows are the only implementation.  The cases cover rows that
are not a multiple of 4 bytes (Ternary 130, 250 and 258), a 258-byte image into a 260-input layer with non-zero trits past the
image, rows of 1792 bytes (k_pad 1792, the largest the dp4a kernel stages), hidden maxima past 2^24, heads of 256 to 300
classes (255 is also ReLUNorm's "no maximum" position, inference.c:25) and an eight-layer chain.

CPU tests pin the oracle to the unmodified reference on every case and check that each case reaches the edges it claims.  GPU
tests run every entry on every case and compare with the reference (the oracle where oracle/_ref is not built), exactly."""
import re
from typing import Callable, NamedTuple

import numpy as np
import pytest

from bitnetmcu_b200 import model as M, pack as P
from restate import emulate, scale_images
from support import engine, lib, plan_line, route, scattered_edge_images, verbose_engine  # noqa: F401  (lib: fixture)

BNM_E_UNSUPPORTED = -3
ROW = "fused path: input row must be a multiple of 16 bytes, <= 1024"
WIDE = "fused path: layer wider than 256 outputs"
DP4A_MAX_KPAD = 1792                 # 128 staged rows of k_pad + 4 bytes fit the SM's 227 kB (launch_fc_dp4a)
N_UNIQUE = 389                       # distinct images per case; batches repeat them, so no 128-image tile is periodic
N_BIG = (1 << 17) + 77               # crosses the C engine's layer-by-layer pass of 2^17 images (kLayerPass, capi.cu)
SIZES = (1, 127, 129, 5 * 128 + 37, N_BIG)


# ---- the cases ---------------------------------------------------------------------------------------------------------------

def _fc(enc, widths, seed, img_bytes=None):
    m = P.random_fc_model(enc, widths, seed=seed)
    if img_bytes is not None:
        m.img_bytes = img_bytes
    return m


def _model(layers, img_bytes):
    m = M.Model(model_class=M.MODEL_FCMNIST, layers=layers, img_bytes=img_bytes)
    m.validate()
    return m


def _codes(enc, w_int):
    return P.codes_from_int_weights(enc, np.asarray(w_int))


def ternary_258_into_260():
    """a 258-byte image into a 260-input layer whose trits 258 and 259 are non-zero in every row: the reference reads those two
    inputs as zero (ref_driver.c clears layer_in before it copies the image in)"""
    rng = np.random.default_rng(258)
    t = rng.integers(-1, 2, size=(64, 260))
    t[:, 258:] = rng.choice([-1, 1], size=(64, 2))
    return _model([P.fc_layer_from_trits("L1", t), P.fc_layer_from_trits("L2", rng.integers(-1, 2, size=(10, 64)))], 258)


def eight_bit_1792():
    """8bit (1792, 288, 257) with hidden row 0 all -128 and row 1 all +127: images at the rails give hidden maxima of
    128 * 128 * 1792 = 29 360 128 > 2^24, a ReLUNorm shift of 18"""
    rng = np.random.default_rng(1792)
    w1 = rng.integers(-128, 128, size=(288, 1792))
    w1[0], w1[1] = -128, 127
    l1 = P.fc_layer_from_codes("L1", M.ENC_8BIT, _codes(M.ENC_8BIT, w1))
    l2 = P.fc_layer_from_codes("L2", M.ENC_8BIT, rng.integers(0, 256, size=(257, 288), dtype=np.uint32))
    return _model([l1, l2], 1792)


def fp130_wide():
    """FP130 (256, 320, 10) with +128 weights in every row of the 320-wide layer (the second weight plane), row 0 all +128"""
    rng = np.random.default_rng(130)
    w1 = P.INT_LUT[M.ENC_FP130][rng.integers(0, 16, size=(320, 256))]
    w1[:, ::7] = 128
    w1[0] = 128
    l1 = P.fc_layer_from_codes("L1", M.ENC_FP130, _codes(M.ENC_FP130, w1))
    l2 = P.fc_layer_from_codes("L2", M.ENC_FP130, rng.integers(0, 16, size=(10, 320), dtype=np.uint32))
    return _model([l1, l2], 256)


def head(C, D):
    """one 8bit layer D -> C whose weights pick input c for class c: the logits are the image's first C bytes, so images place
    maxima and ties at any class"""
    w = np.zeros((C, D), dtype=np.int64)
    w[np.arange(C), np.arange(C)] = 1
    return _model([P.fc_layer_from_codes("L1", M.ENC_8BIT, _codes(M.ENC_8BIT, w))], D)


class Case(NamedTuple):
    name: str
    refusal: str                 # why the fused plan refuses the model (its first failing check)
    make: Callable[[], M.Model]
    emulator_exact: bool = True  # restate.emulate is the emulator bit for bit (not 4bit, not NF4)


CASES = [
    Case("ternary-130", ROW, lambda: _fc(M.ENC_TERNARY, (130, 64, 10), 1)),
    Case("ternary-250-300", ROW, lambda: _fc(M.ENC_TERNARY, (250, 300, 10), 2)),
    Case("ternary-258-into-260", ROW, ternary_258_into_260),
    Case("8bit-196-300", ROW, lambda: _fc(M.ENC_8BIT, (196, 300, 10), 3)),
    Case("4bitsym-200-512-64-300", ROW, lambda: _fc(M.ENC_4BITSYM, (200, 512, 64, 300), 4)),
    Case("binary-1792", ROW, lambda: _fc(M.ENC_BINARY, (1792, 64, 10), 5)),
    Case("8bit-1792-288-257", ROW, eight_bit_1792),
    Case("4bit-1280-256-40", ROW, lambda: _fc(M.ENC_4BIT, (1280, 256, 40), 6), emulator_exact=False),
    Case("fp130-320-wide", WIDE, fp130_wide),
    Case("2bitsym-48-16-260", WIDE, lambda: _fc(M.ENC_2BITSYM, (48, 16, 260), 7)),
    Case("4bitsym-8-layers", WIDE, lambda: _fc(M.ENC_4BITSYM, (64, 96, 304, 64, 48, 32, 32, 32, 10), 8)),
    Case("head-256", ROW, lambda: head(256, 260)),
    Case("head-257", ROW, lambda: head(257, 260)),
    Case("head-300", ROW, lambda: head(300, 300)),
]
CASE_IDS = [c.name for c in CASES]
BY_NAME = {c.name: c for c in CASES}


def fused_refusal(m):
    """the first check of fc_chain_plan_create that model m fails on its shapes, None when it passes them"""
    if m.img_bytes % 16 or m.img_bytes > 1024:
        return ROW
    if any((l.n_out + 15) // 16 * 16 > 256 for l in m.fc_layers):
        return WIDE
    return None


# ---- inputs ------------------------------------------------------------------------------------------------------------------

def head_rows(C, D, seed):
    """int8 images of a head(C, D) model: maxima at class 255, 256 and C - 1, ties between 255 and 256 and between a low class and
    one above 255, near-ties, rows of one value -> (images, the label of each, what each holds)"""
    rng = np.random.default_rng(seed)
    rows, labels, what = [], [], []

    def add(tag, label, top, fill=None):
        """a row whose classes `top` hold 127 and all else `fill` (None: random values below 127)"""
        r = rng.integers(-128, 127, size=D) if fill is None else np.full(D, fill)
        r[list(top)] = 127
        rows.append(r)
        labels.append(label)
        what.append(tag)
    for c in sorted({0, 255, min(256, C - 1), C - 1}):
        add(f"max at {c}", c, [c])
        add(f"max at {c} over 126", c, [c], 126)
    if C > 256:
        add("tie 255 256", 255, [255, 256])
        add(f"tie 3 {C - 1}", 3, [3, C - 1])
        add(f"tie 256 {C - 1}", 256, [256, C - 1])
    add("tie 2 255", 2, [2, 255])
    add(f"tie 255 {C - 1}", 255, [255, C - 1], 126)
    for v in (0, 127, -128, -1):
        add(f"all {v}", 0, [], v)
    r = np.full(D, -128)
    r[C - 1] = -127
    rows.append(r)
    labels.append(C - 1)
    what.append(f"negative maximum at {C - 1}")
    return np.stack(rows).astype(np.int8), np.array(labels, dtype=np.uint32), what


def int8_images(m, seed):
    """N_UNIQUE int8 images: rows at the int8 rails (all 127, all -128, alternating, random signs), all zero, random rows; a head
    model's crafted rows first"""
    D = m.img_bytes
    rng = np.random.default_rng(seed)
    q = rng.integers(-128, 128, size=(N_UNIQUE, D)).astype(np.int8)
    rails = [np.full(D, 127), np.full(D, -128), np.zeros(D), np.where(np.arange(D) % 2, -128, 127),
             np.where(rng.random(D) < 0.5, 127, -128), np.full(D, 1)]
    q[:len(rails)] = np.stack(rails)
    if len(m.fc_layers) == 1:   # a head
        h, _, _ = head_rows(m.n_classes, D, seed)
        q[len(rails):len(rails) + len(h)] = h
    return q


def float_images(m, q, seed):
    """float32 images: the int8 images' first half as floats (their rails and crafted rows survive the scaling), then rows at the
    edges of the input scaling"""
    x = scattered_edge_images(N_UNIQUE, m.img_bytes, seed)
    x[:N_UNIQUE // 2] = q[:N_UNIQUE // 2].astype(np.float32)
    return x


_DATA = {}


def case_data(name, judge):
    """(model, int8 images, logits, labels, float images, logits, labels of their scaled rows, emulator logits), cached per case"""
    if name not in _DATA:
        m = BY_NAME[name].make()
        seed = CASE_IDS.index(name) + 11
        q = int8_images(m, seed)
        lo, la = judge.infer(m, q)
        x = float_images(m, q, seed)
        xlo, xla = judge.infer(m, scale_images(x))
        _DATA[name] = (m, q, lo, la, x, xlo, xla, emulate(m, x))
    return _DATA[name]


def topk_want(logits, k):
    """ranks: highest first, ties to the lower class -> (classes, scores)"""
    order = np.argsort(-logits.astype(np.float64), axis=1, kind="stable")[:, :k]
    return order, np.take_along_axis(logits, order, axis=1)


def top_ks(C):
    return sorted({1, 5} | ({C} if C <= 16 else set()))


# ---- CPU: the cases against the reference, and the edges they reach ---------------------------------------------------------

@pytest.mark.parametrize("name", CASE_IDS)
def test_oracle_matches_reference(oracle, reference, name):
    """the C restatement equals the unmodified reference on every case: rows at the int8 rails, all-zero and random rows"""
    m = BY_NAME[name].make()
    q = int8_images(m, CASE_IDS.index(name) + 11)
    x = float_images(m, q, 3)
    for imgs, what in ((q, "int8"), (scale_images(x), "scaled float")):
        want_lo, want_la = reference.infer(m, imgs)
        lo, la = oracle.infer(m, imgs)
        assert np.array_equal(lo, want_lo), (name, what, "logits")
        assert np.array_equal(la, want_la), (name, what, "labels")


@pytest.mark.parametrize("name", CASE_IDS)
def test_case_shapes(name):
    """each case fails the fused plan's check it names, and every layer fits the dp4a kernel's shared memory"""
    c = BY_NAME[name]
    m = c.make()
    assert fused_refusal(m) == c.refusal, name
    assert all((max(l.n_in, 1) + 31) // 32 * 32 <= DP4A_MAX_KPAD for l in m.fc_layers), name
    if m.img_bytes in (130, 250, 258):
        assert m.img_bytes % 4, name   # the first layer's rows start off 4-byte boundaries


@pytest.mark.parametrize("name", ["head-256", "head-257", "head-300"])
def test_heads_reach_classes_past_255(oracle, name):
    """the crafted rows put the label at 255, 256 and the last class, ties go to the first maximum, rows of one value to class 0"""
    m = BY_NAME[name].make()
    C = m.n_classes
    h, want, what = head_rows(C, m.img_bytes, 1)
    lo, la = oracle.infer(m, h)
    assert np.array_equal(lo, h[:, :C].astype(np.int32)), name   # the logits are the image's first C bytes
    bad = [(tag, int(g)) for tag, g, w in zip(what, la, want) if g != w]
    assert not bad, (name, bad)
    assert {255, C - 1} <= set(la.tolist()) and (C <= 256 or 256 in la.tolist()), name


def test_hidden_maxima_past_2_24(oracle):
    """8bit over 1792 inputs at the rails: hidden maxima past 2^24, ReLUNorm shifts up to 18; FP130's +128 weights sit in a layer
    wider than 256; the Ternary 260-input layer has non-zero trits past the 258-byte image"""
    m = BY_NAME["8bit-1792-288-257"].make()
    q = int8_images(m, 1)
    acc = q.astype(np.int64) @ P.decode_int_weights(m.fc_layers[0]).astype(np.int64).T
    top = acc.max(axis=1)
    assert top.max() == 128 * 128 * 1792 and top.max() > 1 << 24
    assert max(int(t >> 7).bit_length() for t in top) == 18
    f = BY_NAME["fp130-320-wide"].make().fc_layers[0]
    assert f.n_out > 256 and (P.decode_int_weights(f) == 128).any(axis=1).all()
    t = BY_NAME["ternary-258-into-260"].make()
    assert t.img_bytes == 258 and (P.decode_int_weights(t.fc_layers[0])[:, 258:] != 0).all()


# ---- GPU: every entry on every case -----------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def judge(built):
    """the unmodified reference where oracle/_ref is built, else the oracle (pinned to it by test_oracle_matches_reference)"""
    from oracle.oracle import Oracle, Reference
    return Reference() if Reference.available() else Oracle()


class Dev:
    """one case's images and expectations on the device; rows of a batch of n are the case's images i % N_UNIQUE"""

    def __init__(self, name, judge):
        import torch
        self.m, q, lo, la, x, xlo, xla, emu = case_data(name, judge)
        self.name, self.C, self.exact = name, self.m.n_classes, BY_NAME[name].emulator_exact
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
        self.q_np, self.q, self.x = q, t(q), t(x)
        self.lo, self.la, self.xlo, self.xla = t(lo), t(la.astype(np.int32)), t(xlo), t(xla.astype(np.int32))
        self.emu, self.emu_la = t(emu), t(np.argmax(emu, axis=1).astype(np.int32))
        self.lo_np, self.la_np, self.xlo_np, self.emu_np = lo, la, xlo, emu

    def idx(self, n):
        import torch
        return torch.arange(n, device="cuda") % N_UNIQUE

    def check(self, n, got, want, sentinel, what):
        """rows :n of `got` (n + 128 rows) equal want[idx(n)]; the rows past n still hold the sentinel"""
        import torch
        w = want[self.idx(n)]
        g = got[:n].to(w.dtype)
        bad = torch.nonzero((g != w).reshape(n, -1).any(dim=1)).flatten()
        assert bad.numel() == 0, (self.name, n, what, f"{bad.numel()} rows wrong, first {bad[:4].tolist()}")
        assert bool((got[n:] == sentinel).all()), (self.name, n, what, "written past row n")


def out(shape, dtype, sentinel):
    import torch
    return torch.full((shape[0] + 128,) + tuple(shape[1:]), sentinel, dtype=dtype, device="cuda")


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASE_IDS)
def test_no_fused_plan(lib, capfd, monkeypatch, name):
    """the model loads without a fused plan (no plan line, the layered path active, both emulator routes layer by layer), and
    asking for the fused path reports the plan's refusal"""
    from bitnetmcu_b200 import _lib
    c = BY_NAME[name]
    e, err = verbose_engine(capfd, monkeypatch, lambda: engine(c.make()))
    assert plan_line(err) is None and e.active_path == _lib.PATH_LAYERS, (name, err)
    assert route(err, "emulator") == "layer by layer", (name, err)
    assert route(err, "engines") == "bnm_infer_batch_device_f32 + bnm_emulate_batch_device + k_engine_counts", (name, err)
    with pytest.raises(_lib.BnmError, match=f"rc={BNM_E_UNSUPPORTED}.*{re.escape(c.refusal)}"):
        e.set_option(_lib.OPT_PATH, _lib.PATH_TCGEN05)
    assert e.active_path == _lib.PATH_LAYERS, name
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASE_IDS)
def test_host_entries(lib, judge, name):
    """bnm_infer_batch from host memory: the small-batch path (up to 1024 images), the pipeline in chunks of 128 images and of the
    default 65 536; labels only; bnm_infer_topk in chunks of 128"""
    from bitnetmcu_b200 import _lib
    d = Dev(name, judge)
    e = engine(d.m)
    for chunk in (None, 128):
        if chunk:
            e.set_option(_lib.OPT_CHUNK_IMAGES, chunk)
        for n in SIZES if chunk is None else SIZES[:4]:
            i = np.arange(n) % N_UNIQUE
            lo, la = e.infer(d.q_np[i])
            tag = (name, n, chunk)
            assert np.array_equal(lo, d.lo_np[i]), (tag, "logits")
            assert np.array_equal(la, d.la_np[i]), (tag, "labels")
            _, la2 = e.infer(d.q_np[i], want_logits=False)
            assert np.array_equal(la2, la), (tag, "labels only")
    for k in top_ks(d.C):
        i = np.arange(SIZES[3]) % N_UNIQUE
        cls, sc = e.topk(d.q_np[i], k)
        wc, ws = topk_want(d.lo_np[i], k)
        assert np.array_equal(cls, wc) and np.array_equal(sc, ws), (name, "host top-k", k)
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASE_IDS)
def test_device_entries(lib, judge, name):
    """bnm_infer_batch_device with logits and labels, labels only, logits only; bnm_infer_topk_device (k_topk_rows) at k = 1, 5
    and the class count where it is at most 16; every batch size"""
    import torch
    d = Dev(name, judge)
    e = engine(d.m)
    for n in SIZES:
        x = d.q[d.idx(n)]
        for want_lo, want_la in ((True, True), (False, True), (True, False)):
            lo, la = out((n, d.C), torch.int32, -5), out((n,), torch.int32, -7)
            e.infer_device(x, lo[:n] if want_lo else None, la[:n] if want_la else None)
            torch.cuda.synchronize()
            if want_lo:
                d.check(n, lo, d.lo, -5, f"logits (labels too: {want_la})")
            if want_la:
                d.check(n, la, d.la, -7, f"labels (logits too: {want_lo})")
            assert want_lo or bool((lo == -5).all()), (name, n, "logits written")
            assert want_la or bool((la == -7).all()), (name, n, "labels written")
        for k in top_ks(d.C):
            wc, ws = (torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in topk_want(d.lo_np, k))
            cls, sc = out((n, k), torch.int32, -3), out((n, k), torch.int32, -9)
            e.topk_device(x, k, cls[:n], sc[:n])
            torch.cuda.synchronize()
            d.check(n, cls, wc, -3, f"top-{k} classes")
            d.check(n, sc, ws, -9, f"top-{k} scores")
        del x
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASE_IDS)
def test_float_entries(lib, judge, name):
    """bnm_infer_batch_device_f32 against the reference on restate.scale_images of the same rows; the emulator's device entry and
    its top-k against restate.emulate (encodings where it is exact); bnm_compare_engines_device's labels and counts"""
    import torch
    d = Dev(name, judge)
    e = engine(d.m)
    for n in SIZES:
        x = d.x[d.idx(n)]
        lo, la = out((n, d.C), torch.int32, -5), out((n,), torch.int32, -7)
        e.infer_device_f32(x, lo[:n], la[:n])
        torch.cuda.synchronize()
        d.check(n, lo, d.xlo, -5, "float-input logits")
        d.check(n, la, d.xla, -7, "float-input labels")
        k = top_ks(d.C)[-1]
        wc, ws = (torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in topk_want(d.xlo_np, k))
        cls, sc = out((n, k), torch.int32, -3), out((n, k), torch.int32, -9)
        e.topk_device_f32(x, k, cls[:n], sc[:n])
        torch.cuda.synchronize()
        d.check(n, cls, wc, -3, f"float-input top-{k} classes")
        d.check(n, sc, ws, -9, f"float-input top-{k} scores")
        if d.exact:
            elo, ela = out((n, d.C), torch.float64, -12345.5), out((n,), torch.int32, -7)
            e.inference_quantized_device(x, elo[:n], ela[:n])
            torch.cuda.synchronize()
            d.check(n, elo, d.emu, -12345.5, "emulator logits")
            d.check(n, ela, d.emu_la, -7, "emulator labels")
            wc, ws = (torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in topk_want(d.emu_np, k))
            cls, sc = out((n, k), torch.int32, -3), out((n, k), torch.float64, -12345.5)
            e.emulate_topk_device(x, k, cls[:n], sc[:n])
            torch.cuda.synchronize()
            d.check(n, cls, wc, -3, f"emulator top-{k} classes")
            d.check(n, sc, ws, -12345.5, f"emulator top-{k} scores")
        truth = ((torch.arange(n, device="cuda") * 7) % (d.C + 1)).to(torch.int32)
        lc, lp = out((n,), torch.int32, -7), out((n,), torch.int32, -7)
        counts = torch.zeros(4, dtype=torch.int64, device="cuda")
        e.compare_engines_device(x, truth, lc[:n], lp[:n], counts)
        torch.cuda.synchronize()
        d.check(n, lc, d.xla, -7, "engines: C labels")
        wc = d.xla[d.idx(n)]
        got = counts.cpu().tolist()
        assert got[:2] == [n, int((wc == truth).sum())], (name, n, "engines: counts", got)
        if d.exact:
            d.check(n, lp, d.emu_la, -7, "engines: emulator labels")
            wp = d.emu_la[d.idx(n)]
            assert got[2:] == [int((wp == truth).sum()), int((wc != wp).sum())], (name, n, "engines: counts", got)
        del x
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["8bit-196-300", "ternary-130"])
def test_rows_off_16_byte_boundaries(lib, judge, name):
    """device images at a 16-byte offset into their buffer (the entries' alignment rule holds) whose rows of 196 or 130 bytes
    then start off 16-byte (and for 130, off 4-byte) boundaries: int8, float and top-k entries, and the emulator"""
    import torch
    d = Dev(name, judge)
    e = engine(d.m)
    D, n = d.m.img_bytes, SIZES[3]
    buf = torch.zeros(16 + (n + 1) * D, dtype=torch.int8, device="cuda")
    x = buf[16:16 + n * D].view(n, D)
    x.copy_(d.q[d.idx(n)])
    fbuf = torch.zeros(4 + (n + 1) * D, dtype=torch.float32, device="cuda")
    xf = fbuf[4:4 + n * D].view(n, D)
    xf.copy_(d.x[d.idx(n)])
    assert x.data_ptr() % 16 == 0 and xf.data_ptr() % 16 == 0
    lo, la = out((n, d.C), torch.int32, -5), out((n,), torch.int32, -7)
    e.infer_device(x, lo[:n], la[:n])
    torch.cuda.synchronize()
    d.check(n, lo, d.lo, -5, "offset logits")
    d.check(n, la, d.la, -7, "offset labels")
    cls = out((n, 5), torch.int32, -3)
    e.topk_device(x, 5, cls[:n])
    torch.cuda.synchronize()
    d.check(n, cls, torch.from_numpy(topk_want(d.lo_np, 5)[0]).cuda(), -3, "offset top-5")
    e.infer_device_f32(xf, lo[:n], la[:n])
    torch.cuda.synchronize()
    d.check(n, lo, d.xlo, -5, "offset float-input logits")
    d.check(n, la, d.xla, -7, "offset float-input labels")
    elo = out((n, d.C), torch.float64, -12345.5)
    e.inference_quantized_device(xf, elo[:n], la[:n])
    torch.cuda.synchronize()
    d.check(n, elo, d.emu, -12345.5, "offset emulator logits")
    d.check(n, la, d.emu_la, -7, "offset emulator labels")
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("widths", [(1824, 64, 10), (64, 1824, 10)], ids=["first-layer", "hidden-layer"])
def test_dp4a_shared_memory_bound(lib, judge, widths):
    """k_pad 1792 runs (binary-1792, 8bit-1792-288-257 above); a layer of k_pad 1824 loads, and its first call on every entry
    fails with BNM_E_UNSUPPORTED and the layer kernel's message, leaving no error behind for the next call"""
    import torch
    from bitnetmcu_b200 import _lib
    m = _fc(M.ENC_BINARY if widths[0] > 64 else M.ENC_4BITSYM, widths, 1824)
    layer = int(widths[0] < 1824)
    e = engine(m)
    assert e.active_path == _lib.PATH_LAYERS
    n = 129
    q = np.zeros((n, m.img_bytes), dtype=np.int8)
    dq, dx = torch.zeros((n, m.img_bytes), dtype=torch.int8, device="cuda"), torch.zeros((n, m.img_bytes), device="cuda")
    lo, la = torch.zeros((n, 10), dtype=torch.int32, device="cuda"), torch.zeros(n, dtype=torch.int32, device="cuda")
    calls = {
        "host small batch": lambda: e.infer(q),
        "host top-k": lambda: e.topk(q, 3),
        "device": lambda: e.infer_device(dq, lo, la),
        "device top-k": lambda: e.topk_device(dq, 3, lo[:, :3].contiguous()),
        "float": lambda: e.infer_device_f32(dx, lo, la),
        "emulator": lambda: e.inference_quantized_device(dx, None, la),
        "engines": lambda: e.compare_engines_device(dx, labels_c=la),
    }
    msg = f"rc={BNM_E_UNSUPPORTED}.*FC layer {layer}: {widths[layer]} inputs need more shared memory"
    for what, call in calls.items():
        with pytest.raises(_lib.BnmError, match=msg):
            call()
        torch.cuda.synchronize()
    e.close()
    ok = Dev("binary-1792", judge)   # the same process runs the bound's own shape right after
    e = engine(ok.m)
    lo, la = e.infer(ok.q_np)
    assert np.array_equal(lo, ok.lo_np) and np.array_equal(la, ok.la_np)
    e.close()
