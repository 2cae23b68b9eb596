"""The fused FC launches that read what the same call has just written into its own scratch ("fed" launches): float input
scaled by k_quantize_images on a model without a fused float-input form, and every C-engine CNN call, whose FC stage reads the
front-end's features (k_cnn_frontend16 or k_cnn_frontend16_tc).  The window scan, the third fed route, has its own tests
(test_window_scan.py) and runs here once per model.

Models.  CNNMNIST-shaped models as the reference builds them (models.py:100-134): three 8bit depthwise convs, a 2bitsym first
FC layer, then layers of one QuantType.  Every QuantType appears at the reference's default widths (64 channels, 64/64/64/10),
and together the models take the CNN int8 route onto every int8 row of the fused plan, each row from at least two QuantTypes,
and onto the layer-by-layer path (256 channels).  Their heads mix encodings: FP130 residual planes in some layers only,
Ternary layers whose 64 inputs are padded to 70 right after the 2bitsym layer, and an emulator logit scale of 1 where the first
layer's would be 0.5.  C = 10 gives 40 features in rows of 48 bytes whose last 8 bytes the front-ends never write; its first
layer is 8bit, since 40 2bitsym weights do not fill whole words (the reference's exporter refuses them).  The float route
runs on the FC models of kChainKernels that have no float-input form: Binary-160, 2bitsym-96, a 37-class head, 512-byte rows
and a 256-wide model.

CPU tests pin the oracle to the unmodified reference and restate.emulate to the reference's own
QuantizedModel.inference_quantized on these models.  GPU tests check the mode-2 launch decisions of every fed route (the
deterministic guard: a fed launch and the int8 launch after it keep their grid-dependency wait), every row at its ring sweep,
every entry at one grid-filling size against the reference (the oracle where oracle/_ref is not built), exactly, and fed calls
between kernel producers and consumers."""
import functools
import os
import sys
from typing import NamedTuple, Tuple

import numpy as np
import pytest

from bitnetmcu_b200 import model as M, pack as P
from restate import TILE, LEVEL_SHIFT, cnn_stages, emulate, scale_images
from support import CHAIN_ROWS, Sweep, cnn_model, engine, frontends, gather_call, kernel_clone, kernel_copies_are_kernels, \
    kernel_copy, lib, plan_line, plan_ring, quantized_model_list, scattered_edge_images, verbose_engine  # noqa: F401  (lib, kernel_copies_are_kernels: fixtures)

REF_PY = "/root/reference"
N_UNIQUE = 389                        # distinct images per model; batches repeat them (row i is image i % N_UNIQUE)
LAYERED = "layer by layer"
TWO_PASSES = (1 << 20) + 77           # a C-engine pass stages at most 2^20 images (kPass, capi.cu)
LAYER_SIZES = (1, 127, 129, 5 * 128 + 37, (1 << 17) + 77)   # the layered path: across its pass of 2^17 images


# ---- the models ----------------------------------------------------------------------------------------------------------------

class Cnn(NamedTuple):
    name: str
    row: str                  # the int8 row of the fused plan the CNN int8 route reaches, or LAYERED
    channels: int
    enc: int                  # the QuantType of every FC layer after the first
    widths: Tuple[int, ...]   # FC outputs, hidden layers then classes
    seed: int
    nf4_ext: bool = False
    first: int = M.ENC_2BITSYM

    @property
    def exact(self):
        """restate.emulate is the emulator bit for bit (levels the integers fix exactly: not 4bit, not NF4)"""
        return self.enc not in (M.ENC_4BIT, M.ENC_NF4)


DEFAULT = (64, 64, 64, 10)
FIXED = "<64,2,2,16,fixed>"
CNNS = [
    # the reference's default widths, every QuantType
    Cnn("binary-64", FIXED, 64, M.ENC_BINARY, DEFAULT, 1),
    Cnn("ternary-64", FIXED, 64, M.ENC_TERNARY, DEFAULT, 2),
    Cnn("2bitsym-64", FIXED, 64, M.ENC_2BITSYM, DEFAULT, 3),
    Cnn("4bit-64", FIXED, 64, M.ENC_4BIT, DEFAULT, 4),
    Cnn("4bitsym-64", FIXED, 64, M.ENC_4BITSYM, DEFAULT, 5),
    Cnn("8bit-64", FIXED, 64, M.ENC_8BIT, DEFAULT, 6),
    Cnn("nf4-64", FIXED, 64, M.ENC_NF4, DEFAULT, 7),
    Cnn("nf4ext-64", FIXED, 64, M.ENC_NF4, DEFAULT, 8, nf4_ext=True),
    Cnn("fp130-64", "<64,2,2,16>", 64, M.ENC_FP130, DEFAULT, 9),      # +128 past layer 1: residual planes leave the fixed row
    # the other rows
    Cnn("4bit-48-64-64", "<64,2,2,16>", 48, M.ENC_4BIT, (64, 64, 10), 10),
    Cnn("8bit-64-47", "<64,2,2,64>", 64, M.ENC_8BIT, (64, 47), 11),
    Cnn("2bitsym-64-47", "<64,2,2,64>", 64, M.ENC_2BITSYM, (64, 47), 12),
    Cnn("4bitsym-128-64", "<64,1>", 128, M.ENC_4BITSYM, (64, 10), 13),
    Cnn("nf4ext-128-64", "<64,1>", 128, M.ENC_NF4, (64, 10), 14, nf4_ext=True),
    Cnn("fp130-48-96", "<128,1>", 48, M.ENC_FP130, (96, 64, 10), 15),
    Cnn("binary-48-96", "<128,1>", 48, M.ENC_BINARY, (96, 64, 10), 16),
    Cnn("ternary-32-160", "<192,1>", 32, M.ENC_TERNARY, (160, 160, 10), 17),
    Cnn("8bit-32-160", "<192,1>", 32, M.ENC_8BIT, (160, 160, 10), 18),
    Cnn("8bit-64-256", "<256,1>", 64, M.ENC_8BIT, (256, 10), 19),
    Cnn("4bitsym-64-256", "<256,1>", 64, M.ENC_4BITSYM, (256, 10), 20),
    Cnn("2bitsym-256", LAYERED, 256, M.ENC_2BITSYM, DEFAULT, 21),
    Cnn("ternary-256", LAYERED, 256, M.ENC_TERNARY, DEFAULT, 22),
    # feature rows with padding the front-ends never write (C = 10: 40 features, stride 48), and without (C = 12)
    Cnn("8bit-10", "<64,2,2,16>", 10, M.ENC_4BITSYM, (64, 64, 10), 23, first=M.ENC_8BIT),
    Cnn("ternary-12", "<64,2,2,16>", 12, M.ENC_TERNARY, (64, 64, 10), 24),
]
CNN_IDS = [c.name for c in CNNS]
# FC models of kChainKernels without a float-input form: their float input runs k_quantize_images + the int8 form
FLOAT_ROWS = ["<192,1>", "<128,1>", "<64,2,2,64>", "<64,1>", "<256,1>"]
FLOAT_NAMES = {"<192,1>": "binary160", "<128,1>": "2bitsym96", "<64,2,2,64>": "4bitsym-37-classes",
               "<64,1>": "4bitsym-512-byte-rows", "<256,1>": "4bitsym-256-wide"}
FLOAT_IDS = [FLOAT_NAMES[r] for r in FLOAT_ROWS]


def _fc_layer(name, enc, n_in, n_out, rng):
    if enc == M.ENC_TERNARY:
        return P.fc_layer_from_trits(name, rng.integers(-1, 2, size=(n_out, n_in)))
    return P.fc_layer_from_codes(name, enc, rng.integers(0, 1 << P.CODE_BITS[enc], size=(n_out, n_in), dtype=np.uint32))


@functools.lru_cache(maxsize=None)
def make_cnn(name):
    c = CNNS[CNN_IDS.index(name)]
    front = cnn_model(c.channels, 10, seed=c.seed).layers[:5]   # conv, conv, pool, conv, pool: random 8bit taps with +-127
    rng = np.random.default_rng(1000 + c.seed)
    dims = (c.channels * 4,) + c.widths
    fc = [_fc_layer(f"L{11 + 2 * i}", c.first if i == 0 else c.enc, dims[i], dims[i + 1], rng) for i in range(len(c.widths))]
    m = M.Model(model_class=M.MODEL_CNNMNIST, layers=list(front) + fc)
    m.validate()
    return m


@functools.lru_cache(maxsize=None)
def make_float_model(row):
    return dict(CHAIN_ROWS)[row]()


def feat_stride(m):
    """the C engine's feature row: C * 4 int8 features rounded up to 16 bytes"""
    return -(-m.channels * 4 // 16) * 16


# ---- images and expectations ---------------------------------------------------------------------------------------------------

def int8_images(D, seed):
    """N_UNIQUE int8 images: rows at the int8 rails, all zero, one value, then random rows"""
    rng = np.random.default_rng(seed)
    q = rng.integers(-128, 128, size=(N_UNIQUE, D)).astype(np.int8)
    rails = [np.full(D, 127), np.full(D, -128), np.zeros(D), np.where(np.arange(D) % 2, -128, 127),
             np.where(rng.random(D) < 0.5, 127, -128), np.full(D, 1)]
    q[:len(rails)] = np.stack(rails)
    return q


def float_images(q, seed):
    """float32 images: the int8 images' first half as floats, then rows at the edges of the input scaling"""
    x = scattered_edge_images(N_UNIQUE, q.shape[1], seed)
    x[:N_UNIQUE // 2] = q[:N_UNIQUE // 2].astype(np.float32)
    return x


class Judge:
    """the unmodified reference where oracle/_ref is built, else the oracle; the NF4 extension always the oracle (the reference
    has no NF4 decode)"""

    def __init__(self):
        from oracle.oracle import Oracle, Reference
        self.oracle = Oracle()
        self.ref = Reference() if Reference.available() else None

    def infer(self, m, imgs, nf4_ext=False):
        if nf4_ext or self.ref is None:
            return self.oracle.infer(m, imgs, nf4_extension=nf4_ext)
        return self.ref.infer(m, imgs)


@pytest.fixture(scope="module")
def judge(built):
    return Judge()


_DATA = {}


def case_data(kind, name, judge):
    """(model, nf4 extension, exact emulator, int8 images, logits, labels, float images, logits, labels of their scaled rows,
    emulator logits or None), cached per model"""
    if (kind, name) not in _DATA:
        if kind == "cnn":
            c = CNNS[CNN_IDS.index(name)]
            m, ext, exact, seed = make_cnn(name), c.nf4_ext, c.exact, c.seed
        else:
            row = FLOAT_ROWS[FLOAT_IDS.index(name)]
            m, ext, exact, seed = make_float_model(row), False, True, 100 + FLOAT_IDS.index(name)
        q = int8_images(m.img_bytes, seed)
        lo, la = judge.infer(m, q, ext)
        x = float_images(q, seed)
        xlo, xla = judge.infer(m, scale_images(x), ext)
        _DATA[kind, name] = (m, ext, exact, q, lo, la, x, xlo, xla, emulate(m, x) if exact else None)
    return _DATA[kind, name]


# ---- CPU: the models against the reference ------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", [c.name for c in CNNS if not c.nf4_ext])
def test_oracle_matches_reference(oracle, reference, name):
    """the C restatement equals the unmodified reference on every CNN model: int8 rows at the rails, all zero, random, and
    scaled float rows"""
    m = make_cnn(name)
    q = int8_images(256, 7)
    for imgs, what in ((q, "int8"), (scale_images(float_images(q, 8)), "scaled float")):
        want_lo, want_la = reference.infer(m, imgs)
        lo, la = oracle.infer(m, imgs)
        assert np.array_equal(lo, want_lo), (name, what, "logits")
        assert np.array_equal(la, want_la), (name, what, "labels")


@pytest.mark.parametrize("row", FLOAT_ROWS, ids=FLOAT_IDS)
def test_float_models_oracle_matches_reference(oracle, reference, row):
    m = make_float_model(row)
    imgs = scale_images(float_images(int8_images(m.img_bytes, 9), 10))
    want_lo, want_la = reference.infer(m, imgs)
    lo, la = oracle.infer(m, imgs)
    assert np.array_equal(lo, want_lo) and np.array_equal(la, want_la), row


@pytest.mark.skipif(not os.path.isfile(os.path.join(REF_PY, "BitNetMCU.py")), reason="needs the reference's BitNetMCU.py")
@pytest.mark.parametrize("name", [c.name for c in CNNS if c.exact])
def test_emulate_matches_reference_emulator(name):
    """restate.emulate equals the reference's QuantizedModel.inference_quantized on every CNN model whose levels are exact,
    mixed heads included (its last layer's level scale differs from the 2bitsym first layer's), on float rows whose every conv
    stage has a positive maximum (the reference renormalises an all-zero stage by 0/0)"""
    if REF_PY not in sys.path:
        sys.path.append(REF_PY)
    from BitNetMCU import QuantizedModel
    m = make_cnn(name)
    x = float_images(int8_images(256, 11), 12)[::7]
    c1, c2, c3, _ = cnn_stages(m, x)
    keep = [i for i in range(len(x)) if min(c.reshape(len(x), -1)[i].max() for c in (c1, c2, c3)) > 0]
    x = x[keep]
    assert len(x) >= 40, name
    qm = QuantizedModel()
    qm.quantized_model = quantized_model_list(m)
    want = np.asarray(qm.inference_quantized(x), dtype=np.float64)
    assert np.array_equal(emulate(m, x), want), name


@pytest.mark.parametrize("name", CNN_IDS)
def test_model_shapes(name):
    """each model has the shape its row needs: feature rows of C * 4 bytes rounded to 16 (C = 10: 40 features in 48 bytes), a
    first layer of another encoding than the head's (except 2bitsym heads), Ternary inputs padded to tens, FP130 residual planes
    (+128 weights) in the layers past the first only"""
    c = CNNS[CNN_IDS.index(name)]
    m = make_cnn(name)
    fc = m.fc_layers
    assert [l.bitperweight for l in fc] == [c.first] + [c.enc] * (len(fc) - 1)
    assert [l.n_out for l in fc] == list(c.widths) and fc[0].n_in == c.channels * 4
    if c.channels == 10:
        assert feat_stride(m) == 48 and fc[0].n_in == 40
    if c.channels == 12:
        assert feat_stride(m) == 48 == fc[0].n_in
    if c.enc == M.ENC_TERNARY:
        assert all(l.n_in == -(-w // 10) * 10 for l, w in zip(fc[1:], c.widths))
        assert c.widths[0] % 10 == 0 or fc[1].n_in > c.widths[0]
    if c.enc == M.ENC_FP130:
        planes = [1 + int((P.decode_int_weights(l) == 128).any()) for l in fc]
        assert planes == [1] + [2] * (len(fc) - 1), planes
    # the emulator's logits take the last layer's level scale: 1 where the 2bitsym first layer's is 0.5
    if c.first == M.ENC_2BITSYM and c.enc not in (M.ENC_2BITSYM, M.ENC_4BITSYM):
        assert LEVEL_SHIFT.get(fc[0].bitperweight, 0) == 1 and LEVEL_SHIFT.get(fc[-1].bitperweight, 0) == 0


def test_models_cover_every_row_and_quanttype():
    """every QuantType at the reference's default widths; every int8 row and the layered path from at least two QuantTypes"""
    default = {(c.enc, c.nf4_ext) for c in CNNS if c.channels == 64 and c.widths == DEFAULT}
    assert default == {(e, False) for e in P.QUANT_IDS.values()} | {(M.ENC_NF4, True)}
    for row in [r for r, _ in CHAIN_ROWS] + [LAYERED]:
        assert len({c.enc for c in CNNS if c.row == row}) >= 2, row


# ---- GPU helpers ------------------------------------------------------------------------------------------------------------

def decisions(capfd):
    """the `fused launch:` decisions printed since the last call"""
    return [l.split("fused launch: ")[1] for l in capfd.readouterr().err.splitlines() if "fused launch: " in l]


def built_engine(capfd, monkeypatch, m, row, nf4_ext=False, cnn_frontend=None):
    """the model's engine with BNM_VERBOSE; asserts the plan's int8 row (or that no plan serves it) -> (engine, Sweep or None)"""
    from bitnetmcu_b200 import _lib

    def make():
        e = engine(m, cnn_frontend=cnn_frontend)
        if nf4_ext:
            e.set_option(_lib.OPT_NF4_EXTENSION, 1)
        return e
    e, err = verbose_engine(capfd, monkeypatch, make)
    line = plan_line(err)
    if row == LAYERED:
        assert line is None and e.active_path == _lib.PATH_LAYERS, err
        return e, None
    assert line and e.active_path == _lib.PATH_TCGEN05, err
    got, ring = plan_ring(line, "int8")
    assert got == row, line
    return e, ring


class Dev:
    """one model's images and expectations on the device; rows of a batch of n are the model's images i % N_UNIQUE"""

    def __init__(self, kind, name, judge):
        import torch
        self.m, self.ext, self.exact, q, lo, la, x, xlo, xla, emu = case_data(kind, name, judge)
        self.name, self.C = name, self.m.n_classes
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
        self.q_np, self.x_np, self.q, self.x = q, x, t(q), t(x)
        self.lo_np, self.la_np, self.xlo_np, self.xla_np = lo, la, xlo, xla
        self.lo, self.la, self.xlo, self.xla = t(lo), t(la.astype(np.int32)), t(xlo), t(xla.astype(np.int32))
        if emu is not None:
            self.emu, self.emu_la = t(emu), t(np.argmax(emu, axis=1).astype(np.int32))

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


@functools.lru_cache(maxsize=None)
def _sm():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def grid_n():
    """a launch that fills the grid with two tiles per SM and a ragged third round on some CTAs"""
    return 2 * _sm() * TILE + 77


def gather_dst(log, lab, off):
    from bitnetmcu_b200 import _lib
    g = _lib.BnmGather()
    g.n_logits_dst, g.n_labels_dst, g.row_offset = int(log is not None), int(lab is not None), off
    if log is not None:
        g.logits_dst[0] = log.data_ptr()
    if lab is not None:
        g.labels_dst[0] = lab.data_ptr()
    return g


# ---- GPU: the mode-2 decisions of every fed route --------------------------------------------------------------------------

DECISION_CASES = [("float", n) for n in FLOAT_IDS] + [("cnn-int8-cuda-cores", "binary-64"), ("cnn-int8-tensor-cores", "binary-64"),
                                                      ("cnn-float", "ternary-64"), ("cnn-gather", "8bit-64-47")]


@pytest.mark.gpu
@pytest.mark.parametrize("route,name", DECISION_CASES, ids=[f"{r}-{n}" for r, n in DECISION_CASES])
def test_mode2_decisions_of_fed_launches(lib, capfd, monkeypatch, route, name):
    """on one stream: plain int8 -> fed -> plain int8, fed -> fed at two batch sizes, and a fed call of two passes.  In mode 2
    every fed launch and the int8 launch right after one prints `wait`; two plain int8 launches on disjoint buffers still print
    `independent` (FC models; CNN models hold every launch at mode 1).  Modes 0 and 1 always wait."""
    import torch
    from bitnetmcu_b200 import _lib
    cnn = route.startswith("cnn")
    m = make_cnn(name) if cnn else make_float_model(FLOAT_ROWS[FLOAT_IDS.index(name)])
    fe = {"cnn-int8-cuda-cores": _lib.CNN_CUDA_CORES, "cnn-int8-tensor-cores": _lib.CNN_TENSOR_CORES}.get(route)
    e, _ = verbose_engine(capfd, monkeypatch, lambda: engine(m, _lib.PATH_TCGEN05, cnn_frontend=fe))
    C_, D = m.n_classes, m.img_bytes
    s = torch.cuda.Stream()
    ns = (1000, 3000)
    rng = np.random.default_rng(5)
    q = [torch.from_numpy(rng.integers(-128, 128, size=(3000, D)).astype(np.int8)).cuda() for _ in range(2)]
    f = [torch.from_numpy(rng.standard_normal(size=(3000, D)).astype(np.float32)).cuda() for _ in range(2)]
    lo = [torch.empty((TWO_PASSES, C_), dtype=torch.int32, device="cuda") for _ in range(4)]
    la = [torch.empty(TWO_PASSES, dtype=torch.int32, device="cuda") for _ in range(4)]
    dlo = torch.empty((TWO_PASSES, C_), dtype=torch.int32, device="cuda")
    g = gather_dst(dlo, None, 0)

    def plain(k, n=ns[0]):
        return ("plain", lambda: e.infer_device(q[k][:n], lo[k][:n], la[k][:n], stream=s.cuda_stream))

    def fed(k, n, big=None):
        o = (lo[2 + k][:n], la[2 + k][:n])
        if route == "float" or route == "cnn-float":
            x = big if big is not None else f[k][:n]
            return ("fed", lambda: e.infer_device_f32(x, *o, stream=s.cuda_stream))
        x = big if big is not None else q[k][:n]
        if route == "cnn-gather":
            return ("fed", lambda: gather_call(lib, e, x, o[0], o[1], g, s))
        return ("fed", lambda: e.infer_device(x, *o, stream=s.cuda_stream))

    def want(mode, calls):
        """the rule: independent only for a plain FC int8 launch right after another (disjoint buffers) in mode 2"""
        kinds = [k for k, _ in calls]
        return ["independent" if mode == 2 and not cnn and i > 0 and k == "plain" and kinds[i - 1] == "plain" else "wait"
                for i, k in enumerate(kinds)]

    def run(mode, *calls):
        e.set_option(_lib.OPT_LAUNCH_OVERLAP, mode)
        torch.cuda.synchronize()
        decisions(capfd)
        with torch.cuda.stream(s):
            for _, call in calls:
                call()
        s.synchronize()
        return decisions(capfd)

    big = (torch.randn((TWO_PASSES, D), device="cuda") if route in ("float", "cnn-float")
           else torch.randint(-128, 128, (TWO_PASSES, D), dtype=torch.int8, device="cuda"))
    sequences = {
        "plain, plain": [plain(0), plain(1)],
        "plain, fed, plain": [plain(0), fed(0, ns[0]), plain(1)],
        "plain, plain, fed, plain, plain": [plain(0), plain(1), fed(0, ns[0]), plain(0), plain(1)],
        "fed, fed at two sizes": [plain(0), fed(0, ns[0]), fed(1, ns[1]), plain(1)],
        "fed of two passes": [plain(1), fed(0, TWO_PASSES, big), plain(0)],
    }
    for mode in (0, 1, 2):
        for what, calls in sequences.items():
            got = run(mode, *calls)
            # a fed call of two passes is two fed launches
            w = want(mode, calls)
            if what == "fed of two passes":
                w = w[:2] + ["wait"] + w[2:]
            assert got == w, (route, name, mode, what, got)
    e.close()


@pytest.mark.gpu
def test_mode2_captured_fed_sequence(lib, judge, capfd, monkeypatch):
    """Binary-160 in mode 2, captured on one stream: int8, float, int8 on disjoint buffers -> wait (captured) three times; every
    replay equals the eager calls and the reference"""
    import torch
    from bitnetmcu_b200 import _lib
    d = Dev("float", "binary160", judge)
    e, _ = verbose_engine(capfd, monkeypatch, lambda: engine(d.m, _lib.PATH_TCGEN05))
    e.set_option(_lib.OPT_LAUNCH_OVERLAP, 2)
    n = grid_n()
    i = d.idx(n)
    x0, x1, xf = d.q[i].contiguous(), d.q[(i + 7) % N_UNIQUE].contiguous(), d.x[i].contiguous()
    outs = [(torch.empty((n, d.C), dtype=torch.int32, device="cuda"), torch.empty(n, dtype=torch.int32, device="cuda")) for _ in range(3)]

    def seq():
        e.infer_device(x0, *outs[0])
        e.infer_device_f32(xf, *outs[1])
        e.infer_device(x1, *outs[2])
    try:
        torch.cuda.synchronize()
        decisions(capfd)
        seq()
        torch.cuda.synchronize()
        assert decisions(capfd) == ["wait", "wait", "wait"]
        eager = [tuple(kernel_clone(t) for t in o) for o in outs]
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            seq()
        assert decisions(capfd) == ["wait (captured)"] * 3
        for r in range(2):
            for lo, la in outs:
                lo.fill_(-5)
                la.fill_(-7)
            torch.cuda.synchronize()
            graph.replay()
            torch.cuda.synchronize()
            for k, ((lo, la), (elo, ela)) in enumerate(zip(outs, eager)):
                assert torch.equal(lo, elo) and torch.equal(la, ela), ("replay", r, k)
        want = [(d.lo, d.la, i), (d.xlo, d.xla, i), (d.lo, d.la, (i + 7) % N_UNIQUE)]
        for k, ((lo, la), (wlo, wla, wi)) in enumerate(zip(outs, want)):
            assert torch.equal(lo, wlo[wi]) and torch.equal(la, wla[wi]), ("reference", k)
        assert decisions(capfd) == []
        del graph
    finally:
        e.close()


# ---- GPU: every row at its sweep -----------------------------------------------------------------------------------------------

def _sweep(d, ring, row, call, n_sizes, want_lo, want_la, what):
    """call(x, logits, labels) at every size of the row's ring sweep (LAYER_SIZES layer by layer): logits and labels, then
    labels only; sentinels past row n survive"""
    import torch
    sizes = Sweep(row, ring).sizes if ring else LAYER_SIZES
    for n in sizes:
        x = n_sizes(n)
        lo, la = out((n, d.C), torch.int32, -5), out((n,), torch.int32, -7)
        call(x, lo[:n], la[:n])
        torch.cuda.synchronize()
        d.check(n, lo, want_lo, -5, f"{what} logits")
        d.check(n, la, want_la, -7, f"{what} labels")
        la.fill_(-7)
        call(x, None, la[:n])
        torch.cuda.synchronize()
        d.check(n, la, want_la, -7, f"{what} labels only")
        del x


@pytest.mark.gpu
@pytest.mark.parametrize("name", CNN_IDS)
def test_cnn_int8_route_sweep(lib, judge, capfd, monkeypatch, name):
    """the CNN int8 route (front-end features into the fused FC kernel, or layer by layer) on its row's ring sweep"""
    c = CNNS[CNN_IDS.index(name)]
    d = Dev("cnn", name, judge)
    e, ring = built_engine(capfd, monkeypatch, d.m, c.row, c.nf4_ext)
    _sweep(d, ring, c.row, lambda x, lo, la: e.infer_device(x, lo, la), lambda n: d.q[d.idx(n)], d.lo, d.la, "int8")
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("row", FLOAT_ROWS, ids=FLOAT_IDS)
def test_float_route_sweep(lib, judge, capfd, monkeypatch, row):
    """float input on an FC model without a float-input form (k_quantize_images into scratch, then the int8 form) on the row's
    ring sweep"""
    name = FLOAT_IDS[FLOAT_ROWS.index(row)]
    d = Dev("float", name, judge)
    e, ring = built_engine(capfd, monkeypatch, d.m, row)
    _sweep(d, ring, row, lambda x, lo, la: e.infer_device_f32(x, lo, la), lambda n: d.x[d.idx(n)], d.xlo, d.xla, "float")
    e.close()


# ---- GPU: every entry at one grid-filling size -----------------------------------------------------------------------------

def windows_check(e, d, judge, side=None):
    """the window scan at stride 1 on a page with at least two windows per tile of every SM: every window equals the float
    entry on the same window rows, and 389 windows equal the reference on their scaled rows"""
    import torch
    side = side or -(-(16 + int(np.ceil(np.sqrt(grid_n())))) // 4) * 4   # rows of whole 16-byte units
    page = np.random.default_rng(d.C + side).standard_normal(size=(side, side)).astype(np.float32)
    page[::5] *= np.float32(40.0)
    oh = side - 15
    wlo, wla = torch.full((oh, oh, d.C), -5, dtype=torch.int32, device="cuda"), torch.full((oh, oh), -7, dtype=torch.int32, device="cuda")
    plane = torch.from_numpy(page).cuda()
    e.infer_windows_device(plane, 1, wlo, wla)
    torch.cuda.synchronize()
    wins = plane.unfold(0, 16, 1).unfold(1, 16, 1).reshape(-1, 256).contiguous()
    flo, fla = torch.empty((oh * oh, d.C), dtype=torch.int32, device="cuda"), torch.empty(oh * oh, dtype=torch.int32, device="cuda")
    e.infer_device_f32(wins, flo, fla)
    torch.cuda.synchronize()
    assert torch.equal(wlo.reshape(-1, d.C), flo) and torch.equal(wla.reshape(-1), fla), (d.name, "windows vs float entry")
    pick = np.random.default_rng(3).choice(oh * oh, size=N_UNIQUE, replace=False)
    wn = np.lib.stride_tricks.sliding_window_view(page, (16, 16)).reshape(-1, 256)[pick]
    jlo, jla = judge.infer(d.m, scale_images(wn), d.ext)
    assert np.array_equal(flo.cpu().numpy()[pick], jlo) and np.array_equal(fla.cpu().numpy()[pick], jla.astype(np.int32)), \
        (d.name, "windows vs reference")


def float_entries(e, d, n):
    """the float entry, bnm_compare_engines_device (C labels, emulator labels and counts where the emulator is exact) and the
    emulator's logits bit for bit against restate.emulate"""
    import torch
    x = d.x[d.idx(n)]
    lo, la = out((n, d.C), torch.int32, -5), out((n,), torch.int32, -7)
    e.infer_device_f32(x, lo[:n], la[:n])
    torch.cuda.synchronize()
    d.check(n, lo, d.xlo, -5, "float logits")
    d.check(n, la, d.xla, -7, "float labels")
    truth = ((torch.arange(n, device="cuda") * 7) % (d.C + 1)).to(torch.int32)
    lc, lp = out((n,), torch.int32, -7), out((n,), torch.int32, -7)
    counts = torch.zeros(4, dtype=torch.int64, device="cuda")
    e.compare_engines_device(x, truth, lc[:n], lp[:n], counts)
    torch.cuda.synchronize()
    d.check(n, lc, d.xla, -7, "engines: C labels")
    wc = d.xla[d.idx(n)]
    got = counts.cpu().tolist()
    assert got[:2] == [n, int((wc == truth).sum())], (d.name, "engines: counts", got)
    if d.exact:
        d.check(n, lp, d.emu_la, -7, "engines: emulator labels")
        wp = d.emu_la[d.idx(n)]
        assert got[2:] == [int((wp == truth).sum()), int((wc != wp).sum())], (d.name, "engines: counts", got)
        elo, ela = out((n, d.C), torch.float64, -12345.5), out((n,), torch.int32, -7)
        e.inference_quantized_device(x, elo[:n], ela[:n])
        torch.cuda.synchronize()
        d.check(n, elo, d.emu, -12345.5, "emulator logits")
        d.check(n, ela, d.emu_la, -7, "emulator labels")


@pytest.mark.gpu
@pytest.mark.parametrize("name", CNN_IDS)
def test_cnn_entries(lib, judge, capfd, monkeypatch, name):
    """one grid-filling size on every entry that runs the CNN front-end into the FC stage: device int8 on every front-end, float,
    the host pipeline, gather, the window scan, both engines and the emulator"""
    import torch
    c = CNNS[CNN_IDS.index(name)]
    d = Dev("cnn", name, judge)
    n = grid_n()
    i = np.arange(n) % N_UNIQUE
    for fe in frontends(d.m):
        e, _ = built_engine(capfd, monkeypatch, d.m, c.row, c.nf4_ext, cnn_frontend=fe)
        lo, la = out((n, d.C), torch.int32, -5), out((n,), torch.int32, -7)
        e.infer_device(d.q[d.idx(n)], lo[:n], la[:n])
        torch.cuda.synchronize()
        d.check(n, lo, d.lo, -5, f"int8 logits, front-end {fe}")
        d.check(n, la, d.la, -7, f"int8 labels, front-end {fe}")
        e.close()
    e, _ = built_engine(capfd, monkeypatch, d.m, c.row, c.nf4_ext)
    hlo, hla = e.infer(d.q_np[i])
    assert np.array_equal(hlo, d.lo_np[i]) and np.array_equal(hla, d.la_np[i]), (name, "host pipeline")
    if c.row != LAYERED:   # the result exchange is a fused-kernel output
        s = torch.cuda.Stream()
        lo, la = out((n, d.C), torch.int32, -5), out((n,), torch.int32, -7)
        dlo, dla = out((n + 64, d.C), torch.int32, -5), out((n + 64,), torch.int32, -7)
        rc = gather_call(lib, e, d.q[d.idx(n)], lo[:n], la[:n], gather_dst(dlo, dla, 64), s)
        assert rc == 0, (name, "gather", rc)
        d.check(n, lo, d.lo, -5, "gather logits")
        d.check(n, la, d.la, -7, "gather labels")
        d.check(n, dlo[64:], d.lo, -5, "gather logits destination")
        d.check(n, dla[64:], d.la, -7, "gather labels destination")
        assert bool((dlo[:64] == -5).all() and (dla[:64] == -7).all()), (name, "gather rows before the offset")
    float_entries(e, d, n)
    windows_check(e, d, judge)
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("row", FLOAT_ROWS, ids=FLOAT_IDS)
def test_float_model_entries(lib, judge, capfd, monkeypatch, row):
    """one grid-filling size on the float entries of an FC model without a float-input form: float, both engines, the emulator,
    and the window scan where images are 16 x 16"""
    name = FLOAT_IDS[FLOAT_ROWS.index(row)]
    d = Dev("float", name, judge)
    e, _ = built_engine(capfd, monkeypatch, d.m, row)
    float_entries(e, d, grid_n())
    if d.m.img_bytes == 256:
        windows_check(e, d, judge)
    e.close()


# ---- GPU: kernel producers and consumers next to fed calls ------------------------------------------------------------------

NEIGHBOUR_CASES = [("float", "binary160"), ("float", "4bitsym-37-classes"), ("cnn", "ternary-64"), ("cnn", "fp130-48-96")]


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [0, 2])
@pytest.mark.parametrize("kind,name", NEIGHBOUR_CASES, ids=[n for _, n in NEIGHBOUR_CASES])
def test_kernel_neighbours_of_fed_calls(lib, judge, capfd, monkeypatch, kernel_copies_are_kernels, kind, name, mode):
    """fed calls alternate with int8 calls (FC: plain int8; CNN: the CNN int8 call, fed too) at a grid-filling size on one
    stream, with the caller's mode-2 promise kept: double-buffered inputs and outputs, each call's inputs written by a kernel one
    call ahead (before the call before it), its outputs read by kernels right after it.  Every launch waits, every output is
    exact.  Whether a race shows in one run depends on timing; the decision tests above are the guard."""
    import torch
    from bitnetmcu_b200 import _lib
    d = Dev(kind, name, judge)
    row = FLOAT_ROWS[FLOAT_IDS.index(name)] if kind == "float" else CNNS[CNN_IDS.index(name)].row
    e, _ = built_engine(capfd, monkeypatch, d.m, row)
    e.set_option(_lib.OPT_LAUNCH_OVERLAP, mode)
    n, calls = grid_n(), 8
    # call k: even k the float (fed) call, odd k the int8 call; inputs of call k are the images rotated by 11 k
    idx = [(d.idx(n) + 11 * k) % N_UNIQUE for k in range(calls)]
    src = [(d.x if k % 2 == 0 else d.q)[idx[k]].contiguous() for k in range(calls)]
    bufs = [torch.empty_like(src[k]) for k in range(4)]                     # two per kind
    outs = [(torch.empty((n, d.C), dtype=torch.int32, device="cuda"), torch.empty(n, dtype=torch.int32, device="cuda")) for _ in range(4)]
    as_int = lambda t: t.view(torch.int32) if t.dtype == torch.float32 else t
    s = torch.cuda.Stream()
    got = []
    with torch.cuda.stream(s):
        kernel_copy(as_int(bufs[0]), as_int(src[0]))
        torch.cuda.synchronize()
        decisions(capfd)
        for k in range(calls):
            if k + 1 < calls:
                kernel_copy(as_int(bufs[(k + 1) % 4]), as_int(src[k + 1]))
            lo, la = outs[k % 4]
            if k % 2 == 0:
                e.infer_device_f32(bufs[k % 4], lo, la)
            else:
                e.infer_device(bufs[k % 4], lo, la)
            got.append((kernel_clone(lo), kernel_clone(la)))
        s.synchronize()
    assert decisions(capfd) == ["wait"] * calls, (name, mode)
    for k, (lo, la) in enumerate(got):
        wlo, wla = (d.xlo, d.xla) if k % 2 == 0 else (d.lo, d.la)
        assert torch.equal(lo, wlo[idx[k]]), (name, mode, k, "logits")
        assert torch.equal(la, wla[idx[k]]), (name, mode, k, "labels")
    e.close()
