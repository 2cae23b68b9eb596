"""FC models whose layers differ in what the fused plan lays out per layer (fc_chain_plan_create, fc_wgmma.cu): residual weight
planes in some layers only, and encodings that change from layer to layer.

The plan gives each layer its own plane count (2 where an FP130 layer holds a +128 weight, whose residual +1 goes to a second
int8 plane), its own K-steps (Ternary's inputs padded to tens, steps past the previous layer's width dropped) and its own byte
offset in the shared-memory weight image, the running sum over the layers before it.  A wrong offset shows only on a layer after
one with two planes; the fixed-shape row is taken only where every layer has one plane; the emulator's logits take the last
layer's level scale alone.  Models with one encoding throughout (every fixture, random_fc) have plane patterns of all 1s or all
2s, so none of that is visible on them.

Models.  12k_FP130's trained weights with +128 in every subset of its four layers, and the same subsets on a 37-class head;
FP130 models with +128 in the first or in the last layer on every one-pipe row; chains of mixed encodings, every encoding as a
first, a hidden and a last layer, both emulator logit scales after a first layer of the other scale, and a mixed chain of the
fixed shape.

CPU: the plan's weight layout and rows restated in NumPy (restate.plan_of), the coverage of the cases, and the oracle and the
emulator restatement against the unmodified reference where it is present.  GPU (tolerance 0): the plan line against the
restatement, then every entry the plan serves at 1, 129 and a size past two trips round the ring of every form it launches, and
the layer-by-layer path."""
import functools
import os
import re
import sys
from typing import Callable, NamedTuple

import numpy as np
import pytest

from bitnetmcu_b200 import model as M, pack as P
from conftest import load_model
from restate import LEVEL_SHIFT, Plan, emulate, plan_of, scale_images
from support import (Sweep, both_engines, c_float, chain, emulator, fp130_codes, int8_images, lib, out, plan_line, plan_ring,  # noqa: F401
                     quantized_model_list, scattered_edge_images, to_device as t, top_k, verbose_engine,             # (lib: fixture)
                     with_plus128)

REF_PY = "/root/reference"
N_UNIQUE = 389          # distinct images per model; batches repeat them (row i is image i % N_UNIQUE)
B, S2, S4, U4, I8, F, NF4, T = (M.ENC_BINARY, M.ENC_2BITSYM, M.ENC_4BITSYM, M.ENC_4BIT, M.ENC_8BIT, M.ENC_FP130, M.ENC_NF4,
                                M.ENC_TERNARY)
PLUS = True             # an FP130 layer with +128 weights
MAX_TOPK = 16           # the top-k entries take k <= min(n_classes, 16)


FIXED_ROW = "<64,2,2,16,fixed>"


# ---- the models --------------------------------------------------------------------------------------------------------------

def fp130_subset(subset, classes):
    """12k_FP130 with +128 in the layers of `subset`; classes != 10: its first three layers and a random FP130 head"""
    fc = load_model("12k_FP130").fc_layers
    codes = [P.unpack_codes(l.weights[:l.n_out * l.n_in // 8], 4, l.n_out, l.n_in) for l in fc]
    if classes != 10:
        codes[3] = fp130_codes(np.random.default_rng(classes), classes, 64)
    m = M.Model(model_class=M.MODEL_FCMNIST, img_bytes=256,
                layers=[P.fc_layer_from_codes(f"L{i + 1}", F, with_plus128(c, i) if i in subset else c) for i, c in enumerate(codes)])
    m.validate()
    return m


class Case(NamedTuple):
    name: str
    row: str                # the int8 row of the fused plan
    make: Callable
    kind: str               # "subset", "one-pipe" or "mixed"
    nf4_ext: bool = False


def _subset_cases():
    out = []
    for classes in (10, 37):
        for bits in range(16):
            subset = [l for l in range(4) if bits >> l & 1]
            row = "<64,2,2,64>" if classes == 37 else "<64,2,2,16>" if subset else FIXED_ROW
            planes = "".join("2" if l in subset else "1" for l in range(4))
            out.append(Case(f"12k_FP130-{classes}cls-{planes}", row, functools.partial(fp130_subset, tuple(subset), classes), "subset"))
    return out


def _one_pipe_cases():
    out = []
    for row, img, widths in (("<64,1>", 512, (64, 64, 10)), ("<128,1>", 256, (96, 64, 10)), ("<192,1>", 256, (160, 160, 10)),
                             ("<256,1>", 256, (256, 10))):
        for where, at in (("first", 0), ("last", len(widths) - 1)):
            layers = tuple((F, w, PLUS) if i == at else (F, w) for i, w in enumerate(widths))
            out.append(Case(f"fp130-{img}-{'-'.join(map(str, widths))}-{where}", row,
                            functools.partial(chain, img, layers, 100 + len(out)), "one-pipe"))
    return out


MIXED = [
    # the emulator's logit scale 0.5 (4bitsym) after a first layer of scale 1; Ternary's 64 inputs padded to 70
    ("8bit-ternary-binary-4bitsym", FIXED_ROW, 256, ((I8, 64), (T, 64), (B, 64), (S4, 10))),
    ("2bitsym-8bit-fp130+-4bit", "<64,2,2,16>", 256, ((S2, 64), (I8, 64), (F, 64, PLUS), (U4, 10))),
    # the fixed shape, FP130 with -128 but no +128
    ("ternary-fp130-4bitsym-fp130", FIXED_ROW, 256, ((T, 64), (F, 64), (S4, 64), (F, 10))),
    # scale 1 (8bit) after a first layer of scale 0.5; 16 classes
    ("4bitsym-fp130+-binary-8bit", "<64,2,2,16>", 256, ((S4, 64), (F, 64, PLUS), (B, 64), (I8, 16))),
    ("nf4-nf4-fp130+-nf4", "<64,2,2,16>", 256, ((NF4, 64), (NF4, 64), (F, 32, PLUS), (NF4, 12))),
    # Ternary's 32 inputs padded to 40: one K-step
    ("binary-2bitsym-4bit-ternary", "<64,2,2,16>", 256, ((B, 64), (S2, 64), (U4, 32), (T, 10))),
    # a second plane in layer 1 on 128-byte rows; scale 0.5 after 1
    ("fp130+-ternary-2bitsym-128", "<64,2,2,16>", 128, ((F, 64, PLUS), (T, 48), (S2, 16))),
    ("4bit-fp130+-binary", "<64,2,2,16>", 256, ((U4, 32), (F, 64, PLUS), (B, 10))),
    # wider than 64 and more than 16 classes: k_quantize_images and the int8 forms serve their float entries
    ("8bit-fp130+-ternary-96", "<128,1>", 256, ((I8, 96), (F, 64, PLUS), (T, 10))),
    ("2bitsym-4bitsym-fp130+-37cls", "<64,2,2,64>", 256, ((S2, 64), (S4, 64), (F, 37, PLUS))),
]
CASES = _subset_cases() + _one_pipe_cases() + [
    Case(name, row, functools.partial(chain, img, layers, 200 + i), "mixed", nf4_ext=any(l[0] == NF4 for l in layers))
    for i, (name, row, img, layers) in enumerate(MIXED)]
BY_NAME = {c.name: c for c in CASES}
NAMES = list(BY_NAME)


@functools.lru_cache(maxsize=None)
def model(name):
    return BY_NAME[name].make()


@functools.lru_cache(maxsize=None)
def layout(name):
    return plan_of(model(name), BY_NAME[name].nf4_ext)


# ---- CPU: the layout and the cases -----------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", NAMES)
def test_restated_layout(name):
    """each model's restated plan: its stated row, the plane pattern its construction gives, offsets that sum the planes and
    K-steps of every earlier layer, and a weight image that fits"""
    c, m, lay = BY_NAME[name], model(name), layout(name)
    assert isinstance(lay, Plan) and lay.row == c.row, (name, lay)
    fc = m.fc_layers
    assert lay.planes == [1 + int(l.bitperweight == F and (P.decode_int_weights(l) == 128).any()) for l in fc]
    for l in range(1, len(fc)):
        assert lay.b_off[l] - lay.b_off[l - 1] == lay.planes[l - 1] * lay.k_steps[l - 1] * lay.n_pad[l - 1] * 32
    if c.kind == "subset":
        assert lay.planes == [int(ch) for ch in name[-4:]] and lay.float_forms == (m.n_classes == 10)
    for l, layer in enumerate(fc[1:], 1):
        if layer.bitperweight == T and layer.n_in % 32:
            assert lay.k_steps[l] == -(-fc[l - 1].n_out // 32), (name, l)   # the padded trits past the previous width dropped


def test_layout_restatement_edges():
    """the rules on known models: the fixture rows, the fixed shape with residual planes (general row), 512-byte rows (one pipe),
    and a Ternary layer after a 32-wide one (32 inputs padded to 40, K padded to 64: one K-step, from the previous width)"""
    fixed = plan_of(load_model("fc"))
    assert fixed.row == FIXED_ROW and fixed.w_bytes == 27648 and fixed.b_off == [0, 16384, 20480, 24576] and fixed.logit_scale == 0.5
    res = plan_of(load_model("rand_fp130_64"))
    assert res.row == "<64,2,2,16>" and res.planes == [2] * 4 and res.b_off == [0, 32768, 40960, 49152] and res.w_bytes == 53248
    assert res.float_forms and res.logit_scale == 1.0
    wide = plan_of(model("fp130-512-64-64-10-first"))
    assert wide.row == "<64,1>" and wide.k_steps == [16, 2, 2] and wide.planes == [2, 1, 1] and not wide.float_forms
    t = plan_of(chain(256, ((I8, 32), (T, 64), (I8, 10)), 0))
    assert t.k_steps == [8, 1, 2] and t.n_pad == [32, 64, 16] and t.b_off == [0, 8192, 10240]


def test_cases_cover_every_layout():
    """what the GPU tests run: fails when a case that carries one of these goes"""
    lays = {n: layout(n) for n in NAMES}
    # a second plane at every layer position on each 64-wide two-pipe row, and one before a layer with one plane
    for row in ("<64,2,2,16>", "<64,2,2,64>"):
        on = [lays[n] for n in NAMES if lays[n].row == row]
        assert {l for lay in on if len(lay.planes) == 4 for l in range(4) if lay.planes[l] == 2} == {0, 1, 2, 3}, row
        assert any(2 in lay.planes[:-1] and 1 in lay.planes[lay.planes.index(2) + 1:] for lay in on), row
    # the one-kernel float forms run a second plane at every position of a four-layer model, and at the first of another
    on = [lays[n] for n in NAMES if lays[n].float_forms]
    assert {l for lay in on if len(lay.planes) == 4 for l in range(4) if lay.planes[l] == 2} == {0, 1, 2, 3}
    assert any(lay.planes[0] == 2 and lay.planes[1] == 1 for lay in on)
    # a second plane at the first and the last position on each one-pipe row
    for row in ("<64,1>", "<128,1>", "<192,1>", "<256,1>"):
        on = [lays[n].planes for n in NAMES if lays[n].row == row]
        assert any(p[0] == 2 and p[1:] == [1] * (len(p) - 1) for p in on), row
        assert any(p[-1] == 2 and p[:-1] == [1] * (len(p) - 1) for p in on), row
    # the fixed row: one encoding (12k_FP130 as trained) and mixed encodings, every plane 1
    fixed = [n for n in NAMES if lays[n].row == FIXED_ROW]
    assert any(len({l.bitperweight for l in model(n).fc_layers}) >= 3 for n in fixed) and "12k_FP130-10cls-1111" in fixed
    # every encoding as a first, a hidden and a last layer of the mixed chains
    mixed = [n for n in NAMES if BY_NAME[n].kind == "mixed"]
    seen = {(l.bitperweight, "first" if i == 0 else "last" if i + 1 == len(model(n).fc_layers) else "hidden")
            for n in mixed for i, l in enumerate(model(n).fc_layers)}
    assert seen == {(e, p) for e in P.QUANT_IDS.values() for p in ("first", "hidden", "last")}, seen
    # both emulator logit scales after a first layer of the other scale: on the one-kernel float forms, and scale 1 after 0.5
    # on the int8 emulator form too
    def scales(float_forms):
        return {(2.0 ** -LEVEL_SHIFT.get(model(n).fc_layers[0].bitperweight, 0), lays[n].logit_scale) for n in mixed
                if lays[n].float_forms == float_forms}
    assert {(1.0, 0.5), (0.5, 1.0)} <= scales(True), scales(True)
    assert (0.5, 1.0) in scales(False), scales(False)
    # mixed chains past the float forms' limits: wider than 64, more than 16 classes
    assert {lays[n].row for n in mixed if not lays[n].float_forms} == {"<128,1>", "<64,2,2,64>"}
    assert any(BY_NAME[n].nf4_ext for n in mixed)


# ---- CPU: the models against the unmodified reference -------------------------------------------------------------------------

REFERENCE_SAMPLE = [n for n in NAMES if BY_NAME[n].kind != "subset" or n[-4:] in ("1111", "2222", "2111", "1112", "1212")]


@pytest.mark.parametrize("name", [n for n in REFERENCE_SAMPLE if not BY_NAME[n].nf4_ext])
def test_oracle_matches_reference(oracle, reference, name):
    """the C restatement equals the unmodified reference: int8 rows at the rails, all zero, random, and scaled float rows"""
    m = model(name)
    q = int8_images(N_UNIQUE, m.img_bytes, 7)
    for imgs, what in ((q, "int8"), (scale_images(scattered_edge_images(N_UNIQUE, m.img_bytes, 8)), "scaled float")):
        want_lo, want_la = reference.infer(m, imgs)
        lo, la = oracle.infer(m, imgs)
        assert np.array_equal(lo, want_lo) and np.array_equal(la, want_la), (name, what)


@pytest.mark.skipif(not os.path.isfile(os.path.join(REF_PY, "BitNetMCU.py")), reason="needs the reference's BitNetMCU.py")
@pytest.mark.parametrize("name", REFERENCE_SAMPLE)
def test_emulate_matches_reference_emulator(name):
    """restate.emulate equals the reference's QuantizedModel.inference_quantized on the engine's integer levels (4bit and NF4
    layers too, NF4 with the extension where the case has it)"""
    if REF_PY not in sys.path:
        sys.path.append(REF_PY)
    from BitNetMCU import QuantizedModel
    m, ext = model(name), BY_NAME[name].nf4_ext
    x = scattered_edge_images(N_UNIQUE, m.img_bytes, 9)
    qm = QuantizedModel()
    qm.quantized_model = quantized_model_list(m, ext)
    assert np.array_equal(emulate(m, x, nf4_extension=ext), np.asarray(qm.inference_quantized(x), dtype=np.float64)), name


# ---- GPU helpers --------------------------------------------------------------------------------------------------------------

class Data:
    """one model's N_UNIQUE images and expectations on the device; row i of a batch of n is image i % N_UNIQUE"""

    def __init__(self, name, oracle):
        self.name, self.m, self.ext, self.oracle = name, model(name), BY_NAME[name].nf4_ext, oracle
        self.C = self.m.n_classes
        seed = NAMES.index(name)
        self.q_np = int8_images(N_UNIQUE, self.m.img_bytes, seed)
        self.x_np = scattered_edge_images(N_UNIQUE, self.m.img_bytes, seed + 1000)
        self.lo_np, la = oracle.infer(self.m, self.q_np, nf4_extension=self.ext)
        self.la_np = la.astype(np.int32)
        xlo, xla = oracle.infer(self.m, scale_images(self.x_np), nf4_extension=self.ext)
        self.q, self.x, self.lo, self.la, self.xlo, self.xla = map(t, (self.q_np, self.x_np, self.lo_np, self.la_np, xlo, xla.astype(np.int32)))
        self.ks = sorted({1, 5, min(self.C, MAX_TOPK)})
        self.topk_c = {k: tuple(map(t, top_k(self.lo_np, k))) for k in self.ks}
        emu = emulate(self.m, self.x_np, nf4_extension=self.ext)
        self.emu, self.emu_la = t(emu), t(np.argmax(emu, axis=1).astype(np.int32))
        self.topk_py = {k: tuple(map(t, top_k(emu, k))) for k in self.ks}
        self.half = {}   # format -> the float32 entries' results on the widened rows (half_results)

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


_DATA = {}


def data(name, oracle):
    if name not in _DATA:
        _DATA.clear()   # one model's device buffers at a time
        _DATA[name] = Data(name, oracle)
    return _DATA[name]


def built_engine(capfd, monkeypatch, name):
    """the model's engine, its plan line checked against the restatement -> (engine, a batch size past two trips round the ring
    of every form the plan launches)"""
    from bitnetmcu_b200 import _lib
    from bitnetmcu_b200.engine import Engine
    e, err = verbose_engine(capfd, monkeypatch, lambda: Engine(model(name), device=0, nf4_extension=BY_NAME[name].nf4_ext))
    line, lay = plan_line(err), layout(name)
    assert line and e.active_path == _lib.PATH_TCGEN05, err
    row, ring = plan_ring(line, "int8")
    assert row == BY_NAME[name].row == lay.row, (name, line)
    assert int(re.search(r"(\d+) weight bytes", line).group(1)) == lay.w_bytes, (name, line, lay)
    assert int(re.search(r"(\d+) pipes", line).group(1)) == lay.pipes, (name, line)
    assert ("float input <" in line) == lay.float_forms, (name, line)
    rings = [("int8", ring), ("int8 emulator", plan_ring(line, "emul_i8")[1])]
    if lay.float_forms:
        rings += [("float input", plan_ring(line, "float")[1]), ("float emulator", plan_ring(line, "emul")[1])]
    topk = [l for l in err if "fused FC top-k forms" in l][-1]
    rings += [(f"top-k {r}", (1, int(st), 1)) for r, st in re.findall(r"fc_topk_kernel(<[^>]*>) x (\d+) stages", topk)]
    return e, max(Sweep(f"{name} {kind}", r).sizes[-1] for kind, r in rings)


def half_results(e, d, fmt):
    """the float32 entries' results (C engine, emulator) on the N_UNIQUE rows widened from fmt, which the 16-bit entries must
    equal; on the rows that stay finite they equal the oracle and restate.emulate"""
    import torch
    if fmt not in d.half:
        xw = d.x.to(getattr(torch, fmt)).float()
        r = {"lo": torch.empty((N_UNIQUE, d.C), dtype=torch.int32, device="cuda"), "la": torch.empty(N_UNIQUE, dtype=torch.int32, device="cuda")}
        e.infer_device_f32(xw, r["lo"], r["la"])
        r["emu"], r["emu_la"] = torch.empty((N_UNIQUE, d.C), dtype=torch.float64, device="cuda"), torch.empty_like(r["la"])
        e.inference_quantized_device(xw, r["emu"], r["emu_la"])
        torch.cuda.synchronize()
        xw_np = xw.cpu().numpy()
        fin = np.isfinite(xw_np).all(axis=1)
        assert fin.sum() > N_UNIQUE // 2, (d.name, fmt)
        wlo, wla = d.oracle.infer(d.m, scale_images(xw_np[fin]), nf4_extension=d.ext)
        assert np.array_equal(r["lo"].cpu().numpy()[fin], wlo), (d.name, fmt, "float32 logits on the widened rows")
        assert np.array_equal(r["la"].cpu().numpy()[fin], wla.astype(np.int32)), (d.name, fmt, "float32 labels on the widened rows")
        assert np.array_equal(r["emu"].cpu().numpy()[fin], emulate(d.m, xw_np[fin], nf4_extension=d.ext)), \
            (d.name, fmt, "emulator on the widened rows")
        d.half[fmt] = r
    return d.half[fmt]


def top_k_entries(e, d, n, q, x):
    """the C engine's top-k on the int8 rows, and the emulator's on the float rows: classes and scores"""
    import torch
    for k in d.ks:
        for what, fn, imgs, dtype, (want_cls, want_sc) in (("C engine", e.topk_device, q, torch.int32, d.topk_c[k]),
                                                           ("emulator", e.emulate_topk_device, x, torch.float64, d.topk_py[k])):
            cls, sc = out((n, k), torch.int32, -1), out((n, k), dtype, -7)
            fn(imgs, k, cls[:n], sc[:n])
            torch.cuda.synchronize()
            d.check(n, cls, want_cls, -1, f"{what} top-{k} classes")
            d.check(n, sc, want_sc, -7, f"{what} top-{k} scores")


# ---- GPU ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_plan(lib, capfd, monkeypatch, name):
    """the `fused FC plan` line: the restated row, weight bytes and pipes, and the float-input forms where they fit"""
    e, _ = built_engine(capfd, monkeypatch, name)
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_entries(lib, oracle, capfd, monkeypatch, name):
    """every entry the plan serves at 1, 129 and a size past two trips round every form's ring: int8 (logits and labels, labels
    alone), the host pipeline, float32, float16 and bfloat16, the emulator, both engines with counts, and top-k on both engines"""
    import torch
    d = data(name, oracle)
    e, big = built_engine(capfd, monkeypatch, name)
    try:
        for n in (1, 129, big):
            i = d.idx(n)
            q, x = d.q[i], d.x[i]
            lo, la = out((n, d.C), torch.int32, -5), out((n,), torch.int32, -7)
            e.infer_device(q, lo[:n], la[:n])
            torch.cuda.synchronize()
            d.check(n, lo, d.lo, -5, "int8 logits")
            d.check(n, la, d.la, -7, "int8 labels")
            la.fill_(-7)
            e.infer_device(q, None, la[:n])
            torch.cuda.synchronize()
            d.check(n, la, d.la, -7, "int8 labels only")
            hi = np.arange(n) % N_UNIQUE
            hlo, hla = e.infer(d.q_np[hi])
            assert np.array_equal(hlo, d.lo_np[hi]) and np.array_equal(hla.astype(np.int32), d.la_np[hi]), (name, n, "host pipeline")
            c_float(e, d, n, x, d.xlo, d.xla, "float32")
            emulator(e, d, n, x, d.emu, d.emu_la, "float32")
            both_engines(e, d, n, x, d.xla, d.emu_la, "float32")
            for fmt in ("float16", "bfloat16"):
                h, xh = half_results(e, d, fmt), x.to(getattr(torch, fmt))
                c_float(e, d, n, xh, h["lo"], h["la"], fmt)
                emulator(e, d, n, xh, h["emu"], h["emu_la"], fmt)
                both_engines(e, d, n, xh, h["la"], h["emu_la"], fmt)
                del xh
            top_k_entries(e, d, n, q, x)
            del q, x
    finally:
        e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_layered_path(lib, oracle, name):
    """BNM_PATH_LAYERS (one dp4a kernel per layer, each with its own residual plane) gives the same int8, float32 and emulator
    outputs"""
    import torch
    from bitnetmcu_b200 import _lib
    from bitnetmcu_b200.engine import Engine
    d = data(name, oracle)
    e = Engine(d.m, device=0, path=_lib.PATH_LAYERS, nf4_extension=d.ext)
    try:
        assert e.active_path == _lib.PATH_LAYERS
        for n in (1, 129, 5 * 128 + 37):
            i = d.idx(n)
            lo, la = out((n, d.C), torch.int32, -5), out((n,), torch.int32, -7)
            e.infer_device(d.q[i], lo[:n], la[:n])
            torch.cuda.synchronize()
            d.check(n, lo, d.lo, -5, "layered int8 logits")
            d.check(n, la, d.la, -7, "layered int8 labels")
            c_float(e, d, n, d.x[i], d.xlo, d.xla, "layered float32")
            emulator(e, d, n, d.x[i], d.emu, d.emu_la, "layered")
    finally:
        e.close()
