"""The fused FC plan across its shape space (fc_chain_plan_create, fc_wgmma.cu): seeded models at the edges of its rules, every
entry exact.

The plan decides from the layer shapes alone each layer's padded width (n_pad, n_out rounded up to 16) and K-steps (the K of a
layer after the first stops at the previous layer's n_pad, rounded up to 32), the accumulator width, one pipe or two, the
two-pipe row, whether the float-input forms exist, each form's stage count from the shared memory the weight image leaves, and
whether to refuse the model ("weights do not fit in shared memory": the layer-by-layer path serves it).  The kernel has code
that only padded shapes reach: the columns of a 64-wide wgmma piece past n_pad read the zero tile, the weight image is zero from
n_out to n_pad, and K-steps past the previous layer's n_pad multiply activations that must be zero.  Hand-picked models had
hidden layers 16k wide only; these draws have hidden layers 40, 72, 100 or 248 wide feeding K-steps rounded past them.

Models.  N_DRAWS seeded draws (draw()), biased to the edges: hidden widths on each encoding's input grid (8bit: steps of 4;
4bit, 4bitsym, FP130 and NF4: 8; Ternary: any, padded to tens) and not multiples of 16, widths at 16k, 16k + step and 64k +- a
step, a widest layer of 65 to 80 next to narrow ones, 1 to 8 layers, class counts at 16k and 64k +- 1, rows in 16-byte steps
that end inside a 128-byte atom, mixed encodings, FP130 with +128 in some layers only, NF4 with the extension.  Then crafted
models on each side of the shared-memory boundaries, found by searching a hidden width with restate.plan_of: the largest image
that leaves two stages (one pipe), the largest that leaves four stages for two pipes, and the next 16 columns past each.  The
float forms' own shared-memory clause never decides: the largest 64-wide image (eight FP130 layers with +128, 256-byte rows)
still leaves their rings and two stages (test_float_rings_fit_every_64_wide_image), so their boundaries are rows (256 | 272),
classes (16 | 17) and width (64 | 128).

CPU: the coverage of the draws (every class above, or the gap by name), the restated plan on known models, and the oracle
against the unmodified reference.  GPU (tolerance 0): the BNM_VERBOSE plan lines equal restate.plan_lines character for
character, a refused model reports its refusal and runs layer by layer; every entry at 1, 129 and a batch past the first trip
round every form's ring, against the unmodified reference (the oracle for NF4); float16 and bfloat16 on every fourth case.  On
an H100 80GB HBM3 (132 SMs, 700 W power limit) the GPU half of this module (128 tests) takes about 16 s."""
import functools
import re
from typing import NamedTuple

import numpy as np
import pytest

from bitnetmcu_b200 import model as M, pack as P
from restate import (REFUSE_SMEM, SMEM_LIMIT, Plan, batch_size, emulate, plan_lines, plan_of, scale_images,
                     tile_schedule)
from support import (both_engines, c_float, chain, emulator, int8_images, lib, out, plan_line,  # noqa: F401  (lib: fixture)
                     scattered_edge_images, to_device, top_k, verbose_engine)

N_UNIQUE = 389          # distinct images per model; batches repeat them (row i is image i % N_UNIQUE)
N_DRAWS = 48
B, S2, S4, U4, I8, F, NF4, T = (M.ENC_BINARY, M.ENC_2BITSYM, M.ENC_4BITSYM, M.ENC_4BIT, M.ENC_8BIT, M.ENC_FP130, M.ENC_NF4,
                                M.ENC_TERNARY)
ENCODINGS = (B, S2, S4, U4, I8, F, NF4, T)
STEP = {B: 32, S2: 16, S4: 8, U4: 8, F: 8, NF4: 8, I8: 4, T: 2}   # a layer's input grid: rows of whole 32-bit words; Ternary any
CLASSES = (1, 2, 15, 16, 17, 63, 64, 65, 129, 255, 256)
EDGE_ROWS = (16, 112, 144, 240, 272, 400, 640, 752)
THEMES = ("narrow", "acc65", "wide", "deep")
MAX_TOPK = 16


# ---- the models --------------------------------------------------------------------------------------------------------------

def legal(enc, n_in):
    """n_in inputs pack to whole words in enc (exportquant.py's rule); Ternary pads to tens"""
    return enc == T or P.CODE_BITS[enc] * n_in % 32 == 0


def edge_widths(enc, lo=1, hi=256):
    """widths on enc's input grid in [lo, hi]: 16k, 16k + step, 64k +- step, and the grid's points that are not multiples of 16"""
    s = STEP[enc]
    c = {16 * k for k in range(1, 17)} | {16 * k + s for k in range(0, 16)} | {64 * k + d for k in range(1, 5) for d in (-s, s)}
    c |= {w for w in range(s, 257, s) if w % 16}
    return sorted(w for w in c if lo <= w <= hi and legal(enc, w))


def draw(i):
    """draw i: a seeded FC model -> (layers as chain() takes them, image bytes)"""
    rng = np.random.default_rng(9000 + i)
    theme = THEMES[i % len(THEMES)]
    rows = int(rng.choice(EDGE_ROWS)) if rng.random() < 0.6 else 16 * int(rng.integers(1, 49))
    if theme in ("wide", "narrow"):   # narrow: rows the float-input forms take; wide: rows that leave room for wide images
        rows = min(rows, 256 if theme == "narrow" else 400)
    n_layers = int(rng.integers(5, 9)) if theme == "deep" else int(rng.integers(1, 5))
    encs = [int(rng.choice([e for e in ENCODINGS if legal(e, rows)]))] + [int(rng.choice(ENCODINGS)) for _ in range(n_layers - 1)]
    classes = int(rng.choice([c for c in CLASSES if c <= (64 if theme == "acc65" else 16 if theme == "narrow" else 256)]))
    widths = []
    wide_at = int(rng.integers(0, n_layers))   # acc65: the layer 65 to 80 wide (the head when it is the last)
    for l in range(n_layers - 1):
        nxt = encs[l + 1]
        if theme == "acc65":
            w = rng.choice(edge_widths(nxt, 65, 80) or edge_widths(nxt, 65, 96)) if l == wide_at else rng.choice(edge_widths(nxt, 1, 32))
        elif theme == "wide":
            w = rng.choice(edge_widths(nxt, 65, 256))
        else:
            w = rng.choice(edge_widths(nxt, 1, 64 if theme == "narrow" else 96))
        if nxt == T and theme != "acc65" and rng.random() < 0.5:
            # a multiple of 32 into Ternary: its inputs padded to tens round K past the width, and the plan drops that K-step
            w = 32 * rng.integers(1, 3 if theme == "narrow" else 9)
        widths.append(int(w))
    if theme == "acc65" and wide_at == n_layers - 1:
        classes = 65
    layers = tuple((e, w, True) if e == F and rng.random() < 0.5 else (e, w) for e, w in zip(encs, widths + [classes]))
    return layers, rows


def boundary(rows, make, fits):
    """the largest hidden width h (multiples of 16, up to 256) whose model make(h) fits, and h + 16, which does not: rows-byte
    images, make(h) -> layers, fits(plan or refusal) -> bool"""
    ok = [h for h in range(16, 257, 16) if fits(plan_of(chain(rows, make(h), 0)))]
    h = max(ok)
    assert ok == list(range(16, h + 1, 16)) and h < 256, (rows, ok)
    return (make(h), rows), (make(h + 16), rows)


def two_stages(p):
    return isinstance(p, Plan)


def two_pipes(p):
    return isinstance(p, Plan) and p.pipes == 2


# one pipe: the weight image with room for two stages of 512-byte and of 752-byte rows, and 16 columns more (refused)
_ONE_512 = boundary(512, lambda h: ((I8, h), (I8, 10)), two_stages)
_ONE_752 = boundary(752, lambda h: ((U4, h), (F, 16, True)), two_stages)
# two pipes: 384-byte rows with room for four stages (two per pipe), and 16 columns more (one pipe of three stages)
_TWO_384 = boundary(384, lambda h: ((S4, 64), (I8, 64), (I8, h), (I8, 10)), two_pipes)
_TWO_272 = boundary(272, lambda h: ((I8, 64), (F, h, True), (T, 16)), two_pipes)
CRAFTED = {
    "one-pipe-512-fits": _ONE_512[0], "one-pipe-512-refused": _ONE_512[1],
    "one-pipe-752-fits": _ONE_752[0], "one-pipe-752-refused": _ONE_752[1],
    "two-pipes-384-fit": _TWO_384[0], "two-pipes-384-one-pipe": _TWO_384[1],
    "two-pipes-272-fit": _TWO_272[0], "two-pipes-272-one-pipe": _TWO_272[1],
    # the largest 64-wide weight image: the float forms' rings still fit, at two stages
    "float-largest-64-wide": (tuple((F, 64, True) for _ in range(7)) + ((F, 16, True),), 256),
    # the float forms' edges: rows 256 | 272, classes 16 | 17
    "float-rows-256": (((I8, 40), (T, 56), (S4, 10)), 256),
    "float-rows-272": (((I8, 40), (T, 56), (S4, 10)), 272),
    "float-classes-16": (((U4, 56), (I8, 16)), 240),
    "float-classes-17": (((U4, 56), (I8, 17)), 240),
    # 255 classes (ReLUNorm's "no maximum" position) after a narrow Ternary-fed layer
    "head-255": (((I8, 36), (T, 255)), 144),
    # the fixed shape from mixed encodings, and with a 60-wide hidden layer: still the fixed row (n_pad 64), its four padding
    # columns zero
    "fixed-shape": (((T, 64), (I8, 64), (S4, 64), (I8, 16)), 256),
    "fixed-shape-60": (((T, 64), (I8, 60), (I8, 64), (I8, 16)), 256),
}


class Case(NamedTuple):
    name: str
    layers: tuple
    rows: int

    @property
    def nf4_ext(self):
        return any(l[0] == NF4 for l in self.layers)


CASES = [Case(f"draw{i:02d}", *draw(i)) for i in range(N_DRAWS)] + [Case(k, *v) for k, v in CRAFTED.items()]
BY_NAME = {c.name: c for c in CASES}
NAMES = list(BY_NAME)


@functools.lru_cache(maxsize=None)
def model(name):
    c = BY_NAME[name]
    return chain(c.rows, c.layers, NAMES.index(name))


@functools.lru_cache(maxsize=None)
def plan(name):
    return plan_of(model(name), BY_NAME[name].nf4_ext)


def describe(name):
    m, c = model(name), BY_NAME[name]
    layers = " -> ".join(f"{M.ENC_NAMES[l.bitperweight]}{'+' if len(s) > 2 else ''} {l.n_out}" for l, s in zip(m.fc_layers, c.layers))
    return f"{name}: {m.img_bytes}-byte rows, {layers}"


# ---- CPU: what the draws cover -----------------------------------------------------------------------------------------------

def coverage_gaps():
    """the classes of the shape space no case reaches, by name (empty: none)"""
    fused = {n: plan(n) for n in NAMES if isinstance(plan(n), Plan)}
    seen = set()
    for n, p in fused.items():
        m, fc = model(n), model(n).fc_layers
        seen |= {f"max_n {p.max_n}", f"{p.pipes} pipes", f"{len(fc)} layers", f"{m.n_classes} classes"}
        if p.pipes == 2:
            seen.add(f"two-pipe row {p.two_pipe_row}")
        for f in ("int8", "emul_i8", "topk", "float"):
            if f in p.forms and p.forms[f].stages == 2:
                seen.add(f"{f} at 2 stages" + (" x 2 pipes" if f == "int8" and p.pipes == 2 else ""))
        hidden = range(len(fc) - 1)
        if any(fc[l].n_out < p.n_pad[l] for l in hidden):
            seen.add("hidden n_out < n_pad")
            seen |= {f"hidden width off 16 into {M.ENC_NAMES[fc[l + 1].bitperweight]}" for l in hidden if fc[l].n_out % 16}
        if any(32 * p.k_steps[l] > p.n_pad[l - 1] for l in range(1, len(fc))):
            seen.add("K-steps rounded past the previous n_pad")
        if any(-(-fc[l].n_in // 32) > p.k_steps[l] for l in range(1, len(fc))) and n.startswith("draw"):
            seen |= {f"K-steps dropped past the previous n_pad: {p.pipes} pipes"} | \
                ({"K-steps dropped past the previous n_pad: float forms"} if p.float_forms else set())
        if 64 < max(p.n_pad) <= 80 and sorted(p.n_pad)[-2:][0] <= 32:
            seen.add("widest layer 65..80 beside narrow ones")
        if m.img_bytes % 128:
            seen |= {"rows inside an atom: int8", "rows inside an atom: emulator"}
            seen |= {"rows inside an atom: float forms"} if p.float_forms else set()
        if 1 in p.planes and 2 in p.planes:
            seen.add("+128 planes in some layers only")
        if len({l.bitperweight for l in fc}) >= 3:
            seen.add("three or more encodings")
        if BY_NAME[n].nf4_ext:
            seen.add("NF4 with the extension")
        seen.add("float forms" if p.float_forms else "no float forms")
    refused = [n for n in NAMES if plan(n) == REFUSE_SMEM]
    if refused:
        seen.add("refused: weights do not fit")
    # both sides of each boundary: a fitting image within one step of the limit, and its refused neighbour
    for k in ("one-pipe-512", "one-pipe-752"):
        fit, ref = plan(f"{k}-fits"), plan(f"{k}-refused")
        if isinstance(fit, Plan) and ref == REFUSE_SMEM and fit.forms["int8"].stages == 2:
            seen.add(f"{k} boundary")
    for k in ("two-pipes-384", "two-pipes-272"):
        fit, one = plan(f"{k}-fit"), plan(f"{k}-one-pipe")
        if isinstance(fit, Plan) and fit.pipes == 2 and fit.forms["int8"].stages == 2 and isinstance(one, Plan) and one.pipes == 1:
            seen.add(f"{k} boundary")
    for a, b in (("float-rows-256", "float-rows-272"), ("float-classes-16", "float-classes-17")):
        if plan(a).float_forms and not plan(b).float_forms:
            seen.add(f"{a} | {b}")
    want = {f"max_n {n}" for n in (64, 128, 192, 256)} | {"1 pipes", "2 pipes", "int8 at 2 stages x 2 pipes"} | \
        {f"two-pipe row {r}" for r in ("fixed", "last16", "full")} | {f"{n} layers" for n in range(1, 9)} | \
        {f"{c} classes" for c in CLASSES} | {f"{f} at 2 stages" for f in ("int8", "emul_i8", "topk", "float")} | \
        {"hidden n_out < n_pad", "K-steps rounded past the previous n_pad", "K-steps dropped past the previous n_pad: 1 pipes",
         "K-steps dropped past the previous n_pad: 2 pipes", "K-steps dropped past the previous n_pad: float forms",
         "widest layer 65..80 beside narrow ones", "rows inside an atom: int8", "rows inside an atom: float forms",
         "rows inside an atom: emulator", "+128 planes in some layers only", "three or more encodings",
         "NF4 with the extension", "float forms", "no float forms", "refused: weights do not fit"} | \
        {f"hidden width off 16 into {e}" for e in ("8bit", "4bit", "4bitsym", "FP130", "NF4", "Ternary")} | \
        {"one-pipe-512 boundary", "one-pipe-752 boundary", "two-pipes-384 boundary", "two-pipes-272 boundary",
         "float-rows-256 | float-rows-272", "float-classes-16 | float-classes-17"}
    return sorted(want - seen)


def test_draws_cover_the_shape_space():
    """every class of the plan's shape space some case reaches; fails naming the classes none does"""
    assert not coverage_gaps(), coverage_gaps()


def test_cases_are_legal():
    """every layer's inputs pack to whole words in its encoding, as an exporter writes them"""
    assert all(legal(e, w) for c in CASES for (e, *_), w in zip(c.layers[1:], [l[1] for l in c.layers[:-1]]))
    assert all(legal(c.layers[0][0], c.rows) for c in CASES)


def test_float_rings_fit_every_64_wide_image():
    """the float-input forms' shared-memory clause never fails on a model with a 64-wide row: the largest such image (eight
    64-wide FP130 layers, all with a second plane, 256-byte rows, the most a float form takes) leaves their rings and two stages"""
    p = plan("float-largest-64-wide")
    assert p.max_n == 64 and p.planes == [2] * 8 and p.in_atoms == 2 and p.float_forms, p
    assert p.forms["float"].stages == 2 and p.forms["float16"].stages == 3
    assert -(-p.w_bytes // 128) * 128 + 4 * 16384 + 2 * 32768 <= SMEM_LIMIT


def test_plan_restatement_on_known_shapes():
    """the restated rules on hand-computed shapes: a 40-wide 8bit layer into Ternary (n_pad 48, K rounded to 64: two K-steps,
    the second half past the previous width), the fixed shape, and the boundaries' arithmetic"""
    p = plan_of(chain(256, ((I8, 40), (T, 100), (I8, 10)), 0))
    assert p.n_pad == [48, 112, 16] and p.k_steps == [8, 2, 4] and p.planes == [1, 1, 1]
    assert p.b_off == [0, 8 * 48 * 32, 8 * 48 * 32 + 2 * 112 * 32] and p.max_n == 128 and p.pipes == 1 and not p.float_forms
    assert p.w_bytes == 8 * 48 * 32 + 2 * 112 * 32 + 4 * 16 * 32 + 128 * 32
    f = plan("fixed-shape")
    assert f.row == "<64,2,2,16,fixed>" and f.forms["int8"].stages == 2 and f.forms["int8"].smem == 2 * 2 * 32768 + 27648 + 17408 + 1024
    assert plan("fixed-shape-60").row == "<64,2,2,16,fixed>" and plan("fixed-shape-60").n_pad == f.n_pad
    one = plan("one-pipe-512-fits")
    assert one.n_pad == [176, 16] and one.w_bytes + 2 * 65536 == SMEM_LIMIT and plan("one-pipe-512-refused") == REFUSE_SMEM
    lines = plan_lines(plan_of(M.Model.load(_golden("fc"))))
    assert lines[0] == ("bitnetmcu_b200: fused FC plan: 64 accumulator columns, 2 pipes x 2 stages, 27648 weight bytes, 177152 B smem, "
                        "fc_chain_kernel<64,2,2,16,fixed>, float input <64,1,float>, emulator <64,1,float,emul>, float input stages 4, "
                        "int8 emulator fc_emul_i8_kernel<64,1,emul> x 6 stages"), lines[0]


def _golden(name):
    from conftest import GOLDEN
    return f"{GOLDEN}/models/{name}.bnm"


REFERENCE_SAMPLE = [n for i, n in enumerate(NAMES) if i % 3 == 0 or not n.startswith("draw")]


@pytest.mark.parametrize("name", [n for n in REFERENCE_SAMPLE if not BY_NAME[n].nf4_ext])
def test_oracle_matches_reference(oracle, reference, name):
    """the C restatement equals the unmodified reference: int8 rows at the rails, all zero, random, and scaled float rows"""
    m = model(name)
    q = int8_images(N_UNIQUE, m.img_bytes, 7)
    for imgs, what in ((q, "int8"), (scale_images(scattered_edge_images(N_UNIQUE, m.img_bytes, 8)), "scaled float")):
        want_lo, want_la = reference.infer(m, imgs)
        lo, la = oracle.infer(m, imgs)
        assert np.array_equal(lo, want_lo) and np.array_equal(la, want_la), (describe(name), what)


# ---- GPU ---------------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def judge(built):
    """the unmodified reference where oracle/_ref is built, else the oracle (pinned to it by test_oracle_matches_reference)"""
    from oracle.oracle import Reference
    return Reference() if Reference.available() else None


class Data:
    """one model's N_UNIQUE images and expectations on the device; row i of a batch of n is image i % N_UNIQUE"""

    def __init__(self, name, judge, oracle):
        self.name, self.m, self.ext = name, model(name), BY_NAME[name].nf4_ext
        self.C = self.m.n_classes
        infer = oracle.infer if self.ext or judge is None else judge.infer
        kw = {"nf4_extension": True} if self.ext else {}
        seed = NAMES.index(name)
        self.q_np = int8_images(N_UNIQUE, self.m.img_bytes, seed)
        self.x_np = scattered_edge_images(N_UNIQUE, self.m.img_bytes, seed + 1000)
        # 16-bit rows: the same rows clipped to what float16 holds, widened back
        self.xh_np = np.clip(self.x_np, -6e4, 6e4)
        self.lo_np, la = infer(self.m, self.q_np, **kw)
        self.la_np = la.astype(np.int32)
        xlo, xla = infer(self.m, scale_images(self.x_np), **kw)
        self.q, self.x, self.lo, self.la, self.xlo, self.xla = map(to_device, (self.q_np, self.x_np, self.lo_np, self.la_np, xlo,
                                                                                xla.astype(np.int32)))
        self.ks = sorted(k for k in {1, 5, min(self.C, MAX_TOPK)} if k <= self.C)
        self.topk_c = {k: tuple(map(to_device, top_k(self.lo_np, k))) for k in self.ks}
        self.infer, self.kw = infer, kw

    def emulator_reference(self):
        """the emulator's float64 logits on x_np: restate.emulate, NF4 layers decoded as the engine's option says"""
        emu = emulate(self.m, self.x_np, nf4_extension=self.ext)
        self.emu, self.emu_la = to_device(emu), to_device(np.argmax(emu, axis=1).astype(np.int32))
        self.topk_py = {k: tuple(map(to_device, top_k(emu, k))) for k in self.ks}

    def half(self, fmt):
        """the 16-bit rows of fmt on the device and their expectations: (rows, C logits, C labels, emulator logits, labels)"""
        import torch
        xh = to_device(self.xh_np).to(getattr(torch, fmt))
        xw = xh.float().cpu().numpy()
        lo, la = self.infer(self.m, scale_images(xw), **self.kw)
        emu = emulate(self.m, xw, nf4_extension=self.ext)
        return xh, to_device(lo), to_device(la.astype(np.int32)), to_device(emu), to_device(np.argmax(emu, axis=1).astype(np.int32))

    def idx(self, n):
        import torch
        return torch.arange(n, device="cuda") % N_UNIQUE

    def check(self, n, got, want, sentinel, what):
        """rows :n of `got` (n + 128 rows) equal want[idx(n)]; the rows past n still hold the sentinel"""
        import torch
        w = want[self.idx(n)]
        g = got[:n].to(w.dtype)
        bad = torch.nonzero((g != w).reshape(n, -1).any(dim=1)).flatten()
        assert bad.numel() == 0, (describe(self.name), n, what, f"{bad.numel()} rows wrong, first {bad[:4].tolist()}")
        assert bool((got[n:] == sentinel).all()), (describe(self.name), n, what, "written past row n")


def past_first_trip(p, sm):
    """a batch size whose every CTA takes one tile more per pipe than every form's ring holds (pipes x (stages + 1)): each
    ring's first stage is reused, in round 1, on every pipe; the last tile holds 37 images"""
    t = max((p.pipes if f == "int8" else 1) * (form.stages + 1) for f, form in p.forms.items())
    n = batch_size(sm, t, sm, 37)
    for f, form in p.forms.items():
        pipes = p.pipes if f == "int8" else 1
        s = tile_schedule(n, sm, pipes, form.stages, 2 if pipes == 2 else 1)
        assert {(int(pp), int(r)) for pp, r in zip(s.pipe, s.round)} >= {(pp, 1) for pp in range(pipes)}, (f, n)
    return n


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_plan_line(lib, capfd, monkeypatch, name):
    """the BNM_VERBOSE plan lines equal restate.plan_lines exactly (rows, pipes, stages, shared memory, float forms); a refused
    model prints none, runs layer by layer and names the refusal when the fused path is asked for"""
    from bitnetmcu_b200 import _lib
    from bitnetmcu_b200.engine import Engine
    p = plan(name)
    e, err = verbose_engine(capfd, monkeypatch, lambda: Engine(model(name), device=0, nf4_extension=BY_NAME[name].nf4_ext))
    try:
        if isinstance(p, str):
            assert plan_line(err) is None and e.active_path == _lib.PATH_LAYERS, (describe(name), p, err)
            with pytest.raises(_lib.BnmError, match=re.escape(p)):
                e.set_option(_lib.OPT_PATH, _lib.PATH_TCGEN05)
            assert e.active_path == _lib.PATH_LAYERS
            return
        assert e.active_path == _lib.PATH_TCGEN05, (describe(name), err)
        want = plan_lines(p)
        got = (plan_line(err), [l for l in err if "fused FC top-k forms" in l][-1])
        assert got[0] == want[0], (describe(name), "plan line", got[0], want[0])
        assert got[1] == want[1], (describe(name), "top-k line", got[1], want[1])
    finally:
        e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_entries(lib, judge, oracle, name):
    """every entry at 1, 129 and a batch past the first trip round every form's ring: int8 with logits and labels, labels only,
    logits only; the host pipeline; float32; top-k at 1, 5 and min(C, 16); the emulator and its top-k; both engines with counts;
    on every fourth case float16 and bfloat16 too"""
    import torch
    from bitnetmcu_b200.engine import Engine
    d = Data(name, judge, oracle)
    e = Engine(d.m, device=0, nf4_extension=d.ext)
    try:
        p = plan(name)
        big = past_first_trip(p, torch.cuda.get_device_properties(0).multi_processor_count) if isinstance(p, Plan) else 5 * 128 + 37
        d.emulator_reference()
        halves = [(fmt, d.half(fmt)) for fmt in ("float16", "bfloat16")] if NAMES.index(name) % 4 == 0 else []
        for n in (1, 129, big):
            i = d.idx(n)
            q, x = d.q[i], d.x[i]
            for want_lo, want_la in ((True, True), (False, True), (True, False)):
                lo, la = out((n, d.C), torch.int32, -5), out((n,), torch.int32, -7)
                e.infer_device(q, lo[:n] if want_lo else None, la[:n] if want_la else None)
                torch.cuda.synchronize()
                what = "int8 " + ("logits and labels" if want_lo and want_la else "labels only" if want_la else "logits only")
                if want_lo:
                    d.check(n, lo, d.lo, -5, f"{what}: logits")
                if want_la:
                    d.check(n, la, d.la, -7, f"{what}: labels")
                assert (want_lo or bool((lo == -5).all())) and (want_la or bool((la == -7).all())), (describe(name), n, what)
            hi = np.arange(n) % N_UNIQUE
            hlo, hla = e.infer(d.q_np[hi])
            assert np.array_equal(hlo, d.lo_np[hi]) and np.array_equal(hla.astype(np.int32), d.la_np[hi]), (describe(name), n, "host")
            c_float(e, d, n, x, d.xlo, d.xla, "float32")
            emulator(e, d, n, x, d.emu, d.emu_la, "float32")
            both_engines(e, d, n, x, d.xla, d.emu_la, "float32")
            for k in d.ks:
                for what, fn, imgs, dtype, (want_cls, want_sc) in (("C engine", e.topk_device, q, torch.int32, d.topk_c[k]),
                                                                   ("emulator", e.emulate_topk_device, x, torch.float64, d.topk_py[k])):
                    cls, sc = out((n, k), torch.int32, -1), out((n, k), dtype, -7)
                    fn(imgs, k, cls[:n], sc[:n])
                    torch.cuda.synchronize()
                    d.check(n, cls, want_cls, -1, f"{what} top-{k} classes")
                    d.check(n, sc, want_sc, -7, f"{what} top-{k} scores")
            for fmt, (xh, hlo_, hla_, hemu, hemu_la) in halves:
                c_float(e, d, n, xh[i], hlo_, hla_, fmt)
                emulator(e, d, n, xh[i], hemu, hemu_la, fmt)
                both_engines(e, d, n, xh[i], hla_, hemu_la, fmt)
            del q, x
    finally:
        e.close()
