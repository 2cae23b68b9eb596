"""Options changed on a live model (bnm_model_set_option, include/bitnetmcu_b200.h): the NF4 extension's rebuild of the device
weights, path and CNN front-end switches between calls, chunk resizes of the host pipeline, and refused values.

BNM_OPT_NF4_EXTENSION is the one option that replaces device state under a live handle: build_fc_dev frees every decoded plane
and the fused plan, decodes the planes again and makes a new plan, with the overlap mode re-applied.  Scratch and planes share a
pool that never returns memory, so a stale plane or weight image would not fault: it would silently give the old weights'
results.  The other options only set fields of the model, read by the calls made after them; a refused value must leave them
all, and the route, as they were.

Models.  For the rules: an FC model with a fused plan (4bitsym-64), one without (a 300-wide layer), CNN-48 and a 144-channel CNN
(no tensor-core front-end, the layered emulator).  For the NF4 toggles: rand_nf4_64, a mixed chain with NF4 in the middle
layer and an FP130 layer with +128 weights (a residual plane) at the end, a CNN with an NF4 head, an NF4 model with no plan (a
304-wide layer), and 4bitsym-64, which has no NF4 layer.  For the front-end switches: CNN-48 with conv3 on IDP.2A (the fixture,
conv3 bound 24581) and a random CNN-48 past 65535 (IMAD).

CPU: restate.emulate against the reference's QuantizedModel.inference_quantized on the engine's integer levels, for 4bit
layers and NF4 layers with the extension off and on.  GPU (tolerance 0, against the oracle with the extension the model has at
the time of the call and restate.emulate): the rules on four models; the toggle sequence off -> on -> on -> off -> on with every
entry family at 1, 700 and 2^17 + 77 images (past the layer-by-layer pass and seven tiles per CTA) after each step, and a fresh
engine with the same option; a toggle in BNM_PATH_LAYERS and in overlap mode 2 (the wait decisions under BNM_VERBOSE); path
and front-end switches between calls queued on one stream; graphs captured under one front-end and replayed under another; and
one engine's host pipeline through chunks of 65536, 128, 1000, 300000 and 128 images."""
import functools
import os
import sys

import numpy as np
import pytest

from bitnetmcu_b200 import model as M
from conftest import load_model
from restate import Plan, cnn_stages, conv3_bound, emulate, plan_lines, plan_of, scale_images
from support import (both_engines, c_float, chain, cnn_model, emulator, gather_call, int8_images, kernel_copies_are_kernels,  # noqa: F401
                     kernel_copy, lib, out, quantized_model_list, scattered_edge_images, to_device, top_k,  # (lib,
                     verbose_engine)                                                                        # kernel_copies_are_kernels: fixtures)

REF_PY = "/root/reference"
B, S2, S4, U4, I8, F, NF4, T = (M.ENC_BINARY, M.ENC_2BITSYM, M.ENC_4BITSYM, M.ENC_4BIT, M.ENC_8BIT, M.ENC_FP130, M.ENC_NF4,
                                M.ENC_TERNARY)
PLUS = True                     # an FP130 layer with +128 weights
N_UNIQUE = 389                  # distinct images per model; row i of a batch is image i % N_UNIQUE
SIZES = (1, 700, (1 << 17) + 77)
E_ARG, E_UNSUPPORTED = -1, -3   # BNM_E_ARG, BNM_E_UNSUPPORTED (capi.cu)
OPT_PATH, OPT_NF4, OPT_CHUNK, OPT_OVERLAP, OPT_FRONTEND = 1, 2, 3, 4, 5
OPTIONS = (OPT_PATH, OPT_NF4, OPT_CHUNK, OPT_OVERLAP, OPT_FRONTEND)
OPT_NAMES = {OPT_PATH: "BNM_OPT_PATH", OPT_NF4: "BNM_OPT_NF4_EXTENSION", OPT_CHUNK: "BNM_OPT_CHUNK_IMAGES",
             OPT_OVERLAP: "BNM_OPT_LAUNCH_OVERLAP", OPT_FRONTEND: "BNM_OPT_CNN_FRONTEND"}


# ---- the models ----------------------------------------------------------------------------------------------------------------

def cnn_with_head(channels, layers, seed):
    """cnn_model's random front-end (8bit taps with +-127, conv3 on IMAD) and the FC head chain() draws for `layers`"""
    head = chain(channels * 4, layers, seed).fc_layers
    for i, l in enumerate(head):
        l.name = f"L{11 + 2 * i}"
    m = M.Model(model_class=M.MODEL_CNNMNIST, layers=list(cnn_model(channels, 10, seed).layers[:5]) + head)
    m.validate()
    return m


MODELS = {
    "fc": lambda: load_model("fc"),                                     # FC 4bitsym-64, the fixed-shape row; no NF4 layer
    "fc-no-plan": lambda: chain(256, ((I8, 300), (I8, 10)), 1),         # a 300-wide layer: layer by layer only
    "cnn48": lambda: load_model("cnn_48"),                              # conv3 bound 24581: IDP.2A
    "cnn48-imad": lambda: cnn_model(48, 10, seed=48),                   # conv3 bound past 65535: IMAD
    "cnn144": lambda: cnn_model(144, 10, seed=144),                     # CUDA-core front-end only, the layered emulator
    "nf4": lambda: load_model("rand_nf4_64"),
    "nf4-mixed": lambda: chain(256, ((S4, 64), (NF4, 64), (F, 10, PLUS)), 3),
    "nf4-cnn": lambda: cnn_with_head(64, ((S2, 64), (NF4, 64), (NF4, 10)), 7),
    "nf4-no-plan": lambda: chain(256, ((NF4, 304), (NF4, 10)), 4),
    "4bit": lambda: chain(256, ((U4, 64), (S4, 64), (U4, 10)), 5),
    "4bit-cnn": lambda: cnn_with_head(48, ((S2, 64), (U4, 64), (U4, 10)), 9),
}
NAMES = list(MODELS)


@functools.lru_cache(maxsize=None)
def model(name):
    return MODELS[name]()


def fc_view(m):
    """the FC chain a model's fused plan is made for: CNN models feed it rows of C * 4 features rounded up to 16 bytes"""
    if m.model_class == M.MODEL_FCMNIST:
        return m
    return M.Model(model_class=M.MODEL_FCMNIST, layers=m.fc_layers, img_bytes=-(-m.channels * 4 // 16) * 16)


def plan(name, ext=False):
    return plan_of(fc_view(model(name)), ext)


def has_nf4(name):
    return any(l.bitperweight == NF4 for l in model(name).fc_layers)


def test_models():
    """each model is what the module says: plans, conv3 bounds, NF4 and FP130 layers"""
    assert isinstance(plan("fc"), Plan) and plan("fc").row == "<64,2,2,16,fixed>" and not has_nf4("fc")
    assert not isinstance(plan("fc-no-plan"), Plan) and not isinstance(plan("nf4-no-plan", True), Plan)
    assert conv3_bound(model("cnn48")) <= 65535 < conv3_bound(model("cnn48-imad"))
    assert model("cnn144").channels == 144 and isinstance(plan("cnn144"), Plan)
    for name in ("nf4", "nf4-mixed", "nf4-cnn"):
        assert has_nf4(name) and isinstance(plan(name, True), Plan), name
    assert [l.bitperweight for l in model("nf4-mixed").fc_layers] == [S4, NF4, F] and plan("nf4-mixed", True).planes == [1, 1, 2]
    assert all(m.img_bytes == 256 for m in map(model, NAMES))


# ---- CPU: the emulator restatement on 4bit and NF4 layers against the reference ---------------------------------------------

RESTATE_CASES = [("4bit", False), ("4bit-cnn", False), ("nf4", False), ("nf4", True), ("nf4-mixed", False), ("nf4-mixed", True),
                 ("nf4-cnn", False), ("nf4-cnn", True)]


@pytest.mark.skipif(not os.path.isfile(os.path.join(REF_PY, "BitNetMCU.py")), reason="needs the reference's BitNetMCU.py")
@pytest.mark.parametrize("name,ext", RESTATE_CASES, ids=[f"{n}-ext{int(e)}" for n, e in RESTATE_CASES])
def test_emulate_is_the_reference_emulator_on_integer_levels(name, ext):
    """the emulator's rule on 4bit and NF4 layers (INTEGRATION.md section 5): the reference's
    QuantizedModel.inference_quantized given the engine's integer levels -- 4bit's integers, NF4's zeros without the extension
    and its LUT with it -- is restate.emulate(..., nf4_extension) bit for bit.  CNN rows whose every conv stage has a positive
    maximum (the reference renormalises an all-zero stage by 0/0)"""
    if REF_PY not in sys.path:
        sys.path.append(REF_PY)
    from BitNetMCU import QuantizedModel
    m = model(name)
    x = scattered_edge_images(N_UNIQUE, 256, 11)
    if m.model_class == M.MODEL_CNNMNIST:
        c1, c2, c3, _ = cnn_stages(m, x)
        x = x[[i for i in range(len(x)) if min(c.reshape(len(x), -1)[i].max() for c in (c1, c2, c3)) > 0]]
        assert len(x) >= 40, name
    qm = QuantizedModel()
    qm.quantized_model = quantized_model_list(m, ext)
    want = np.asarray(qm.inference_quantized(x), dtype=np.float64)
    got = emulate(m, x, nf4_extension=ext)
    assert np.array_equal(got, want), (name, ext)
    # the extension decides the NF4 layers' levels: without it they are zeros, and the logits of an all-NF4 chain with them
    if has_nf4(name):
        assert not np.array_equal(got, emulate(m, x, nf4_extension=not ext)), (name, ext)
    if name == "nf4":
        assert (not got.any()) == (not ext), (name, ext)


# ---- the option rules ------------------------------------------------------------------------------------------------------------

def rule(option, value, has_plan, tc_frontend):
    """bnm_model_set_option restated: (return code, a fragment of bnm_last_error() or None, what get_option then reports)"""
    if option == OPT_PATH:
        if not 0 <= value <= 2:
            return E_ARG, f"bad path {value}", None
        if value == 2 and not has_plan:
            return E_UNSUPPORTED, "fused tensor-core path unavailable for this model", None
        return 0, None, value
    if option == OPT_NF4:
        return 0, None, int(value != 0)
    if option == OPT_CHUNK:
        return (E_ARG, "chunk must be >= 128 images", None) if value < 128 else (0, None, value)
    if option == OPT_OVERLAP:
        return (E_ARG, "launch overlap mode must be 0, 1 or 2", None) if not 0 <= value <= 2 else (0, None, value)
    if option == OPT_FRONTEND:
        if not 0 <= value <= 2:
            return E_ARG, "CNN front-end must be 0 (auto), 1 (CUDA cores) or 2 (tensor cores)", None
        if value == 2 and not tc_frontend:
            return E_UNSUPPORTED, "tensor-core CNN front-end needs a 16x16 CNN model", None
        return 0, None, value
    return E_ARG, f"unknown option {option}", None


# legal, boundary and illegal values of every option, and unknown options
VALUES = {OPT_PATH: (-1, 0, 1, 2, 3), OPT_NF4: (0, 1, 7, -1), OPT_CHUNK: (-1, 0, 127, 128, 1000, 1 << 40),
          OPT_OVERLAP: (-1, 0, 1, 2, 3), OPT_FRONTEND: (-1, 0, 1, 2, 3), 0: (0, 1), 6: (0,), 99: (1,)}
RULE_MODELS = ["fc", "fc-no-plan", "cnn48", "cnn144"]


def test_rules_table():
    """the restated rules on the four models: what each refuses"""
    refused = {n: sorted((o, v) for o, vs in VALUES.items() for v in vs
                         if rule(o, v, isinstance(plan(n), Plan), n == "cnn48")[0]) for n in RULE_MODELS}
    common = [(0, 0), (0, 1), (1, -1), (1, 3), (3, -1), (3, 0), (3, 127), (4, -1), (4, 3), (5, -1), (5, 2), (5, 3), (6, 0), (99, 1)]
    assert refused["fc"] == refused["cnn144"] == common
    assert refused["fc-no-plan"] == sorted(common + [(1, 2)])
    assert refused["cnn48"] == [r for r in common if r != (5, 2)]


# ---- GPU helpers -------------------------------------------------------------------------------------------------------------------

def windows_of(pages, sy, sx):
    """the 16 x 16 windows of a [P, H, W] stack on a stride grid, flattened in the window entries' order"""
    p_, h, w = pages.shape
    return np.stack([pages[p, r:r + 16, c:c + 16].reshape(256) for p in range(p_) for r in range(0, h - 15, sy)
                     for c in range(0, w - 15, sx)])


WINDOW_STRIDE = (2, 2)
PAD = (7, 8, 3, 5)             # left, right, top, bottom: torch.nn.functional.pad's order


@functools.lru_cache(maxsize=None)
def oracle_lib():
    from oracle.oracle import Oracle
    return Oracle()


@functools.lru_cache(maxsize=None)
def expect(name, ext):
    """NumPy expectations of model `name` with the NF4 extension on or off: the N_UNIQUE int8 and float rows, the oracle's logits
    and labels, restate.emulate's logits for float32, float16 and bfloat16 rows (widened), and the windows of a one-window page,
    a three-page stack and that stack padded by reflection"""
    import torch
    m, seed = model(name), NAMES.index(name)
    c = lambda imgs: tuple(a.astype(np.int32) for a in oracle_lib().infer(m, imgs, nf4_extension=ext))
    q = int8_images(N_UNIQUE, 256, seed)
    x = scattered_edge_images(N_UNIQUE, 256, seed + 100)
    r = {"q": q, "x": x, "int8": c(q)}
    for fmt in ("float32", "float16", "bfloat16"):
        xw = torch.from_numpy(x).to(getattr(torch, fmt)).float().numpy()
        emu = emulate(m, xw, nf4_extension=ext)
        r[fmt] = c(scale_images(xw)) + (emu, np.argmax(emu, axis=1).astype(np.int32))
    rng = np.random.default_rng(seed + 200)
    pages = {"one": rng.normal(size=(1, 16, 16)).astype(np.float32), "stack": rng.normal(size=(3, 40, 40)).astype(np.float32)}
    pages["stack"][1, 5:30, 7:20] = 0.0
    r["pages"] = pages
    padded = np.pad(pages["stack"], ((0, 0), (PAD[2], PAD[3]), (PAD[0], PAD[1])), mode="reflect")
    for key, wins in (("one", windows_of(pages["one"], 1, 1)), ("stack", windows_of(pages["stack"], *WINDOW_STRIDE)),
                      ("padded", windows_of(padded, *WINDOW_STRIDE))):
        r["win", key] = c(scale_images(wins)) + (emulate(m, wins, nf4_extension=ext),)
    return r


class Dev:
    """one model's expectations with the NF4 extension on or off on the device; row i of a batch of n is image i % N_UNIQUE.
    name, C, idx and check are what support's entry checks (c_float, emulator, both_engines) take"""

    def __init__(self, name, ext):
        import torch
        self.model, self.ext, self.m = name, ext, model(name)
        self.name, self.C = f"{name}, NF4 extension {'on' if ext else 'off'}", self.m.n_classes
        x = self.host = expect(name, ext)
        self.q, self.x = to_device(x["q"]), to_device(x["x"])
        self.inputs = {fmt: self.x.to(getattr(torch, fmt)) for fmt in ("float32", "float16", "bfloat16")}
        self.lo, self.la = map(to_device, x["int8"])
        self.want = {fmt: tuple(map(to_device, x[fmt])) for fmt in self.inputs}
        self.ks = [k for k in (1, 5) if k <= self.C]
        self.topk_c = {k: tuple(map(to_device, top_k(x["int8"][0], k))) for k in self.ks}
        self.topk_py = {k: tuple(map(to_device, top_k(x["float32"][2], k))) for k in self.ks}
        self.pages = {k: to_device(v) for k, v in x["pages"].items()}

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


def sync():
    import torch
    torch.cuda.synchronize()


def int8_entries(e, d, n, what):
    """the int8 device entry with logits and labels, labels only, top-k at k = 1 and 5, and the host entry"""
    import torch
    q = d.q[d.idx(n)]
    lo, la = out((n, d.C), torch.int32, -5), out((n,), torch.int32, -7)
    e.infer_device(q, lo[:n], la[:n])
    sync()
    d.check(n, lo, d.lo, -5, f"{what}: int8 device logits")
    d.check(n, la, d.la, -7, f"{what}: int8 device labels")
    la.fill_(-7)
    e.infer_device(q, None, la[:n])
    sync()
    d.check(n, la, d.la, -7, f"{what}: int8 device labels only")
    for k in d.ks:
        cls, sc = out((n, k), torch.int32, -1), out((n, k), torch.int32, -7)
        e.topk_device(q, k, cls[:n], sc[:n])
        sync()
        d.check(n, cls, d.topk_c[k][0], -1, f"{what}: int8 top-{k} classes")
        d.check(n, sc, d.topk_c[k][1], -7, f"{what}: int8 top-{k} scores")
    hi = np.arange(n) % N_UNIQUE
    hlo, hla = e.infer(d.host["q"][hi])
    path = "small batch" if n <= 1024 else "chunked"
    assert np.array_equal(hlo, d.host["int8"][0][hi]), (d.name, n, f"{what}: int8 host ({path}) logits")
    assert np.array_equal(hla.astype(np.int32), d.host["int8"][1][hi]), (d.name, n, f"{what}: int8 host ({path}) labels")


def float_entries(e, d, n, what):
    """the float entries on float32, float16 and bfloat16 rows: the C engine, the emulator, its top-k (float32), both engines"""
    import torch
    i = d.idx(n)
    for fmt, xs in d.inputs.items():
        lo, la, emu, emu_la = d.want[fmt]
        x = xs[i]
        c_float(e, d, n, x, lo, la, f"{what}: {fmt}")
        emulator(e, d, n, x, emu, emu_la, f"{what}: {fmt}")
        both_engines(e, d, n, x, la, emu_la, f"{what}: {fmt}")
        if fmt == "float32":
            for k in d.ks:
                cls, sc = out((n, k), torch.int32, -1), out((n, k), torch.float64, -7)
                e.emulate_topk_device(x, k, cls[:n], sc[:n])
                sync()
                d.check(n, cls, d.topk_py[k][0], -1, f"{what}: emulator top-{k} classes")
                d.check(n, sc, d.topk_py[k][1], -7, f"{what}: emulator top-{k} scores")
        del x


def window_entries(e, d, what):
    """the stacked window entries (C engine, emulator) on a one-window page and a three-page stack, and the padded ones"""
    import torch
    from bitnetmcu_b200.engine import window_grid

    def same(got, want, part):
        g = got.cpu().numpy().reshape(want.shape[0], -1)
        assert np.array_equal(g, want.reshape(want.shape[0], -1).astype(g.dtype)), (d.name, f"{what}: windows {part}")
    for key, pages, pad in (("one", d.pages["one"], None), ("stack", d.pages["stack"], None), ("padded", d.pages["stack"], PAD)):
        lo, la, emu = d.host["win", key]
        sy, sx = (1, 1) if key == "one" else WINDOW_STRIDE
        kw = {"padding": pad, "pad_mode": "reflect"} if pad else {}
        n = lo.shape[0]
        c_lo, c_la = torch.full((n, d.C), -5, dtype=torch.int32, device="cuda"), torch.full((n,), -7, dtype=torch.int32, device="cuda")
        p_lo, p_la = torch.full((n, d.C), np.nan, dtype=torch.float64, device="cuda"), torch.full_like(c_la, -7)
        grid = (pages.shape[0],) + window_grid(pages.shape[1], pages.shape[2], (sy, sx), pad)
        e.scan_windows_device(pages, (sy, sx), c_lo.view(grid + (d.C,)), c_la.view(grid), **kw)
        e.emulate_windows_device(pages, (sy, sx), p_lo.view(grid + (d.C,)), p_la.view(grid), **kw)
        k = d.ks[-1]
        cls, sc = torch.full((n, k), -1, dtype=torch.int32, device="cuda"), torch.full((n, k), -7, dtype=torch.int32, device="cuda")
        e.scan_windows_topk_device(pages, (sy, sx), k, cls.view(grid + (k,)), sc.view(grid + (k,)), **kw)
        sync()
        same(c_lo, lo, f"{key}: C logits")
        same(c_la, la, f"{key}: C labels")
        same(p_lo, emu, f"{key}: emulator logits")
        same(p_la, np.argmax(emu, axis=1), f"{key}: emulator labels")
        want_cls, want_sc = top_k(lo, k)
        same(cls, want_cls, f"{key}: C top-{k} classes")
        same(sc, want_sc, f"{key}: C top-{k} scores")


def gather_entry(lib, e, d, n, what):
    """bnm_infer_batch_device_gather into same-GPU destinations at row offset 3, besides the call's own labels"""
    import torch
    from bitnetmcu_b200 import _lib
    dst_lo, dst_la = out((n + 3, d.C), torch.int32, -5), out((n + 3,), torch.int32, -7)
    la = out((n,), torch.int32, -7)
    g = _lib.BnmGather()
    g.n_logits_dst, g.n_labels_dst, g.row_offset = 1, 1, 3
    g.logits_dst[0], g.labels_dst[0] = dst_lo.data_ptr(), dst_la.data_ptr()
    rc = gather_call(lib, e, d.q[d.idx(n)], None, la[:n], g, torch.cuda.current_stream())
    assert rc == 0, (d.name, n, f"{what}: gather", lib.bnm_last_error())
    d.check(n, la, d.la, -7, f"{what}: gather: own labels")
    assert bool((dst_lo[:3] == -5).all()) and bool((dst_la[:3] == -7).all()), (d.name, n, f"{what}: gather: rows before the offset")
    d.check(n, dst_lo[3:], d.lo, -5, f"{what}: gather: destination logits")
    d.check(n, dst_la[3:], d.la, -7, f"{what}: gather: destination labels")


def every_family(lib, e, d, what, sizes=SIZES):
    """every entry family at each size (the window entries once), against d's expectations"""
    from bitnetmcu_b200 import _lib
    for n in sizes:
        int8_entries(e, d, n, what)
        float_entries(e, d, n, what)
        if e.active_path == _lib.PATH_TCGEN05:
            gather_entry(lib, e, d, n, what)
    window_entries(e, d, what)


def set_rc(lib, e, option, value):
    """bnm_model_set_option's return code and, when it refuses, bnm_last_error()"""
    rc = lib.bnm_model_set_option(e.handle, option, int(value))
    return rc, (lib.bnm_last_error().decode() if rc else "")


def options(lib, e):
    return {OPT_NAMES[o]: int(lib.bnm_model_get_option(e.handle, o)) for o in OPTIONS}


def err_lines(capfd, what):
    return [l for l in capfd.readouterr().err.splitlines() if what in l]


def topk_route(capfd, e, d):
    """the `topk route:` line of one int8 top-k call"""
    import torch
    capfd.readouterr()
    cls = torch.empty((1, 1), dtype=torch.int32, device="cuda")
    e.topk_device(d.q[:1], 1, cls)
    sync()
    lines = err_lines(capfd, "topk route: ")
    assert len(lines) == 1, (d.name, lines)
    return lines[0].split("topk route: bnm_infer_topk_device: ")[1]


def want_topk_route(name, ext, path):
    from bitnetmcu_b200 import _lib
    p = plan(name, ext)
    front = "k_cnn_frontend16 + " if model(name).channels == 144 else "k_cnn_frontend16_tc + " if model(name).model_class else ""
    if path == _lib.PATH_LAYERS or not isinstance(p, Plan):
        return front + "layer by layer + k_topk_rows<int32>"
    return front + p.forms["topk"].row


# ---- GPU: the rules ----------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("name", RULE_MODELS)
def test_option_rules(lib, name):
    """every option at legal, boundary and illegal values, and unknown options: the return code, bnm_last_error(), every
    get_option and active_path afterwards; a refused value leaves every option and the route as they were, and the call after it
    gives what the call before it gave.  The options start away from their defaults, so a refusal that resets one shows"""
    import torch
    from bitnetmcu_b200 import _lib
    from bitnetmcu_b200.engine import Engine
    has_plan, tc = isinstance(plan(name), Plan), name == "cnn48"
    d = Dev(name, False)
    e = Engine(d.m, device=0)
    n = 300
    try:
        assert options(lib, e) == {"BNM_OPT_PATH": 0, "BNM_OPT_NF4_EXTENSION": 0, "BNM_OPT_CHUNK_IMAGES": 65536,
                                   "BNM_OPT_LAUNCH_OVERLAP": 0, "BNM_OPT_CNN_FRONTEND": 0}, name
        assert lib.bnm_model_get_option(e.handle, 0) == lib.bnm_model_get_option(e.handle, 6) == -1
        base = {OPT_PATH: 2 if has_plan else 1, OPT_NF4: 0, OPT_CHUNK: 1000, OPT_OVERLAP: 1, OPT_FRONTEND: 1}

        def reset():
            for o, v in base.items():
                assert set_rc(lib, e, o, v) == (0, ""), (name, OPT_NAMES[o], v)
        reset()
        state = options(lib, e)

        def call():
            lo, la = out((n, d.C), torch.int32, -5), out((n,), torch.int32, -7)
            e.infer_device(d.q[d.idx(n)], lo[:n], la[:n])
            sync()
            return lo.cpu().numpy(), la.cpu().numpy()
        for option, values in VALUES.items():
            opt = OPT_NAMES.get(option, f"option {option}")
            for value in values:
                what = (name, f"{opt} = {value}")
                want_rc, fragment, want_get = rule(option, value, has_plan, tc)
                before = call()
                rc, err = set_rc(lib, e, option, value)
                assert rc == want_rc, what + (rc, err)
                if rc:
                    assert fragment in err, what + (err,)
                    assert options(lib, e) == state, what + ("options after the refusal", options(lib, e), state)
                    assert e.active_path == base[OPT_PATH], what + ("active path after the refusal",)
                    after = call()
                    assert all(np.array_equal(a, b) for a, b in zip(before, after)), what + ("the call after the refusal",)
                    assert np.array_equal(after[0][:n], d.host["int8"][0][np.arange(n) % N_UNIQUE]), what + ("int8 logits",)
                    continue
                got = options(lib, e)
                assert got[opt] == want_get, what + (got,)
                assert {k: v for k, v in got.items() if k != opt} == {k: v for k, v in state.items() if k != opt}, what + (got,)
                want_path = (1 if value == 1 else 2 if has_plan else 1) if option == OPT_PATH else base[OPT_PATH]
                assert e.active_path == want_path, what + ("active path", e.active_path)
                after = call()
                assert np.array_equal(after[0][:n], d.host["int8"][0][np.arange(n) % N_UNIQUE]), what + ("int8 logits",)
                reset()
                assert options(lib, e) == state, what + ("options after the reset",)
    finally:
        e.close()


# ---- GPU: the NF4 extension's rebuild -------------------------------------------------------------------------------------------

TOGGLE_MODELS = ["nf4", "nf4-mixed", "nf4-cnn", "nf4-no-plan", "fc"]
TOGGLES = (0, 1, 1, 0, 1)      # off -> on -> on (no change) -> off -> on


def plan_check(err, name, ext, changed, what):
    """the lines a toggle printed (err) on a model created with BNM_VERBOSE: a rebuild prints the plan restate.plan_of predicts
    (none without a plan); no change, nothing"""
    lines = [l for l in err if "fused FC plan" in l or "fused FC top-k forms" in l]
    p = plan(name, ext)
    if not changed or not isinstance(p, Plan):
        assert lines == [], (name, what, "no plan lines expected", lines)
    else:
        assert tuple(lines) == plan_lines(p), (name, what, "plan lines of the rebuild", lines, plan_lines(p))


@pytest.mark.gpu
@pytest.mark.parametrize("name", TOGGLE_MODELS)
def test_nf4_toggles(lib, capfd, monkeypatch, name):
    """BNM_OPT_NF4_EXTENSION off -> on -> on -> off -> on on a model created with BNM_VERBOSE: after each step get_option, the
    active path, the plan lines the rebuild prints and the top-k route name what restate.plan_of predicts, and every entry family
    at 1, 700 and 2^17 + 77 images equals the oracle and restate.emulate with the extension then in force, and a fresh engine
    made with it"""
    from bitnetmcu_b200 import _lib
    from bitnetmcu_b200.engine import Engine
    e, _ = verbose_engine(capfd, monkeypatch, lambda: Engine(model(name), device=0))
    devs = {ext: Dev(name, ext) for ext in (False, True)}
    if not has_nf4(name):   # the rebuild must change nothing
        assert all(np.array_equal(a, b) for a, b in zip(devs[0].host["int8"], devs[1].host["int8"])), name
    try:
        ext = 0
        for step, value in enumerate(TOGGLES):
            capfd.readouterr()
            what = f"step {step}: {OPT_NAMES[OPT_NF4]} = {value}"
            assert set_rc(lib, e, OPT_NF4, value) == (0, ""), (name, what)
            printed = capfd.readouterr().err.splitlines()
            assert options(lib, e)["BNM_OPT_NF4_EXTENSION"] == value, (name, what)
            p = plan(name, value)
            assert e.active_path == (_lib.PATH_TCGEN05 if isinstance(p, Plan) else _lib.PATH_LAYERS), (name, what)
            d = devs[bool(value)]
            assert topk_route(capfd, e, d) == want_topk_route(name, value, _lib.PATH_AUTO), (name, what)
            every_family(lib, e, d, what)
            fresh = Engine(d.m, device=0, nf4_extension=bool(value))
            try:
                int8_entries(fresh, d, 700, f"{what}: a fresh engine")
                float_entries(fresh, d, 700, f"{what}: a fresh engine")
            finally:
                fresh.close()
            plan_check(printed, name, value, value != ext, what)
            ext = value
            capfd.readouterr()
    finally:
        e.close()


@pytest.mark.gpu
def test_nf4_toggle_on_the_layered_path(lib, capfd, monkeypatch):
    """a toggle while BNM_OPT_PATH = BNM_PATH_LAYERS keeps the path; back on AUTO the new plan serves every entry"""
    from bitnetmcu_b200 import _lib
    from bitnetmcu_b200.engine import Engine
    name = "nf4-mixed"
    e, _ = verbose_engine(capfd, monkeypatch, lambda: Engine(model(name), device=0, path=_lib.PATH_LAYERS))
    try:
        for value in (1, 0, 1):
            d = Dev(name, bool(value))
            what = f"{OPT_NAMES[OPT_NF4]} = {value} on BNM_PATH_LAYERS"
            capfd.readouterr()
            assert set_rc(lib, e, OPT_NF4, value) == (0, ""), what
            plan_check(capfd.readouterr().err.splitlines(), name, value, True, what)
            assert options(lib, e)["BNM_OPT_PATH"] == _lib.PATH_LAYERS and e.active_path == _lib.PATH_LAYERS, what
            assert topk_route(capfd, e, d) == want_topk_route(name, value, _lib.PATH_LAYERS), what
            every_family(lib, e, d, what, sizes=SIZES[:2])
        assert set_rc(lib, e, OPT_PATH, _lib.PATH_AUTO) == (0, "")
        assert e.active_path == _lib.PATH_TCGEN05
        assert topk_route(capfd, e, d) == want_topk_route(name, 1, _lib.PATH_AUTO)
        every_family(lib, e, d, f"{OPT_NAMES[OPT_NF4]} = 1, then BNM_PATH_AUTO")
    finally:
        e.close()


def decisions(capfd):
    """the `fused launch:` decisions printed since the last call"""
    return [l.split("fused launch: ")[1] for l in capfd.readouterr().err.splitlines() if "fused launch: " in l]


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["nf4", "nf4-cnn"])
def test_nf4_toggle_in_overlap_mode_2(lib, capfd, monkeypatch, name, kernel_copies_are_kernels):
    """BNM_OPT_LAUNCH_OVERLAP = 2 survives the rebuild.  FC: back-to-back launches on disjoint buffers after each toggle, the
    first waits (a new plan), the next is declared independent.  CNN: the mode stays effectively 1 (the front-end feeds the FC
    kernel), every launch waits, and a chain where a kernel writes each call's images right before it reads what it wrote"""
    import torch
    from bitnetmcu_b200.engine import Engine
    e, _ = verbose_engine(capfd, monkeypatch, lambda: Engine(model(name), device=0))
    cnn = model(name).model_class == M.MODEL_CNNMNIST
    n = 1000
    s = torch.cuda.Stream()
    try:
        assert set_rc(lib, e, OPT_OVERLAP, 2) == (0, "")
        for value in (1, 0, 1):
            capfd.readouterr()
            assert set_rc(lib, e, OPT_NF4, value) == (0, ""), (name, value)
            d = Dev(name, bool(value))
            what = (name, f"{OPT_NAMES[OPT_OVERLAP]} = 2, then {OPT_NAMES[OPT_NF4]} = {value}")
            assert options(lib, e)["BNM_OPT_LAUNCH_OVERLAP"] == 2, what
            srcs = [d.q[(d.idx(n) + 17 * j) % N_UNIQUE] for j in range(4)]
            imgs = [srcs[0].clone(), srcs[1].clone()]
            lo = [out((n, d.C), torch.int32, -5) for _ in range(4)]
            la = [out((n,), torch.int32, -7) for _ in range(4)]
            sync()
            capfd.readouterr()
            with torch.cuda.stream(s):
                for j in range(4):
                    if cnn:   # the call's images written by a kernel on the same stream right before it
                        kernel_copy(imgs[j % 2], srcs[j])
                    e.infer_device(imgs[j % 2] if cnn else srcs[j % 2], lo[j][:n], la[j][:n], stream=s.cuda_stream)
            sync()
            got = decisions(capfd)
            # FC: the first launch of a new plan waits; each launch after it shares no buffer with the one right before
            want = ["wait"] * 4 if cnn else ["wait", "independent", "independent", "independent"]
            assert got == want, what + ("fused launch decisions", got, want)
            for j in range(4):
                rows = ((d.idx(n) + 17 * (j if cnn else j % 2)) % N_UNIQUE)
                assert torch.equal(lo[j][:n], d.lo[rows]) and torch.equal(la[j][:n], d.la[rows]), what + (f"launch {j}",)
    finally:
        e.close()


# ---- GPU: path and front-end switches between calls ------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("name", ["fc", "cnn48"])
def test_path_switches_between_queued_calls(lib, capfd, monkeypatch, name):
    """BNM_OPT_PATH AUTO -> LAYERS -> TCGEN05 -> AUTO with calls of every device family in between, all queued on one stream
    without a synchronisation: each call takes the route of the path set before it (its top-k route line) and gives the same
    results"""
    import torch
    from bitnetmcu_b200 import _lib
    from bitnetmcu_b200.engine import Engine
    e, _ = verbose_engine(capfd, monkeypatch, lambda: Engine(model(name), device=0))
    d = Dev(name, False)
    n, s = 700, torch.cuda.Stream()
    i = d.idx(n)
    q, x, xh = d.q[i], d.x[i], d.inputs["float16"][i]
    k = d.ks[-1]
    results = []
    try:
        sync()
        capfd.readouterr()
        with torch.cuda.stream(s):
            for path in (_lib.PATH_AUTO, _lib.PATH_LAYERS, _lib.PATH_TCGEN05, _lib.PATH_AUTO):
                assert set_rc(lib, e, OPT_PATH, path) == (0, ""), (name, path)
                r = {"path": path, "lo": out((n, d.C), torch.int32, -5), "la": out((n,), torch.int32, -7),
                     "la_only": out((n,), torch.int32, -7), "cls": out((n, k), torch.int32, -1), "sc": out((n, k), torch.int32, -7),
                     "f_lo": out((n, d.C), torch.int32, -5), "h_la": out((n,), torch.int32, -7),
                     "emu": out((n, d.C), torch.float64, -7), "emu_la": out((n,), torch.int32, -7),
                     "pcls": out((n, k), torch.int32, -1), "psc": out((n, k), torch.float64, -7)}
                st = s.cuda_stream
                e.infer_device(q, r["lo"][:n], r["la"][:n], stream=st)
                e.infer_device(q, None, r["la_only"][:n], stream=st)
                e.topk_device(q, k, r["cls"][:n], r["sc"][:n], stream=st)
                e.infer_device_f32(x, r["f_lo"][:n], None, stream=st)
                e.infer_device_f32(xh, None, r["h_la"][:n], stream=st)
                e.inference_quantized_device(x, r["emu"][:n], r["emu_la"][:n], stream=st)
                e.emulate_topk_device(x, k, r["pcls"][:n], r["psc"][:n], stream=st)
                results.append(r)
        sync()
        routes = [l.split("topk route: ")[1] for l in capfd.readouterr().err.splitlines() if "topk route: " in l]
        layered = ["layer by layer" in r for r in routes]
        assert layered == [False, False, True, True, False, False, False, False], (name, routes)   # C engine, emulator per path
        lo, la, emu, emu_la = d.want["float32"]
        h_la = d.want["float16"][1]
        for r in results:
            what = f"{OPT_NAMES[OPT_PATH]} = {r['path']}, queued"
            d.check(n, r["lo"], d.lo, -5, f"{what}: int8 logits")
            d.check(n, r["la"], d.la, -7, f"{what}: int8 labels")
            d.check(n, r["la_only"], d.la, -7, f"{what}: int8 labels only")
            d.check(n, r["cls"], d.topk_c[k][0], -1, f"{what}: top-{k} classes")
            d.check(n, r["sc"], d.topk_c[k][1], -7, f"{what}: top-{k} scores")
            d.check(n, r["f_lo"], lo, -5, f"{what}: float32 logits")
            d.check(n, r["h_la"], h_la, -7, f"{what}: float16 labels")
            d.check(n, r["emu"], emu, -7, f"{what}: emulator logits")
            d.check(n, r["emu_la"], emu_la, -7, f"{what}: emulator labels")
            d.check(n, r["pcls"], d.topk_py[k][0], -1, f"{what}: emulator top-{k} classes")
            d.check(n, r["psc"], d.topk_py[k][1], -7, f"{what}: emulator top-{k} scores")
    finally:
        e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["cnn48", "cnn48-imad"])
def test_frontend_switches(lib, capfd, monkeypatch, name):
    """BNM_OPT_CNN_FRONTEND 0 -> 1 -> 2 -> 0 on CNN-48, with conv3 on IDP.2A and on IMAD: the top-k route names the front-end
    kernel, and every entry family gives the same results"""
    from bitnetmcu_b200.engine import Engine
    e, err = verbose_engine(capfd, monkeypatch, lambda: Engine(model(name), device=0))
    packed = conv3_bound(model(name)) <= 65535
    assert [l for l in err if "conv3 on " + ("IDP.2A" if packed else "IMAD") in l], (name, err)
    d = Dev(name, False)
    row = plan(name).forms["topk"].row
    try:
        for value in (0, 1, 2, 0):
            what = f"{OPT_NAMES[OPT_FRONTEND]} = {value} (conv3 on {'IDP.2A' if packed else 'IMAD'})"
            assert set_rc(lib, e, OPT_FRONTEND, value) == (0, ""), (name, what)
            assert options(lib, e)["BNM_OPT_CNN_FRONTEND"] == value, (name, what)
            front = "k_cnn_frontend16 + " if value == 1 else "k_cnn_frontend16_tc + "
            assert topk_route(capfd, e, d) == front + row, (name, what)
            every_family(lib, e, d, what, sizes=SIZES[:2])
            capfd.readouterr()
    finally:
        e.close()


@pytest.mark.gpu
def test_graph_keeps_its_frontend(lib, capfd, monkeypatch):
    """the int8, top-k and float entries captured under front-end 2 (tensor cores), then BNM_OPT_CNN_FRONTEND = 1: each replay
    equals its eager call on the same buffers, prints no route line, and the eager calls name k_cnn_frontend16"""
    import torch
    from bitnetmcu_b200.engine import Engine
    name = "cnn48"
    e, _ = verbose_engine(capfd, monkeypatch, lambda: Engine(model(name), device=0))
    d = Dev(name, False)
    n, k = 700, 5
    q, x = d.q[d.idx(n)].clone(), d.x[d.idx(n)].clone()

    def bufs():
        return [out((n, d.C), torch.int32, -5), out((n,), torch.int32, -7), out((n, k), torch.int32, -1),
                out((n, k), torch.int32, -7), out((n, d.C), torch.int32, -5)]

    def calls(b):
        e.infer_device(q, b[0][:n], b[1][:n])
        e.topk_device(q, k, b[2][:n], b[3][:n])
        e.infer_device_f32(x, b[4][:n], None)
    try:
        assert set_rc(lib, e, OPT_FRONTEND, 2) == (0, "")
        g_out = bufs()
        sync()
        capfd.readouterr()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            calls(g_out)
        captured = err_lines(capfd, "topk route: ")
        assert len(captured) == 1 and "k_cnn_frontend16_tc + " in captured[0], captured
        assert set_rc(lib, e, OPT_FRONTEND, 1) == (0, "")
        for seed in (1, 2):   # new images in the captured buffers
            j = (d.idx(n) * seed + seed) % N_UNIQUE
            q.copy_(d.q[j])
            x.copy_(d.x[j])
            for b in g_out:
                b.fill_(-9)
            g.replay()
            sync()
            assert err_lines(capfd, "route") == [], seed
            eager = bufs()
            calls(eager)
            sync()
            routes = err_lines(capfd, "topk route: ")
            assert len(routes) == 1 and "k_cnn_frontend16 + " in routes[0], routes
            what = f"graph captured under {OPT_NAMES[OPT_FRONTEND]} = 2, replayed under 1, images {seed}"
            for part, a, b in zip(("int8 logits", "int8 labels", "top-k classes", "top-k scores", "float32 logits"), g_out, eager):
                assert torch.equal(a[:n], b[:n]), (what, part, "replay vs eager")
            assert torch.equal(eager[0][:n], d.lo[j]) and torch.equal(eager[1][:n], d.la[j]), (what, "eager int8 vs the oracle")
            assert torch.equal(eager[4][:n], d.want["float32"][0][j]), (what, "eager float32 vs the oracle")
        del g
    finally:
        e.close()


# ---- GPU: chunk resizes on one engine ---------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_chunk_resizes(lib):
    """one engine's host pipeline through BNM_OPT_CHUNK_IMAGES 65536 (emulator), 128 (int8), 1000 (top-k), 300000 (emulator)
    and 128 (int8): its slot buffers grow for the largest chunk and serve smaller chunks of another element size after it.  At
    each step n = 3 chunks + 17 images (at most 300017) and a 700-image int8 call, against the oracle and restate.emulate"""
    from bitnetmcu_b200.engine import Engine
    name = "fc"
    e = Engine(model(name), device=0)
    x = expect(name, False)
    lo, la = x["int8"]
    emu = x["float32"][2]
    try:
        for chunk, entry in ((65536, "emulator"), (128, "int8"), (1000, "top-k"), (300000, "emulator"), (128, "int8")):
            assert set_rc(lib, e, OPT_CHUNK, chunk) == (0, "")
            assert options(lib, e)["BNM_OPT_CHUNK_IMAGES"] == chunk
            n = min(3 * chunk + 17, 300017)
            what = f"{OPT_NAMES[OPT_CHUNK]} = {chunk}, {n} images"
            i = np.arange(n) % N_UNIQUE
            if entry == "emulator":
                got = e.inference_quantized(x["x"][i])
                assert np.array_equal(got, emu[i]), (what, "host emulator logits")
            elif entry == "int8":
                glo, gla = e.infer(x["q"][i])
                assert np.array_equal(glo, lo[i]) and np.array_equal(gla.astype(np.int32), la[i]), (what, "host int8")
            else:
                cls, sc = e.topk(x["q"][i], 5)
                wc, ws = top_k(lo, 5)
                assert np.array_equal(cls.astype(np.int32), wc[i]) and np.array_equal(sc, ws[i]), (what, "host top-5")
            j = np.arange(700) % N_UNIQUE
            glo, gla = e.infer(x["q"][j])
            assert np.array_equal(glo, lo[j]) and np.array_equal(gla.astype(np.int32), la[j]), (what, "host int8, 700 images")
    finally:
        e.close()
