"""Window scan of a stack of float16 or bfloat16 pages (include/bitnetmcu_b200.h section 12): bnm_scan_windows_device_f16,
bnm_scan_windows_topk_device_f16, bnm_emulate_windows_device_f16 and bnm_emulate_windows_topk_device_f16.

Each entry is defined as its section 10 sibling on the stack widened to float32 (an exact conversion), so every GPU case runs both
on the same pages, the sibling on ``pages.float()``, and compares every output with tolerance 0.  The siblings are verified against
the oracle and the emulator restatement elsewhere.  The CPU tests check the symbols, the descriptor's layout, the failure without a
device, the scaling kernel's SASS, and a NumPy restatement of widening followed by the window scaling (column maxima, then a
16-wide sliding maximum) against the reference's per-image scaling on the widened windows."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from conftest import ROOT, load_model
from restate import scale_images
from support import instructions, lib, local_memory, random_fc, sass_functions, verbose_engine  # noqa: F401 (lib: fixture)

FORMATS = ["float16", "bfloat16"]
MODELS = ["fc", "12k_FP130", "ternary64", "binary160", "2bitsym96", "cnn_48", "cnn_letters", "rand_nf4_64"]
STRIDES = [(1, 1), (2, 3), (16, 16), (17, 5)]
STACKS = [(1, 37, 53), (3, 50, 18), (7, 41, 67)]   # planes, height, width: odd pages; out_w below 4 in the second
ENTRIES = ["scan", "scan_topk", "emulate", "emulate_topk"]
NAMES = {"scan": "bnm_scan_windows_device", "scan_topk": "bnm_scan_windows_topk_device", "emulate": "bnm_emulate_windows_device",
         "emulate_topk": "bnm_emulate_windows_topk_device"}
SENTINEL = -7
BNM_E_ARG, BNM_E_NODEV, BNM_E_UNSUPPORTED = -1, -2, -3


# ---- restatements ------------------------------------------------------------------------------------------------------------

def widen(bits, fmt):
    """the exact widening of 16-bit patterns (uint16) to float32, with integer arithmetic: bfloat16 is the top half of a float32;
    float16 moves its exponent and mantissa into float32's, normalising subnormals"""
    b = np.asarray(bits, dtype=np.uint32)
    if fmt == "bfloat16":
        return (b << 16).view(np.float32)
    sign, exp, man = (b >> 15) << 31, (b >> 10) & 0x1F, b & 0x3FF
    out = np.where(exp == 0x1F, (0xFF << 23) | (man << 13), ((exp + 112) << 23) | (man << 13))   # inf / NaN, normal
    sub = man.astype(np.float64) * 2.0 ** -24                                                   # subnormal and zero: exact
    out = np.where(exp == 0, sub.astype(np.float32).view(np.uint32), out)
    return (out | sign).astype(np.uint32).view(np.float32)


def stacked_windows_np(buf, planes, h, w, pitch, plane_pitch, sy, sx):
    """the windows of a stack held in the flat array buf (plane p at p * plane_pitch, rows pitch apart), numbered plane by plane,
    then row-major, each flattened row-major: [planes * out_h * out_w, 256]"""
    from numpy.lib.stride_tricks import as_strided
    if planes == 0 or h < 16 or w < 16:
        return np.zeros((0, 256), dtype=buf.dtype)
    oh, ow = (h - 16) // sy + 1, (w - 16) // sx + 1
    e = buf.itemsize
    v = as_strided(buf, shape=(planes, oh, ow, 16, 16), strides=(plane_pitch * e, sy * pitch * e, sx * e, pitch * e, e), writeable=False)
    return np.ascontiguousarray(v).reshape(-1, 256)


def window_scaling(page, sy, sx):
    """the window scaling kernel's steps on one float32 page [h, w]: every column's max |x| over a window row's 16 rows, the max of
    16 of them per window, scale = 127 / max(that, 1e-5), each pixel round_half_even(x * scale) clipped, all in float32.  Its
    maxima carry NaN, as NumPy's do, and a NaN product (a NaN pixel, or inf times a scale of 0) scales to 0: a window holding a
    NaN or an infinity is the all-zero row -> int8 [windows, 256]"""
    h, w = page.shape
    oh, ow = (h - 16) // sy + 1, (w - 16) // sx + 1
    out = np.empty((oh, ow, 256), dtype=np.int8)
    for r, c in np.ndindex(oh, ow):
        band = page[r * sy:r * sy + 16]
        col = np.abs(band).max(axis=0)
        m = col[c * sx:c * sx + 16].max()
        scale = np.float32(127.0) / np.maximum(m, np.float32(1e-5))
        with np.errstate(invalid="ignore"):
            y = np.round(band[:, c * sx:c * sx + 16] * scale).clip(-128, 127).reshape(256)
        out[r, c] = np.where(np.isnan(y), 0, y).astype(np.int8)
    return out.reshape(-1, 256)


def edge_page_bits(fmt, h=48, w=64, seed=0):
    """a 16-bit page (uint16 patterns [h, w]) of normal pixels with blocks of the scaling edges: zeros of both signs, subnormals,
    the largest finite value of the format, infinities, NaN and maxima below 1e-5"""
    import torch
    rng = np.random.default_rng(seed)
    x = torch.from_numpy(rng.standard_normal((h, w), dtype=np.float32)).to(getattr(torch, fmt))
    bits = x.view(torch.int16).numpy().view(np.uint16).copy()
    big = 0x7BFF if fmt == "float16" else 0x7F7F          # 65504 / the largest finite bfloat16
    inf, nan = (0x7C00, 0x7E00) if fmt == "float16" else (0x7F80, 0x7FC0)
    sign = lambda: rng.integers(0, 2, (16, 16)) << 15
    bits[0:16, 0:16] = 0x0000                             # whole windows at every stride: zeros, subnormals, maxima below 1e-5
    bits[2:10, 2:10] = 0x8000                             # -0.0
    bits[16:32, 0:16] = rng.integers(0, 0x0400 if fmt == "float16" else 0x0080, size=(16, 16)) | sign()
    bits[22, 3] = 0x0001                                  # the smallest subnormal of either format
    bits[0:16, 16:32] = (widen_inverse(np.float32(3e-6), fmt) + rng.integers(0, 8, size=(16, 16))) | sign()
    bits[5, 50], bits[30, 52] = big, big | 0x8000
    bits[40, 30], bits[44, 60] = inf, inf | 0x8000
    bits[25, 45], bits[46, 10] = nan, nan | 0x8000
    return bits


def edge_pages_bits(fmt):
    """edge_page_bits and its mirror image with every sign flipped: two planes [2, 48, 64]"""
    bits = edge_page_bits(fmt)
    return np.ascontiguousarray(np.stack([bits, bits[::-1, ::-1] ^ np.uint16(0x8000)]))


def widen_inverse(v, fmt):
    """the 16-bit pattern nearest float32 v (round to nearest even), as an int"""
    if fmt == "float16":
        return int(np.float16(v).view(np.uint16))
    u = int(np.float32(v).view(np.uint32))
    return (u + 0x7FFF + ((u >> 16) & 1)) >> 16


# ---- CPU ----------------------------------------------------------------------------------------------------------------------

def test_entries_are_declared_and_exported(built):
    from bitnetmcu_b200 import _lib
    text = open(os.path.join(ROOT, "include", "bitnetmcu_b200.h")).read()
    assert "typedef struct bnm_windows_f16" in text
    lib = _lib.load()
    for name in NAMES.values():
        assert re.search(rf"BNM_API int {name}_f16\(bnm_model \*m, const bnm_windows_f16 \*windows, int format,", text), name
        assert name + "_f16" in _lib.EXPORTED and hasattr(lib, name + "_f16"), name


def test_descriptor_layout(built):
    """bnm_windows_f16 declares the fields of bnm_windows in the same order and types, the image's element type aside, so
    _lib.BnmWindows (48 bytes) serves both"""
    from bitnetmcu_b200 import _lib
    text = open(os.path.join(ROOT, "include", "bitnetmcu_b200.h")).read()

    def fields(name):
        body = re.search(rf"typedef struct {name} \{{(.*?)\}} {name};", text, re.S).group(1)
        body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
        out = []
        for decl in filter(None, (d.strip() for d in body.split(";"))):
            t, names = decl.rsplit(" ", 1) if "," not in decl else decl.split(" ", 1)
            for n in names.split(","):
                n = n.strip()
                out.append((t.strip() + " *" * n.startswith("*"), n.lstrip("*")))
        return out
    f32, f16 = fields("bnm_windows"), fields("bnm_windows_f16")
    assert [n for _, n in f32] == [n for _, n in f16] == [n for n, _ in _lib.BnmWindows._fields_]
    assert f32[0] == ("const float *", "image") and f16[0] == ("const uint16_t *", "image")
    assert f32[1:] == f16[1:]
    assert C.sizeof(_lib.BnmWindows) == 48
    src = open(os.path.join(ROOT, "bitnetmcu_b200", "csrc", "capi.cu")).read()
    for n, _ in _lib.BnmWindows._fields_:
        assert f"offsetof(bnm_windows_f16, {n}) == offsetof(bnm_windows, {n})" in src, n


def test_entries_fail_without_a_device(built):
    from bitnetmcu_b200 import _lib
    lib = _lib.load()
    if lib.bnm_device_count() > 0:
        pytest.skip("a CUDA device is present")
    img = np.zeros(4 * 64 * 64, dtype=np.uint16)
    d = _lib.BnmWindows(img.ctypes.data, 2, 64, 64, 64, 64 * 64, 16, 16)
    out = np.full(64, 7, dtype=np.uint32)
    o = C.c_void_p(out.ctypes.data)
    for fmt in (_lib.FLOAT16, _lib.BFLOAT16):
        for rc in (lib.bnm_scan_windows_device_f16(None, C.byref(d), fmt, None, o, None),
                   lib.bnm_scan_windows_topk_device_f16(None, C.byref(d), fmt, 1, o, None, None),
                   lib.bnm_emulate_windows_device_f16(None, C.byref(d), fmt, None, o, None),
                   lib.bnm_emulate_windows_topk_device_f16(None, C.byref(d), fmt, 1, o, None, None)):
            assert rc == BNM_E_NODEV and b"no CUDA device" in lib.bnm_last_error()
    assert (out == 7).all()


def test_window_kernel_is_one_function_without_local_memory(built):
    """the element kind is a runtime field of k_quantize_windows, as planes are: one function serves float32, float16 and
    bfloat16 planes"""
    funcs = {k: v for k, v in sass_functions().items() if "k_quantize_windows" in k}
    assert list(funcs) == ["_ZN3bnm18k_quantize_windowsENS_9WindowRunE"], list(funcs)
    ins = instructions(next(iter(funcs.values())))
    assert not local_memory(ins)
    loads = [i for i in ins if "LDG" in i]
    assert any("LDG.E.U16" in i for i in loads) and any(re.search(r"LDG\.E\.CONSTANT\b", i) for i in loads), loads


def test_widening_restatement_matches_numpy():
    """all 65 536 patterns: float16 as NumPy widens np.float16; bfloat16 as the top 16 bits of the float32 it was cut from"""
    bits = np.arange(1 << 16, dtype=np.uint32).astype(np.uint16)
    want = bits.view(np.float16).astype(np.float32)
    got = widen(bits, "float16")
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan) and np.array_equal(got[~nan].view(np.uint32), want[~nan].view(np.uint32))
    f = np.random.default_rng(0).uniform(-3e38, 3e38, 4096).astype(np.float32)
    assert np.array_equal(widen((f.view(np.uint32) >> 16).astype(np.uint16), "bfloat16").view(np.uint32), f.view(np.uint32) & 0xFFFF0000)


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("sy,sx", [(1, 1), (3, 2), (16, 16), (7, 5)])
def test_window_scaling_restatement_on_widened_windows(fmt, sy, sx):
    """widening, then the window scaling (column maxima, sliding maximum) equals restate.scale_images on the widened windows
    extracted one by one, on a page with zeros of both signs, subnormals, maxima below 1e-5, the format's largest finite value,
    infinities and NaN; every window holding a NaN or an infinity is the all-zero row"""
    bits = edge_page_bits(fmt)
    page = widen(bits, fmt)
    got = window_scaling(page, sy, sx)
    wins = stacked_windows_np(page.reshape(-1), 1, *page.shape, page.shape[1], 0, sy, sx)
    assert got.shape == wins.shape and len(got) > 0
    assert np.array_equal(got, scale_images(wins))
    poisoned = ~np.isfinite(wins).all(axis=1)
    assert poisoned.any() and (~poisoned).any() and np.isnan(wins).any() and np.isinf(wins).any()
    assert not got[poisoned].any()
    # the finite cases are there too: a window whose maximum is a subnormal, one below 1e-5 but normal, one at the format's
    # largest value
    m = np.abs(wins[~poisoned]).max(axis=1)
    assert (m[m > 0] < np.float32(1.2e-38) if fmt == "bfloat16" else m[m > 0] < np.float32(6.1e-5)).any()
    assert ((m > 0) & (m < np.float32(1e-5))).any()
    assert (m == widen(np.uint16(0x7BFF if fmt == "float16" else 0x7F7F), fmt)).any()


# ---- GPU ----------------------------------------------------------------------------------------------------------------------

def _engine(name, path=0):
    from bitnetmcu_b200.engine import Engine
    m = load_model(name) if isinstance(name, str) else name
    return Engine(m, device=0, path=path, nf4_extension=(name == "rand_nf4_64"))


def page_np(h, w, seed):
    """normal pixels with MNIST-normalised patches and a dark margin, float32 [h, w]"""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal(size=(h, w), dtype=np.float32)
    for _ in range(max(1, h * w // 4000)):
        r, c = rng.integers(0, max(1, h - 20)), rng.integers(0, max(1, w - 20))
        x[r:r + 20, c:c + 20] = (rng.integers(0, 256, size=(min(20, h - r), min(20, w - c))) / 255.0 - 0.1307).astype(np.float32) / np.float32(0.3081)
    x[:, :3] *= np.float32(0.01)
    return x


def pages_np(planes, h, w, seed):
    return np.stack([page_np(h, w, seed=seed + 7 * p) for p in range(planes)])


def stack(pages, dtype, fill=0.0, gap=0, pad=0, below=0):
    """pages (a CPU tensor or NumPy array [P, h, w]) as a CUDA stack of dtype [P, h, w] inside one allocation: rows 16 bytes
    rounded + pad elements apart, `below` rows past each page and `gap` elements between planes, all that padding filled with
    fill ("nan-inf": NaN and infinity alternating)"""
    import torch
    src = torch.as_tensor(pages)
    p, h, w = src.shape
    per = 16 // torch.empty((), dtype=dtype).element_size()
    pitch = (w + per - 1) // per * per + pad
    plane_pitch = (h + below) * pitch + gap
    buf = torch.full((max(p, 1) * plane_pitch,), float("nan") if fill == "nan-inf" else fill, dtype=dtype, device="cuda")
    if fill == "nan-inf":
        buf[::2] = float("inf")
    view = buf.as_strided((p, h, w), (plane_pitch, pitch, 1))
    view.copy_(src.to(dtype))
    return view


def half_stack(planes, h, w, seed, fmt, **kw):
    import torch
    return stack(pages_np(planes, h, w, seed), getattr(torch, fmt), **kw)


def widened(pages):
    """a 16-bit CUDA stack widened to float32, in a float32 stack of its own: what a caller passes today, ``pages.float()``"""
    import torch
    return stack(pages.float().cpu(), torch.float32)


def _k(e):
    return min(e.n_classes, 5)


def run_stack(e, entry, pages, stride, k=None, first=True, second=True, stream=None, sync=True):
    """a stacked entry on a CUDA stack (its dtype picks the entry) -> its two outputs as NumPy, flattened to [windows, ...]
    (None where not asked): (logits, labels) or (classes, scores)"""
    import torch
    from bitnetmcu_b200.engine import window_grid
    grid = (pages.shape[0] if pages.dim() == 3 else 1,) + window_grid(pages.shape[-2], pages.shape[-1], stride)
    emul, topk = entry.startswith("emulate"), entry.endswith("topk")
    ldt = torch.float64 if emul else torch.int32
    if topk:
        k = k or _k(e)
        a = torch.full(grid + (k,), SENTINEL, dtype=torch.int32, device="cuda") if first else None
        b = torch.full(grid + (k,), SENTINEL, dtype=ldt, device="cuda") if second else None
        (e.emulate_windows_topk_device if emul else e.scan_windows_topk_device)(pages, stride, k, a, b, stream=stream)
    else:
        a = torch.full(grid + (e.n_classes,), SENTINEL, dtype=ldt, device="cuda") if first else None
        b = torch.full(grid, SENTINEL, dtype=torch.int32, device="cuda") if second else None
        (e.emulate_windows_device if emul else e.scan_windows_device)(pages, stride, a, b, stream=stream)
    if not sync:
        return a, b
    torch.cuda.synchronize()
    n = int(np.prod(grid))
    return tuple(None if t is None else t.reshape(n, -1).cpu().numpy() for t in (a, b))


def assert_same(got, want, what):
    for g, w, kind in zip(got, want, ("first", "second")):
        if g is None or w is None:
            continue
        assert g.shape == w.shape, (what, kind, g.shape, w.shape)
        same = (g == w) | (np.isnan(g) & np.isnan(w)) if g.dtype.kind == "f" else g == w
        bad = np.flatnonzero(~same.reshape(len(w), -1).all(axis=1))
        assert bad.size == 0, (what, kind, f"{bad.size} of {len(w)} windows differ, first {bad[:6].tolist()}")


def assert_sibling(e, entry, pages, stride, what, **kw):
    """the 16-bit entry on pages equals its float32 sibling on pages.float(), and writes something"""
    got = run_stack(e, entry, pages, stride, **kw)
    assert_same(got, run_stack(e, entry, widened(pages), stride, **kw), what)
    assert all(g is None or len(g) == 0 or (g != SENTINEL).any() for g in got), what
    return got


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("name", MODELS)
def test_entries_equal_the_float32_siblings(lib, name, fmt):
    """every entry, stride and stack, on the default path and BNM_PATH_LAYERS: the float32 sibling on pages.float()"""
    from bitnetmcu_b200 import _lib
    e = _engine(name)
    for path in (_lib.PATH_AUTO, _lib.PATH_LAYERS):
        e.set_option(_lib.OPT_PATH, path)
        for planes, h, w in STACKS:
            pages = half_stack(planes, h, w, planes * 100 + h, fmt, gap=8 * planes)
            for stride in STRIDES:
                for entry in ENTRIES:
                    assert_sibling(e, entry, pages, stride, (name, fmt, path, planes, stride, entry))
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("name", ["fc", "cnn_letters", "binary160"])
def test_outputs_and_k(lib, name, fmt):
    """labels only, logits only and both; top-k with and without scores at k = 1 and min(n_classes, 16): each the sibling's"""
    e = _engine(name)
    pages = half_stack(3, 50, 70, 1, fmt)
    for entry in ENTRIES:
        if entry.endswith("topk"):
            for k in (1, min(e.n_classes, 16)):
                for second in (True, False):
                    assert_sibling(e, entry, pages, (1, 2), (entry, k, second), k=k, second=second)
        else:
            for first, second in ((True, True), (False, True), (True, False)):
                assert_sibling(e, entry, pages, (1, 2), (entry, first, second), first=first, second=second)
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("name", ["fc", "binary160", "cnn_48"])
def test_only_the_window_pixels_count(lib, name, fmt):
    """stacks whose row padding, rows below each page and gaps between planes hold NaN and infinity: the results of the clean
    stack (a band that read past a window's rows or the plane's width would see them)"""
    import torch
    e = _engine(name)
    for planes, h, w in STACKS:
        x = pages_np(planes, h, w, seed=h + w)
        clean = stack(x, getattr(torch, fmt))
        dirty = stack(x, getattr(torch, fmt), fill="nan-inf", gap=40, pad=8, below=9)
        assert dirty.stride(0) > dirty.shape[1] * dirty.stride(1) and dirty.stride(1) > dirty.shape[2]
        for stride in STRIDES:
            for entry in ENTRIES:
                assert_same(run_stack(e, entry, dirty, stride), run_stack(e, entry, clean, stride), (name, fmt, planes, stride, entry))
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("name", ["fc", "binary160", "cnn_48"])
def test_scaling_edges(lib, name, fmt):
    """windows whose maximum is a subnormal or below 1e-5, windows holding infinities or NaN, and the format's largest finite
    value, through every entry: the sibling's results"""
    import torch
    pages = stack(torch.from_numpy(edge_pages_bits(fmt).view(np.int16)).view(getattr(torch, fmt)), getattr(torch, fmt))
    e = _engine(name)
    for stride in [(1, 1), (2, 3), (16, 16)]:
        for entry in ENTRIES:
            assert_sibling(e, entry, pages, stride, (name, fmt, "edges", stride, entry))
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", FORMATS)
def test_scaling_edges_follow_numpy(lib, fmt):
    """the rows the GPU scaled from the edge pages are the NumPy rule's (window_scaling, pinned to the reference expression on
    the CPU): the C engine's logits of each window equal its int8-input logits of the restated rows, and every window holding a
    NaN or an infinity has the all-zero row's logits"""
    import torch
    bits = edge_pages_bits(fmt)
    pages = stack(torch.from_numpy(bits.view(np.int16)).view(getattr(torch, fmt)), getattr(torch, fmt))
    e = _engine("fc")
    zero = torch.zeros((1, 256), dtype=torch.int8, device="cuda")
    zlo = torch.empty((1, 10), dtype=torch.int32, device="cuda")
    e.infer_device(zero, zlo, None)
    for stride in [(1, 1), (2, 3), (16, 16)]:
        lo, _ = run_stack(e, "scan", pages, stride)
        page_rows = [window_scaling(widen(b, fmt), *stride) for b in bits]
        rows = np.concatenate(page_rows)
        want = torch.empty((len(rows), 10), dtype=torch.int32, device="cuda")
        e.infer_device(torch.from_numpy(rows).cuda(), want, None)
        torch.cuda.synchronize()
        assert np.array_equal(lo, want.cpu().numpy()), (fmt, stride)
        wins = np.concatenate([stacked_windows_np(widen(b, fmt).reshape(-1), 1, *b.shape, b.shape[1], 0, *stride) for b in bits])
        poisoned = ~np.isfinite(wins).all(axis=1)
        assert poisoned.any() and (~poisoned).any(), (fmt, stride)
        assert (lo[poisoned] == zlo.cpu().numpy()).all(), (fmt, stride)
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", FORMATS)
def test_pass_boundary_inside_a_plane_and_a_window_row(lib, fmt):
    """three planes of 601 x 701 windows at stride 1: window 2^20, where the second pass starts, is in row 293 of the third
    plane, column 581"""
    import torch
    pages = half_stack(3, 16 + 600, 16 + 700, 41, fmt)
    w0 = 1 << 20
    p, r, c = w0 // (601 * 701), w0 % (601 * 701) // 701, w0 % 701
    assert (p, r, c) == (2, 293, 581)
    e = _engine("fc")
    for entry in ("scan", "scan_topk", "emulate"):
        got = assert_sibling(e, entry, pages, 1, (fmt, entry, "pass"))
        assert got[0].shape[0] == 3 * 601 * 701 > w0
        torch.cuda.empty_cache()
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", FORMATS)
def test_last_plane_past_2_31_elements(lib, fmt):
    """two 16-bit planes 2^31 + 256 elements apart: the second starts past 2^31 elements and past 4 GiB; every entry equals the
    sibling on the two planes widened"""
    import torch
    dt = getattr(torch, fmt)
    plane_pitch = (1 << 31) + 256
    h, w = 40, 64
    buf = torch.full((plane_pitch + h * w,), float("nan"), dtype=dt, device="cuda")
    pages = buf.as_strided((2, h, w), (plane_pitch, w, 1))
    pages.copy_(torch.from_numpy(pages_np(2, h, w, seed=64)).to(dt))
    assert pages[1].data_ptr() - pages.data_ptr() > 4 << 30
    for name in ("fc", "cnn_48"):
        e = _engine(name)
        for entry in ENTRIES:
            assert_sibling(e, entry, pages, (2, 3), (name, fmt, entry, "past 2^31"))
        e.close()
    del pages, buf
    torch.cuda.empty_cache()


@pytest.mark.gpu
def test_argument_errors(lib):
    """each argument error gives its code and writes nothing: a format other than 1 or 2 whatever the descriptor holds, pitches
    that are not a multiple of 8 elements, a misaligned image, a bad k, no output, a model whose images are not 256 elements"""
    import torch
    from bitnetmcu_b200 import _lib
    e = _engine("fc")
    img = torch.zeros((4 * 64 * 64 + 64,), dtype=torch.float16, device="cuda")
    lo = torch.full((4 * 49 * 49 * 10 + 64,), SENTINEL, dtype=torch.float64, device="cuda")   # room for every output type
    la = torch.full((4 * 49 * 49 * 16 + 64,), SENTINEL, dtype=torch.int32, device="cuda")
    P = lambda t, off=0: C.c_void_p(t.data_ptr() + off)

    def desc(planes=2, h=64, w=64, pitch=64, plane_pitch=64 * 64, sy=1, sx=1, off=0):
        return _lib.BnmWindows(img.data_ptr() + off, planes, h, w, pitch, plane_pitch, sy, sx)

    calls = {
        "scan": lambda d, f, a, b, k: lib.bnm_scan_windows_device_f16(e.handle, d, f, a, b, None),
        "scan_topk": lambda d, f, a, b, k: lib.bnm_scan_windows_topk_device_f16(e.handle, d, f, k, b, a, None),
        "emulate": lambda d, f, a, b, k: lib.bnm_emulate_windows_device_f16(e.handle, d, f, a, b, None),
        "emulate_topk": lambda d, f, a, b, k: lib.bnm_emulate_windows_topk_device_f16(e.handle, d, f, k, b, a, None),
    }
    for entry, call in calls.items():
        topk = entry.endswith("topk")
        for bad in (0, 3):
            for d in (C.byref(desc()), C.byref(desc(planes=0)), None):
                assert call(d, bad, P(lo), P(la), 3) == BNM_E_ARG and b"format" in lib.bnm_last_error(), (entry, bad)
        for fmt in (_lib.FLOAT16, _lib.BFLOAT16):
            cases = {
                "null descriptor": call(None, fmt, P(lo), P(la), 3),
                "zero stride": call(C.byref(desc(sy=0)), fmt, P(lo), P(la), 3),
                "pitch < width": call(C.byref(desc(pitch=56)), fmt, P(lo), P(la), 3),
                "pitch % 8 (a multiple of 4)": call(C.byref(desc(w=60, pitch=60)), fmt, P(lo), P(la), 3),
                "plane pitch % 8 (a multiple of 4)": call(C.byref(desc(plane_pitch=64 * 64 + 4)), fmt, P(lo), P(la), 3),
                "image misaligned by 8 bytes": call(C.byref(desc(off=8)), fmt, P(lo), P(la), 3),
                "logits / scores misaligned": call(C.byref(desc()), fmt, P(lo, 2 if entry == "scan_topk" else 4), P(la), 3),
                "no output": call(C.byref(desc()), fmt, None, None, 3),
            }
            if topk:
                cases.update({"k = 0": call(C.byref(desc()), fmt, P(lo), P(la), 0), "k = 11": call(C.byref(desc()), fmt, P(lo), P(la), 11),
                              "k = 0, no windows": call(C.byref(desc(planes=0)), fmt, P(lo), P(la), 0)})
            assert cases == {k: BNM_E_ARG for k in cases}, (entry, fmt, cases)
            call(C.byref(desc(w=60, pitch=60)), fmt, P(lo), P(la), 3)
            assert b"multiple of 8 elements" in lib.bnm_last_error()
            for d in (desc(planes=0), desc(h=15), desc(w=15)):
                assert call(C.byref(d), fmt, P(lo), P(la), 3) == 0, entry
            # one plane ignores the plane pitch
            assert call(C.byref(desc(planes=1, h=15, plane_pitch=3)), fmt, P(lo), P(la), 3) == 0, entry
    wide = _engine(random_fc(4, (512, 64, 64, 10), 1))
    for fmt in (_lib.FLOAT16, _lib.BFLOAT16):
        assert lib.bnm_scan_windows_device_f16(wide.handle, C.byref(desc()), fmt, P(lo), P(la), None) == BNM_E_UNSUPPORTED
        assert b"16x16" in lib.bnm_last_error()
        assert lib.bnm_emulate_windows_device_f16(wide.handle, C.byref(desc()), fmt, P(lo), P(la), None) == BNM_E_UNSUPPORTED
        assert lib.bnm_scan_windows_topk_device_f16(wide.handle, C.byref(desc()), fmt, 3, P(la), P(lo), None) == BNM_E_UNSUPPORTED
        assert lib.bnm_emulate_windows_topk_device_f16(wide.handle, C.byref(desc()), fmt, 3, P(la), P(lo), None) == BNM_E_UNSUPPORTED
    wide.close()
    torch.cuda.synchronize()
    assert (lo == SENTINEL).all() and (la == SENTINEL).all()
    e.close()


ROUTE_CASES = [("fc", lambda: load_model("fc"), 0), ("37 classes", lambda: random_fc(4, (256, 64, 64, 37), 2), 0),
               ("binary160", lambda: load_model("binary160"), 0), ("cnn_48", lambda: load_model("cnn_48"), 0),
               ("layers", lambda: load_model("fc"), 1), ("cnn layers", lambda: load_model("cnn_48"), 1)]


@pytest.mark.gpu
def test_routes_name_the_16bit_scaling_step(lib, capfd, monkeypatch):
    """each 16-bit entry prints one windows route line: the float32 sibling's route with k_quantize_windows<float16> or
    <bfloat16> as its scaling step, and the float32 line unchanged"""
    import torch
    for what, make, path in ROUTE_CASES:
        e, _ = verbose_engine(capfd, monkeypatch, lambda: _engine(make(), path=path))
        for fmt in FORMATS:
            pages = half_stack(2, 40, 40, 2, fmt)
            for entry in ENTRIES:
                lines = {}
                for kind, p in ((fmt, pages), ("float32", widened(pages))):
                    torch.cuda.synchronize()
                    capfd.readouterr()
                    run_stack(e, entry, p, 3)
                    got = [l for l in capfd.readouterr().err.splitlines() if "route: " in l]
                    assert len(got) == 1, (what, entry, kind, got)
                    name = NAMES[entry] + ("_f16" if kind != "float32" else "")
                    assert f"windows route: {name}: " in got[0], (what, entry, kind, got)
                    lines[kind] = got[0].split(f"windows route: {name}: ")[1]
                assert lines["float32"].startswith("k_quantize_windows + "), (what, entry, lines)
                assert lines[fmt] == lines["float32"].replace("k_quantize_windows + ", f"k_quantize_windows<{fmt}> + ", 1), (what, entry, lines)
        e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["fc", "cnn_48", "binary160"])
def test_graph_replay_and_two_streams(lib, name):
    """a captured 16-bit call replays as the eager call on the pages' contents at replay time; calls on two streams give each
    stack's own results"""
    import torch
    e = _engine(name)
    shape, stride = (3, 150, 100), (2, 1)
    for fmt in FORMATS:
        for entry in ENTRIES:
            pages = half_stack(*shape, 4, fmt)
            run_stack(e, entry, pages, stride, sync=False)   # warm: the pool and the kernels' attributes
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=torch.cuda.Stream()):
                outs = run_stack(e, entry, pages, stride, sync=False)
            pages.copy_(torch.from_numpy(pages_np(*shape, seed=5)).to(pages.dtype))
            g.replay()
            torch.cuda.synchronize()
            got = tuple(t.reshape(outs[1].shape[:3].numel(), -1).cpu().numpy() for t in outs)
            assert_same(got, run_stack(e, entry, pages, stride), (name, fmt, entry, "replay"))
            assert_same(got, run_stack(e, entry, widened(pages), stride), (name, fmt, entry, "replay, float32"))
            del g
            stacks = [half_stack(*shape, 10 + k, fmt) for k in range(2)]
            alone = [run_stack(e, entry, p, stride) for p in stacks]
            streams = [torch.cuda.Stream(), torch.cuda.Stream()]
            torch.cuda.synchronize()
            for _ in range(3):
                res = []
                for p, st in zip(stacks, streams):
                    with torch.cuda.stream(st):
                        res.append(run_stack(e, entry, p, stride, sync=False))
            torch.cuda.synchronize()
            for k, outs in enumerate(res):
                assert_same(tuple(t.reshape(outs[1].shape[:3].numel(), -1).cpu().numpy() for t in outs), alone[k], (name, fmt, entry, "stream", k))
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", FORMATS)
def test_mode2_int8_launch_after_a_16bit_window_call_waits(lib, oracle, capfd, monkeypatch, fmt):
    """in mode 2 a 16-bit window call between two int8 launches is a launch of another kind: its own fused launch and the int8
    launch after it keep their wait"""
    import torch
    from bitnetmcu_b200 import _lib
    e, _ = verbose_engine(capfd, monkeypatch, lambda: _engine("fc"))
    e.set_option(_lib.OPT_LAUNCH_OVERLAP, 2)
    rng = np.random.default_rng(8)
    xs = [rng.integers(-128, 128, size=(148 * 128 * 2 + 77, 256)).astype(np.int8) for _ in range(2)]
    wants = [oracle.infer(e.model, x) for x in xs]
    d_x = [torch.from_numpy(x).cuda() for x in xs]
    outs = [(torch.empty((x.shape[0], 10), dtype=torch.int32, device="cuda"), torch.empty(x.shape[0], dtype=torch.int32, device="cuda")) for x in xs]
    pages = half_stack(3, 200, 300, 6, fmt)
    wlo = torch.empty((3, 185, 285, 10), dtype=torch.int32, device="cuda")
    wla = torch.empty((3, 185, 285), dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    capfd.readouterr()
    e.infer_device(d_x[0], *outs[0])
    e.infer_device(d_x[1], *outs[1])
    e.scan_windows_device(pages, 1, wlo, wla)
    e.infer_device(d_x[0], *outs[0])
    torch.cuda.synchronize()
    got = [l.split("fused launch: ")[1] for l in capfd.readouterr().err.splitlines() if "fused launch: " in l]
    assert got == ["wait", "independent", "wait", "wait"], got
    for (lo, la), (wl, wb) in zip(outs, wants):
        assert np.array_equal(lo.cpu().numpy(), wl) and np.array_equal(la.cpu().numpy().astype(np.uint32), wb)
    e.set_option(_lib.OPT_LAUNCH_OVERLAP, 0)
    assert_same((wlo.reshape(-1, 10).cpu().numpy(), wla.reshape(-1, 1).cpu().numpy()), run_stack(e, "scan", widened(pages), 1), "mode 2")
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("name", ["fc", "cnn_48"])
def test_engine_methods_on_16bit_tensors(lib, name, fmt):
    """the Engine's window methods on torch.float16 / torch.bfloat16 pages (a [P, H, W] stack, one [H, W] page, and a plane for
    infer_windows_device) equal their float32 results on pages.float(), output shapes included"""
    import torch
    from bitnetmcu_b200.engine import window_grid
    e = _engine(name)
    pages = half_stack(3, 45, 61, 21, fmt)
    f32 = widened(pages)
    for stride in [(1, 1), (3, 2)]:
        for entry in ENTRIES:
            for p16, p32 in ((pages, f32), (pages[1], f32[1])):
                assert_same(run_stack(e, entry, p16, stride), run_stack(e, entry, p32, stride), (name, fmt, entry, p16.dim()))
        oh, ow = window_grid(45, 61, stride)
        res = []
        for plane in (pages[2], f32[2]):
            lo = torch.full((oh, ow, e.n_classes), SENTINEL, dtype=torch.int32, device="cuda")
            la = torch.full((oh, ow), SENTINEL, dtype=torch.int32, device="cuda")
            e.infer_windows_device(plane, stride, lo, la)
            only = torch.full((oh, ow), SENTINEL, dtype=torch.int32, device="cuda")
            e.infer_windows_device(plane, stride, None, only)
            torch.cuda.synchronize()
            assert torch.equal(only, la)
            res.append((lo.cpu().numpy(), la.cpu().numpy()))
        assert np.array_equal(res[0][0], res[1][0]) and np.array_equal(res[0][1], res[1][1]), (name, fmt, stride)
        assert (res[0][1] != SENTINEL).all()
    e.close()
