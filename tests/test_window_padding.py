"""Window scan of padded pages (include/bitnetmcu_b200.h section 13): bnm_scan_windows_padded_device,
bnm_scan_windows_topk_padded_device, bnm_emulate_windows_padded_device, bnm_emulate_windows_topk_padded_device and their _f16
forms.

Each entry is defined as its unpadded sibling (sections 10 and 12) on ``F.pad(pages.float(), (left, right, top, bottom), mode,
value)``, so every GPU case runs the padded entry on the pages and the float32 sibling on that padded copy, and compares every
output with tolerance 0.  The siblings are verified against the oracle and the emulator restatement elsewhere.  The CPU tests check
the declarations, the padding structure's layout, the failure without a device, window_grid, and a NumPy restatement of the
scaling kernel's padded band (each band row and column mapped to the page's, or to the fill value) against the reference's
per-image scaling on windows cut from ``np.pad``."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from conftest import ROOT, load_model
from restate import scale_images
from support import lib, random_fc, verbose_engine  # noqa: F401 (lib: fixture)

FORMATS = ["float32", "float16", "bfloat16"]
MODES = ["constant", "replicate", "reflect"]
NP_MODES = {"constant": "constant", "replicate": "edge", "reflect": "reflect"}   # NumPy's names for torch's modes
MODELS = ["fc", "12k_FP130", "ternary64", "binary160", "2bitsym96", "cnn_48", "cnn_letters", "rand_nf4_64"]
ENTRIES = ["scan", "scan_topk", "emulate", "emulate_topk"]
STEMS = {"scan": "bnm_scan_windows", "scan_topk": "bnm_scan_windows_topk", "emulate": "bnm_emulate_windows",
         "emulate_topk": "bnm_emulate_windows_topk"}
# (planes, height, width), stride, padding (left, right, top, bottom): odd pages, pages under 16 pixels that have windows only
# through their padding, every side from 0 to 15, strides under and over 16; every case is valid for reflect (each pad < the side)
CASES = [((1, 37, 53), (1, 1), (7, 8, 7, 8)),
         ((3, 9, 12), (2, 3), (7, 8, 7, 8)),
         ((2, 41, 67), (16, 16), (15, 0, 3, 15)),
         ((3, 50, 18), (17, 5), (0, 15, 15, 0)),
         ((2, 14, 30), (1, 2), (1, 2, 0, 13))]
PAD_VALUES = {"constant": [0.0, 1.5, -3.25], "replicate": [0.0], "reflect": [0.0]}
SENTINEL = -7
BNM_E_ARG, BNM_E_NODEV = -1, -2


def entry_name(entry, fmt, padded=True):
    return STEMS[entry] + ("_padded" if padded else "") + "_device" + ("" if fmt == "float32" else "_f16")


# ---- restatements ------------------------------------------------------------------------------------------------------------

def pad_index(i, n, mode):
    """the page index of padded indices i (counted from the page's first pixel) on a side of n pixels: i on the page, else the
    edge pixel (replicate), the mirror image about the edge pixel (reflect), or -1 for the fill value (constant)"""
    i = np.asarray(i, dtype=np.int64)
    if mode == "replicate":
        return np.clip(i, 0, n - 1)
    if mode == "reflect":
        return np.where(i < 0, -i, np.where(i >= n, 2 * (n - 1) - i, i))
    return np.where((i >= 0) & (i < n), i, -1)


def padded_window_scaling(page, pad, mode, value, sy, sx):
    """the scaling kernel on a padded float32 page [h, w]: per window row, a band of 16 padded rows whose rows and columns are
    mapped to the page's with pad_index (the fill value where either is -1), every column's max |x| over the band, the max of 16 of
    them per window, scale = 127 / max(that, 1e-5), each pixel round_half_even(x * scale) clipped, a NaN product 0 -> int8
    [windows, 256]"""
    h, w = page.shape
    left, right, top, bottom = pad
    ph, pw = h + top + bottom, w + left + right
    if ph < 16 or pw < 16:
        return np.zeros((0, 256), dtype=np.int8)
    oh, ow = (ph - 16) // sy + 1, (pw - 16) // sx + 1
    cols = pad_index(np.arange(pw) - left, w, mode)
    out = np.empty((oh, ow, 256), dtype=np.int8)
    for r in range(oh):
        rows = pad_index(r * sy + np.arange(16) - top, h, mode)
        band = page[np.clip(rows, 0, h - 1)][:, np.clip(cols, 0, w - 1)]
        band = np.where((rows[:, None] < 0) | (cols[None, :] < 0), np.float32(value), band).astype(np.float32)
        col = np.abs(band).max(axis=0)
        for c in range(ow):
            m = col[c * sx:c * sx + 16].max()
            scale = np.float32(127.0) / np.maximum(m, np.float32(1e-5))
            with np.errstate(invalid="ignore", over="ignore"):
                y = np.round(band[:, c * sx:c * sx + 16] * scale).clip(-128, 127).reshape(256)
            out[r, c] = np.where(np.isnan(y), 0, y).astype(np.int8)
    return out.reshape(-1, 256)


def windows_of(page, sy, sx):
    """every 16x16 window of a float32 page on the stride grid, flattened row-major: [windows, 256]"""
    h, w = page.shape
    if h < 16 or w < 16:
        return np.zeros((0, 256), dtype=np.float32)
    oh, ow = (h - 16) // sy + 1, (w - 16) // sx + 1
    return np.stack([page[r * sy:r * sy + 16, c * sx:c * sx + 16].reshape(256) for r in range(oh) for c in range(ow)])


def edge_page(h=40, w=52, seed=0):
    """a float32 page of normal pixels with the scaling edges on and next to its edges: subnormals and maxima below 1e-5 in
    corner blocks, -0.0, NaN on the left edge and one pixel in (reflect mirrors the second, not the first), +inf on the bottom
    edge, -inf on the right edge, NaN one row above the bottom"""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((h, w), dtype=np.float32)
    x[0:4, 0:16] = (rng.integers(1, 1 << 20, size=(4, 16)) * (2.0 ** -149)).astype(np.float32) * rng.choice([-1, 1], (4, 16)).astype(np.float32)
    x[0:16, w - 16:w] = np.float32(3e-6) * rng.uniform(0.5, 1.0, (16, 16)).astype(np.float32)
    x[h - 6:h, 0:6] = np.float32(-0.0)
    x[h // 2, 0] = np.nan
    x[h // 3, 1] = np.nan
    x[h - 1, w // 2] = np.inf
    x[h // 4, w - 1] = -np.inf
    x[h - 2, w // 3] = np.nan
    return x


def small_page(h=9, w=12, seed=1):
    """a page under 16 pixels either way, normal pixels and a dark corner"""
    x = np.random.default_rng(seed).standard_normal((h, w), dtype=np.float32)
    x[:3, :3] *= np.float32(1e-7)
    return x


# ---- CPU ----------------------------------------------------------------------------------------------------------------------

def _header():
    return open(os.path.join(ROOT, "include", "bitnetmcu_b200.h")).read()


def _struct_fields(text, name):
    body = re.search(rf"typedef struct {name} \{{(.*?)\}} {name};", text, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    out = []
    for decl in filter(None, (d.strip() for d in body.split(";"))):
        t, names = decl.rsplit(" ", 1) if "," not in decl else decl.split(" ", 1)
        for n in names.split(","):
            out.append((t.strip(), n.strip()))
    return out


def test_entries_struct_and_enum_are_declared_and_exported(built):
    from bitnetmcu_b200 import _lib
    text = _header()
    assert re.search(r"enum \{ BNM_PAD_CONSTANT = 0, BNM_PAD_REPLICATE = 1, BNM_PAD_REFLECT = 2 \};", text)
    assert (_lib.PAD_CONSTANT, _lib.PAD_REPLICATE, _lib.PAD_REFLECT) == (0, 1, 2)
    l = _lib.load()
    for entry in ENTRIES:
        for fmt in ("float32", "float16"):
            name = entry_name(entry, fmt)
            head = (r"const bnm_windows \*windows, const bnm_window_padding \*padding," if fmt == "float32" else
                    r"const bnm_windows_f16 \*windows, int format,\s+const bnm_window_padding \*padding,")
            assert re.search(rf"BNM_API int {name}\(bnm_model \*m, {head}", text), name
            assert name in _lib.EXPORTED and hasattr(l, name), name
    # each padded entry is named in the header's list of entries a graph may capture
    graphs = text[text.index(" * Graphs."):text.index("may be captured into a CUDA graph")]
    assert "bnm_scan_windows_padded_device" in graphs and "section 13" in graphs


def test_padding_structure_layout(built):
    """_lib.BnmWindowPadding declares the header's fields in the same order with the same types (24 bytes)"""
    from bitnetmcu_b200 import _lib
    fields = _struct_fields(_header(), "bnm_window_padding")
    ctypes_of = {"uint32_t": C.c_uint32, "float": C.c_float}
    assert [n for _, n in fields] == [n for n, _ in _lib.BnmWindowPadding._fields_] == ["left", "right", "top", "bottom", "mode", "value"]
    assert [ctypes_of[t] for t, _ in fields] == [t for _, t in _lib.BnmWindowPadding._fields_]
    assert C.sizeof(_lib.BnmWindowPadding) == 24


def test_entries_fail_without_a_device(built):
    from bitnetmcu_b200 import _lib
    l = _lib.load()
    if l.bnm_device_count() > 0:
        pytest.skip("a CUDA device is present")
    img = np.zeros(4 * 64 * 64, dtype=np.float32)
    d = _lib.BnmWindows(img.ctypes.data, 2, 64, 64, 64, 64 * 64, 16, 16)
    pad = _lib.BnmWindowPadding(7, 8, 7, 8, _lib.PAD_REPLICATE, 0.0)
    out = np.full(64, 7, dtype=np.uint32)
    o = C.c_void_p(out.ctypes.data)
    for entry in ENTRIES:
        for fmt in ("float32", "float16", "bfloat16"):
            fn = getattr(l, entry_name(entry, fmt))
            lead = (C.byref(d),) if fmt == "float32" else (C.byref(d), _lib.FLOAT16 if fmt == "float16" else _lib.BFLOAT16)
            rc = fn(None, *lead, C.byref(pad), 1, o, None, None) if entry.endswith("topk") else fn(None, *lead, C.byref(pad), None, o, None)
            assert rc == BNM_E_NODEV and b"no CUDA device" in l.bnm_last_error(), (entry, fmt)
    assert (out == 7).all()


def test_window_grid_with_padding():
    """window_grid over the padded page: 7 + 8 pixels at stride 1 give one window per pixel; pages under 16 pixels get windows
    through their padding only; a page of no pixels has none"""
    from bitnetmcu_b200.engine import window_grid
    assert window_grid(4096, 4096, 1, (7, 8, 7, 8)) == (4096, 4096)
    assert window_grid(9, 12, 1, (7, 8, 7, 8)) == (9, 12)
    assert window_grid(9, 12, 1) == (0, 0)
    assert window_grid(10, 12, (2, 3), 3) == (1, 1) and window_grid(9, 12, (2, 3), 3) == (0, 0)
    assert window_grid(37, 53, (16, 16), (15, 0, 3, 15)) == (3, 4)
    assert window_grid(50, 18, (17, 5), (0, 15, 15, 0)) == (3, 4)
    assert window_grid(0, 40, 1, 15) == (0, 0) and window_grid(40, 0, 1, 15) == (0, 0)
    assert window_grid(40, 40, 1, 0) == window_grid(40, 40, 1) == (25, 25)
    with pytest.raises(ValueError):
        window_grid(40, 40, 1, (1, 2, 3))


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("pad", [(7, 8, 7, 8), (0, 15, 15, 0), (15, 0, 0, 15), (3, 1, 0, 2)])
def test_padded_scaling_restatement_matches_numpy(mode, pad):
    """the padded band scaling equals restate.scale_images on windows cut from np.pad(page, ..., mode) at strides (1, 1),
    (2, 3), (16, 16) and (17, 5), on a page with NaN, +-inf, subnormal and below-1e-5 blocks at its edges and on a page under 16
    pixels; windows covering a copy of a NaN or an infinity are the all-zero row"""
    pages = [edge_page()] + ([small_page()] if mode != "reflect" or max(pad) < 9 else [])
    values = {"constant": [0.0, 2.5, np.nan], "replicate": [0.0], "reflect": [0.0]}[mode]
    seen_poisoned = seen_finite = False
    for page in pages:
        for value in values:
            kw = {"constant_values": np.float32(value)} if mode == "constant" else {}
            padded = np.pad(page, ((pad[2], pad[3]), (pad[0], pad[1])), mode=NP_MODES[mode], **kw)
            for sy, sx in [(1, 1), (2, 3), (16, 16), (17, 5)]:
                got = padded_window_scaling(page, pad, mode, value, sy, sx)
                wins = windows_of(padded, sy, sx)
                assert got.shape == wins.shape, (mode, pad, value, (sy, sx))
                assert np.array_equal(got, scale_images(wins)), (mode, pad, value, (sy, sx))
                poisoned = ~np.isfinite(wins).all(axis=1)
                assert not got[poisoned].any()
                seen_poisoned |= bool(poisoned.any())
                seen_finite |= bool((~poisoned).any())
    assert seen_poisoned and seen_finite


def test_reflect_and_replicate_copy_edge_pixels():
    """the restatement's mapping on the edges it is meant to cover: replicate repeats the edge pixel, reflect mirrors about it
    (the NaN in column 0 is repeated by replicate only, the one in column 1 mirrored by reflect only)"""
    page = edge_page()
    h = page.shape[0]
    cols_rep = pad_index(np.arange(-3, 0), page.shape[1], "replicate")
    cols_ref = pad_index(np.arange(-3, 0), page.shape[1], "reflect")
    assert cols_rep.tolist() == [0, 0, 0] and cols_ref.tolist() == [3, 2, 1]
    assert np.isnan(page[h // 2, cols_rep]).all() and not np.isnan(page[h // 2, cols_ref]).any()
    assert np.isnan(page[h // 3, cols_ref]).any() and not np.isnan(page[h // 3, cols_rep]).any()
    assert pad_index([-1, 12, 13], 12, "constant").tolist() == [-1, -1, -1] and pad_index([12, 13], 12, "reflect").tolist() == [10, 9]


# ---- GPU ----------------------------------------------------------------------------------------------------------------------

def _engine(name, path=0):
    from bitnetmcu_b200.engine import Engine
    m = load_model(name) if isinstance(name, str) else name
    return Engine(m, device=0, path=path, nf4_extension=(name == "rand_nf4_64"))


def _dtype(fmt):
    import torch
    return getattr(torch, fmt)


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
    """pages (a CPU or CUDA tensor or NumPy array [P, h, w]) as a CUDA stack of dtype [P, h, w] inside one allocation: rows 16
    bytes rounded + pad elements apart, `below` rows past each page and `gap` elements between planes, all that padding filled
    with fill ("nan-inf": NaN and infinity alternating)"""
    import torch
    src = torch.as_tensor(pages)
    p, h, w = src.shape
    per = 16 // torch.empty((), dtype=dtype).element_size()
    pitch = max(per, (w + per - 1) // per * per + pad)
    plane_pitch = (h + below) * pitch + gap
    buf = torch.full((max(p, 1) * max(plane_pitch, 1),), float("nan") if fill == "nan-inf" else fill, dtype=dtype, device="cuda")
    if fill == "nan-inf":
        buf[::2] = float("inf")
    view = buf.as_strided((p, h, w), (plane_pitch, pitch, 1))
    view.copy_(src.to(device="cuda", dtype=dtype))
    return view


def make_stack(planes, h, w, seed, fmt, **kw):
    return stack(pages_np(planes, h, w, seed), _dtype(fmt), **kw)


def padded_copy(pages, pad, mode, value):
    """what a caller passes the unpadded sibling today: F.pad(pages.float(), pad, mode, value), in a float32 stack of its own"""
    import torch
    import torch.nn.functional as F
    x = pages.float()
    x = F.pad(x, pad, mode="constant", value=value) if mode == "constant" else F.pad(x, pad, mode=mode)
    return stack(x, torch.float32)


def _k(e):
    return min(e.n_classes, 5)


def run_stack(e, entry, pages, stride, padding=None, mode="constant", value=0.0, k=None, first=True, second=True, stream=None,
              sync=True):
    """an entry through the Engine on a CUDA stack (its dtype picks the 16-bit form, padding the padded one) -> its two outputs
    as NumPy, flattened to [windows, ...] (None where not asked): (logits, labels) or (classes, scores)"""
    import torch
    from bitnetmcu_b200.engine import window_grid
    grid = (pages.shape[0] if pages.dim() == 3 else 1,) + window_grid(pages.shape[-2], pages.shape[-1], stride, padding)
    emul, topk = entry.startswith("emulate"), entry.endswith("topk")
    ldt = torch.float64 if emul else torch.int32
    kw = {} if padding is None else {"padding": padding, "pad_mode": mode, "pad_value": value}
    if topk:
        k = k or _k(e)
        a = torch.full(grid + (k,), SENTINEL, dtype=torch.int32, device="cuda") if first else None
        b = torch.full(grid + (k,), SENTINEL, dtype=ldt, device="cuda") if second else None
        (e.emulate_windows_topk_device if emul else e.scan_windows_topk_device)(pages, stride, k, a, b, stream=stream, **kw)
    else:
        a = torch.full(grid + (e.n_classes,), SENTINEL, dtype=ldt, device="cuda") if first else None
        b = torch.full(grid, SENTINEL, dtype=torch.int32, device="cuda") if second else None
        (e.emulate_windows_device if emul else e.scan_windows_device)(pages, stride, a, b, stream=stream, **kw)
    if not sync:
        return a, b
    torch.cuda.synchronize()
    n = int(np.prod(grid))
    return tuple(None if t is None else t.reshape(n, -1).cpu().numpy() for t in (a, b))


def flat(outs):
    return tuple(None if t is None else t.reshape(int(np.prod(t.shape[:3])), -1).cpu().numpy() for t in outs)


def assert_same(got, want, what):
    for g, w, kind in zip(got, want, ("first", "second")):
        if g is None or w is None:
            continue
        assert g.shape == w.shape, (what, kind, g.shape, w.shape)
        same = (g == w) | (np.isnan(g) & np.isnan(w)) if g.dtype.kind == "f" else g == w
        bad = np.flatnonzero(~same.reshape(len(w), -1).all(axis=1))
        assert bad.size == 0, (what, kind, f"{bad.size} of {len(w)} windows differ, first {bad[:6].tolist()}")


def assert_padded(e, entry, pages, stride, pad, mode, value, what, **kw):
    """the padded entry on pages equals its float32 sibling on F.pad(pages.float(), ...), and writes every window"""
    got = run_stack(e, entry, pages, stride, pad, mode, value, **kw)
    assert_same(got, run_stack(e, entry, padded_copy(pages, pad, mode, value), stride, **kw), what)
    # classes and labels are never the sentinel (a score or a logit may be)
    written = got[0] if entry.endswith("topk") or got[1] is None else got[1]
    assert (written != SENTINEL).any(axis=-1).all(), what
    return got


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("name", MODELS)
def test_entries_equal_the_sibling_on_padded_pages(lib, name, fmt):
    """every padded entry, mode and case on the default path, and one case per mode on BNM_PATH_LAYERS: the float32 sibling on
    F.pad(pages.float(), ...); fill values 0, 1.5 and -3.25 in constant mode"""
    from bitnetmcu_b200 import _lib
    e = _engine(name)
    for mi, mode in enumerate(MODES):
        for ci, (shape, stride, pad) in enumerate(CASES):
            pages = make_stack(*shape, seed=ci * 10 + mi, fmt=fmt, gap=8 * shape[0])
            value = PAD_VALUES[mode][ci % len(PAD_VALUES[mode])]
            for entry in ENTRIES:
                assert_padded(e, entry, pages, stride, pad, mode, value, (name, fmt, mode, shape, stride, pad, entry))
    e.set_option(_lib.OPT_PATH, _lib.PATH_LAYERS)
    for mi, mode in enumerate(MODES):
        shape, stride, pad = CASES[(mi + 1) % len(CASES)]
        pages = make_stack(*shape, seed=99 + mi, fmt=fmt)
        for entry in ENTRIES:
            assert_padded(e, entry, pages, stride, pad, mode, 0.75, (name, fmt, "layers", mode, entry))
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["fc", "cnn_letters", "binary160"])
def test_outputs_and_k(lib, name):
    """labels only, logits only and both; top-k with and without scores at k = 1 and min(n_classes, 16): each the sibling's on
    the padded copy"""
    e = _engine(name)
    for fmt, mode in zip(FORMATS, MODES):
        pages = make_stack(2, 30, 41, 3, fmt)
        for entry in ENTRIES:
            if entry.endswith("topk"):
                for k in (1, min(e.n_classes, 16)):
                    for second in (True, False):
                        assert_padded(e, entry, pages, (1, 2), (7, 8, 7, 8), mode, 0.5, (fmt, entry, k, second), k=k, second=second)
            else:
                for first, second in ((True, True), (False, True), (True, False)):
                    assert_padded(e, entry, pages, (1, 2), (7, 8, 7, 8), mode, 0.5, (fmt, entry, first, second), first=first, second=second)
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", FORMATS)
def test_zero_padding_is_the_sibling(lib, fmt):
    """all-zero padding in every mode (any fill value) gives the unpadded entry's results on the same pages, bit for bit"""
    for name in ("fc", "binary160", "cnn_48"):
        e = _engine(name)
        for shape, stride, _ in CASES:
            if min(shape[1:]) < 16:
                continue
            pages = make_stack(*shape, seed=5, fmt=fmt, gap=16)
            for entry in ENTRIES:
                want = run_stack(e, entry, pages, stride)
                for mode in MODES:
                    got = run_stack(e, entry, pages, stride, (0, 0, 0, 0), mode, float("nan"))
                    assert_same(got, want, (name, fmt, shape, stride, entry, mode))
        e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("fmt", FORMATS)
def test_reads_stay_on_the_page(lib, fmt, mode):
    """stacks whose row padding, rows below each page and gaps between planes hold 1e30 (float16: its largest value, 65504), or
    NaN and infinity: the results of the clean stack (a border that read past the page's rows or width would see them)"""
    for name in ("fc", "cnn_48"):
        e = _engine(name)
        for ci, (shape, stride, pad) in enumerate(CASES):
            x = pages_np(*shape, seed=ci + 31)
            clean = stack(x, _dtype(fmt))
            want = {entry: run_stack(e, entry, clean, stride, pad, mode, 2.0) for entry in ENTRIES}
            for fill in (65504.0 if fmt == "float16" else 1e30, "nan-inf"):
                dirty = stack(x, _dtype(fmt), fill=fill, gap=40, pad=8, below=9)
                assert dirty.stride(0) > dirty.shape[1] * dirty.stride(1) and dirty.stride(1) > dirty.shape[2]
                for entry in ENTRIES:
                    assert_same(run_stack(e, entry, dirty, stride, pad, mode, 2.0), want[entry], (name, fmt, mode, shape, fill, entry))
        e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", FORMATS)
def test_nonfinite_fill_and_edges(lib, fmt):
    """NaN and +-inf fill values zero every window touching the border; NaN and infinite pixels on the edges, repeated by
    replicate and mirrored by reflect, zero every window covering a copy: each the sibling's on the padded copy, and the zero
    row's logits where the padded copy's window is not finite"""
    import torch
    import torch.nn.functional as F
    e = _engine("fc")
    zero = torch.zeros((1, 256), dtype=torch.int8, device="cuda")
    zlo = torch.empty((1, 10), dtype=torch.int32, device="cuda")
    e.infer_device(zero, zlo, None)
    pages = stack(np.stack([edge_page(), edge_page(seed=3)[::-1, ::-1].copy()]), _dtype(fmt))
    cases = [("constant", v) for v in (float("nan"), float("inf"), float("-inf"))] + [("replicate", 0.0), ("reflect", 0.0)]
    for mode, value in cases:
        for stride, pad in [((1, 1), (7, 8, 7, 8)), ((2, 3), (15, 1, 0, 15)), ((16, 16), (8, 8, 8, 8))]:
            for e_name in ("fc", "cnn_48"):
                eng = e if e_name == "fc" else _engine(e_name)
                for entry in ENTRIES:
                    assert_padded(eng, entry, pages, stride, pad, mode, value, (fmt, mode, value, stride, pad, e_name, entry))
                if eng is not e:
                    eng.close()
            lo, _ = run_stack(e, "scan", pages, stride, pad, mode, value)
            x = pages.float()
            x = F.pad(x, pad, mode="constant", value=value) if mode == "constant" else F.pad(x, pad, mode=mode)
            wins = np.concatenate([windows_of(p, *stride) for p in x.cpu().numpy()])
            poisoned = ~np.isfinite(wins).all(axis=1)
            assert poisoned.any() and (~poisoned).any(), (fmt, mode, value, stride)
            assert (lo[poisoned] == zlo.cpu().numpy()).all(), (fmt, mode, value, stride)
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", FORMATS)
def test_pass_boundary_inside_a_plane_and_a_window_row(lib, fmt):
    """three 593 x 693 planes padded by 7 + 8 at stride 1: 593 x 693 windows each, and window 2^20, where the second pass
    starts, is in row 327 of the third plane, column 67; the layered emulator's passes of 65 536 also start inside rows"""
    import torch
    mode = MODES[FORMATS.index(fmt)]
    pages = make_stack(3, 593, 693, 41, fmt)
    w0 = 1 << 20
    p, r, c = w0 // (593 * 693), w0 % (593 * 693) // 693, w0 % 693
    assert (p, r, c) == (2, 327, 67)
    e = _engine("fc")
    for entry in ("scan", "scan_topk", "emulate"):
        got = assert_padded(e, entry, pages, 1, (7, 8, 7, 8), mode, -1.0, (fmt, entry, "pass"))
        assert got[0].shape[0] == 3 * 593 * 693 > w0
        torch.cuda.empty_cache()
    e.close()


def _c_entry(l, entry, fmt):
    """the padded C entry as f(handle, descriptor, padding, first, second, k) with section 10's argument order"""
    from bitnetmcu_b200 import _lib
    fn = getattr(l, entry_name(entry, fmt))
    lead = () if fmt == "float32" else (_lib.FLOAT16 if fmt == "float16" else _lib.BFLOAT16,)
    if entry.endswith("topk"):
        return lambda h, d, pad, a, b, k: fn(h, d, *lead, pad, k, b, a, None)   # a: scores, b: classes
    return lambda h, d, pad, a, b, k: fn(h, d, *lead, pad, a, b, None)


@pytest.mark.gpu
def test_argument_errors(lib):
    """each argument error gives BNM_E_ARG and writes nothing: a NULL padding, a side of 16, a mode outside BNM_PAD_*, reflect
    with a pad >= the page's height or width, a padded page past 2^32 - 1 pixels (checked before any pixel is read); pages of
    no pixels return 0 whatever the reflect pads"""
    import torch
    from bitnetmcu_b200 import _lib
    e = _engine("fc")
    lo = torch.full((4 * 80 * 80 * 16 + 64,), SENTINEL, dtype=torch.float64, device="cuda")   # room for every output type
    la = torch.full((4 * 80 * 80 * 16 + 64,), SENTINEL, dtype=torch.int32, device="cuda")
    P = lambda t: C.c_void_p(t.data_ptr())
    for fmt in FORMATS:
        img = torch.zeros((4 * 64 * 64 + 64,), dtype=_dtype(fmt), device="cuda")

        def desc(planes=2, h=20, w=24, pitch=64, plane_pitch=64 * 64):
            return _lib.BnmWindows(img.data_ptr(), planes, h, w, pitch, plane_pitch, 1, 1)

        def padding(left=7, right=8, top=7, bottom=8, mode=_lib.PAD_REPLICATE, value=0.0):
            return C.byref(_lib.BnmWindowPadding(left, right, top, bottom, mode, value))

        for entry in ENTRIES:
            call = _c_entry(lib, entry, fmt)
            d = C.byref(desc())
            cases = {
                "null padding": call(e.handle, d, None, P(lo), P(la), 3),
                "left 16": call(e.handle, d, padding(left=16), P(lo), P(la), 3),
                "right 16": call(e.handle, d, padding(right=16), P(lo), P(la), 3),
                "top 16": call(e.handle, d, padding(top=16), P(lo), P(la), 3),
                "bottom 16": call(e.handle, d, padding(bottom=16), P(lo), P(la), 3),
                "mode 3": call(e.handle, d, padding(mode=3), P(lo), P(la), 3),
                "mode 2^32 - 1": call(e.handle, d, padding(mode=0xFFFFFFFF), P(lo), P(la), 3),
                "reflect top = height": call(e.handle, C.byref(desc(h=7)), padding(top=7, bottom=0, mode=_lib.PAD_REFLECT), P(lo), P(la), 3),
                "reflect bottom > height": call(e.handle, C.byref(desc(h=7)), padding(top=0, bottom=9, mode=_lib.PAD_REFLECT), P(lo), P(la), 3),
                "reflect left = width": call(e.handle, C.byref(desc(w=8)), padding(left=8, right=0, mode=_lib.PAD_REFLECT), P(lo), P(la), 3),
                "reflect right > width": call(e.handle, C.byref(desc(w=8)), padding(left=0, right=15, mode=_lib.PAD_REFLECT), P(lo), P(la), 3),
                "padded height over 2^32 - 1": call(e.handle, C.byref(desc(planes=1, h=0xFFFFFFF8)), padding(top=4, bottom=4),
                                                    P(lo), P(la), 3),
                "padded width over 2^32 - 1": call(e.handle, C.byref(desc(planes=1, w=0xFFFFFFF0, pitch=0xFFFFFFF0)),
                                                   padding(left=15, right=1), P(lo), P(la), 3),
                "null descriptor": call(e.handle, None, padding(), P(lo), P(la), 3),
                "no output": call(e.handle, d, padding(), None, None, 3),
            }
            assert cases == {k: BNM_E_ARG for k in cases}, (entry, fmt, cases)
            call(e.handle, d, None, P(lo), P(la), 3)
            assert b"null padding" in lib.bnm_last_error()
            call(e.handle, d, padding(mode=3), P(lo), P(la), 3)
            assert b"padding mode 3" in lib.bnm_last_error()
            call(e.handle, C.byref(desc(h=7)), padding(top=7, bottom=0, mode=_lib.PAD_REFLECT), P(lo), P(la), 3)
            assert b"reflect" in lib.bnm_last_error()
            # pages of no pixels: no windows, whatever the padding would reflect; reflect just under the sides is valid
            for dz in (desc(planes=0), desc(h=0), desc(w=0)):
                assert call(e.handle, C.byref(dz), padding(15, 15, 15, 15, _lib.PAD_REFLECT), P(lo), P(la), 3) == 0, (entry, fmt)
            assert call(e.handle, C.byref(desc(planes=0)), padding(15, 15, 15, 15, _lib.PAD_CONSTANT), P(lo), P(la), 3) == 0
            assert call(e.handle, C.byref(desc(h=1, w=1)), padding(0, 0, 0, 0, _lib.PAD_REFLECT), P(lo), P(la), 3) == 0
            if entry.endswith("topk"):
                assert call(e.handle, d, padding(), P(lo), P(la), 0) == BNM_E_ARG
                assert call(e.handle, C.byref(desc(planes=0)), padding(), P(lo), P(la), 0) == BNM_E_ARG
    torch.cuda.synchronize()
    assert (lo == SENTINEL).all() and (la == SENTINEL).all()
    # a 16-bit padded entry checks its format first, as the unpadded 16-bit entries do
    fn = lib.bnm_scan_windows_padded_device_f16
    pad = _lib.BnmWindowPadding(1, 1, 1, 1, 0, 0.0)
    assert fn(e.handle, None, 3, C.byref(pad), P(lo), P(la), None) == BNM_E_ARG and b"format" in lib.bnm_last_error()
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["fc", "cnn_48", "binary160"])
def test_graph_replay(lib, name):
    """each padded entry captured into a CUDA graph: a replay equals the eager call on the pages' contents at replay time, and
    the sibling on their padded copy"""
    import torch
    e = _engine(name)
    shape, stride, pad = (3, 40, 37), (2, 1), (7, 8, 7, 8)
    for fmt, mode in zip(FORMATS, MODES):
        for entry in ENTRIES:
            pages = make_stack(*shape, seed=4, fmt=fmt)
            run_stack(e, entry, pages, stride, pad, mode, 0.25, sync=False)   # warm: the pool and the kernels' attributes
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=torch.cuda.Stream()):
                outs = run_stack(e, entry, pages, stride, pad, mode, 0.25, sync=False)
            pages.copy_(torch.from_numpy(pages_np(*shape, seed=5)).to(pages.dtype))
            g.replay()
            torch.cuda.synchronize()
            got = flat(outs)
            assert_same(got, run_stack(e, entry, pages, stride, pad, mode, 0.25), (name, fmt, entry, "replay"))
            assert_same(got, run_stack(e, entry, padded_copy(pages, pad, mode, 0.25), stride), (name, fmt, entry, "replay, sibling"))
            del g
    e.close()


ROUTE_CASES = [("fc", lambda: load_model("fc"), 0), ("37 classes", lambda: random_fc(4, (256, 64, 64, 37), 2), 0),
               ("binary160", lambda: load_model("binary160"), 0), ("cnn_48", lambda: load_model("cnn_48"), 0),
               ("layers", lambda: load_model("fc"), 1), ("cnn layers", lambda: load_model("cnn_48"), 1)]


@pytest.mark.gpu
def test_routes_are_the_siblings(lib, capfd, monkeypatch):
    """each padded entry prints one windows route line: the unpadded sibling's line under the padded entry's name, with the same
    scaling kernel"""
    import torch
    for what, make, path in ROUTE_CASES:
        e, _ = verbose_engine(capfd, monkeypatch, lambda: _engine(make(), path=path))
        for fmt in FORMATS:
            pages = make_stack(2, 30, 40, 2, fmt)
            for entry in ENTRIES:
                lines = {}
                for padded in (True, False):
                    torch.cuda.synchronize()
                    capfd.readouterr()
                    run_stack(e, entry, pages, 3, (7, 8, 7, 8) if padded else None, "reflect")
                    got = [l for l in capfd.readouterr().err.splitlines() if "route: " in l]
                    assert len(got) == 1, (what, entry, fmt, padded, got)
                    name = entry_name(entry, fmt, padded)
                    assert f"windows route: {name}: " in got[0], (what, entry, fmt, padded, got)
                    lines[padded] = got[0].split(f"windows route: {name}: ")[1]
                assert lines[True] == lines[False] and lines[True].startswith("k_quantize_windows"), (what, entry, fmt, lines)
        e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["float32", "bfloat16"])
def test_mode2_int8_launch_after_a_padded_call_waits(lib, oracle, capfd, monkeypatch, fmt):
    """in mode 2 a padded window call between two int8 launches is a launch of another kind: its own fused launch and the int8
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
    pages = make_stack(3, 200, 300, 6, fmt)
    wlo = torch.empty((3, 200, 300, 10), dtype=torch.int32, device="cuda")
    wla = torch.empty((3, 200, 300), dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    capfd.readouterr()
    e.infer_device(d_x[0], *outs[0])
    e.infer_device(d_x[1], *outs[1])
    e.scan_windows_device(pages, 1, wlo, wla, padding=(7, 8, 7, 8), pad_mode="replicate")
    e.infer_device(d_x[0], *outs[0])
    torch.cuda.synchronize()
    got = [l.split("fused launch: ")[1] for l in capfd.readouterr().err.splitlines() if "fused launch: " in l]
    assert got == ["wait", "independent", "wait", "wait"], got
    for (lo, la), (wl, wb) in zip(outs, wants):
        assert np.array_equal(lo.cpu().numpy(), wl) and np.array_equal(la.cpu().numpy().astype(np.uint32), wb)
    e.set_option(_lib.OPT_LAUNCH_OVERLAP, 0)
    want = run_stack(e, "scan", padded_copy(pages, (7, 8, 7, 8), "replicate", 0.0), 1)
    assert_same((wlo.reshape(-1, 10).cpu().numpy(), wla.reshape(-1, 1).cpu().numpy()), want, "mode 2")
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["fc", "cnn_48"])
def test_engine_methods_equal_the_c_entries(lib, name):
    """the Engine's window methods with padding= (an int or a 4-tuple, every pad_mode) equal the C entries called directly, on a
    [P, H, W] stack and one [H, W] page; window_grid with the padding is the outputs' shape; padding=None is the unpadded entry"""
    import torch
    from bitnetmcu_b200 import _lib
    from bitnetmcu_b200.engine import window_grid
    e = _engine(name)
    codes = {"constant": _lib.PAD_CONSTANT, "replicate": _lib.PAD_REPLICATE, "reflect": _lib.PAD_REFLECT}
    for fmt in FORMATS:
        pages = make_stack(3, 21, 30, 21, fmt)
        for padding, mode in ((5, "reflect"), ((7, 8, 7, 8), "replicate"), ((0, 3, 15, 1), "constant")):
            sides = (padding,) * 4 if isinstance(padding, int) else padding
            stride = (1, 2)
            oh, ow = window_grid(21, 30, stride, padding)
            assert (oh, ow) == ((21 + sides[2] + sides[3] - 16) // 1 + 1, (30 + sides[0] + sides[1] - 16) // 2 + 1)
            for entry in ENTRIES:
                topk = entry.endswith("topk")
                k = _k(e)
                tail = (k,) if topk else (e.n_classes,)
                ldt = torch.float64 if entry.startswith("emulate") else torch.int32
                a = torch.full((3, oh, ow) + tail, SENTINEL, dtype=ldt, device="cuda")
                b = torch.full((3, oh, ow) + ((k,) if topk else ()), SENTINEL, dtype=torch.int32, device="cuda")
                d = _lib.BnmWindows(pages.data_ptr(), 3, 21, 30, pages.stride(1), pages.stride(0), *stride)
                pad = _lib.BnmWindowPadding(*sides, codes[mode], -2.0)
                rc = _c_entry(lib, entry, fmt)(e.handle, C.byref(d), C.byref(pad), C.c_void_p(a.data_ptr()), C.c_void_p(b.data_ptr()), k)
                assert rc == 0, (fmt, entry, lib.bnm_last_error())
                torch.cuda.synchronize()
                want = (b, a) if topk else (a, b)   # the Engine's order: (classes, scores) / (logits, labels)
                got = run_stack(e, entry, pages, stride, padding, mode, -2.0)
                assert_same(got, flat(want), (name, fmt, entry, padding, mode))
                one = run_stack(e, entry, pages[1], stride, padding, mode, -2.0)
                n1 = oh * ow
                assert_same(one, tuple(t[n1:2 * n1] for t in got), (name, fmt, entry, padding, mode, "one page"))
        assert_same(run_stack(e, "scan", pages, 3, None), run_stack(e, "scan", pages, 3, (0, 0, 0, 0), "reflect"), (name, fmt, "none"))
        with pytest.raises(ValueError):
            run_stack(e, "scan", pages, 3, 4, "circular")
    e.close()
