"""Window scan of page stacks in host memory (include/bitnetmcu_b200.h section 14): bnm_scan_windows, bnm_scan_windows_topk,
bnm_emulate_windows and bnm_emulate_windows_topk, through Engine.scan_windows, scan_windows_topk, emulate_windows and
emulate_windows_topk.

Each host entry is defined as its device sibling (sections 10, 12 and 13) on the same stack copied to the GPU, so every GPU case
runs the host method on NumPy arrays or CPU tensors and the matching *_device method on the stack uploaded with torch, and compares
every output with tolerance 0.  The siblings are verified against the oracle and the emulator restatement elsewhere.  The CPU tests
check the declarations, the descriptor's layout, the failure without a device, and the band rule restated here: that every band's
staged rows hold every page row its windows read, the border rows that replicate or reflect padding maps onto included."""
import ctypes as C
import os
import re
import threading

import numpy as np
import pytest

from conftest import ROOT, load_model
from support import lib, verbose_engine  # noqa: F401 (lib: fixture)

ENTRIES = ["scan", "scan_topk", "emulate", "emulate_topk"]
STEMS = {"scan": "bnm_scan_windows", "scan_topk": "bnm_scan_windows_topk", "emulate": "bnm_emulate_windows",
         "emulate_topk": "bnm_emulate_windows_topk"}
MODES = ["constant", "replicate", "reflect"]
FORMATS = ["float32", "float16", "bfloat16"]
SENTINEL = -7
BNM_E_ARG, BNM_E_NODEV = -1, -2
MIN_CHUNK = 128   # BNM_OPT_CHUNK_IMAGES at its minimum: 128 KiB of page pixels per band


# ---- the band rule (header section 14), restated ------------------------------------------------------------------------------

def pad_index(i, n, mode):
    """the page index of padded indices i on a side of n pixels (the scaling kernel's rule): i on the page, else the edge pixel
    (replicate), its mirror image about the edge pixel (reflect), or -1 for the fill value (constant)"""
    i = np.asarray(i, dtype=np.int64)
    if mode == "replicate":
        return np.clip(i, 0, n - 1)
    if mode == "reflect":
        return np.where(i < 0, -i, np.where(i >= n, 2 * (n - 1) - i, i))
    return np.where((i >= 0) & (i < n), i, -1)


def _sides(padding):
    from bitnetmcu_b200.engine import _pad_sides
    return (0, 0, 0, 0) if padding is None else _pad_sides(padding)


def band_rows(h, top, sy, r0, r1, mode):
    """the page rows [a, e) that window rows r0 .. r1 - 1 read: those their windows cover, and with reflect down to the mirror
    image of the topmost border row they read"""
    y0 = r0 * sy - top
    a, e = max(0, y0), min(h, (r1 - 1) * sy - top + 16)
    return a, (max(e, min(h, 1 - y0)) if mode == "reflect" and y0 < 0 else e)


def band_rule(planes, h, w, elem, stride, padding=None, mode="constant", chunk=65536):
    """[(first plane, planes, first window row, window rows)] of a host window call, as the header states the rule"""
    from bitnetmcu_b200.engine import window_grid
    sy, sx = (stride, stride) if isinstance(stride, int) else stride
    _, _, top, _ = _sides(padding)
    oh, ow = window_grid(h, w, (sy, sx), padding)
    if planes == 0 or oh == 0 or ow == 0:
        return []
    budget, most = chunk * 1024, 1 << 20
    a, e = band_rows(h, top, sy, 0, oh, mode)
    plane_bytes = (e - a) * w * elem
    if plane_bytes <= budget and oh * ow <= most:
        per = min(budget // plane_bytes, most // (oh * ow))
        return [(p, min(per, planes - p), 0, oh) for p in range(0, planes, per)]
    rows = budget // (w * elem) - 16
    R = max(1, min((rows // sy if rows >= 0 else -1) + 1, most // ow))
    head = -(-top // sy)
    t = oh
    over = (oh - 1) * sy - top + 16 - h
    if over > 0:
        t = (h + top - 16) // sy + 1 if h + top >= 16 else 0
        if mode == "reflect":
            t = min(t, (h - 1 - over + top) // sy)
    out = []
    for p in range(planes):
        s = 0
        while s < oh:
            end = s + R if s else max(R, head)
            if end > t or end >= oh:
                end = oh
            out.append((p, 1, s, end - s))
            s = end
    return out


CONFIGS = [((3, 300, 200), 4, 1, None, "constant"),
           ((2, 300, 200), 4, 3, (15, 15, 15, 15), "reflect"),
           ((2, 300, 200), 4, 17, (1, 1, 1, 1), "replicate"),
           ((1, 40, 3000), 4, 1, (15, 0, 15, 15), "reflect"),
           ((2, 260, 2100), 2, (2, 5), (7, 8, 7, 8), "reflect"),
           ((5, 20, 40), 4, 16, (0, 15, 0, 15), "constant"),
           ((1, 600, 640), 4, 1, (7, 8, 7, 8), "replicate"),
           ((3, 17, 5000), 2, 1, (15, 15, 15, 15), "reflect"),
           ((2, 20, 40), 4, 16, (0, 0, 8, 0), "reflect"),        # out_h = 1: the window reads row 8, covers rows 0 .. 7
           ((2, 20, 5000), 4, 16, (0, 0, 8, 0), "reflect"),
           ((2, 20, 40), 4, 10, (0, 0, 15, 0), "reflect"),       # out_h = 2: rows 0 .. 15 read, 0 .. 14 covered
           ((2, 20, 5000), 4, 10, (0, 0, 15, 0), "reflect"),
           ((2, 40, 5000), 4, (1, 3), (3, 0, 15, 15), "reflect")]


@pytest.mark.parametrize("shape,elem,stride,padding,mode", CONFIGS)
def test_band_rule_covers_every_read(shape, elem, stride, padding, mode):
    """at the minimum chunk: the bands cover the grid in window order, each a run of whole planes or of rows in one plane, each
    within the budget unless it is one window row or an edge band the padding forces; and in band coordinates (the band's rows
    staged from its first covered row, its top border what lies above the page) every row a window reads maps to the page row the
    whole page maps it to, so the scaling kernel sees the same pixels on the band as on the page"""
    from bitnetmcu_b200.engine import window_grid
    planes, h, w = shape
    sy = stride if isinstance(stride, int) else stride[0]
    _, _, top, _ = _sides(padding)
    oh, ow = window_grid(h, w, stride, padding)
    bands = band_rule(planes, h, w, elem, stride, padding, mode, MIN_CHUNK)
    seen = []
    for p, n_p, r0, nr in bands:
        assert n_p == 1 or (r0, nr) == (0, oh)
        seen += [(q, r) for q in range(p, p + n_p) for r in range(r0, r0 + nr)]
        a, e = band_rows(h, top, sy, r0, r0 + nr, mode)
        band_top = a - (r0 * sy - top)
        assert band_top == 0 or r0 == 0
        for r in range(r0, r0 + nr):
            i = np.arange(16)
            on_page = pad_index(r * sy + i - top, h, mode)
            on_band = pad_index((r - r0) * sy + i - band_top, e - a, mode)
            assert ((on_band >= 0) & (on_band < e - a) | (on_band == -1)).all()
            assert np.array_equal(np.where(on_band < 0, -1, on_band + a), on_page), (p, r0, nr, r)
    assert seen == [(q, r) for q in range(planes) for r in range(oh)]


def test_band_rule_whole_planes_and_rows():
    """small planes share bands (2^20 windows or the budget, whichever ends first); large ones are cut into runs of rows"""
    assert band_rule(64, 1024, 1024, 4, 16) == [(p, 16, 0, 64) for p in range(0, 64, 16)]
    assert band_rule(64, 1024, 1024, 4, 1) == [(p, 1, 0, 1009) for p in range(64)]
    assert len(band_rule(16, 4096, 4096, 4, 1)) == 16 * -(-4081 // 256)
    assert band_rule(16, 4096, 4096, 4, 16) == [(p, 1, 0, 256) for p in range(16)]
    assert band_rule(2, 8192, 8192, 4, 16)[:2] == [(0, 1, 0, 128), (0, 1, 128, 128)]


# ---- CPU ----------------------------------------------------------------------------------------------------------------------

def _header():
    return open(os.path.join(ROOT, "include", "bitnetmcu_b200.h")).read()


def test_entries_and_descriptor_are_declared(built):
    from bitnetmcu_b200 import _lib
    text = _header()
    assert "#define BNM_FLOAT32 3" in text and _lib.FLOAT32 == 3
    l = _lib.load()
    for entry in ENTRIES:
        name = STEMS[entry]
        assert re.search(rf"BNM_API int {name}\(bnm_model \*m, const bnm_windows_host \*windows, const bnm_window_padding \*padding,",
                         text), name
        assert name in _lib.EXPORTED and hasattr(l, name), name
    body = re.search(r"typedef struct bnm_windows_host \{(.*?)\} bnm_windows_host;", text, re.S).group(1)
    names = re.findall(r"(\w+)(?:,\s*(\w+))?;", re.sub(r"/\*.*?\*/", "", body, flags=re.S))
    fields = [n for pair in names for n in pair if n]
    assert fields == [n for n, _ in _lib.BnmWindowsHost._fields_]
    assert C.sizeof(_lib.BnmWindowsHost) == 48


def test_entries_fail_without_a_device(built):
    from bitnetmcu_b200 import _lib
    l = _lib.load()
    if l.bnm_device_count() > 0:
        pytest.skip("a CUDA device is present")
    img = np.zeros((2, 64, 64), dtype=np.float32)
    d = _lib.BnmWindowsHost(img.ctypes.data, _lib.FLOAT32, 2, 64, 64, 64, 64 * 64, 16, 16)
    out = np.full(64, 7, dtype=np.uint32)
    o = C.c_void_p(out.ctypes.data)
    for entry in ENTRIES:
        fn = getattr(l, STEMS[entry])
        rc = fn(None, C.byref(d), None, 1, o, None) if entry.endswith("topk") else fn(None, C.byref(d), None, None, o)
        assert rc == BNM_E_NODEV and b"no CUDA device" in l.bnm_last_error(), entry
    assert (out == 7).all()


def test_16bit_entries_reject_float32_format(built):
    """BNM_FLOAT32 is no format of the 16-bit device entries: they reject it as any other value, before anything else"""
    from bitnetmcu_b200 import _lib
    l = _lib.load()
    out = np.zeros(4, dtype=np.uint32)
    rc = l.bnm_scan_windows_device_f16(None, None, _lib.FLOAT32, None, C.c_void_p(out.ctypes.data), None)
    assert rc == BNM_E_ARG
    assert l.bnm_last_error() == b"bnm_scan_windows_device_f16: format 3, must be BNM_FLOAT16 (1) or BNM_BFLOAT16 (2)"


# ---- GPU ----------------------------------------------------------------------------------------------------------------------

def _torch():
    import torch
    return torch


def head37():
    from bitnetmcu_b200 import pack
    return pack.random_fc_model(4, (256, 64, 64, 64, 37), seed=37)


MODELS = {"fc": lambda: load_model("fc"), "head37": head37, "binary160": lambda: load_model("binary160"),
          "cnn_48": lambda: load_model("cnn_48")}


def _engine(name, chunk=None):
    from bitnetmcu_b200 import _lib
    from bitnetmcu_b200.engine import Engine
    e = Engine(MODELS[name]() if isinstance(name, str) else name, device=0)
    if chunk is not None:
        e.set_option(_lib.OPT_CHUNK_IMAGES, chunk)
    return e


def pages_np(planes, h, w, seed):
    """float32 [planes, h, w]: normal pixels with MNIST-normalised patches and a dark margin"""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal(size=(planes, h, w), dtype=np.float32)
    for p in range(planes):
        for _ in range(max(1, h * w // 4000)):
            r, c = rng.integers(0, max(1, h - 20)), rng.integers(0, max(1, w - 20))
            x[p, r:r + 20, c:c + 20] = (rng.integers(0, 256, size=x[p, r:r + 20, c:c + 20].shape) / 255.0 - 0.1307) / 0.3081
    x[:, :, :3] *= np.float32(0.01)
    return x


def host_pages(x, fmt, kind="numpy", pinned=False):
    """float32 pages x as host pages of fmt: a NumPy array (float32 / float16) or a CPU tensor, pinned or not"""
    torch = _torch()
    if kind == "numpy":
        assert not pinned and fmt != "bfloat16"
        return x.astype(np.float16) if fmt == "float16" else x
    t = torch.from_numpy(x).to(getattr(torch, fmt))
    return t.pin_memory() if pinned else t


def device_stack(pages):
    """host pages (NumPy or CPU tensor) uploaded with torch into a CUDA stack whose rows are 16 bytes apart, the device entries'
    pitch rule: a view [P, h, w]"""
    torch = _torch()
    t = pages if isinstance(pages, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(pages))
    t = t if t.dim() == 3 else t.unsqueeze(0)
    p, h, w = t.shape
    per = 16 // t.element_size()
    pitch = max(per, -(-w // per) * per)
    buf = torch.zeros((max(p, 1), max(h, 1), pitch), dtype=t.dtype, device="cuda")
    view = buf[:p, :h, :w]
    view.copy_(t)
    return view


def _k(e, k):
    return min(e.n_classes, k)


def run_host(e, entry, pages, stride, padding=None, mode="constant", value=0.0, k=5, first=True, second=True):
    """the host method -> its two outputs flattened to [windows, ...] (None where not asked): (logits, labels) or (classes, scores)"""
    kw = {} if padding is None else {"padding": padding, "pad_mode": mode, "pad_value": value}
    if entry.endswith("topk"):
        fn = e.emulate_windows_topk if entry.startswith("emulate") else e.scan_windows_topk
        outs = fn(pages, stride, _k(e, k), want_scores=second, **kw)
    else:
        fn = e.emulate_windows if entry.startswith("emulate") else e.scan_windows
        outs = fn(pages, stride, want_labels=second, want_logits=first, **kw)
    return tuple(None if t is None else t.reshape((int(np.prod(t.shape[:3])),) + t.shape[3:]) for t in outs)


def run_device(e, entry, pages, stride, padding=None, mode="constant", value=0.0, k=5, first=True, second=True):
    """the matching device method on the pages uploaded with torch -> its outputs as run_host returns them"""
    torch = _torch()
    from bitnetmcu_b200.engine import window_grid
    d = device_stack(pages)
    grid = (d.shape[0],) + window_grid(d.shape[1], d.shape[2], stride, padding)
    kw = {} if padding is None else {"padding": padding, "pad_mode": mode, "pad_value": value}
    ldt = torch.float64 if entry.startswith("emulate") else torch.int32
    if entry.endswith("topk"):
        kk = _k(e, k)
        a = torch.full(grid + (kk,), SENTINEL, dtype=torch.int32, device="cuda")
        b = torch.full(grid + (kk,), SENTINEL, dtype=ldt, device="cuda") if second else None
        (e.emulate_windows_topk_device if entry.startswith("emulate") else e.scan_windows_topk_device)(d, stride, kk, a, b, **kw)
    else:
        a = torch.full(grid + (e.n_classes,), SENTINEL, dtype=ldt, device="cuda") if first else None
        b = torch.full(grid, SENTINEL, dtype=torch.int32, device="cuda") if second else None
        (e.emulate_windows_device if entry.startswith("emulate") else e.scan_windows_device)(d, stride, a, b, **kw)
    torch.cuda.synchronize()
    n = int(np.prod(grid))
    return tuple(None if t is None else t.reshape((n,) + tuple(t.shape[3:])).cpu().numpy() for t in (a, b))


def assert_same(got, want, what):
    for g, w, kind in zip(got, want, ("first", "second")):
        assert (g is None) == (w is None), (what, kind)
        if g is None:
            continue
        if w.dtype == np.int32 and g.dtype == np.uint32:
            g = g.view(np.int32)
        assert g.shape == w.shape and g.dtype == w.dtype, (what, kind, g.shape, w.shape, g.dtype, w.dtype)
        if w.size == 0:
            continue
        same = (g == w) | (np.isnan(g) & np.isnan(w)) if g.dtype.kind == "f" else g == w
        bad = np.flatnonzero(~same.reshape(len(w), -1).all(axis=1))
        assert bad.size == 0, (what, kind, f"{bad.size} of {len(w)} windows differ, first {bad[:6].tolist()}")


def check(e, entry, pages, stride, what, **kw):
    got = run_host(e, entry, pages, stride, **kw)
    assert_same(got, run_device(e, entry, pages, stride, **kw), what)
    return got


def host_windows_lines(err):
    return [l for l in err if "host windows: " in l]


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(MODELS))
def test_models_and_outputs(lib, name):
    """every entry on each model, at the default chunk and at the minimum (many row bands): labels only, logits only, both; top-1
    and top-5 with and without scores"""
    x = pages_np(2, 300, 200, seed=3)
    for chunk in (None, MIN_CHUNK):
        e = _engine(name, chunk)
        for entry in ENTRIES:
            if entry.endswith("topk"):
                for k in (1, 5):
                    for second in (True, False):
                        check(e, entry, x, (1, 2), (name, chunk, entry, k, second), k=k, second=second)
            else:
                for first, second in ((True, True), (False, True), (True, False)):
                    check(e, entry, x, (1, 2), (name, chunk, entry, first, second), first=first, second=second)
        e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", FORMATS)
def test_formats_arrays_tensors_pinned(lib, fmt):
    """float32, float16 and bfloat16 pages as NumPy arrays (float32, float16) and as CPU tensors, pageable and pinned"""
    x = pages_np(3, 150, 230, seed=11)
    kinds = [("tensor", False), ("tensor", True)] + ([("numpy", False)] if fmt != "bfloat16" else [])
    for name in ("fc", "cnn_48"):
        e = _engine(name, MIN_CHUNK)
        for kind, pinned in kinds:
            pages = host_pages(x, fmt, kind, pinned)
            for entry in ENTRIES:
                check(e, entry, pages, (1, 3), (name, fmt, kind, pinned, entry))
            check(e, "scan", pages, 4, (name, fmt, kind, pinned, "padded"), padding=(7, 8, 7, 8), mode="replicate")
        e.close()


GRIDS = [((2, 100, 90), 1), ((2, 100, 90), 3), ((3, 130, 77), 16), ((3, 130, 77), 17), ((2, 61, 300), (2, 5)),
         ((2, 61, 300), (5, 1)), ((4, 12, 40), 1), ((2, 40, 9), 2), ((0, 40, 40), 1), ((1, 500, 250), 1), ((40, 30, 33), 2)]


@pytest.mark.gpu
def test_grids(lib):
    """strides 1, 3, 16 and 17 (rows the grid skips), stride_y != stride_x, pages under 16 pixels either way (no windows), no
    planes, one plane, and stacks of many small planes, at the default and the minimum chunk"""
    for chunk in (None, MIN_CHUNK):
        e = _engine("fc", chunk)
        for shape, stride in GRIDS:
            x = pages_np(*shape, seed=shape[1] + shape[2])
            for entry in ("scan", "scan_topk"):
                got = check(e, entry, x, stride, (chunk, shape, stride, entry))
                if min(shape) == 0 or min(shape[1:]) < 16:
                    assert got[0].shape[0] == 0
            check(e, "emulate", x[0] if shape[0] == 1 else x, stride, (chunk, shape, stride, "emulate"))
        e.close()


BAND_CASES = [((40, 30, 33), 4, 1, None, "constant"),          # many small planes: bands of whole planes
              ((3, 400, 300), 4, 1, None, "constant"),          # planes cut into runs of rows
              ((2, 400, 300), 2, 3, (15, 15, 15, 15), "reflect"),
              ((2, 330, 200), 4, 17, (1, 1, 1, 1), "replicate"),
              ((2, 300, 2100), 4, (2, 5), (7, 8, 7, 8), "reflect")]


@pytest.mark.gpu
@pytest.mark.parametrize("case", range(len(BAND_CASES)))
def test_band_count_follows_the_rule(lib, capfd, monkeypatch, case):
    """at the minimum chunk, the `host windows:` line of each call gives the band count of the restated rule and the window
    route; the results are the device sibling's.  The cases have bands of whole planes, and planes cut into bands of rows"""
    from bitnetmcu_b200 import _lib
    shape, elem, stride, padding, mode = BAND_CASES[case]
    fmt = "float32" if elem == 4 else "float16"
    x = host_pages(pages_np(*shape, seed=case), fmt)
    e, _ = verbose_engine(capfd, monkeypatch, lambda: _engine("fc"))
    e.set_option(_lib.OPT_CHUNK_IMAGES, MIN_CHUNK)
    want = band_rule(*shape, elem, stride, padding, mode, MIN_CHUNK)
    assert len(want) > 1
    assert any(n_p > 1 for _, n_p, _, _ in want) == (case == 0)
    for entry in ("scan", "emulate_topk"):
        capfd.readouterr()
        got = run_host(e, entry, x, stride, padding=padding, mode=mode, value=0.5)
        lines = host_windows_lines(capfd.readouterr().err.splitlines())
        assert len(lines) == 1, lines
        assert f"host windows: {STEMS[entry]}: {len(want)} bands: k_quantize_windows" in lines[0], (lines[0], len(want))
        assert_same(got, run_device(e, entry, x, stride, padding=padding, mode=mode, value=0.5), (case, entry))
    e.close()


PAD_CASES = [(0, 0, 0, 0), (1, 1, 1, 1), (7, 8, 7, 8), (15, 15, 15, 15), (15, 0, 0, 15), (0, 15, 15, 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
def test_padding(lib, mode):
    """constant (fill 0, 2.5 and NaN), replicate and reflect with sides 0, 1, 7 + 8 and 15 on planes the minimum chunk cuts into
    bands: reflect by 15 rows makes a plane's first and last bands hold rows their windows do not cover"""
    values = [0.0, 2.5, float("nan")] if mode == "constant" else [0.0]
    e = _engine("fc", MIN_CHUNK)
    x = pages_np(2, 260, 300, seed=5)
    x[0, 0, 5] = np.nan
    x[1, -2, 7] = np.inf
    for i, pad in enumerate(PAD_CASES):
        for stride in (1, (3, 2), 16):
            value = values[i % len(values)]
            assert len(band_rule(2, 260, 300, 4, stride, pad, mode, MIN_CHUNK)) > 2 or stride == 16
            for entry in ("scan", "emulate"):
                check(e, entry, x, stride, (mode, pad, stride, value, entry), padding=pad, mode=mode, value=value)
    e.close()


SHORT_REFLECT = [((2, 20, 40), 16, (0, 0, 8, 0)), ((2, 20, 40), 10, (0, 0, 15, 0)), ((3, 17, 61), (16, 3), (15, 2, 15, 15)),
                 ((2, 20, 5000), 16, (0, 0, 8, 0)), ((2, 20, 5000), 10, (0, 0, 15, 0)), ((2, 40, 5000), (1, 3), (3, 0, 15, 15))]


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["float32", "float16"])
def test_reflect_reads_rows_the_windows_do_not_cover(lib, fmt):
    """reflect padding on pages whose few window rows read mirrored rows below the ones they cover (out_h * stride_y small next
    to top), in bands of several whole planes (where a short staging would read the next plane's first rows) and in row bands of
    wide pages at the minimum chunk: the padded device sibling's results.  Each page's row just past the covered ones differs
    from the rows around it, so a band that lacked it would give other results"""
    for chunk in (None, MIN_CHUNK):
        e = _engine("fc", chunk)
        for ci, (shape, stride, pad) in enumerate(SHORT_REFLECT):
            x = pages_np(*shape, seed=70 + ci)
            x[:, :16] *= np.float32(0.05)
            x[:, pad[2]] = np.float32(40.0)   # the mirror image of the topmost border row
            pages = host_pages(x, fmt)
            bands = band_rule(*shape, 4 if fmt == "float32" else 2, stride, pad, "reflect", chunk or 65536)
            assert bands, (shape, stride, pad)
            for entry in ("scan", "emulate_topk"):
                check(e, entry, pages, stride, (fmt, chunk, shape, stride, pad, entry), padding=pad, mode="reflect")
        e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", FORMATS)
def test_pitch_and_plane_gaps_are_never_read(lib, fmt):
    """pages as strided views, rows wider than the page and gaps between planes holding NaN and 1e30 (float16: 65504): the
    results of a compact copy"""
    torch = _torch()
    x = pages_np(3, 140, 90, seed=9)
    big = 65504.0 if fmt == "float16" else 1e30
    buf = torch.full((3, 150, 101), float("nan"), dtype=getattr(torch, fmt))
    buf[:, :, 1::2] = big
    buf[:, 140:] = big
    view = buf[:, :140, :90]
    view.copy_(torch.from_numpy(x))
    assert view.stride(1) > 90 and view.stride(0) > 140 * view.stride(1)
    compact = view.contiguous()
    e = _engine("fc", MIN_CHUNK)
    for entry in ENTRIES:
        for stride, pad, mode in ((1, None, "constant"), (3, (15, 15, 15, 15), "reflect"), (16, (7, 8, 7, 8), "replicate")):
            got = run_host(e, entry, view, stride, padding=pad, mode=mode)
            assert_same(got, run_host(e, entry, compact, stride, padding=pad, mode=mode), (fmt, entry, stride, pad))
            assert_same(got, run_device(e, entry, compact, stride, padding=pad, mode=mode), (fmt, entry, stride, pad, "device"))
    if fmt != "bfloat16":
        a = np.full((3, 150, 101), np.nan, dtype=np.float16 if fmt == "float16" else np.float32)
        a[:, :140, :90] = x
        got = run_host(e, "scan", a[:, :140, :90], 2)
        assert_same(got, run_host(e, "scan", np.ascontiguousarray(a[:, :140, :90]), 2), (fmt, "numpy view"))
        broadcast = np.broadcast_to(a[0, 3, :90], (2, 40, 90))   # row stride 0: copied, as rows may not overlap
        assert_same(run_host(e, "scan", broadcast, 2), run_host(e, "scan", np.ascontiguousarray(broadcast), 2), (fmt, "broadcast"))
    expanded = view[0, 3].expand(2, 40, 90)
    assert_same(run_host(e, "scan", expanded, 2), run_device(e, "scan", expanded.contiguous(), 2), (fmt, "expanded"))
    e.close()


def _host_fn(l, entry):
    """the host entry as f(handle, descriptor, padding, first, second, k) in section 10's argument order"""
    fn = getattr(l, STEMS[entry])
    if entry.endswith("topk"):
        return lambda h, d, pad, a, b, k: fn(h, d, pad, k, b, a)   # a: scores, b: classes
    return lambda h, d, pad, a, b, k: fn(h, d, pad, a, b)


def _device_fn(l, entry):
    fn = getattr(l, STEMS[entry] + "_device")
    if entry.endswith("topk"):
        return lambda h, d, a, b, k: fn(h, d, k, b, a, None)
    return lambda h, d, a, b, k: fn(h, d, a, b, None)


def _padded_fn(l, entry):
    fn = getattr(l, STEMS[entry] + "_padded_device")
    if entry.endswith("topk"):
        return lambda h, d, pad, a, b, k: fn(h, d, pad, k, b, a, None)
    return lambda h, d, pad, a, b, k: fn(h, d, pad, a, b, None)


@pytest.mark.gpu
def test_argument_errors(lib):
    """a NULL descriptor, an unknown format, a zero stride, pitch < width, no output, a bad k and reflect padding too wide for the
    page: the device sibling's code and text (the entry's name in place of the sibling's; pitch: no 16-byte rule for host rows),
    and nothing written"""
    torch = _torch()
    from bitnetmcu_b200 import _lib
    e = _engine("fc")
    h = e.handle
    x = pages_np(2, 40, 40, seed=1)
    d_x = torch.from_numpy(x).cuda()
    out = np.full(2 * 25 * 25 * 16, SENTINEL, dtype=np.float64)
    d_out = torch.full((2 * 25 * 25 * 16,), SENTINEL, dtype=torch.float64, device="cuda")
    o, d_o = C.c_void_p(out.ctypes.data), C.c_void_p(d_out.data_ptr())

    def host_desc(**kw):
        f = dict(image=x.ctypes.data, format=_lib.FLOAT32, planes=2, height=40, width=40, pitch=40, plane_pitch=1600, stride_y=1,
                 stride_x=1)
        f.update(kw)
        return _lib.BnmWindowsHost(**f)

    def dev_desc(**kw):
        f = dict(image=d_x.data_ptr(), planes=2, height=40, width=40, pitch=40, plane_pitch=1600, stride_y=1, stride_x=1)
        f.update({k: v for k, v in kw.items() if k != "format"})
        return _lib.BnmWindows(**f)

    def errs(entry, kw, first, second, k, pad=None):
        kw = dict(kw)
        null = kw.pop("null", False)
        hd, dd = host_desc(**kw), dev_desc(**kw)
        hp = None if pad is None else C.byref(pad)
        a, b, da, db = (o if first else None), (o if second else None), (d_o if first else None), (d_o if second else None)
        rc = _host_fn(lib, entry)(h, None if null else C.byref(hd), hp, a, b, k)
        text = lib.bnm_last_error().decode()
        if pad is None:
            drc = _device_fn(lib, entry)(h, None if null else C.byref(dd), da, db, k)
        else:
            drc = _padded_fn(lib, entry)(h, C.byref(dd), hp, da, db, k)
        dtext = lib.bnm_last_error().decode()
        return rc, text, drc, dtext.replace(STEMS[entry] + ("_padded" if pad is not None else "") + "_device", STEMS[entry])

    for entry in ENTRIES:
        topk = entry.endswith("topk")
        cases = [({"null": True}, True, True, 1, None), ({"stride_y": 0}, True, True, 1, None), ({}, False, False, 1, None),
                 ({}, True, True, 0, None) if topk else None, ({}, True, True, 17, None) if topk else None,
                 ({"height": 10}, True, True, 1, _lib.BnmWindowPadding(1, 1, 12, 0, _lib.PAD_REFLECT, 0.0)),
                 ({"width": 12}, True, True, 1, _lib.BnmWindowPadding(0, 13, 0, 0, _lib.PAD_REFLECT, 0.0)),
                 ({}, True, True, 1, _lib.BnmWindowPadding(16, 0, 0, 0, _lib.PAD_CONSTANT, 0.0))]
        for kw, first, second, k, pad in filter(None, cases):
            rc, text, drc, dtext = errs(entry, kw, first, second, k, pad)
            assert rc == drc == BNM_E_ARG and text == dtext, (entry, kw, k, text, dtext)
        rc, text, drc, dtext = errs(entry, {"pitch": 39}, True, True, 1)
        assert rc == drc == BNM_E_ARG and text == f"{STEMS[entry]}: pitch 39 must be >= width 40" and dtext.startswith(text), (text, dtext)
        for fmt in (0, 4, -1):
            hd = host_desc(format=fmt)
            rc = _host_fn(lib, entry)(h, C.byref(hd), None, o, o, 1)
            assert rc == BNM_E_ARG and lib.bnm_last_error().decode() == \
                f"{STEMS[entry]}: format {fmt}, must be BNM_FLOAT32 (3), BNM_FLOAT16 (1) or BNM_BFLOAT16 (2)", (entry, fmt)
    assert (out == SENTINEL).all() and bool((d_out == SENTINEL).all())
    e.close()


@pytest.mark.gpu
def test_two_threads_on_one_model(lib):
    """two threads' host scans on one model at the minimum chunk, several calls each: every result the sibling's"""
    e = _engine("fc", MIN_CHUNK)
    stacks = [pages_np(2, 220, 180, seed=20 + t) for t in range(2)]
    want = [run_device(e, "scan", s, (1, 2)) for s in stacks]
    errors = []

    def worker(t):
        try:
            for _ in range(4):
                assert_same(run_host(e, "scan", stacks[t], (1, 2)), want[t], ("thread", t))
        except BaseException as ex:   # noqa: BLE001 - reported by the main thread
            errors.append(ex)

    threads = [threading.Thread(target=worker, args=(t,)) for t in range(2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    e.close()


@pytest.mark.gpu
def test_host_scan_while_another_thread_captures(lib):
    """a host scan on one thread while the main thread captures a device window scan into a torch.cuda.graph in global mode: the
    capture stays valid, its replay and the host scan both give the sibling's results"""
    torch = _torch()
    e = _engine("fc", MIN_CHUNK)
    x = pages_np(2, 220, 180, seed=31)
    want = run_device(e, "scan", x, (1, 2))
    g_x = device_stack(pages_np(1, 64, 80, seed=32))
    g_la = torch.full((1, 49, 65), SENTINEL, dtype=torch.int32, device="cuda")
    capturing, done = threading.Event(), threading.Event()
    errors, got = [], []

    def host():
        try:
            assert capturing.wait(600)
            got.append(run_host(e, "scan", x, (1, 2)))
        except BaseException as ex:   # noqa: BLE001 - reported by the main thread
            errors.append(ex)
        finally:
            done.set()

    t = threading.Thread(target=host)
    t.start()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):                    # capture_error_mode="global"
        e.scan_windows_device(g_x, 1, None, g_la)
        capturing.set()
        assert done.wait(600)
    t.join()
    assert not errors, errors
    assert_same(got[0], want, "host scan during capture")
    g.replay()
    torch.cuda.synchronize()
    ref = torch.full_like(g_la, SENTINEL)
    e.scan_windows_device(g_x, 1, None, ref)
    torch.cuda.synchronize()
    assert torch.equal(g_la, ref) and bool((g_la != SENTINEL).all())
    del g
    e.close()


def _mem_available():
    try:
        with open("/proc/meminfo") as f:
            return next(int(l.split()[1]) * 1024 for l in f if l.startswith("MemAvailable:"))
    except (OSError, StopIteration):
        return 0


@pytest.mark.gpu
def test_host_span_past_2_to_32_bytes(lib):
    """17 float32 pages of 8192 x 8192 (4.25 GiB; the last plane starts at byte 2^32) at stride 16, labels only: the sibling's
    labels on the stack uploaded with torch.  Planes differ (a random 97 x 89 tile per plane), so a read displaced by a wrapped
    32-bit offset changes the labels"""
    torch = _torch()
    P, H, W = 17, 8192, 8192
    need = P * H * W * 4
    if _mem_available() < 3 * need:
        pytest.skip(f"needs {3 * need / 2**30:.1f} GiB of host memory")
    if torch.cuda.mem_get_info()[0] < need + (4 << 30):
        pytest.skip(f"needs {need / 2**30 + 4:.1f} GiB of device memory")
    rng = np.random.default_rng(17)
    x = np.empty((P, H, W), dtype=np.float32)
    for p in range(P):
        tile = rng.standard_normal((97, 89), dtype=np.float32)
        x[p] = np.tile(tile, (H // 97 + 1, W // 89 + 1))[:H, :W]
    assert x[16].ctypes.data - x.ctypes.data == 1 << 32
    e = _engine("fc")
    _, labels = e.scan_windows(x, 16, want_logits=False)
    d = torch.from_numpy(x).cuda()
    want = torch.full((P, 512, 512), SENTINEL, dtype=torch.int32, device="cuda")
    e.scan_windows_device(d, 16, None, want)
    torch.cuda.synchronize()
    w = want.cpu().numpy().view(np.uint32)
    assert np.array_equal(labels, w)
    assert not np.array_equal(labels[16], labels[0])
    del d, want
    torch.cuda.empty_cache()
    e.close()
