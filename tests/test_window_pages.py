"""Window scan of a stack of pages (include/bitnetmcu_b200.h section 10): bnm_scan_windows_device, bnm_scan_windows_topk_device,
bnm_emulate_windows_device and bnm_emulate_windows_topk_device classify every 16x16 window of every plane of a stack in one call.
Each entry's contract is bit-exactness with its per-image counterpart (bnm_infer_batch_device_f32, bnm_infer_topk_device_f32,
bnm_emulate_batch_device, bnm_emulate_topk_device) on the windows extracted plane by plane and concatenated, which pins it to the
oracle and the emulator restatement through entries that are already verified.  The CPU tests check the stacked window order, the
exported symbols, the failure without a device and the scaling kernels' SASS; the GPU tests check the results on every model and
route, against the oracle and the restatement, across pass and plane boundaries, the pixels a window may read, 64-bit plane
offsets, the scaling edges, the outputs and arguments, the routes, graphs, streams and mode 2."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from conftest import ROOT, load_model
from support import instructions, lib, local_memory, random_fc, sass_functions, verbose_engine  # noqa: F401 (lib: fixture)

MODELS = ["fc", "12k_FP130", "ternary64", "binary160", "2bitsym96", "cnn_48", "cnn_letters", "rand_nf4_64"]   # as the window scan's
STRIDES = [(1, 1), (2, 3), (16, 16), (17, 5)]
STACKS = [(1, 37, 53), (3, 50, 18), (7, 41, 67)]   # planes, height, width: odd pages; out_w below 4 in the second
ENTRIES = ["scan", "scan_topk", "emulate", "emulate_topk"]
SENTINEL = -7


def stacked_windows_np(buf, planes, h, w, pitch, plane_pitch, sy, sx):
    """the windows of a stack held in the flat array buf (plane p at p * plane_pitch, rows pitch apart) in the stacked window
    order, each flattened row-major: [planes * out_h * out_w, 256]"""
    from numpy.lib.stride_tricks import as_strided
    if planes == 0 or h < 16 or w < 16:
        return np.zeros((0, 256), dtype=buf.dtype)
    oh, ow = (h - 16) // sy + 1, (w - 16) // sx + 1
    e = buf.itemsize
    v = as_strided(buf, shape=(planes, oh, ow, 16, 16), strides=(plane_pitch * e, sy * pitch * e, sx * e, pitch * e, e), writeable=False)
    return np.ascontiguousarray(v).reshape(-1, 256)


def page_np(h, w, seed):
    """normal pixels with MNIST-normalised patches and a dark margin, float32 [h, w]"""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal(size=(h, w), dtype=np.float32)
    for _ in range(max(1, h * w // 4000)):
        r, c = rng.integers(0, max(1, h - 20)), rng.integers(0, max(1, w - 20))
        x[r:r + 20, c:c + 20] = (rng.integers(0, 256, size=(min(20, h - r), min(20, w - c))) / 255.0 - 0.1307).astype(np.float32) / np.float32(0.3081)
    x[:, :3] *= np.float32(0.01)
    return x


# ---- CPU ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("planes,h,w,pitch,gap,sy,sx", [(1, 16, 16, 16, 0, 1, 1), (3, 37, 53, 56, 0, 2, 3), (2, 40, 41, 44, 100, 17, 5),
                                                        (4, 31, 70, 72, 8, 1, 40), (3, 19, 16, 16, 4, 3, 7), (0, 40, 40, 40, 0, 1, 1)])
def test_stacked_window_order_equals_a_loop(planes, h, w, pitch, gap, sy, sx):
    """plane_pitch = h * pitch + gap (gap > 0: planes further apart than their rows): window (p * out_h + r) * out_w + c is rows
    r*sy .. +15, columns c*sx .. +15 of plane p"""
    plane_pitch = h * pitch + gap
    buf = np.arange(max(planes, 1) * plane_pitch, dtype=np.float32)
    oh, ow = (h - 16) // sy + 1, (w - 16) // sx + 1
    loop = [np.array([buf[p * plane_pitch + (r * sy + y) * pitch + c * sx + x] for y in range(16) for x in range(16)])
            for p in range(planes) for r in range(oh) for c in range(ow)]
    got = stacked_windows_np(buf, planes, h, w, pitch, plane_pitch, sy, sx)
    assert got.shape == (planes * oh * ow, 256)
    assert np.array_equal(got, np.array(loop).reshape(-1, 256))


def test_stacked_entries_are_declared_and_exported(built):
    from bitnetmcu_b200 import _lib
    text = open(os.path.join(ROOT, "include", "bitnetmcu_b200.h")).read()
    assert "typedef struct bnm_windows" in text
    lib = _lib.load()
    for name in ("bnm_scan_windows_device", "bnm_scan_windows_topk_device", "bnm_emulate_windows_device", "bnm_emulate_windows_topk_device"):
        assert re.search(rf"BNM_API int {name}\(", text), name
        assert name in _lib.EXPORTED and hasattr(lib, name), name
    assert C.sizeof(_lib.BnmWindows) == 48


def test_stacked_entries_fail_without_a_device(built):
    from bitnetmcu_b200 import _lib
    lib = _lib.load()
    if lib.bnm_device_count() > 0:
        pytest.skip("a CUDA device is present")
    img = np.zeros(4 * 64 * 64, dtype=np.float32)
    d = _lib.BnmWindows(img.ctypes.data, 2, 64, 64, 64, 64 * 64, 16, 16)
    out = np.full(64, 7, dtype=np.uint32)
    o = C.c_void_p(out.ctypes.data)
    for rc in (lib.bnm_scan_windows_device(None, C.byref(d), None, o, None),
               lib.bnm_scan_windows_topk_device(None, C.byref(d), 1, o, None, None),
               lib.bnm_emulate_windows_device(None, C.byref(d), None, o, None),
               lib.bnm_emulate_windows_topk_device(None, C.byref(d), 1, o, None, None)):
        assert rc == -2 and b"no CUDA device" in lib.bnm_last_error()
    assert (out == 7).all()


def test_scaling_kernels_have_no_local_memory(built):
    """k_quantize_windows is still one function (planes and plane pitch are runtime fields), and the emulator's int8-input CNN
    front-end is one function of its own next to the float one"""
    kernels = sass_functions()
    for key in ("k_quantize_windows", "_ZN3bnm22k_cnn_emul_frontend_i8", "_ZN3bnm19k_cnn_emul_frontendE"):
        funcs = {k: v for k, v in kernels.items() if key in k}
        assert len(funcs) == 1, (key, list(funcs))
        for name, text in funcs.items():
            ins = instructions(text)
            assert len(ins) > 100 and not local_memory(ins), name


# ---- GPU ---------------------------------------------------------------------------------------------------------------------

def _engine(name, path=0):
    from bitnetmcu_b200.engine import Engine
    m = load_model(name) if isinstance(name, str) else name
    return Engine(m, device=0, path=path, nf4_extension=(name == "rand_nf4_64"))


def stack(pages, fill=0.0, gap=0, pad=0, below=0):
    """pages (NumPy [P, h, w]) as a CUDA stack [P, h, w] inside one allocation: rows (w rounded up to 4) + pad floats apart, `below`
    rows past each page and `gap` floats between planes, all that padding filled with fill"""
    import torch
    p, h, w = pages.shape
    pitch = (w + 3) // 4 * 4 + pad
    plane_pitch = (h + below) * pitch + gap
    buf = torch.full((max(p, 1) * plane_pitch,), fill, dtype=torch.float32, device="cuda")
    view = buf.as_strided((p, h, w), (plane_pitch, pitch, 1))
    view.copy_(torch.from_numpy(pages))
    return view


def unfold(pages, sy, sx):
    """the windows of a CUDA stack extracted plane by plane and concatenated: float32 [P * out_h * out_w, 256], contiguous"""
    import torch
    return torch.cat([pages[p].unfold(0, 16, sy).unfold(1, 16, sx).reshape(-1, 256) for p in range(pages.shape[0])]).contiguous()


def _k(e):
    return min(e.n_classes, 5)


def run_stack(e, entry, pages, stride, k=None, first=True, second=True, stream=None, sync=True):
    """a stacked entry on a CUDA stack -> its two outputs as NumPy, flattened to [windows, ...] (None where not asked):
    (logits, labels) or (classes, scores)"""
    import torch
    from bitnetmcu_b200.engine import window_grid
    grid = (pages.shape[0],) + window_grid(pages.shape[-2], pages.shape[-1], stride)
    emul, topk = entry.startswith("emulate"), entry.endswith("topk")
    ldt = torch.float64 if emul else torch.int32
    if topk:
        k = k or _k(e)
        a = torch.full(grid + (k,), SENTINEL, dtype=torch.int32, device="cuda") if first else None
        b = torch.full(grid + (k,), SENTINEL, dtype=ldt, device="cuda") if second else None
        fn = e.emulate_windows_topk_device if emul else e.scan_windows_topk_device
        fn(pages, stride, k, a, b, stream=stream)
    else:
        a = torch.full(grid + (e.n_classes,), SENTINEL, dtype=ldt, device="cuda") if first else None
        b = torch.full(grid, SENTINEL, dtype=torch.int32, device="cuda") if second else None
        (e.emulate_windows_device if emul else e.scan_windows_device)(pages, stride, a, b, stream=stream)
    if not sync:
        return a, b
    torch.cuda.synchronize()
    n = int(np.prod(grid))
    return tuple(None if t is None else t.reshape(n, -1).cpu().numpy() for t in (a, b))


def run_rows(e, entry, rows, k=None):
    """the per-image counterpart of a stacked entry on float rows [n, 256] (CUDA) -> the same two outputs as NumPy"""
    import torch
    n = rows.shape[0]
    emul, topk = entry.startswith("emulate"), entry.endswith("topk")
    ldt = torch.float64 if emul else torch.int32
    if topk:
        k = k or _k(e)
        a = torch.full((n, k), SENTINEL, dtype=torch.int32, device="cuda")
        b = torch.full((n, k), SENTINEL, dtype=ldt, device="cuda")
        if n:
            (e.emulate_topk_device if emul else e.topk_device_f32)(rows, k, a, b)
    else:
        a = torch.full((n, e.n_classes), SENTINEL, dtype=ldt, device="cuda")
        b = torch.full((n,), SENTINEL, dtype=torch.int32, device="cuda")
        if n:
            (e.inference_quantized_device if emul else e.infer_device_f32)(rows, a, b)
    torch.cuda.synchronize()
    return a.reshape(n, -1).cpu().numpy(), b.reshape(n, -1).cpu().numpy()


def assert_same(got, want, what):
    for g, w, kind in zip(got, want, ("first", "second")):
        if g is None or w is None:
            continue
        assert g.shape == w.shape, (what, kind, g.shape, w.shape)
        bad = np.flatnonzero((g != w).reshape(len(w), -1).any(axis=1))
        assert bad.size == 0, (what, kind, f"{bad.size} of {len(w)} windows differ, first {bad[:6].tolist()}")


def pages_np(planes, h, w, seed):
    return np.stack([page_np(h, w, seed=seed + 7 * p) for p in range(planes)]) if planes else np.zeros((0, h, w), dtype=np.float32)


@pytest.mark.gpu
@pytest.mark.parametrize("name", MODELS)
def test_stacked_entries_equal_their_counterparts(lib, name):
    """every entry, stride and stack, on the default path and BNM_PATH_LAYERS: the counterpart on the unfolded windows; one plane:
    infer_windows_device"""
    import torch
    from bitnetmcu_b200 import _lib
    from bitnetmcu_b200.engine import window_grid
    e = _engine(name)
    for path in (_lib.PATH_AUTO, _lib.PATH_LAYERS):
        e.set_option(_lib.OPT_PATH, path)
        for planes, h, w in STACKS:
            pages = stack(pages_np(planes, h, w, seed=planes * 100 + h), gap=4 * planes)
            for stride in STRIDES:
                rows = unfold(pages, *stride)
                assert rows.shape[0] == planes * len(range(0, h - 15, stride[0])) * len(range(0, w - 15, stride[1]))
                for entry in ENTRIES:
                    assert_same(run_stack(e, entry, pages, stride), run_rows(e, entry, rows), (name, path, planes, stride, entry))
                if planes == 1:
                    oh, ow = window_grid(h, w, stride)
                    lo = torch.empty((oh, ow, e.n_classes), dtype=torch.int32, device="cuda")
                    la = torch.empty((oh, ow), dtype=torch.int32, device="cuda")
                    e.infer_windows_device(pages[0], stride, lo, la)
                    torch.cuda.synchronize()
                    want = (lo.reshape(-1, e.n_classes).cpu().numpy(), la.reshape(-1, 1).cpu().numpy())
                    assert_same(run_stack(e, "scan", pages, stride), want, (name, path, "one plane", stride))
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["fc", "binary160", "cnn_letters"])
def test_topk_windows_equal_the_oracle(lib, oracle, name):
    """the C engine's top-k of every window: a stable sort of the oracle's logits on the scaled windows"""
    from bitnetmcu_b200.engine import quantize_images
    e = _engine(name)
    pages = pages_np(3, 45, 61, seed=9)
    for sy, sx in [(1, 1), (3, 2)]:
        k = min(e.n_classes, 16)
        cls, sc = run_stack(e, "scan_topk", stack(pages), (sy, sx), k=k)
        x = stacked_windows_np(pages.reshape(-1), 3, 45, 61, 61, 45 * 61, sy, sx)
        logits, _ = oracle.infer(e.model, quantize_images(x))
        order = np.argsort(-logits.astype(np.int64), axis=1, kind="stable")[:, :k]
        assert np.array_equal(cls.astype(np.int64), order), (name, (sy, sx))
        assert np.array_equal(sc, np.take_along_axis(logits, order, axis=1)), (name, (sy, sx))
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["fc", "cnn_48", "cnn_16small"])
def test_emulated_windows_equal_the_restatement(lib, name):
    from restate import emulate
    e = _engine(name)
    pages = pages_np(3, 40, 52, seed=12)
    for sy, sx in [(1, 1), (5, 3)]:
        lo, la = run_stack(e, "emulate", stack(pages), (sy, sx))
        want = emulate(e.model, stacked_windows_np(pages.reshape(-1), 3, 40, 52, 52, 40 * 52, sy, sx))
        assert np.array_equal(lo, want), (name, (sy, sx), np.argwhere(lo != want)[:5])
        assert np.array_equal(la[:, 0], np.argmax(want, axis=1)), (name, (sy, sx))
    e.close()


def _sliced(e, entry, pages, got, rows_per_plane):
    """got (the stacked entry's outputs on pages at stride 1) against the counterpart, plane by plane, in slices of window rows"""
    import torch
    oh, ow = pages.shape[1] - 15, pages.shape[2] - 15
    for p in range(pages.shape[0]):
        for r0 in range(0, oh, rows_per_plane):
            r1 = min(oh, r0 + rows_per_plane)
            want = run_rows(e, entry, pages[p, r0:r1 + 15].unfold(0, 16, 1).unfold(1, 16, 1).reshape(-1, 256).contiguous())
            sl = slice((p * oh + r0) * ow, (p * oh + r1) * ow)
            assert_same(tuple(g[sl] for g in got), want, (entry, "plane", p, "rows", r0))
        torch.cuda.empty_cache()


@pytest.mark.gpu
def test_pass_boundaries_across_planes(lib):
    """planes of 601 x 701 windows (421 301 each) at stride 1: the passes of 2^20 windows start inside a plane and inside a window
    row; five planes on the C engine (labels and logits, top-k), three on the CNN emulator's int8 front-end"""
    e = _engine("fc")
    pages = stack(pages_np(5, 16 + 600, 16 + 700, seed=41))
    for entry in ("scan", "scan_topk"):
        got = run_stack(e, entry, pages, 1)
        assert got[0].shape[0] == 5 * 421301 > 2 * (1 << 20)
        _sliced(e, entry, pages, got, 301)
    e.close()
    e = _engine("cnn_48")
    pages = pages[:3]
    _sliced(e, "emulate", pages, run_stack(e, "emulate", pages, 1), 301)
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["fc", "binary160", "cnn_48"])
def test_only_the_window_pixels_count(lib, name):
    """stacks inside one allocation whose row padding, rows below each page and gap between planes hold 1e30: the results of the
    clean stack (a band or a plane offset that reached past a window would see them)"""
    e = _engine(name)
    for planes, h, w in STACKS:
        x = pages_np(planes, h, w, seed=h + w)
        clean, dirty = stack(x), stack(x, fill=1e30, gap=36, pad=8, below=9)
        assert dirty.stride(0) > dirty.shape[1] * dirty.stride(1)
        for stride in STRIDES:
            for entry in ENTRIES:
                assert_same(run_stack(e, entry, dirty, stride), run_stack(e, entry, clean, stride), (name, planes, stride, entry))
    e.close()


@pytest.mark.gpu
def test_plane_offsets_past_4_gib(lib):
    """two planes 2^30 + 256 elements apart: the second one's byte offset is past 4 GiB; every entry equals the per-plane calls"""
    import torch
    plane_pitch = (1 << 30) + 256
    h, w = 40, 64
    buf = torch.full((plane_pitch + h * w,), 1e30, dtype=torch.float32, device="cuda")
    pages = buf.as_strided((2, h, w), (plane_pitch, w, 1))
    pages.copy_(torch.from_numpy(pages_np(2, h, w, seed=64)))
    assert pages[1].data_ptr() - pages.data_ptr() > 4 << 30
    for name in ("fc", "cnn_48"):
        e = _engine(name)
        for entry in ENTRIES:
            got = run_stack(e, entry, pages, (2, 3))
            alone = [run_stack(e, entry, pages[p:p + 1].clone(), (2, 3)) for p in range(2)]
            assert_same(got, tuple(np.concatenate([a[i] for a in alone]) for i in range(2)), (name, entry, "4 GiB"))
        e.close()
    del pages, buf
    torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["fc", "binary160", "cnn_48"])
def test_scaling_edges(lib, name):
    """windows that are all zero, all negative, hold +-1e30, subnormals or -0.0, through every entry"""
    x = page_np(96, 96, seed=3)
    x[0:24, 0:24] = 0.0
    x[0:24, 30:60] = -np.abs(x[0:24, 30:60]) - np.float32(0.5)
    x[30:34, 5] = np.float32(1e30)
    x[40, 40] = np.float32(-1e30)
    x[50:80, 50:80] = np.float32(1e-40) * np.sign(x[50:80, 50:80])
    x[60:90, 0:30] = np.float32(-0.0)
    x[62, 3] = np.float32(2e-45)
    x[70:72, 10:12] = np.float32(0.5) / np.float32(127.0) * np.arange(4, dtype=np.float32).reshape(2, 2)
    pages = stack(np.stack([x, -x[::-1].copy()]))
    e = _engine(name)
    for stride in [(1, 1), (2, 3), (16, 16)]:
        rows = unfold(pages, *stride)
        for entry in ENTRIES:
            assert_same(run_stack(e, entry, pages, stride), run_rows(e, entry, rows), (name, "edges", stride, entry))
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["fc", "cnn_letters", "binary160"])
def test_outputs_and_k(lib, name):
    """labels only, logits only, scores NULL, k = 1 and min(n_classes, 16)"""
    e = _engine(name)
    pages = stack(pages_np(3, 50, 70, seed=1))
    for entry in ENTRIES:
        if entry.endswith("topk"):
            for k in (1, min(e.n_classes, 16)):
                both = run_stack(e, entry, pages, (1, 2), k=k)
                assert np.array_equal(run_stack(e, entry, pages, (1, 2), k=k, second=False)[0], both[0]), (entry, k)
                if k == 1:
                    labels = run_stack(e, entry.replace("_topk", ""), pages, (1, 2), first=False)[1]
                    assert np.array_equal(both[0].astype(np.int64), labels.astype(np.int64)), (entry, "rank 0 is the label")
        else:
            both = run_stack(e, entry, pages, (1, 2))
            assert np.array_equal(run_stack(e, entry, pages, (1, 2), first=False)[1], both[1]), entry
            assert np.array_equal(run_stack(e, entry, pages, (1, 2), second=False)[0], both[0]), entry
    e.close()


@pytest.mark.gpu
def test_argument_errors(lib):
    """each argument error gives its code and writes nothing; no windows returns 0 and writes nothing; a top-k call checks k and
    alignment even then"""
    import torch
    from bitnetmcu_b200 import _lib
    e = _engine("fc")
    img = torch.zeros((4 * 64 * 64 + 64,), dtype=torch.float32, device="cuda")
    lo = torch.full((4 * 49 * 49 * 10 + 64,), SENTINEL, dtype=torch.float64, device="cuda")   # room for every output type
    la = torch.full((4 * 49 * 49 * 16 + 64,), SENTINEL, dtype=torch.int32, device="cuda")
    P = lambda t, off=0: C.c_void_p(t.data_ptr() + off)

    def desc(planes=2, h=64, w=64, pitch=64, plane_pitch=64 * 64, sy=1, sx=1, off=0):
        return _lib.BnmWindows(img.data_ptr() + off, planes, h, w, pitch, plane_pitch, sy, sx)

    calls = {
        "scan": lambda d, a, b, k: lib.bnm_scan_windows_device(e.handle, d, a, b, None),
        "scan_topk": lambda d, a, b, k: lib.bnm_scan_windows_topk_device(e.handle, d, k, b, a, None),
        "emulate": lambda d, a, b, k: lib.bnm_emulate_windows_device(e.handle, d, a, b, None),
        "emulate_topk": lambda d, a, b, k: lib.bnm_emulate_windows_topk_device(e.handle, d, k, b, a, None),
    }
    for entry, call in calls.items():
        topk = entry.endswith("topk")
        cases = {
            "null descriptor": call(None, P(lo), P(la), 3),
            "zero stride y": call(C.byref(desc(sy=0)), P(lo), P(la), 3),
            "zero stride x": call(C.byref(desc(sx=0)), P(lo), P(la), 3),
            "pitch < width": call(C.byref(desc(pitch=60)), P(lo), P(la), 3),
            "pitch % 4": call(C.byref(desc(w=62, pitch=63)), P(lo), P(la), 3),
            "plane pitch % 4": call(C.byref(desc(plane_pitch=64 * 64 + 2)), P(lo), P(la), 3),
            "image misaligned": call(C.byref(desc(off=4)), P(lo), P(la), 3),
            "logits / scores misaligned": call(C.byref(desc()), P(lo, 2 if topk and entry == "scan_topk" else 4), P(la), 3),
            "no output": call(C.byref(desc()), None, None, 3),
        }
        if topk:
            cases.update({"k = 0": call(C.byref(desc()), P(lo), P(la), 0), "k = 11": call(C.byref(desc()), P(lo), P(la), 11),
                          "k = 17": call(C.byref(desc()), P(lo), P(la), 17),
                          "k = 0, no windows": call(C.byref(desc(planes=0)), P(lo), P(la), 0),
                          "scores misaligned, no windows": call(C.byref(desc(planes=0)), P(lo, 2), P(la), 3)})
        assert cases == {k: -1 for k in cases}, (entry, cases)
        for d in (desc(planes=0), desc(h=15), desc(w=15), desc(planes=0, h=0, w=0)):
            assert call(C.byref(d), P(lo), P(la), 3) == 0, entry
        # one plane ignores the plane pitch
        assert call(C.byref(desc(planes=1, h=15, plane_pitch=3)), P(lo), P(la), 3) == 0, entry
    wide = _engine(random_fc(4, (512, 64, 64, 10), 1))
    for entry in calls:
        call = {"scan": lib.bnm_scan_windows_device, "emulate": lib.bnm_emulate_windows_device}.get(entry)
        if call is not None:
            assert call(wide.handle, C.byref(desc()), P(lo), P(la), None) == -3 and b"16x16" in lib.bnm_last_error()
    assert lib.bnm_scan_windows_topk_device(wide.handle, C.byref(desc()), 3, P(la), P(lo), None) == -3
    assert lib.bnm_emulate_windows_topk_device(wide.handle, C.byref(desc()), 3, P(la), P(lo), None) == -3
    wide.close()
    torch.cuda.synchronize()
    assert (lo == SENTINEL).all() and (la == SENTINEL).all()
    e.close()


ROUTE_CASES = [("fc", lambda: load_model("fc"), 0), ("37 classes", lambda: random_fc(4, (256, 64, 64, 37), 2), 0),
               ("binary160", lambda: load_model("binary160"), 0), ("cnn_48", lambda: load_model("cnn_48"), 0),
               ("layers", lambda: load_model("fc"), 1), ("cnn layers", lambda: load_model("cnn_48"), 1)]


@pytest.mark.gpu
def test_routes_name_the_window_kernels(lib, capfd, monkeypatch):
    pages = stack(pages_np(2, 40, 40, seed=2))
    names = {"scan": "bnm_scan_windows_device", "scan_topk": "bnm_scan_windows_topk_device", "emulate": "bnm_emulate_windows_device",
             "emulate_topk": "bnm_emulate_windows_topk_device"}
    for what, make, path in ROUTE_CASES:
        e, _ = verbose_engine(capfd, monkeypatch, lambda: _engine(make(), path=path))
        for entry in ENTRIES:
            capfd.readouterr()
            run_stack(e, entry, pages, 3)
            lines = [l for l in capfd.readouterr().err.splitlines() if "route: " in l]
            assert len(lines) == 1 and f"windows route: {names[entry]}: " in lines[0], (what, entry, lines)
            r = lines[0].split(f"windows route: {names[entry]}: ")[1]
            emul, topk, cnn = entry.startswith("emulate"), entry.endswith("topk"), what.startswith("cnn")
            assert r.startswith("k_quantize_windows + ") and ",float" not in r, (what, entry, r)
            if path:
                assert "layer by layer" in r and ("k_topk_rows" in r) == topk, (what, entry, r)
                continue
            if emul and cnn:
                assert r.startswith("k_quantize_windows + k_cnn_emul_frontend_i8 + "), (what, entry, r)
            assert ("k_cnn_frontend16" in r) == (cnn and not emul), (what, entry, r)
            kernel = r.split(" + ")[-1]
            want = ("fc_topk_kernel<" if topk else "fc_emul_i8_kernel<" if emul else "fc_chain_kernel<")
            assert kernel.startswith(want) and (",emul" in kernel) == emul, (what, entry, r)
        e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["fc", "cnn_48", "binary160"])
def test_graph_replay_and_two_streams(lib, name):
    import torch
    e = _engine(name)
    shape, stride = (3, 150, 100), (2, 1)
    for entry in ENTRIES:
        pages = stack(pages_np(*shape, seed=4))
        outs = run_stack(e, entry, pages, stride, sync=False)   # warm: the pool and the kernels' attributes
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=torch.cuda.Stream()):
            outs = run_stack(e, entry, pages, stride, sync=False)
        pages.copy_(torch.from_numpy(pages_np(*shape, seed=5)))
        g.replay()
        torch.cuda.synchronize()
        got = tuple(t.reshape(outs[1].shape[:3].numel(), -1).cpu().numpy() for t in outs)
        assert_same(got, run_stack(e, entry, pages, stride), (name, entry, "replay"))
        del g
        stacks = [stack(pages_np(*shape, seed=10 + k)) for k in range(2)]
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
            assert_same(tuple(t.reshape(outs[1].shape[:3].numel(), -1).cpu().numpy() for t in outs), alone[k], (name, entry, "stream", k))
    e.close()


@pytest.mark.gpu
def test_mode2_int8_launch_after_a_stacked_window_call_waits(lib, oracle, capfd, monkeypatch):
    """in mode 2 a stacked window call between two int8 launches is a launch of another kind: its own fused launch and the int8
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
    pages = stack(pages_np(3, 200, 300, seed=6))
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
    assert_same((wlo.reshape(-1, 10).cpu().numpy(), wla.reshape(-1, 1).cpu().numpy()), run_rows(e, "scan", unfold(pages, 1, 1)), "mode 2")
    e.close()
