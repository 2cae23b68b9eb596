"""Window scan (include/bitnetmcu_b200.h section 9): bnm_infer_windows_device_f32 classifies every 16x16 window of a float plane on a
stride grid.  Its contract is bit-exactness with bnm_infer_batch_device_f32 on the extracted windows in row-major window order,
which pins it to the oracle through an entry that is already verified.  The CPU tests check the window restatement, the grid
formula, the exported symbol and the failure without a device; the GPU tests check the results on every route, the pixels a
window may read, the scaling edges, several passes, the outputs, the routes, the arguments, graphs, streams and mode 2."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from conftest import ROOT, load_model
from support import instructions, lib, local_memory, random_fc, sass_functions, verbose_engine  # noqa: F401 (lib: fixture)

STRIDES = [(1, 1), (2, 3), (4, 4), (16, 16), (17, 5), (1, 40)]
PAGES = [(16, 16), (37, 53), (300, 520), (50, 18)]   # one window; odd; large; out_w below 4 (one window per band at most strides)
MODELS = ["fc", "12k_FP130", "ternary64", "binary160", "2bitsym96", "cnn_48", "cnn_letters", "rand_nf4_64"]
LABEL_SENTINEL, LOGIT_SENTINEL = -7, -123456789


def windows_np(page, sy, sx):
    """the windows of page in window order, each flattened row-major: float32 [out_h * out_w, 256]"""
    from numpy.lib.stride_tricks import sliding_window_view
    if page.shape[0] < 16 or page.shape[1] < 16:
        return np.zeros((0, 256), dtype=page.dtype)
    return np.ascontiguousarray(sliding_window_view(page, (16, 16))[::sy, ::sx]).reshape(-1, 256)


def page_np(h, w, seed):
    """normal pixels with MNIST-normalised patches and a dark margin, float32 [h, w]"""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal(size=(h, w), dtype=np.float32)
    for _ in range(max(1, h * w // 4000)):
        r, c = rng.integers(0, max(1, h - 20)), rng.integers(0, max(1, w - 20))
        x[r:r + 20, c:c + 20] = (rng.integers(0, 256, size=(min(20, h - r), min(20, w - c))) / 255.0 - 0.1307).astype(np.float32) / np.float32(0.3081)
    x[:, :3] *= np.float32(0.01)
    return x


def plane(x, fill=0.0):
    """x (NumPy [h, w]) as a CUDA plane whose rows are a multiple of 4 floats apart (16-byte rows), the padding filled with fill"""
    import torch
    h, w = x.shape
    buf = torch.full((h, (w + 3) // 4 * 4), fill, dtype=torch.float32, device="cuda")
    buf[:, :w] = torch.from_numpy(x)
    return buf[:, :w]


# ---- CPU ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("h,w,sy,sx", [(16, 16, 1, 1), (17, 19, 1, 2), (37, 53, 2, 3), (40, 41, 17, 5), (31, 70, 1, 40), (16, 90, 3, 7)])
def test_window_restatement_equals_a_loop(h, w, sy, sx):
    from bitnetmcu_b200.engine import window_grid
    page = np.arange(h * w, dtype=np.float32).reshape(h, w)
    out_h, out_w = window_grid(h, w, (sy, sx))
    assert (out_h, out_w) == ((h - 16) // sy + 1, (w - 16) // sx + 1)
    loop = np.array([page[r * sy:r * sy + 16, c * sx:c * sx + 16].reshape(256) for r in range(out_h) for c in range(out_w)])
    assert np.array_equal(windows_np(page, sy, sx), loop)
    # the last window ends inside the page, one more step would not
    assert (out_h - 1) * sy + 16 <= h < out_h * sy + 16 and (out_w - 1) * sx + 16 <= w < out_w * sx + 16


def test_window_grid_edges():
    from bitnetmcu_b200.engine import window_grid
    assert window_grid(15, 100, 1) == (0, 0) and window_grid(100, 15, 1) == (0, 0)
    assert window_grid(16, 16, 5) == (1, 1) and window_grid(31, 31, 16) == (1, 1) and window_grid(32, 33, 16) == (2, 2)
    assert window_grid(4096, 4096, 1) == (4081, 4081) and window_grid(4096, 4096, (2, 4)) == (2041, 1021)
    with pytest.raises(ValueError):
        window_grid(32, 32, (0, 1))


def test_window_entry_is_declared_and_exported(built):
    from bitnetmcu_b200 import _lib
    text = open(os.path.join(ROOT, "include", "bitnetmcu_b200.h")).read()
    assert re.search(r"BNM_API int bnm_infer_windows_device_f32\(", text)
    assert "bnm_infer_windows_device_f32" in _lib.EXPORTED
    assert hasattr(_lib.load(), "bnm_infer_windows_device_f32")


def test_window_entry_fails_without_a_device(built):
    from bitnetmcu_b200 import _lib
    lib = _lib.load()
    if lib.bnm_device_count() > 0:
        pytest.skip("a CUDA device is present")
    labels = np.full(4, 7, dtype=np.uint32)
    rc = lib.bnm_infer_windows_device_f32(None, None, 32, 32, 32, 16, 16, None, C.c_void_p(labels.ctypes.data), None)
    assert rc == -2 and b"no CUDA device" in lib.bnm_last_error()
    assert (labels == 7).all()


def test_window_kernel_has_no_local_memory(built):
    funcs = {k: v for k, v in sass_functions().items() if "k_quantize_windows" in k}
    assert len(funcs) == 1, list(funcs)
    for name, text in funcs.items():
        assert not local_memory(instructions(text)), name


# ---- GPU ---------------------------------------------------------------------------------------------------------------------

def _engine(name):
    from bitnetmcu_b200.engine import Engine
    m = load_model(name) if isinstance(name, str) else name
    return Engine(m, device=0, nf4_extension=(name == "rand_nf4_64"))


def run_windows(e, image, stride, logits=True, labels=True, stream=None):
    """the window entry on a CUDA plane -> (logits [out_h*out_w, C], labels [out_h*out_w]) as NumPy (None when not asked)"""
    import torch
    from bitnetmcu_b200.engine import window_grid
    oh, ow = window_grid(image.shape[0], image.shape[1], stride)
    lo = torch.full((oh, ow, e.n_classes), LOGIT_SENTINEL, dtype=torch.int32, device="cuda") if logits else None
    la = torch.full((oh, ow), LABEL_SENTINEL, dtype=torch.int32, device="cuda") if labels else None
    e.infer_windows_device(image, stride, lo, la, stream=stream)
    torch.cuda.synchronize()
    return (lo.reshape(-1, e.n_classes).cpu().numpy() if logits else None), (la.reshape(-1).cpu().numpy() if labels else None)


def run_f32(e, rows):
    """bnm_infer_batch_device_f32 on float rows [n, 256] (CUDA) -> (logits, labels) as NumPy"""
    import torch
    n = rows.shape[0]
    lo = torch.empty((n, e.n_classes), dtype=torch.int32, device="cuda")
    la = torch.empty((n,), dtype=torch.int32, device="cuda")
    if n:
        e.infer_device_f32(rows.contiguous(), lo, la)
    torch.cuda.synchronize()
    return lo.cpu().numpy(), la.cpu().numpy()


def torch_windows(image, sy, sx):
    """the torch extraction a caller makes today: float32 [out_h * out_w, 256] on the image's device"""
    return image.unfold(0, 16, sy).unfold(1, 16, sx).reshape(-1, 256)


def assert_same(got, want, what):
    for g, w, k in zip(got, want, ("logits", "labels")):
        bad = np.flatnonzero((g != w).reshape(len(w), -1).any(axis=1))
        assert bad.size == 0, (what, k, f"{bad.size} of {len(w)} windows differ, first {bad[:6].tolist()}")


@pytest.mark.gpu
@pytest.mark.parametrize("name", MODELS)
def test_windows_equal_the_f32_entry(lib, name):
    import torch
    e = _engine(name)
    for h, w in PAGES:
        page = plane(page_np(h, w, seed=h * 1000 + w))
        for sy, sx in STRIDES:
            got = run_windows(e, page, (sy, sx))
            want = run_f32(e, torch_windows(page, sy, sx))
            assert got[1].size == want[1].size == len(range(0, h - 15, sy)) * len(range(0, w - 15, sx))
            assert_same(got, want, (name, (h, w), (sy, sx)))
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["fc", "binary160", "cnn_letters", "rand_nf4_64"])
def test_windows_equal_the_oracle(lib, oracle, name):
    import torch
    from bitnetmcu_b200.engine import quantize_images
    e = _engine(name)
    page = page_np(45, 61, seed=9)
    for sy, sx in [(1, 1), (3, 2)]:
        got = run_windows(e, plane(page), (sy, sx))
        q = quantize_images(windows_np(page, sy, sx))
        want = oracle.infer(e.model, q, nf4_extension=(name == "rand_nf4_64"))
        assert_same(got, (want[0], want[1].astype(np.int32)), (name, "oracle", (sy, sx)))
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["fc", "binary160", "cnn_48"])
def test_only_the_window_pixels_count(lib, name):
    """the page inside a larger allocation whose pitch padding and rows past the page hold 1e30: the same results as the clean
    page (a box or a sliding max that reached past a window would see them)"""
    import torch
    e = _engine(name)
    for h, w in [(37, 53), (300, 520), (50, 18)]:
        page = plane(page_np(h, w, seed=w))
        pitch = (w + 3) // 4 * 4 + 8
        big = torch.full((h + 9, pitch), 1e30, dtype=torch.float32, device="cuda")
        big[:h, :w] = page
        view = big[:h, :w]
        assert view.stride(0) == pitch
        for stride in STRIDES:
            assert_same(run_windows(e, view, stride), run_windows(e, page, stride), (name, (h, w), stride, "padded"))
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["fc", "binary160", "cnn_48"])
def test_scaling_edges(lib, name):
    """windows that are all zero, all negative, hold +-1e30, subnormals or -0.0: the f32 entry's results"""
    import torch
    x = page_np(96, 96, seed=3)
    x[0:24, 0:24] = 0.0
    x[0:24, 30:60] = -np.abs(x[0:24, 30:60]) - np.float32(0.5)
    x[30:34, 5] = np.float32(1e30)
    x[40, 40] = np.float32(-1e30)
    x[50:80, 50:80] = np.float32(1e-40) * np.sign(x[50:80, 50:80])      # subnormals (and their signs)
    x[60:90, 0:30] = np.float32(-0.0)
    x[62, 3] = np.float32(2e-45)
    x[70:72, 10:12] = np.float32(0.5) / np.float32(127.0) * np.arange(4, dtype=np.float32).reshape(2, 2)   # .5 ties after scaling
    e = _engine(name)
    page = plane(x)
    for sy, sx in [(1, 1), (2, 3), (16, 16)]:
        assert_same(run_windows(e, page, (sy, sx)), run_f32(e, torch_windows(page, sy, sx)), (name, "edges", (sy, sx)))
    e.close()


@pytest.mark.gpu
def test_several_passes_and_partial_tiles(lib):
    """2^22 windows (four passes of 2^20, every CTA of the FC kernel on several tiles), then grids of window counts that are not a
    multiple of 128"""
    import torch
    e = _engine("fc")
    page = plane(page_np(2063, 2063, seed=22))
    got = run_windows(e, page, 1)
    assert got[1].size == 1 << 22
    for r0 in range(0, 2048, 512):   # the reference in slices of window rows: 512 x 2048 windows each
        want = run_f32(e, torch_windows(page[r0:r0 + 512 + 15], 1, 1))
        sl = slice(r0 * 2048, (r0 + 512) * 2048)
        assert_same((got[0][sl], got[1][sl]), want, ("2^22", r0))
    for h, w, s in [(16, 16 + 128, 1), (16 + 128, 16, 1), (47, 29, (2, 1)), (19, 1000, 3)]:
        p = plane(page_np(h, w, seed=h + w))
        assert_same(run_windows(e, p, s), run_f32(e, torch_windows(p, *((s, s) if isinstance(s, int) else s))), ("partial", h, w, s))
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["binary160", "fc"])
def test_pass_boundaries_inside_a_window_row(lib, name):
    """out_w = 2047, which does not divide the 2^20-window pass: a scaling CTA's run of windows straddles each pass boundary, and
    only its part in the pass is written"""
    e = _engine(name)
    page = plane(page_np(16 + 1100, 2062, seed=31))
    got = run_windows(e, page, 1)
    assert got[1].size == 1101 * 2047 > 2 * (1 << 20)
    for r0 in range(0, 1101, 367):
        want = run_f32(e, torch_windows(page[r0:r0 + 367 + 15], 1, 1))
        sl = slice(r0 * 2047, (r0 + 367) * 2047)
        assert_same((got[0][sl], got[1][sl]), want, (name, "pass boundary", r0))
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["fc", "cnn_letters", "binary160"])
def test_labels_only_and_logits_only(lib, name):
    import torch
    e = _engine(name)
    page = plane(page_np(70, 90, seed=1))
    both = run_windows(e, page, (1, 2))
    assert np.array_equal(run_windows(e, page, (1, 2), logits=False)[1], both[1])
    assert np.array_equal(run_windows(e, page, (1, 2), labels=False)[0], both[0])
    e.close()


@pytest.mark.gpu
def test_routes_name_the_window_kernel(lib, capfd, monkeypatch):
    import torch
    from bitnetmcu_b200 import _lib
    page = plane(page_np(40, 40, seed=2))
    cases = [("fc", load_model("fc"), 0), ("37 classes", random_fc(4, (256, 64, 64, 37), 2), 0),
             ("binary160", load_model("binary160"), 0), ("cnn_48", load_model("cnn_48"), 0), ("layers", load_model("fc"), _lib.PATH_LAYERS)]
    for what, m, path in cases:
        e, _ = verbose_engine(capfd, monkeypatch, lambda: _engine(m))
        if path:
            e.set_option(_lib.OPT_PATH, path)
        capfd.readouterr()
        run_windows(e, page, 3)
        lines = [l for l in capfd.readouterr().err.splitlines() if "windows route: " in l]
        assert len(lines) == 1, (what, lines)
        r = lines[0].split("windows route: bnm_infer_windows_device_f32: ")[1]
        assert r.startswith("k_quantize_windows + "), (what, r)
        assert ("layer by layer" in r) == (path == _lib.PATH_LAYERS), (what, r)
        assert ("k_cnn_frontend" in r) == (what == "cnn_48"), (what, r)
        e.close()


@pytest.mark.gpu
def test_argument_errors(lib):
    import torch
    e = _engine("fc")
    f = lib.bnm_infer_windows_device_f32
    page = torch.zeros((64, 64), dtype=torch.float32, device="cuda")
    lo = torch.full((49 * 49 * 10 + 8,), LOGIT_SENTINEL, dtype=torch.int32, device="cuda")
    la = torch.full((49 * 49 + 8,), LABEL_SENTINEL, dtype=torch.int32, device="cuda")
    P = lambda t, off=0: C.c_void_p(t.data_ptr() + off)
    call = lambda img, h, w, pitch, sy, sx, lg, lb: f(e.handle, img, h, w, pitch, sy, sx, lg, lb, None)
    cases = {
        "zero stride y": call(P(page), 64, 64, 64, 0, 1, P(lo), P(la)),
        "zero stride x": call(P(page), 64, 64, 64, 1, 0, P(lo), P(la)),
        "pitch < width": call(P(page), 64, 64, 60, 1, 1, P(lo), P(la)),
        "pitch % 4": call(P(page), 32, 62, 63, 1, 1, P(lo), P(la)),
        "image misaligned": call(P(page, 4), 32, 32, 64, 1, 1, P(lo), P(la)),
        "logits misaligned": call(P(page), 32, 32, 64, 1, 1, P(lo, 4), P(la)),
        "no output": call(P(page), 32, 32, 64, 1, 1, None, None),
        "null image": call(None, 32, 32, 64, 1, 1, P(lo), P(la)),
    }
    assert cases == {k: -1 for k in cases}, cases
    wide = _engine(random_fc(4, (512, 64, 64, 10), 1))
    assert f(wide.handle, P(page), 64, 64, 64, 1, 1, P(lo), P(la), None) == -3
    assert b"16x16" in lib.bnm_last_error()
    wide.close()
    for h, w in [(15, 64), (64, 15), (0, 0)]:
        assert call(P(page), h, w, 64, 1, 1, P(lo), P(la)) == 0
    torch.cuda.synchronize()
    assert (lo == LOGIT_SENTINEL).all() and (la == LABEL_SENTINEL).all()
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["fc", "cnn_48", "binary160"])
def test_graph_replay_and_two_streams(lib, name):
    import torch
    e = _engine(name)
    h, w, stride = 300, 200, (2, 1)
    oh, ow = (h - 16) // 2 + 1, w - 15
    page = plane(page_np(h, w, seed=4))
    lo = torch.empty((oh, ow, e.n_classes), dtype=torch.int32, device="cuda")
    la = torch.empty((oh, ow), dtype=torch.int32, device="cuda")
    e.infer_windows_device(page, stride, lo, la)   # warm: the pool and the kernels' attributes
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    with torch.cuda.graph(g, stream=s):
        e.infer_windows_device(page, stride, lo, la)
    page.copy_(torch.from_numpy(page_np(h, w, seed=5)))
    g.replay()
    torch.cuda.synchronize()
    want = run_windows(e, page, stride)
    assert_same((lo.reshape(-1, e.n_classes).cpu().numpy(), la.reshape(-1).cpu().numpy()), want, (name, "replay"))
    del g
    # two pages on two streams at once
    pages = [plane(page_np(h, w, seed=10 + k)) for k in range(2)]
    alone = [run_windows(e, p, stride) for p in pages]
    outs = [(torch.empty_like(lo), torch.empty_like(la)) for _ in range(2)]
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    torch.cuda.synchronize()
    for _ in range(3):
        for p, (o1, o2), st in zip(pages, outs, streams):
            with torch.cuda.stream(st):
                e.infer_windows_device(p, stride, o1, o2)
    torch.cuda.synchronize()
    for k, (o1, o2) in enumerate(outs):
        assert_same((o1.reshape(-1, e.n_classes).cpu().numpy(), o2.reshape(-1).cpu().numpy()), alone[k], (name, "stream", k))
    e.close()


@pytest.mark.gpu
def test_mode2_int8_launch_after_a_window_launch_waits(lib, oracle, capfd, monkeypatch):
    """in mode 2, two int8 launches on disjoint buffers are independent; a window call in between is a launch of another kind:
    its own fused launch and the int8 launch after it keep their wait, and every result is right"""
    import torch
    from bitnetmcu_b200 import _lib
    e, _ = verbose_engine(capfd, monkeypatch, lambda: _engine("fc"))
    e.set_option(_lib.OPT_LAUNCH_OVERLAP, 2)
    rng = np.random.default_rng(8)
    xs = [rng.integers(-128, 128, size=(148 * 128 * 2 + 77, 256)).astype(np.int8) for _ in range(2)]
    wants = [oracle.infer(e.model, x) for x in xs]
    d_x = [torch.from_numpy(x).cuda() for x in xs]
    outs = [(torch.empty((x.shape[0], 10), dtype=torch.int32, device="cuda"), torch.empty(x.shape[0], dtype=torch.int32, device="cuda")) for x in xs]
    page = plane(page_np(400, 300, seed=6))
    wlo = torch.empty((385, 285, 10), dtype=torch.int32, device="cuda")
    wla = torch.empty((385, 285), dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    capfd.readouterr()
    e.infer_device(d_x[0], *outs[0])
    e.infer_device(d_x[1], *outs[1])
    e.infer_windows_device(page, 1, wlo, wla)
    e.infer_device(d_x[0], *outs[0])
    torch.cuda.synchronize()
    got = [l.split("fused launch: ")[1] for l in capfd.readouterr().err.splitlines() if "fused launch: " in l]
    assert got == ["wait", "independent", "wait", "wait"], got
    for (lo, la), (wl, wb) in zip(outs, wants):
        assert np.array_equal(lo.cpu().numpy(), wl) and np.array_equal(la.cpu().numpy().astype(np.uint32), wb)
    assert_same((wlo.reshape(-1, 10).cpu().numpy(), wla.reshape(-1).cpu().numpy()), run_f32(e, torch_windows(page, 1, 1)), "mode 2 windows")
    e.close()
