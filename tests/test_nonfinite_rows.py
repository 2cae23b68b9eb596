"""Rows holding NaN or infinity through the input scaling of every float entry and route (include/bitnetmcu_b200.h sections 5,
9, 11 and 12).

The reference caller scales a row with NumPy (test_inference.py:140-145): scale = 127 / max(max|x|, 1e-5), then
round(x * scale).clip(-128, 127) in float32 and .astype(np.int8).  On a row with any non-finite element that is the all-zero
int8 row: max and np.maximum carry a NaN into the scale, an infinity makes the scale 0 (inf * 0 is NaN, any finite pixel +-0),
and NaN casts to 0.  The CPU tests pin restate.scale_images to that literal expression on crafted float32, float16 and bfloat16
rows.  The GPU tests (tolerance 0, sentinel-filled outputs) place such rows among finite ones -- the first and last row, every
position of a 128-row tile, past the first trip round the fused kernels' tile ring -- and check:

* the scaling entries (bnm_quantize_images, _device, _device_f16): the restated int8 rows;
* the C engine's float entries (logits, labels, top-k, both engines' labels and counts) on the fused one-kernel forms, the
  scaling kernel followed by the int8 form, BNM_PATH_LAYERS and both CNN front-ends: the oracle on the restated rows;
* the emulator's entries on the same routes: restate.emulate, which gives a poisoned row the emulator's result on the zero row,
  logits all 0.0 and label 0.  The reference emulator itself carries the NaN into its logits, and np.argmax of an all-NaN row
  is 0; the label agrees, the logits deliberately do not (the engine writes no NaN logits);
* the window entries: every window covering a NaN or infinite pixel is the zero row's result, and the windows beside it, one
  pixel away in either direction at strides 1, 2 and 16, are those of the clean page.

Every route is asserted through its BNM_VERBOSE route line or plan line, so a case cannot silently run another route."""
import numpy as np
import pytest

from conftest import load_model
from restate import TILE, emulate, scale_images
from support import engine, frontends, lib, random_fc, route, scattered_edge_images, top_k, verbose_engine  # noqa: F401 (lib: fixture)

FORMATS = ["float32", "float16", "bfloat16"]
U_FINITE = 389                      # distinct finite rows of a batch
SENTINEL = -7
F32_SNAN, F32_NEG_SNAN, F32_NAN_PAYLOAD = 0x7F800001, 0xFF800001, 0x7FC12345
HALF_NAN = {"float16": (0x7E00, 0xFE00, 0x7C01, 0xFC01, 0x7D55), "bfloat16": (0x7FC0, 0xFFC0, 0x7F81, 0xFF81, 0x7FAA)}


# ---- rows ---------------------------------------------------------------------------------------------------------------------

def _bits32(u):
    return np.uint32(u).view(np.float32)


def crafted_rows(d, seed=0):
    """float32 rows [k, d] that each hold a NaN or an infinity (float16 also overflows 1e5 to inf): both NaN signs, signalling and
    payload NaN, +-inf, in lane 0, the last lane and the last 4-element group, all-NaN and all-inf rows, and rows whose finite
    maximum is below the 1e-5 floor or zero"""
    rng = np.random.default_rng(seed)
    base = lambda: rng.standard_normal(d).astype(np.float32)
    rows = []

    def put(r, at, v):
        r = r.copy()
        r[at] = v
        rows.append(r)
    for v in (np.float32(np.nan), -np.float32(np.nan), _bits32(F32_SNAN), _bits32(F32_NEG_SNAN), _bits32(F32_NAN_PAYLOAD),
              np.float32(np.inf), -np.float32(np.inf)):
        put(base(), int(rng.integers(0, d)), v)
        put(base(), d - 1, v)                          # the last lane
        put(base(), d - 3, v)                          # inside the last 4-element group
        put(base(), 0, v)
    put(base(), [0, d - 1], [np.inf, np.nan])         # both kinds
    rows.append(np.full(d, np.nan, dtype=np.float32))
    rows.append(np.full(d, -np.inf, dtype=np.float32))
    tiny = (rng.uniform(-1, 1, d) * 3e-6).astype(np.float32)   # the finite maximum below the 1e-5 floor
    put(tiny, d // 2, np.nan)
    put(tiny, d - 1, -np.inf)
    put(np.zeros(d, dtype=np.float32), 5, np.nan)      # the finite maximum 0
    put(np.zeros(d, dtype=np.float32), d - 2, np.inf)
    put(base() * np.float32(1e4), d - 1, np.float32(1e5))   # finite in float32 and bfloat16, inf in float16
    return np.stack(rows)


def to_format(x, fmt, nan_rows=True):
    """float32 rows -> (16-bit patterns uint16 or None, the rows the kernels see: float32, or the 16-bit values widened).  The
    16-bit rows round to nearest even, as torch converts; with nan_rows, rows 0 .. 4 (crafted rows wherever this is used) then
    get one explicit NaN pattern each: both signs, signalling, payload."""
    if fmt == "float32":
        return None, np.ascontiguousarray(x, dtype=np.float32)
    import torch
    bits = torch.from_numpy(np.ascontiguousarray(x)).to(getattr(torch, fmt)).view(torch.int16).numpy().view(np.uint16).copy()
    d = bits.shape[1]
    for i, b in enumerate(HALF_NAN[fmt] if nan_rows else ()):
        bits[i, [i % d, d - 1][i % 2]] = b
    return bits, widen(bits, fmt)


def widen(bits, fmt):
    """16-bit patterns -> float32: bfloat16 is the top half of a float32; float16 as NumPy widens np.float16"""
    if fmt == "bfloat16":
        return (bits.astype(np.uint32) << 16).view(np.float32)
    return bits.view(np.float16).astype(np.float32)


def literal(x):
    """test_inference.py:140-145 as written, .astype(np.int8) included"""
    with np.errstate(invalid="ignore", over="ignore"):
        scale = 127.0 / np.maximum(np.abs(x).max(axis=-1, keepdims=True), 1e-5)
        return np.round(x * scale).clip(-128, 127).astype(np.int8)


class Batch:
    """U distinct rows (the crafted ones first, then finite ones) and a batch of n rows drawn from them: row i is base[idx[i]].
    Poisoned rows sit at row 0, row n - 1 and every 129th row (129 j is position j % 128 of its tile: every position of a tile,
    in tiles all through the batch); the other rows cycle through the finite ones."""

    def __init__(self, n, d, seed=0):
        self.crafted = crafted_rows(d, seed)
        k = len(self.crafted)
        self.base = np.concatenate([self.crafted, scattered_edge_images(U_FINITE, d, seed + 1)])
        self.idx = k + np.arange(n) % U_FINITE
        pos = sorted(set(range(0, n, 129)) | {0, n - 1}) if n else []
        self.idx[pos] = np.arange(len(pos)) % k
        self.n, self.d = n, d

    def rows(self, fmt):
        """(device images of fmt [n, d], the float32 rows the kernels see [U, d])"""
        import torch
        bits, seen = to_format(self.base, fmt)
        dev_idx = torch.from_numpy(self.idx).cuda()
        if bits is None:
            x = torch.from_numpy(seen).cuda()
        else:
            x = torch.from_numpy(bits.view(np.int16)).cuda().view(getattr(torch, fmt))
        return x[dev_idx].contiguous(), seen

    def poisoned(self, seen):
        return ~np.isfinite(seen).all(axis=1)


# ---- CPU ----------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("d", [256, 100, 16])
def test_restatement_is_the_reference_expression(fmt, d):
    """restate.scale_images equals the reference caller's literal expression on the crafted rows and finite ones, widened from
    float16 / bfloat16 where asked, and every row holding a NaN or an infinity is the all-zero row"""
    k = len(crafted_rows(d))
    x = np.concatenate([crafted_rows(d), scattered_edge_images(64, d, 3)])
    bits, seen = to_format(x, fmt)
    got = scale_images(seen)
    assert np.array_equal(got, literal(seen))
    bad = ~np.isfinite(seen).all(axis=1)
    assert not got[bad].any()
    assert bad[:k - 1].all() and bad[k - 1] == (fmt == "float16")   # 1e5 overflows float16 only
    assert got[~bad].any(axis=1).mean() > 0.5                         # the finite rows are there too
    assert np.isnan(seen).any(axis=1).sum() >= 20 and np.isinf(seen).any(axis=1).sum() >= 10
    if bits is not None:
        assert {int(b) for b in bits.ravel()} >= set(HALF_NAN[fmt])


def test_the_one_sentence_rule():
    """the table of the two cases that tell the rules apart, and a NaN next to the floor"""
    x = np.array([[np.nan, 1, 2], [np.inf, 1, -3], [-np.inf, 0, 0], [np.nan, 1e-6, 0], [1, 2, 4]], dtype=np.float32)
    assert scale_images(x).tolist() == [[0, 0, 0], [0, 0, 0], [0, 0, 0], [0, 0, 0], [32, 64, 127]]
    assert np.array_equal(scale_images(x), literal(x))


def test_batch_layout():
    """poisoned rows at the first and last row and at every position of a tile, past the first ring round"""
    b = Batch(5 * 132 * TILE + 77, 256)
    seen = b.base
    p = np.flatnonzero(~np.isfinite(seen[b.idx]).all(axis=1))
    assert p[0] == 0 and p[-1] == b.n - 1
    assert set((p % TILE).tolist()) == set(range(TILE))
    assert (p // TILE).max() > 4 * 132


# ---- GPU: scaling and batch entries -------------------------------------------------------------------------------------------

def _ring_n():
    """past the first trip round every float-input form's ring: five tiles per CTA plus a ragged tile"""
    import torch
    return 5 * torch.cuda.get_device_properties(0).multi_processor_count * TILE + 77


def _eq(got, want, what):
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    same = (got == want).reshape(len(want), -1).all(axis=1)
    bad = np.flatnonzero(~same)
    assert bad.size == 0, (what, f"{bad.size} of {len(want)} rows differ, first {bad[:6].tolist()}")


def _full(shape, dtype, fill):
    import torch
    return torch.full(shape, fill, dtype=dtype, device="cuda")


@pytest.mark.gpu
@pytest.mark.parametrize("d", [256, 100, 784])
def test_scaling_entries(lib, d):
    """bnm_quantize_images (host, float32), bnm_quantize_images_device and _device_f16: the restated int8 rows"""
    import torch
    from bitnetmcu_b200 import engine as E
    b = Batch(_ring_n() if d == 256 else 3000, d, seed=d)
    for fmt in FORMATS:
        x, seen = b.rows(fmt)
        want = scale_images(seen)[b.idx]
        assert not want[b.poisoned(seen)[b.idx]].any()
        q = _full(x.shape, torch.int8, 99)
        E.quantize_images_device(x, q)
        torch.cuda.synchronize()
        _eq(q.cpu().numpy(), want, (fmt, d, "device"))
        if fmt == "float32":
            _eq(E.quantize_images(x.cpu().numpy()), want, (d, "host"))


# route case -> (model, path, CNN front-end, the emulator route line at creation (the default path's; None on BNM_PATH_LAYERS,
# whose routes the top-k lines name per call), the start of the C engine's float top-k route line)
def _route_cases():
    from bitnetmcu_b200 import _lib
    return {
        "fused": ("fc", 0, None, "fc_emul_kernel<64,1,float,emul>", "k_quantize_images + fc_topk_kernel<64,"),
        "scaling, 37 classes": ("fc37", 0, None, "k_quantize_images + fc_emul_i8_kernel<64,1,emul>", "k_quantize_images + fc_topk_kernel<64,"),
        "scaling, binary160": ("binary160", 0, None, "k_quantize_images + fc_emul_i8_kernel<192,1,emul>", "k_quantize_images + fc_topk_kernel<192,"),
        "layers": ("fc", _lib.PATH_LAYERS, None, None, "k_quantize_images + layer by layer + k_topk_rows<int32>"),
        "cnn, front-end 1": ("cnn_48", 0, _lib.CNN_CUDA_CORES, "k_cnn_emul_frontend + fc_emul_i8_kernel<128,1,emul>",
                             "k_quantize_images + k_cnn_frontend16 + fc_topk_kernel<"),
        "cnn, front-end 2": ("cnn_48", 0, _lib.CNN_TENSOR_CORES, "k_cnn_emul_frontend + fc_emul_i8_kernel<128,1,emul>",
                             "k_quantize_images + k_cnn_frontend16_tc + fc_topk_kernel<"),
        "cnn, layers": ("cnn_48", _lib.PATH_LAYERS, None, None, "k_quantize_images + k_cnn_frontend16"),
    }


ROUTES = ["fused", "scaling, 37 classes", "scaling, binary160", "layers", "cnn, front-end 1", "cnn, front-end 2", "cnn, layers"]


def _model(name):
    return random_fc(4, (256, 64, 64, 37), 2) if name == "fc37" else load_model(name)


def _route_engine(capfd, monkeypatch, case):
    """the case's engine with BNM_VERBOSE, its creation lines checked: the path, and on the default path the plan's float-input
    forms (on the fused case only) and the emulator route"""
    from bitnetmcu_b200 import _lib
    name, path, fe, emul_route, _ = _route_cases()[case]
    m = _model(name)
    e, err = verbose_engine(capfd, monkeypatch, lambda: engine(m, path=path, cnn_frontend=fe))
    assert e.active_path == (_lib.PATH_LAYERS if path == _lib.PATH_LAYERS else _lib.PATH_TCGEN05), (case, err)
    if emul_route is not None:
        assert any("float input <64,1,float>" in l for l in err) == (case == "fused"), (case, err)
        assert route(err, "emulator") == emul_route, (case, err)
    if fe is not None:
        assert fe in frontends(m), case
    return e, m


def _topk_line(capfd, call, entry):
    """the `topk route:` line one top-k call prints"""
    import torch
    torch.cuda.synchronize()
    capfd.readouterr()
    call()
    torch.cuda.synchronize()
    lines = [l for l in capfd.readouterr().err.splitlines() if "topk route: " in l]
    assert len(lines) == 1, (entry, lines)
    assert f"topk route: {entry}: " in lines[0], (entry, lines)
    return lines[0].split(f"topk route: {entry}: ")[1]


def _scale_name(fmt):
    return "k_quantize_images" if fmt == "float32" else f"k_quantize_images<{fmt}>"


@pytest.mark.gpu
@pytest.mark.parametrize("case", ROUTES)
def test_c_engine_routes(lib, oracle, capfd, monkeypatch, case):
    """bnm_infer_batch_device_f32 / _f16 (logits and labels, labels only), the top-k entries (k = 1 and 5, with and without
    scores) and bnm_compare_engines_device / _f16 (both labels, the counts over a truth vector): the oracle on the restated rows,
    the emulator's labels those of restate.emulate"""
    import torch
    e, m = _route_engine(capfd, monkeypatch, case)
    want_topk_route = _route_cases()[case][4]
    C = m.n_classes
    b = Batch(_ring_n(), m.img_bytes, seed=len(case))
    n, idx = b.n, b.idx
    for fmt in FORMATS:
        x, seen = b.rows(fmt)
        poisoned = b.poisoned(seen)
        assert poisoned[idx].sum() >= TILE, (case, fmt)
        q = scale_images(seen)
        lo, la = oracle.infer(m, q)
        zlo, zla = oracle.infer(m, np.zeros((1, m.img_bytes), dtype=np.int8))
        assert (lo[poisoned] == zlo).all() and (la[poisoned] == zla[0]).all()
        py = np.argmax(emulate(m, seen), axis=1)
        assert (py[poisoned] == 0).all()
        want_lo, want_la, want_py = lo[idx], la[idx].astype(np.int32), py[idx].astype(np.int32)
        tag = (case, fmt)

        glo, gla = _full((n, C), torch.int32, SENTINEL), _full((n,), torch.int32, SENTINEL)
        e.infer_device_f32(x, glo, gla)
        only = _full((n,), torch.int32, SENTINEL)
        e.infer_device_f32(x, None, only)
        torch.cuda.synchronize()
        _eq(glo.cpu().numpy(), want_lo, tag + ("logits",))
        _eq(gla.cpu().numpy(), want_la, tag + ("labels",))
        _eq(only.cpu().numpy(), want_la, tag + ("labels only",))

        for k in (1, min(5, C)):
            wc, ws = top_k(want_lo, k)
            for scores in (True, False):
                cl = _full((n, k), torch.int32, SENTINEL)
                sc = _full((n, k), torch.int32, SENTINEL) if scores else None
                entry = "bnm_infer_topk_device_f32" if fmt == "float32" else "bnm_infer_topk_device_f16"
                line = _topk_line(capfd, lambda: e.topk_device_f32(x, k, cl, sc), entry)
                assert line.startswith(want_topk_route.replace("k_quantize_images", _scale_name(fmt), 1)), (tag, line)
                _eq(cl.cpu().numpy(), wc, tag + ("top-k classes", k, scores))
                if scores:
                    _eq(sc.cpu().numpy(), ws, tag + ("top-k scores", k))

        truth = torch.from_numpy((np.arange(n) * 7 % (C + 1)).astype(np.int32)).cuda()
        lc, lp = _full((n,), torch.int32, SENTINEL), _full((n,), torch.int32, SENTINEL)
        counts = torch.zeros(4, dtype=torch.int64, device="cuda")
        e.compare_engines_device(x, truth, lc, lp, counts)
        torch.cuda.synchronize()
        _eq(lc.cpu().numpy(), want_la, tag + ("engines: C labels",))
        _eq(lp.cpu().numpy(), want_py, tag + ("engines: emulator labels",))
        t = truth.cpu().numpy()
        assert counts.cpu().tolist() == [n, int((want_la == t).sum()), int((want_py == t).sum()), int((want_la != want_py).sum())], tag
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["fused", "scaling, binary160", "layers", "cnn, front-end 1", "cnn, layers"])
def test_emulator_routes(lib, capfd, monkeypatch, case):
    """bnm_emulate_batch_device / _f16 (logits and labels), bnm_emulate_inference_quantized (host) and bnm_emulate_topk_device /
    _f16: restate.emulate, whose poisoned rows are the zero row's -- logits all 0.0, label 0"""
    import torch
    e, m = _route_engine(capfd, monkeypatch, case)
    C = m.n_classes
    b = Batch(_ring_n(), m.img_bytes, seed=len(case) + 1)
    n, idx = b.n, b.idx
    for fmt in FORMATS:
        x, seen = b.rows(fmt)
        poisoned = b.poisoned(seen)
        want = emulate(m, seen)
        assert (want[poisoned] == 0.0).all()
        assert (np.argmax(want, axis=1)[poisoned] == 0).all()
        want_lo, want_la = want[idx], np.argmax(want, axis=1).astype(np.int32)[idx]
        tag = (case, fmt)
        lo, la = _full((n, C), torch.float64, -12345.5), _full((n,), torch.int32, SENTINEL)
        e.inference_quantized_device(x, lo, la)
        torch.cuda.synchronize()
        _eq(lo.cpu().numpy(), want_lo, tag + ("emulator logits",))
        _eq(la.cpu().numpy(), want_la, tag + ("emulator labels",))
        if fmt == "float32":
            _eq(e.inference_quantized(x.cpu().numpy()), want_lo, tag + ("host emulator logits",))
        k = min(5, C)
        wc, ws = top_k(want_lo, k)
        cl, sc = _full((n, k), torch.int32, SENTINEL), _full((n, k), torch.float64, -12345.5)
        entry = "bnm_emulate_topk_device" if fmt == "float32" else "bnm_emulate_topk_device_f16"
        line = _topk_line(capfd, lambda: e.emulate_topk_device(x, k, cl, sc), entry)
        if case in ("layers", "cnn, layers"):
            assert line == "layer by layer + k_topk_rows<double>", (tag, line)
        elif case.startswith("cnn"):
            want_line = "k_cnn_emul_frontend + " if fmt == "float32" else f"{_scale_name(fmt)} + k_cnn_emul_frontend_i8 + "
            assert line.startswith(want_line), (tag, line)
        else:
            assert line.startswith(_scale_name(fmt) + " + fc_topk_kernel<"), (tag, line)
        _eq(cl.cpu().numpy(), wc, tag + ("emulator top-k classes",))
        _eq(sc.cpu().numpy(), ws, tag + ("emulator top-k scores",))
    e.close()


# ---- GPU: windows -------------------------------------------------------------------------------------------------------------

H = W = 64
STRIDES = [(1, 1), (2, 2), (16, 16), (2, 16)]
# one non-finite pixel per poisoned plane (plane 0 is clean): rows and columns 31 and 32, so at every stride some window ends one
# pixel before the pixel and some starts one pixel after it, in both directions; the last plane's 1e5 is inf in float16 only
PIXELS = [(31, 31, np.nan), (32, 32, -np.inf), (31, 32, np.inf), (32, 31, _bits32(F32_SNAN)), (17, 47, np.float32(1e5))]


def _pages(fmt):
    """the stack [1 + len(PIXELS), H, W] of fmt on the device and the float32 planes the kernels see"""
    import torch
    rng = np.random.default_rng(5)
    clean = rng.standard_normal((H, W)).astype(np.float32)
    clean[:, :8] *= np.float32(1e-3)
    planes = np.stack([clean] + [clean.copy() for _ in PIXELS])
    for p, (y, x, v) in enumerate(PIXELS, 1):
        planes[p, y, x] = v
    bits, seen = to_format(planes.reshape(-1, W), fmt, nan_rows=False)
    if bits is None:
        return torch.from_numpy(planes).cuda(), planes
    bits = bits.reshape(planes.shape)
    bits[4, 32, 31] = HALF_NAN[fmt][2]   # plane 4's NaN as the format's signalling NaN
    return torch.from_numpy(bits.view(np.int16)).cuda().view(getattr(torch, fmt)), widen(bits, fmt)


def _window_masks(seen, sy, sx):
    """per plane and window [P, oh, ow]: covers a non-finite pixel; and the windows one pixel short of a poisoned plane's pixel,
    per direction"""
    P = seen.shape[0]
    oh, ow = (H - 16) // sy + 1, (W - 16) // sx + 1
    r0, c0 = np.arange(oh)[:, None] * sy, np.arange(ow)[None, :] * sx
    cover = np.zeros((P, oh, ow), dtype=bool)
    near = {k: np.zeros((P, oh, ow), dtype=bool) for k in ("above", "below", "left", "right")}
    for p in range(P):
        for y, x in zip(*np.nonzero(~np.isfinite(seen[p]))):
            iny, inx = (r0 <= y) & (y < r0 + 16), (c0 <= x) & (x < c0 + 16)
            cover[p] |= iny & inx
            near["above"][p] |= (r0 + 16 == y) & inx
            near["below"][p] |= (r0 == y + 1) & inx
            near["left"][p] |= iny & (c0 + 16 == x)
            near["right"][p] |= iny & (c0 == x + 1)
    return cover, near


def _run_windows(e, entry, pages, stride, k):
    """one stacked entry -> its two outputs [P, oh, ow, ...] as NumPy"""
    import torch
    from bitnetmcu_b200.engine import window_grid
    grid = (pages.shape[0],) + window_grid(H, W, stride)
    emul = entry.startswith("emulate")
    ldt, lfill = (torch.float64, -12345.5) if emul else (torch.int32, SENTINEL)
    if entry.endswith("topk"):
        a, b = _full(grid + (k,), torch.int32, SENTINEL), _full(grid + (k,), ldt, lfill)
        (e.emulate_windows_topk_device if emul else e.scan_windows_topk_device)(pages, stride, k, a, b)
    elif entry == "single":
        a, b = _full(grid + (e.n_classes,), ldt, lfill), _full(grid, torch.int32, SENTINEL)
        for p in range(pages.shape[0]):
            e.infer_windows_device(pages[p], stride, a[p], b[p])
    else:
        a, b = _full(grid + (e.n_classes,), ldt, lfill), _full(grid, torch.int32, SENTINEL)
        (e.emulate_windows_device if emul else e.scan_windows_device)(pages, stride, a, b)
    torch.cuda.synchronize()
    return a.cpu().numpy(), b.cpu().numpy()


WINDOW_ENTRIES = ["single", "scan", "scan_topk", "emulate", "emulate_topk"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["fc", "binary160", "cnn_48"])
def test_windows(lib, oracle, capfd, monkeypatch, name):
    """single page (bnm_infer_windows_device_f32, or the 16-bit scan on one plane) and stacked entries, C engine and emulator,
    float32 and 16-bit: a window covering a NaN or infinite pixel is the zero row's result; every other window, those one pixel
    away in each direction included, is the clean plane's; the clean plane's C-engine results are the oracle's"""
    m = load_model(name)
    e, _ = verbose_engine(capfd, monkeypatch, lambda: engine(m))
    C, k = m.n_classes, min(5, m.n_classes)
    zlo, zla = oracle.infer(m, np.zeros((1, 256), dtype=np.int8))
    zero = {"c": (zlo[0], int(zla[0])), "emul": (np.zeros(C), 0)}
    for fmt in FORMATS:
        pages, seen = _pages(fmt)
        assert (~np.isfinite(seen[-1])).any() == (fmt == "float16")
        for stride in STRIDES:
            cover, near = _window_masks(seen, *stride)
            assert all(v.any() for v in near.values()), (stride, {d: int(v.sum()) for d, v in near.items()})
            assert cover[1:len(PIXELS)].any(axis=(1, 2)).all() and not cover[0].any()
            planes = len(PIXELS) + (fmt == "float16")   # the last plane is another page where its pixel is finite
            cover, near = cover[:planes], {d: v[:planes] for d, v in near.items()}
            for entry in WINDOW_ENTRIES:
                tag = (name, fmt, stride, entry)
                capfd.readouterr()
                a, b = (t[:planes] for t in _run_windows(e, entry, pages, stride, k))
                lines = [l for l in capfd.readouterr().err.splitlines() if "windows route: " in l]
                assert lines and all(l.split(": ", 3)[-1].startswith("k_quantize_windows") for l in lines), (tag, lines)
                zlogit, zlabel = zero["emul" if entry.startswith("emulate") else "c"]
                if entry.endswith("topk"):
                    zc, zs = top_k(zlogit[None], k)
                    za, zb = zc[0], zs[0]
                else:
                    za, zb = zlogit, zlabel
                for got, z in ((a, za), (b, zb)):
                    assert (got[cover] == z).all(), (tag, "covering windows", int((got[cover] != z).any(axis=-1).sum()) if got.ndim > 3 else None)
                    clean = np.broadcast_to(got[0], got.shape)
                    _eq(got[~cover], clean[~cover], tag + ("windows off the pixel",))
                    for d, mask in near.items():
                        assert (got[mask] == clean[mask]).all(), (tag, d)
                if entry == "scan" and stride == (2, 16):
                    from numpy.lib.stride_tricks import sliding_window_view
                    wins = sliding_window_view(seen[0], (16, 16))[::stride[0], ::stride[1]].reshape(-1, 256)
                    lo, la = oracle.infer(m, scale_images(wins))
                    _eq(a[0].reshape(-1, C), lo, tag + ("clean plane vs oracle",))
    e.close()
