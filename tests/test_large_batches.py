"""Every inference route on batches whose byte offsets pass 2^31 and 2^32, and the split of a fused int8 batch into launches the
kernel takes.

Inputs are periodic: U = 8191 unique rows (an odd prime), and row i of a batch is unique row i mod U, built on the device by
index_select, so nothing of GB size crosses the host (but for the host entry's own case).  The expected result of a batch is
the same entry on the U unique rows, pinned to the oracle (the C engine) or to restate (scaling, the emulator) in the same
test, then tiled; the comparison runs on the device, in slices, and names the first rows that differ.  A window scan's pages
are periodic in both directions with period 89 instead, each plane at its own phase.

A 32-bit product anywhere in an offset would displace a read or a write by 2^31 or 2^32 bytes.  With U odd that lands on
another unique row: test_a_wrapped_offset_shows checks, on the CPU and for every case, that the expected result there
differs for most rows.  Every output buffer holds a sentinel, checked past row n; the input is checked unchanged.

Each case closes its engine (a model's scratch pool keeps what it took), frees its tensors, states the device memory it needs,
skips with that figure when the GPU has less free, and prints its n, peak device memory and wall time."""
import functools

import numpy as np
import pytest

from conftest import load_model
from restate import emulate, scale_images
from support import (WRAPS, GiB, P, SENTINEL_I32, SPARE, U, Case, Spec, check_input, check_tiled,  # noqa: F401
                     check_wrapped_offsets, lib, need, normal_images, outputs, periodic, random_fc, row_uid, verbose_engine, views,
                     want_on_device)
# (lib: a fixture)

PAGE = 4096                     # a window-scan page is PAGE x PAGE floats
N22, N23, N24, N25 = ((1 << b) + 77 for b in (22, 23, 24, 25))
K_FUSED_PASS = 1 << 28          # images per fused FC launch (kFusedPass, capi.cu)
N_GATHER = 2 * 148 * 128 + 77

MODELS = {
    "fc": lambda: load_model("fc"),                                 # 4bitsym-64, the fixed-shape row
    "head47": lambda: random_fc(16, (256, 64, 47), 47),             # 64-wide 8bit, 47 classes: the general two-pipe row
    "2bitsym96": lambda: load_model("2bitsym96"),                   # <128,1>
    "binary160": lambda: load_model("binary160"),                   # <192,1>
    "cnn_48": lambda: load_model("cnn_48"),
    "fc16": lambda: random_fc(16, (16, 16, 10), 16),                # 16-byte rows: a fused launch of 2^28 images is 4 GiB
}


@functools.lru_cache(maxsize=None)
def model(name):
    return MODELS[name]()


# ---- the unique rows and what every entry gives on them (CPU) -------------------------------------------------------------------

@functools.lru_cache(maxsize=None)
def rows_i8(name):
    m = model(name)
    return np.random.default_rng(len(name) * 1009 + m.img_bytes).integers(-128, 128, size=(U, m.img_bytes), dtype=np.int8)


@functools.lru_cache(maxsize=None)
def rows_f32(name):
    return normal_images(U, seed=len(name) * 7 + 3, elems=model(name).img_bytes)


@functools.lru_cache(maxsize=None)
def tile():
    """the P x P floats a window-scan page repeats"""
    return np.random.default_rng(89).standard_normal((P, P), dtype=np.float32)


def small_page():
    """(P + 15)^2 floats whose P^2 windows at stride 1 are the unique windows, window (y, x) unique window y P + x"""
    i = np.arange(P + 15) % P
    return np.ascontiguousarray(tile()[i][:, i])


def unique_windows():
    return np.lib.stride_tricks.sliding_window_view(small_page(), (16, 16)).reshape(P * P, 256)


def _topk(logits, k):
    order = np.argsort(-logits.astype(np.int64), axis=1, kind="stable")[:, :k]
    return {"classes": order.astype(np.uint32), "scores": np.take_along_axis(logits, order, axis=1)}


_EXPECTED = {}


def expected(oracle, kind, name):
    """what entry `kind` gives on the unique rows of model `name` (the unique windows for the window kinds): {output: NumPy
    [unique, ...]}.  C engine: the oracle on the int8 rows, or on the scaled float rows (f32); emulator: restate.emulate"""
    key = (kind, name)
    if key not in _EXPECTED:
        m = model(name)
        if kind == "c":
            lo, la = oracle.infer(m, rows_i8(name))
            r = {"logits": lo, "labels": la}
        elif kind == "topk":
            r = _topk(expected(oracle, "c", name)["logits"], 16)
        elif kind == "c_f32":
            lo, la = oracle.infer(m, scale_images(rows_f32(name)))
            r = {"logits": lo, "labels": la}
        elif kind == "emul":
            lo = emulate(m, rows_f32(name))
            r = {"logits": lo, "labels": np.argmax(lo, axis=1).astype(np.uint32)}
        elif kind == "engines":
            r = {"labels_c": expected(oracle, "c_f32", name)["labels"], "labels_py": expected(oracle, "emul", name)["labels"]}
        elif kind == "win":
            lo, la = oracle.infer(m, scale_images(unique_windows()))
            r = {"logits": lo, "labels": la}
        elif kind == "win_topk":
            r = _topk(expected(oracle, "win", name)["logits"], 16)
        elif kind == "win_emul":
            lo = emulate(m, unique_windows())
            r = {"logits": lo, "labels": np.argmax(lo, axis=1).astype(np.uint32)}
        _EXPECTED[key] = r
    return _EXPECTED[key]


def window_uid(rows):
    """the unique window of windows of a stack of pages at stride 1, plane p at phase (7 p, 3 p)"""
    per = (PAGE - 15) * (PAGE - 15)
    p, r = rows // per, rows % per
    return ((r // (PAGE - 15) + 7 * p) % P) * P + (r % (PAGE - 15) + 3 * p) % P


SPECS = {
    "int8 fc": Spec("c", "fc", N24, 256, ("logits", "labels")),
    "int8 fc labels only": Spec("c", "fc", N24, 256, ("labels",)),
    "int8 head47": Spec("c", "head47", N24, 256, ("logits", "labels")),
    "int8 2bitsym96": Spec("c", "2bitsym96", N24, 256, ("logits", "labels")),
    "int8 binary160": Spec("c", "binary160", N24, 256, ("logits", "labels")),
    "topk head47": Spec("topk", "head47", N25, 256, ("classes", "scores")),
    "f32 fc": Spec("c_f32", "fc", N22, 1024, ("logits", "labels")),
    "emulator fc": Spec("emul", "fc", N22, 1024, ("logits", "labels")),
    "engines fc": Spec("engines", "fc", N22, 1024, ("labels_c", "labels_py")),
    "f32 binary160": Spec("c_f32", "binary160", N22, 1024, ("logits", "labels")),
    "emulator head47": Spec("emul", "head47", N23, 1024, ("logits", "labels")),
    "cnn_48": Spec("c", "cnn_48", N24, 256, ("logits", "labels")),
    "emulator cnn_48": Spec("emul", "cnn_48", N22, 1024, ("logits", "labels")),
    "layers fc": Spec("c", "fc", N23, 256, ("logits", "labels")),
    "host fc labels only": Spec("c", "fc", N23, 256, ("labels",)),
    "windows head47": Spec("win", "head47", (PAGE - 15) ** 2, None, ("logits", "labels"), window_uid),
    # three pages: 16 classes and 16 scores per window pass 2^31 bytes past 33.6 M windows
    "windows topk head47": Spec("win_topk", "head47", 3 * (PAGE - 15) ** 2, None, ("classes", "scores"), window_uid, 3),
    "windows emulator head47": Spec("win_emul", "head47", (PAGE - 15) ** 2, None, ("logits", "labels"), window_uid),
    "split fc16 labels only": Spec("c", "fc16", K_FUSED_PASS + 77, 16, ("labels",)),
}

# gather destinations: (what, bytes per row, row_offset, the byte offset its rows straddle); the call writes N_GATHER rows from
# row_offset on.  The logits rows straddle 2^32 bytes, all of them past 2^31.
GATHERS = [("labels u8", 1, (1 << 32) - 1000, 1 << 32), ("labels", 4, (1 << 29) - 500, 1 << 31),
           ("logits", 40, (1 << 32) // 40 - 500, 1 << 32)]


# ---- CPU: a wrapped offset would show ----------------------------------------------------------------------------------------

@pytest.mark.parametrize("case", list(SPECS))
def test_a_wrapped_offset_shows(oracle, case):
    """for every read and write whose offsets pass a wrap W (2^31 or 2^32 bytes), the result a read or write displaced by W
    would give differs from the expected one for most rows: reads of input row a - W / in_bytes, and the bytes a wrapped write
    of row a would put over the rows there, on the labels of a labels-only call and on every output of the others"""
    s = SPECS[case]
    check_wrapped_offsets(case, s, expected(oracle, s.kind, s.name))


def test_wrapped_gather_rows_land_on_sentinels():
    """a gather destination written from row_offset on: its rows straddle 2^31 or 2^32 bytes, and a write displaced by 2^31 or
    2^32 bytes lands before them (inside the buffer or before it), where the check of the whole buffer's sentinel sees it"""
    for what, rb, row0, cross in GATHERS:
        end = (row0 + N_GATHER) * rb
        assert row0 * rb < cross < end, what
        for w in WRAPS:
            if end > w:
                assert end - w <= row0 * rb, (what, w)


# ---- GPU helpers ---------------------------------------------------------------------------------------------------------------

def _engine(name, path=0, frontend=None):
    from bitnetmcu_b200 import _lib
    from bitnetmcu_b200.engine import Engine
    e = Engine(model(name), device=0, path=path)
    if frontend is not None:
        e.set_option(_lib.OPT_CNN_FRONTEND, frontend)
    return e


def run(e, kind, x, o):
    """the device entry of `kind` on images x into the output views o"""
    if kind == "c":
        e.infer_device(x, o.get("logits"), o.get("labels"))
    elif kind == "c_f32":
        e.infer_device_f32(x, o.get("logits"), o.get("labels"))
    elif kind == "emul":
        e.inference_quantized_device(x, o.get("logits"), o.get("labels"))
    elif kind == "topk":
        e.topk_device(x, 16, o["classes"], o["scores"])
    elif kind == "engines":
        e.compare_engines_device(x, labels_c=o["labels_c"], labels_py=o["labels_py"])


def rows_of(s):
    return rows_f32(s.name) if s.kind in ("c_f32", "emul", "engines") else rows_i8(s.name)


def entry_case(oracle, case, e_factory, what=None):
    """case `case` of SPECS through its device entry on the engine e_factory() makes: the small call on the unique rows pinned
    to the reference, the periodic batch of n rows against it tiled, the sentinels, the input"""
    import torch
    s = SPECS[case]
    res = expected(oracle, s.kind, s.name)
    what = what or case
    with Case(what, s.n, need(s, res)) as c:
        e = c.engine(e_factory)
        u = rows_of(s)
        small = outputs(res, s.outputs, U)
        run(e, s.kind, torch.from_numpy(u).cuda(), views(small, U))
        torch.cuda.synchronize()
        want = want_on_device(small, res, what)
        x = periodic(u, s.n)
        got = outputs(res, s.outputs, s.n)
        run(e, s.kind, x, views(got, s.n))
        torch.cuda.synchronize()
        check_tiled(got, want, s.n, s.uid, what)
        check_input(x, u, what)
        del x, got, small, want


# ---- GPU: the int8 C engine ----------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("case,row", [("int8 fc", "<64,2,2,16,fixed>"), ("int8 fc labels only", "<64,2,2,16,fixed>"),
                                      ("int8 head47", "<64,2,2,64>"), ("int8 2bitsym96", "<128,1>"),
                                      ("int8 binary160", "<192,1>")])
def test_int8_rows(lib, oracle, capfd, monkeypatch, case, row):
    """the int8 entry on the fused plan's rows, input past 4 GiB (and the 47-class logits past 2 GiB)"""
    from support import plan_line, plan_ring
    e, err = verbose_engine(capfd, monkeypatch, lambda: _engine(SPECS[case].name))
    assert plan_ring(plan_line(err), "int8")[0] == row, err
    e.close()
    entry_case(oracle, case, lambda: _engine(SPECS[case].name))


@pytest.mark.gpu
def test_topk(lib, oracle):
    """the 16 best classes and their scores of 2^25 + 77 images: both outputs past 2 GiB"""
    entry_case(oracle, "topk head47", lambda: _engine("head47"))


@pytest.mark.gpu
@pytest.mark.parametrize("frontend", [1, 2])
def test_cnn_int8(lib, oracle, frontend):
    """the C engine's CNN route, input past 4 GiB, on the CUDA-core and the tensor-core front-end"""
    entry_case(oracle, "cnn_48", lambda: _engine("cnn_48", frontend=frontend), f"cnn_48 front-end {frontend}")


@pytest.mark.gpu
def test_layer_path(lib, oracle):
    """BNM_PATH_LAYERS: passes of 2^17 images whose offsets pass 2^31 bytes"""
    from bitnetmcu_b200 import _lib
    entry_case(oracle, "layers fc", lambda: _engine("fc", path=_lib.PATH_LAYERS))


# ---- GPU: float input and the emulator --------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_float_fused_forms(lib, oracle, capfd, monkeypatch):
    """the three fused float-input forms of fc, float input past 4 GiB: the C engine's, the emulator's and the two engines'
    one kernel (labels of both engines, and the counts: every image, and the mismatches of the tiled labels)"""
    import torch
    from support import route
    e, err = verbose_engine(capfd, monkeypatch, lambda: _engine("fc"))
    assert "k_quantize_images" not in route(err, "emulator") and "k_quantize_images" not in route(err, "engines"), err
    e.close()
    for case in ("f32 fc", "emulator fc", "engines fc"):
        entry_case(oracle, case, lambda: _engine("fc"))
    s = SPECS["engines fc"]
    res = expected(oracle, "engines", "fc")
    with Case("engines fc counts", s.n, s.n * 1024 + GiB) as c:
        e = c.engine(lambda: _engine("fc"))
        x = periodic(rows_f32("fc"), s.n)
        counts = torch.zeros(4, dtype=torch.int64, device="cuda")
        e.compare_engines_device(x, counts=counts)
        times = np.full(U, s.n // U) + (np.arange(U) < s.n % U)   # how often each unique row occurs
        mismatches = int((times * (res["labels_c"] != res["labels_py"])).sum())
        got = counts.tolist()
        assert got[0] == s.n and got[3] == mismatches, (got, s.n, mismatches)
        del x


@pytest.mark.gpu
def test_float_passes(lib, oracle):
    """float input through k_quantize_images passes of 2^20 images, whose offsets b * in_bytes pass 4 GiB"""
    entry_case(oracle, "f32 binary160", lambda: _engine("binary160"))


@pytest.mark.gpu
def test_emulator_int8_route(lib, oracle):
    """the emulator's scaling kernel and fc_emul_i8_kernel on 8 GiB of float input, float64 logits past 2 GiB"""
    entry_case(oracle, "emulator head47", lambda: _engine("head47"))


@pytest.mark.gpu
def test_cnn_emulator(lib, oracle):
    """the emulator's fused CNN front-end (k_cnn_emul_frontend) on float input past 4 GiB"""
    entry_case(oracle, "emulator cnn_48", lambda: _engine("cnn_48"))


# ---- GPU: the result exchange, the window scan, the host pipeline -------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("what,rb,row0,cross", GATHERS)
def test_gather_rows_past_2_31(lib, oracle, what, rb, row0, cross):
    """one destination written from row_offset on, its rows straddling 2^31 or 2^32 bytes: they equal the tiled labels or
    logits, every other row of the buffer keeps its sentinel"""
    import torch
    from bitnetmcu_b200 import _lib
    from support import gather_call
    res = expected(oracle, "c", "fc")
    rows = row0 + N_GATHER + SPARE
    with Case(f"gather {what} at row {row0}", N_GATHER, rows * rb + GiB) as c:
        e = c.engine(lambda: _engine("fc"))
        x = periodic(rows_i8("fc"), N_GATHER)
        logits = what == "logits"
        dt, sent = (torch.uint8, 0xA5) if rb == 1 else (torch.int32, SENTINEL_I32)
        dst = torch.full((rows, 10) if logits else (rows,), sent, dtype=dt, device="cuda")
        g = _lib.BnmGather()
        g.n_logits_dst, g.n_labels_dst, g.row_offset, g.labels_u8 = int(logits), int(not logits), row0, int(rb == 1)
        (g.logits_dst if logits else g.labels_dst)[0] = dst.data_ptr()
        assert gather_call(lib, e, x, None, None, g, torch.cuda.current_stream()) == 0, lib.bnm_last_error()
        want = torch.from_numpy(res["logits"] if logits else res["labels"].astype(np.int32)).cuda().to(dt)
        bad = (dst[row0:row0 + N_GATHER] != want.index_select(0, row_uid(torch.arange(N_GATHER, device="cuda")))).reshape(N_GATHER, -1)
        bad = bad.any(dim=1)
        assert not bool(bad.any()), (what, f"{int(bad.sum())} rows wrong, first", (torch.nonzero(bad)[:6, 0] + row0).tolist())
        for a, b in ((0, row0), (row0 + N_GATHER, rows)):
            for r in range(a, b, 1 << 26):
                assert bool((dst[r:min(b, r + (1 << 26))] == sent).all()), (what, "a row outside the call's rows was written", r)
        check_input(x, rows_i8("fc"), what)
        del x, dst


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["windows head47", "windows topk head47", "windows emulator head47"])
def test_window_scan(lib, oracle, case):
    """every 16 x 16 window at stride 1 of 4096 x 4096 pages (one; three for top-k), its outputs past 2^31 bytes: the window
    scan of the small page whose windows are the unique ones, pinned to the reference, tiled"""
    import torch
    s = SPECS[case]
    res = expected(oracle, s.kind, s.name)
    emul, topk = s.kind == "win_emul", s.kind == "win_topk"
    with Case(case, s.n, need(s, res, s.planes * PAGE * PAGE * 4)) as c:
        e = c.engine(lambda: _engine(s.name))

        def scan(pages, n, o):
            grid = (pages.shape[0], pages.shape[1] - 15, pages.shape[2] - 15)
            v = views(o, n, grid)
            if topk:
                e.scan_windows_topk_device(pages, 1, 16, v["classes"], v["scores"])
            else:
                (e.emulate_windows_device if emul else e.scan_windows_device)(pages, 1, v["logits"], v["labels"])
            torch.cuda.synchronize()

        small = outputs(res, s.outputs, P * P)
        scan(torch.from_numpy(small_page()).cuda()[None], P * P, small)
        want = want_on_device(small, res, case)
        t = torch.from_numpy(tile()).cuda()
        ar = torch.arange(PAGE, device="cuda")
        pages = torch.stack([t.index_select(0, (ar + 7 * p) % P).index_select(1, (ar + 3 * p) % P) for p in range(s.planes)])
        got = outputs(res, s.outputs, s.n)
        scan(pages, s.n, got)
        check_tiled(got, want, s.n, s.uid, case)
        del pages, got, small, want


@pytest.mark.gpu
def test_host_pipeline(lib, oracle):
    """bnm_infer_batch from a host array of 2^23 + 77 images, labels only: chunk offsets past 2^31 bytes"""
    s = SPECS["host fc labels only"]
    res = expected(oracle, "c", "fc")
    with Case("host fc labels only", s.n, GiB) as c:
        e = c.engine(lambda: _engine("fc"))
        u = rows_i8("fc")
        _, small = e.infer(u, want_logits=False)
        assert np.array_equal(small, res["labels"]), "small call"
        idx = row_uid(np.arange(s.n))
        x = np.take(u, idx, axis=0)
        sent = np.uint32(SENTINEL_I32 & 0xFFFFFFFF)
        labels = np.full(s.n + SPARE, sent, dtype=np.uint32)
        e.infer(x, want_logits=False, out_labels=labels[:s.n])
        bad = np.flatnonzero(labels[:s.n] != small[idx])
        assert bad.size == 0, (f"{bad.size} rows wrong, first {bad[:6].tolist()}", f"byte offsets {(bad[:6] * 256).tolist()}")
        assert (labels[s.n:] == sent).all(), "written past row n"
        for r in range(0, s.n, 1 << 22):
            assert np.array_equal(x[r:r + (1 << 22)], u[idx[r:r + (1 << 22)]]), ("input changed", r)


# ---- GPU: a fused int8 batch past one launch ------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_fused_batch_splits_into_launches(lib, oracle, capfd, monkeypatch):
    """16-byte rows on the fused plan: bnm_infer_launch_count is 1 at 2^28 images and 2 just past it; labels only at 2^28 + 77
    run as two launches (two BNM_VERBOSE launch lines) and equal the tiled small call, sentinels and input intact.  In launch
    overlap mode 2, after a call on other buffers, the call's first launch is independent and its second keeps its wait."""
    import torch
    from bitnetmcu_b200 import _lib
    from support import plan_line
    s = SPECS["split fc16 labels only"]
    res = expected(oracle, "c", "fc16")
    with Case("split fc16 labels only", s.n, need(s, res)) as c:
        e, err = verbose_engine(capfd, monkeypatch, lambda: c.engine(lambda: _engine("fc16")))
        assert plan_line(err) and e.active_path == _lib.PATH_TCGEN05, err
        assert [e.launch_count(n) for n in (1, K_FUSED_PASS, K_FUSED_PASS + 1, s.n, 2 * K_FUSED_PASS + 1)] == [1, 1, 2, 2, 3]
        u = rows_i8("fc16")
        x_small = torch.from_numpy(u).cuda()
        small = outputs(res, s.outputs, U)
        run(e, "c", x_small, views(small, U))
        torch.cuda.synchronize()
        want = want_on_device(small, res, "fc16")
        x = periodic(u, s.n)
        got = outputs(res, s.outputs, s.n)
        torch.cuda.synchronize()
        capfd.readouterr()
        run(e, "c", x, views(got, s.n))
        torch.cuda.synchronize()
        lines = [l.split("fused launch: ")[1] for l in capfd.readouterr().err.splitlines() if "fused launch: " in l]
        assert lines == ["wait", "wait"], lines
        check_tiled(got, want, s.n, row_uid, "two launches")
        # mode 2: a call on other buffers, then the large call
        e.set_option(_lib.OPT_LAUNCH_OVERLAP, 2)
        got["labels"].fill_(SENTINEL_I32)
        torch.cuda.synchronize()
        capfd.readouterr()
        run(e, "c", x_small, views(small, U))
        run(e, "c", x, views(got, s.n))
        torch.cuda.synchronize()
        lines = [l.split("fused launch: ")[1] for l in capfd.readouterr().err.splitlines() if "fused launch: " in l]
        assert lines == ["wait", "independent", "wait"], lines
        check_tiled(got, want, s.n, row_uid, "two launches, mode 2")
        check_input(x, u, "fc16")
        del x, got
