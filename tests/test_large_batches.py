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
import gc
import time
from typing import Callable, NamedTuple, Optional, Tuple

import numpy as np
import pytest

from conftest import load_model
from restate import emulate, scale_images
from support import lib, normal_images, random_fc, verbose_engine  # noqa: F401  (lib: a fixture)

U = 8191                        # unique rows of a batch, an odd prime
P = 89                          # period of a window-scan page in both directions, an odd prime
PAGE = 4096                     # a window-scan page is PAGE x PAGE floats
N22, N23, N24, N25 = ((1 << b) + 77 for b in (22, 23, 24, 25))
K_FUSED_PASS = 1 << 28          # images per fused FC launch (kFusedPass, capi.cu)
N_GATHER = 2 * 148 * 128 + 77
SPARE = 128                     # sentinel rows past n in every output buffer
SLICE_BYTES = 256 << 20         # bytes of a row slice the device builds or compares at a time
GiB = 1 << 30
SENTINEL_I32, SENTINEL_F64 = -0x3C3C3C3D, -7.25e300   # fill of every output buffer
WRAPS = (1 << 31, 1 << 32)      # the byte displacements of a wrapped 32-bit offset

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


def row_uid(rows):
    """the unique row of batch rows (NumPy or torch integers)"""
    return rows % U


def window_uid(rows):
    """the unique window of windows of a stack of pages at stride 1, plane p at phase (7 p, 3 p)"""
    per = (PAGE - 15) * (PAGE - 15)
    p, r = rows // per, rows % per
    return ((r // (PAGE - 15) + 7 * p) % P) * P + (r % (PAGE - 15) + 3 * p) % P


class Spec(NamedTuple):
    kind: str                     # the entry's key in expected()
    name: str                     # the model
    n: int                        # images or windows
    in_bytes: Optional[int]       # bytes per input row (None: the window scan, whose pages stay small)
    outputs: Tuple[str, ...]      # what the call writes
    uid: Callable = row_uid
    planes: int = 1               # window scan: pages in the stack


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

def _differ(a, b):
    return (a != b).reshape(len(a), -1).any(axis=1)


@pytest.mark.parametrize("case", list(SPECS))
def test_a_wrapped_offset_shows(oracle, case):
    """for every read and write whose offsets pass a wrap W (2^31 or 2^32 bytes), the result a read or write displaced by W
    would give differs from the expected one for most rows: reads of input row a - W / in_bytes, and the bytes a wrapped write
    of row a would put over the rows there, on the labels of a labels-only call and on every output of the others"""
    s = SPECS[case]
    res = expected(oracle, s.kind, s.name)
    checked = 0
    for w in WRAPS:
        if s.in_bytes and s.n * s.in_bytes > w:
            assert w % s.in_bytes == 0
            d = w // s.in_bytes
            a = np.arange(d, min(s.n, d + U))
            diff = np.zeros(a.size, dtype=bool)
            for o in s.outputs:
                diff |= _differ(res[o][s.uid(a)], res[o][s.uid(a - d)])
            assert diff.mean() > 0.5, (case, "input", w, d, diff.mean())
            checked += 1
        for o in s.outputs:
            e = np.ascontiguousarray(res[o])
            rb = e[0].nbytes
            if s.n * rb <= w:
                continue
            b = e.view(np.uint8).reshape(e.shape[0], rb)
            a = np.arange(-(-w // rb), min(s.n, -(-w // rb) + U))
            pos = (a * rb - w)[:, None] + np.arange(rb)
            under = b[s.uid(pos // rb), pos % rb]          # what the rows there hold
            diff = _differ(b[s.uid(a)], under)
            assert diff.mean() > 0.5, (case, o, w, diff.mean())
            checked += 1
    assert checked, (case, "no offset of this case passes 2^31 bytes")
    assert s.in_bytes is None or (s.n - 77) & (s.n - 78) == 0, (case, "n is not 77 past a power of two")


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

def _free():
    import torch
    gc.collect()
    torch.cuda.empty_cache()
    return torch.cuda.mem_get_info()[0]


class Case:
    """one case: its need checked against the free device memory (skip with the figure); on exit its engines closed and its
    peak device memory (torch's tensors, and what the library held, as the device sees it) and wall time printed"""

    def __init__(self, what, n, need):
        self.what, self.n, self.need = what, n, need
        self.engines = []

    def engine(self, make):
        self.engines.append(make())
        return self.engines[-1]

    def __enter__(self):
        import torch
        free = _free()
        if free < self.need:
            pytest.skip(f"{self.what}: needs {self.need / GiB:.1f} GiB of device memory, {free / GiB:.1f} GiB free")
        torch.cuda.reset_peak_memory_stats()
        self.free0, self.reserved0 = free, torch.cuda.memory_reserved()
        self.t0 = time.perf_counter()
        return self

    def __exit__(self, *exc):
        import torch
        torch.cuda.synchronize()
        # the library's scratch pools keep their high-water mark until the engine closes
        held = (self.free0 - torch.cuda.mem_get_info()[0]) - (torch.cuda.memory_reserved() - self.reserved0)
        for e in self.engines:
            e.close()
        if exc[0] is None:
            peak = torch.cuda.max_memory_reserved() - self.reserved0 + held
            print(f"large batch: {self.what}: n = {self.n}, peak device memory {peak / GiB:.2f} GiB, "
                  f"wall {time.perf_counter() - self.t0:.2f} s")
        _free()
        return False


def _dtype(a):
    import torch
    return torch.float64 if a.dtype == np.float64 else torch.int32


def slices(t, n):
    """(start, end) of row slices of about SLICE_BYTES of tensor t, up to row n"""
    step = max(1, SLICE_BYTES // (t[0].numel() * t.element_size()))
    return [(s, min(n, s + step)) for s in range(0, n, step)]


def periodic(unique, n):
    """the CUDA batch [n, ...] whose row i is unique row i mod U, built slice by slice with index_select"""
    import torch
    u = torch.from_numpy(np.ascontiguousarray(unique)).cuda()
    out = torch.empty((n,) + tuple(u.shape[1:]), dtype=u.dtype, device="cuda")
    for s, e in slices(out, n):
        torch.index_select(u, 0, row_uid(torch.arange(s, e, device="cuda")), out=out[s:e])
    return out


def _sentinel(dtype):
    import torch
    return SENTINEL_F64 if dtype == torch.float64 else SENTINEL_I32


def outputs(res, names, n):
    """{output: CUDA tensor [n + SPARE, ...] filled with the sentinel}, shaped like the expected rows"""
    import torch
    return {o: torch.full((n + SPARE,) + res[o].shape[1:], _sentinel(_dtype(res[o])), dtype=_dtype(res[o]), device="cuda")
            for o in names}


def views(outs, n, lead=None):
    """rows :n of every output buffer (reshaped to lead + row shape when given)"""
    return {o: (t[:n] if lead is None else t[:n].reshape(lead + tuple(t.shape[1:]))) for o, t in outs.items()}


def want_on_device(got, res, what):
    """the small call's outputs (CUDA, rows :U') equal the expected NumPy rows: -> them as CUDA tensors"""
    import torch
    out = {}
    for o, t in got.items():
        w = res[o]
        g = t[:w.shape[0]].cpu().numpy()
        bad = np.flatnonzero(_differ(g.astype(w.dtype) if w.dtype == np.uint32 else g, w))
        assert bad.size == 0, (what, o, "small call", f"{bad.size} unique rows differ from the reference, first {bad[:6].tolist()}")
        out[o] = t[:w.shape[0]].clone()
    return out


def check_tiled(got, want, n, uid, what):
    """rows :n of got equal want[uid(row)], compared on the device in slices; rows n: still hold the sentinel"""
    import torch
    for o, t in got.items():
        w = want[o]
        for s, e in slices(t, n):
            bad = (t[s:e] != w.index_select(0, uid(torch.arange(s, e, device="cuda")))).reshape(e - s, -1).any(dim=1)
            if bool(bad.any()):
                rows = (torch.nonzero(bad)[:6, 0] + s).tolist()
                raise AssertionError((what, o, f"{int(bad.sum())} rows of {s}..{e} wrong, first {rows}",
                                      f"byte offsets {[r * t[0].numel() * t.element_size() for r in rows]}"))
        assert bool((t[n:] == _sentinel(t.dtype)).all()), (what, o, "written past row n")


def check_input(x, unique, what):
    """the periodic batch x still holds its rows"""
    import torch
    u = torch.from_numpy(np.ascontiguousarray(unique)).cuda()
    for s, e in slices(x, x.shape[0]):
        assert torch.equal(x[s:e], u.index_select(0, row_uid(torch.arange(s, e, device="cuda")))), (what, "input changed", s)


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


def need(s, res, extra=0):
    """device bytes of a case: the batch, the outputs with their sentinel rows, and 1 GiB for a comparison slice, the unique rows'
    results and the library's scratch and planes"""
    per_row = sum(res[o][0].nbytes for o in s.outputs)
    return s.n * (s.in_bytes or 0) + (s.n + SPARE) * per_row + GiB + extra


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
