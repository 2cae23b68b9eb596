"""CUDA graphs of the C ABI's device entries (include/bitnetmcu_b200.h, "Graphs"; DESIGN.md 4.6).

Every case runs its entry eagerly on R contents of the input buffers, then captures it once and replays the graph R times,
refilling the inputs in place before each replay.  Each replay must give exactly what the eager call gave on the same contents,
and those results must equal the oracle (the C engine) or tests/restate.py (the emulator) on a prefix of the rows.  The sizes are
1 image, N_MANY, and one more than a pass on the routes that run in passes, so that one graph holds several passes of scratch
allocation and free nodes.  Further tests pin the launch-overlap (mode 2) decisions of captured launches, host calls made while
another thread captures, two graphs of one model replayed at once, and a graph that keeps its route after the path option
changes."""
import ctypes as C
import threading
from typing import Callable, List, NamedTuple, Optional

import numpy as np
import pytest

from conftest import load_model
from restate import emulate, scale_images
from support import N_MANY, engine, lib, random_fc, verbose_engine

pytestmark = pytest.mark.gpu

R = 3                                         # contents, eager calls and replays per case
BIG, BIG_LAYERS = (1 << 20) + 129, (1 << 17) + 3
PREFIX = 1024                                 # rows checked against the oracle or the restatement
SENTINEL = -7


def _torch():
    import torch
    return torch


def graph_of(fn, mode="global"):
    """fn() captured through torch.cuda.graph (capture on torch's side stream, which is the current stream inside)"""
    torch = _torch()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, capture_error_mode=mode):
        fn()
    return g


# ---- the driver API, for captures on a stream of the test's choosing ------------------------------------------------------------

class Driver:
    """cuStreamBeginCapture / cuStreamEndCapture / cuGraphInstantiate / cuGraphLaunch on torch's stream handles"""
    GLOBAL, THREAD_LOCAL, RELAXED = 0, 1, 2

    def __init__(self):
        self.cu = C.CDLL("libcuda.so.1")

    def _ok(self, rc, what):
        assert rc == 0, f"{what}: CUresult {rc}"

    def begin(self, stream, mode=GLOBAL):
        self._ok(self.cu.cuStreamBeginCapture_v2(C.c_void_p(stream.cuda_stream), C.c_int(mode)), "cuStreamBeginCapture")

    def end(self, stream):
        """-> (graph, exec): the captured graph and its instantiation"""
        graph, exe = C.c_void_p(), C.c_void_p()
        self._ok(self.cu.cuStreamEndCapture(C.c_void_p(stream.cuda_stream), C.byref(graph)), "cuStreamEndCapture")
        self._ok(self.cu.cuGraphInstantiateWithFlags(C.byref(exe), graph, C.c_ulonglong(0)), "cuGraphInstantiate")
        return graph, exe

    def launch(self, exe, stream):
        self._ok(self.cu.cuGraphLaunch(exe, C.c_void_p(stream.cuda_stream)), "cuGraphLaunch")

    def destroy(self, graph, exe):
        self._ok(self.cu.cuGraphExecDestroy(exe), "cuGraphExecDestroy")
        self._ok(self.cu.cuGraphDestroy(graph), "cuGraphDestroy")

    def version(self):
        v = C.c_int(0)
        self._ok(self.cu.cuDriverGetVersion(C.byref(v)), "cuDriverGetVersion")
        return v.value

    def kernel_edges(self, graph):
        """the edge types (CUgraphEdgeData.type: 0 default, 1 programmatic) of the graph's kernel-to-kernel edges"""
        class EdgeData(C.Structure):
            _fields_ = [("from_port", C.c_ubyte), ("to_port", C.c_ubyte), ("type", C.c_ubyte), ("reserved", C.c_ubyte * 5)]
        get = self.cu.cuGraphGetEdges_v2
        n = C.c_size_t(0)
        self._ok(get(graph, None, None, None, C.byref(n)), "cuGraphGetEdges_v2")
        frm, to, data = (C.c_void_p * n.value)(), (C.c_void_p * n.value)(), (EdgeData * n.value)()
        self._ok(get(graph, frm, to, data, C.byref(n)), "cuGraphGetEdges_v2")

        def kernel(node):
            t = C.c_int(-1)
            self._ok(self.cu.cuGraphNodeGetType(C.c_void_p(node), C.byref(t)), "cuGraphNodeGetType")
            return t.value == 0   # CU_GRAPH_NODE_TYPE_KERNEL
        return [data[i].type for i in range(n.value) if kernel(frm[i]) and kernel(to[i])]


# ---- models and engines -------------------------------------------------------------------------------------------------------

MODELS = {
    "fc": lambda: load_model("fc"),                           # FC 4bitsym-64: the fixed-shape row and the one-kernel float forms
    "binary160": lambda: load_model("binary160"),             # one pipe, 192 wide
    "wide37": lambda: random_fc(4, (256, 64, 64, 37), 2),     # 37 classes: scaling kernel + fc_emul_i8_kernel, the general row
    "cnn48": lambda: load_model("cnn_48"),
}


@pytest.fixture(scope="module")
def engines(lib):
    """(model name, path, CNN front-end) -> (model, engine), built once; closed when the module ends, after its graphs"""
    from bitnetmcu_b200 import _lib
    made = {}

    def get(name, layers=False, frontend=None):
        key = (name, layers, frontend)
        if key not in made:
            m = MODELS[name]()
            made[key] = (m, engine(m, _lib.PATH_LAYERS if layers else 0, frontend))
        return made[key]
    yield get
    for _, e in made.values():
        e.close()


def images(n, width, f32, seed):
    """seeded device images: int8 uniform, or float32 normal"""
    torch = _torch()
    g = torch.Generator(device="cuda").manual_seed(seed)
    if f32:
        return torch.randn((n, width), generator=g, device="cuda", dtype=torch.float32)
    return torch.randint(-128, 128, (n, width), generator=g, device="cuda", dtype=torch.int8)


# ---- one entry's call on static buffers ---------------------------------------------------------------------------------------

class Entry(NamedTuple):
    call: Callable[[], None]          # issues the entry on torch's current stream
    x: object                         # the input buffer, refilled in place
    outs: List[object]                # output buffers, reset to their fill before each call
    fills: List[float]
    want: Callable                    # (x prefix as NumPy, p) -> expected prefixes of outs (None: not checked there)


def _oracle_c(oracle, m, x):
    return oracle.infer(m, x)


def _topk(logits, k):
    cls = np.argsort(-logits, axis=1, kind="stable")[:, :k]
    return cls, np.take_along_axis(logits, cls, axis=1)


def make_entry(kind, m, e, n, oracle, k=0, scores=True, offset=False, labels_only=False, gather_off=0):
    """the buffers and the call of one entry: kind "int8", "f32", "emul", "engines", "topk", "topk_f32", "emul_topk", "gather",
    "quantize".  offset: logits 8 bytes past a 16-byte boundary (the fixed-shape FC model's general row)."""
    torch = _torch()
    nc, w = m.n_classes, m.img_bytes
    f32 = kind in ("f32", "emul", "engines", "topk_f32", "emul_topk", "quantize")
    x = images(n, w, f32, 0)
    i32 = lambda *s: torch.empty(s, dtype=torch.int32, device="cuda")
    f64 = lambda *s: torch.empty(s, dtype=torch.float64, device="cuda")

    def c_ref(xp):
        return _oracle_c(oracle, m, scale_images(xp) if f32 else xp)

    if kind in ("int8", "f32"):
        lo = None
        if not labels_only:
            if offset:   # logits 8 bytes past a 16-byte boundary
                lo = i32(n * nc + 2)[2:].view(n, nc)
                assert lo.data_ptr() % 16 == 8
            else:
                lo = i32(n, nc)
                assert lo.data_ptr() % 16 == 0
        la = i32(n)
        fn = e.infer_device if kind == "int8" else e.infer_device_f32
        outs = [la] + ([lo] if lo is not None else [])
        return Entry(lambda: fn(x, lo, la), x, outs, [SENTINEL] * len(outs),
                     lambda xp: (lambda r: [r[1]] + ([r[0]] if lo is not None else []))(c_ref(xp)))
    if kind == "gather":
        from bitnetmcu_b200 import _lib
        from bitnetmcu_b200.engine import N
        dst_lo, dst_la = i32(n + gather_off, nc), i32(n + gather_off)
        lo, la = i32(n, nc), i32(n)
        g = _lib.BnmGather()
        g.n_logits_dst, g.n_labels_dst, g.row_offset = 1, 1, gather_off
        g.logits_dst[0], g.labels_dst[0] = dst_lo.data_ptr(), dst_la.data_ptr()
        call = lambda: e._device_call(e.lib.bnm_infer_batch_device_gather, x, torch.int8,
                                      [(lo, torch.int32, (N, nc)), (la, 4, N), C.byref(g)], None)

        def want(xp):
            rlo, rla = c_ref(xp)
            return [rlo, rla, None, None]   # the destinations are compared with the eager call's (their rows sit at an offset)
        return Entry(call, x, [lo, la, dst_lo[gather_off:], dst_la[gather_off:]], [SENTINEL] * 4, want)
    if kind == "emul":
        lo, la = f64(n, nc), i32(n)

        def want(xp):
            r = emulate(m, xp)
            return [r, np.argmax(r, axis=1)]
        return Entry(lambda: e.inference_quantized_device(x, lo, la), x, [lo, la], [np.nan, SENTINEL], want)
    if kind == "engines":
        truth = torch.randint(0, nc, (n,), dtype=torch.int32, device="cuda")
        lc, lp, counts = i32(n), i32(n), torch.empty(4, dtype=torch.int64, device="cuda")

        def want(xp):
            return [c_ref(xp)[1], np.argmax(emulate(m, xp), axis=1), None]
        return Entry(lambda: e.compare_engines_device(x, truth, lc, lp, counts), x, [lc, lp, counts], [SENTINEL, SENTINEL, 0], want)
    if kind in ("topk", "topk_f32", "emul_topk"):
        cls = i32(n, k)
        sc = (f64(n, k) if kind == "emul_topk" else i32(n, k)) if scores else None
        fn = {"topk": e.topk_device, "topk_f32": e.topk_device_f32, "emul_topk": e.emulate_topk_device}[kind]

        def want(xp):
            c, s = _topk(emulate(m, xp) if kind == "emul_topk" else c_ref(xp)[0], k)
            return [c] + ([s] if scores else [])
        return Entry(lambda: fn(x, k, cls, sc), x, [cls] + ([sc] if scores else []), [SENTINEL] * (2 if scores else 1), want)
    if kind == "quantize":
        from bitnetmcu_b200.engine import quantize_images_device
        q = torch.empty((n, w), dtype=torch.int8, device="cuda")
        return Entry(lambda: quantize_images_device(x, q), x, [q], [0], lambda xp: [scale_images(xp)])
    raise ValueError(kind)


def run_calls(ent: Entry, fn, seeds) -> list:
    """per seed: refill the input in place, reset the outputs, fn(), wait -> the outputs as NumPy"""
    torch = _torch()
    got = []
    for s in seeds:
        ent.x.copy_(images(*ent.x.shape, ent.x.dtype == torch.float32, s))
        for o, f in zip(ent.outs, ent.fills):
            o.fill_(f)
        torch.cuda.synchronize()
        fn()
        torch.cuda.synchronize()
        got.append([o.cpu().numpy().copy() for o in ent.outs])
    return got


def assert_equal(got, want, what):
    got, want = np.asarray(got), np.asarray(want)
    if want.dtype.kind != "f":
        got, want = got.astype(np.int64), want.astype(np.int64)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    bad = np.flatnonzero((got != want).reshape(len(want), -1).any(axis=1)) if want.ndim else np.flatnonzero(got != want)
    assert bad.size == 0, (what, f"{bad.size} of {len(want)} rows differ, first {bad[:4].tolist()}")


def replay_matches_eager(ent: Entry, tag, mode="global"):
    """R eager calls, one capture, R replays on the same R contents: equal outputs, and the eager ones equal the reference on the
    first PREFIX rows.  -> the eager outputs"""
    seeds = [11 + r for r in range(R)]
    eager = run_calls(ent, ent.call, seeds)
    g = graph_of(ent.call, mode)
    replays = run_calls(ent, g.replay, seeds)
    for r, s in enumerate(seeds):
        for j, (a, b) in enumerate(zip(eager[r], replays[r])):
            assert_equal(b, a, (tag, "replay", r, "output", j))
        xp = images(*ent.x.shape, ent.x.dtype == _torch().float32, s)[:PREFIX].cpu().numpy()
        for j, w in enumerate(ent.want(xp)):
            if w is not None:
                assert_equal(eager[r][j][:PREFIX], w, (tag, "reference", r, "output", j))
    del g
    return eager


# ---- every device entry x route ---------------------------------------------------------------------------------------------

# (id, model, entry kind, options, sizes beyond 1 and N_MANY)
CASES = [
    ("fc-fixed", "fc", "int8", {}, []),
    ("fc-general", "fc", "int8", {"offset": True}, []),
    ("fc-labels", "fc", "int8", {"labels_only": True}, []),
    ("fc-gather", "fc", "gather", {"gather_off": 37}, []),
    ("fc-f32", "fc", "f32", {}, []),
    ("fc-emul", "fc", "emul", {}, []),
    ("fc-engines", "fc", "engines", {}, []),
    ("fc-topk1", "fc", "topk", {"k": 1, "scores": False}, []),
    ("fc-topk5", "fc", "topk", {"k": 5}, []),
    ("fc-topk5-f32", "fc", "topk_f32", {"k": 5, "scores": False}, []),
    ("fc-emul-topk5", "fc", "emul_topk", {"k": 5}, []),
    ("fc-quantize", "fc", "quantize", {}, []),
    ("binary160", "binary160", "int8", {}, []),
    ("binary160-emul", "binary160", "emul", {}, [BIG]),
    ("wide37", "wide37", "int8", {}, []),
    ("wide37-f32", "wide37", "f32", {}, [BIG]),
    ("wide37-emul", "wide37", "emul", {}, []),
    ("wide37-engines", "wide37", "engines", {}, [BIG]),
    ("wide37-topk5", "wide37", "topk", {"k": 5}, []),
    ("wide37-emul-topk1", "wide37", "emul_topk", {"k": 1, "scores": False}, []),
    ("cnn48-frontend0", "cnn48", "int8", {"frontend": 0}, [BIG]),
    ("cnn48-frontend1", "cnn48", "int8", {"frontend": 1}, [BIG]),
    ("cnn48-emul", "cnn48", "emul", {}, []),
    ("cnn48-topk5", "cnn48", "topk", {"k": 5}, []),
    ("fc-layers", "fc", "int8", {"layers": True}, [BIG_LAYERS]),
    ("fc-layers-emul", "fc", "emul", {"layers": True}, [BIG_LAYERS]),
    ("fc-layers-topk5", "fc", "topk", {"k": 5, "layers": True}, []),
    ("fc-layers-emul-topk5", "fc", "emul_topk", {"k": 5, "layers": True}, []),
]
PARAMS = [pytest.param(c, n, id=f"{c[0]}-{n}") for c in CASES for n in [1, N_MANY] + c[4]]


@pytest.mark.parametrize("case,n", PARAMS)
def test_replay_equals_eager_call(engines, oracle, case, n):
    cid, name, kind, opts, _ = case
    opts = dict(opts)
    m, e = engines(name, opts.pop("layers", False), opts.pop("frontend", None))
    replay_matches_eager(make_entry(kind, m, e, n, oracle, **opts), (cid, n))


def test_engine_counts_add_up_over_replays(engines, oracle):
    """bnm_compare_engines_device adds to counts on every replay: R replays on unchanged images give R times one call's counts"""
    torch = _torch()
    m, e = engines("wide37")
    ent = make_entry("engines", m, e, N_MANY, oracle)
    one = run_calls(ent, ent.call, [5])[0][2]
    assert one[0] == N_MANY
    g = graph_of(ent.call)
    ent.outs[2].zero_()
    for _ in range(R):
        g.replay()
    torch.cuda.synchronize()
    assert ent.outs[2].cpu().numpy().tolist() == (R * one).tolist()


@pytest.mark.parametrize("mode", ["thread_local", "relaxed"])
def test_other_capture_modes(engines, oracle, mode):
    """the CNN route, whose scratch becomes graph allocations, captured in the two other capture modes"""
    m, e = engines("cnn48")
    replay_matches_eager(make_entry("int8", m, e, N_MANY, oracle), mode, mode)


def test_quantize_infer_topk_chain(engines, oracle):
    """quantize_images_device -> infer_device -> topk_device in one graph (INTEGRATION.md 4)"""
    torch = _torch()
    from bitnetmcu_b200.engine import quantize_images_device
    m, e = engines("fc")
    n = 4096
    x = images(n, m.img_bytes, True, 0)
    q = torch.empty((n, m.img_bytes), dtype=torch.int8, device="cuda")
    la = torch.empty(n, dtype=torch.int32, device="cuda")
    cls = torch.empty((n, 5), dtype=torch.int32, device="cuda")

    def chain():
        quantize_images_device(x, q)
        e.infer_device(q, None, la)
        e.topk_device(q, 5, cls)
    chain()
    g = graph_of(chain)
    for s in range(R):
        x.copy_(images(n, m.img_bytes, True, 40 + s))
        la.fill_(SENTINEL)
        cls.fill_(SENTINEL)
        g.replay()
        torch.cuda.synchronize()
        lo, want = oracle.infer(m, scale_images(x.cpu().numpy()))
        assert_equal(la.cpu().numpy(), want, ("chain labels", s))
        assert_equal(cls.cpu().numpy(), _topk(lo, 5)[0], ("chain classes", s))


# ---- mode 2 (BNM_OPT_LAUNCH_OVERLAP) inside graphs ----------------------------------------------------------------------------

def decisions(capfd):
    return [l.split("fused launch: ")[1] for l in capfd.readouterr().err.splitlines() if "fused launch: " in l]


def _overlap_engine(capfd, monkeypatch):
    from bitnetmcu_b200 import _lib
    m = MODELS["fc"]()
    e, _ = verbose_engine(capfd, monkeypatch, lambda: engine(m, _lib.PATH_TCGEN05))
    e.set_option(_lib.OPT_LAUNCH_OVERLAP, 2)
    return m, e


def test_mode2_captured_decisions(lib, oracle, capfd, monkeypatch):
    """three captured launches on distinct buffers: wait, independent, independent (captured); a captured launch that reads the
    images of the captured launch before it: wait (captured); every replay bit-exact"""
    torch = _torch()
    m, e = _overlap_engine(capfd, monkeypatch)
    n, nc = N_MANY, m.n_classes
    xs = [images(n, m.img_bytes, False, 60 + i) for i in range(3)]
    los = [torch.empty((n, nc), dtype=torch.int32, device="cuda") for _ in range(3)]
    las = [torch.empty(n, dtype=torch.int32, device="cuda") for _ in range(3)]
    try:
        capfd.readouterr()
        g = graph_of(lambda: [e.infer_device(xs[i], los[i], las[i]) for i in range(3)])
        assert decisions(capfd) == ["wait (captured)", "independent (captured)", "independent (captured)"]
        g2 = graph_of(lambda: [e.infer_device(xs[0], los[i], las[i]) for i in range(2)])
        assert decisions(capfd) == ["wait (captured)", "wait (captured)"]
        for s in range(R):
            for i, x in enumerate(xs):
                x.copy_(images(n, m.img_bytes, False, 70 + 3 * s + i))
            for t in los + las:
                t.fill_(SENTINEL)
            torch.cuda.synchronize()
            g.replay()
            torch.cuda.synchronize()
            for i in range(3):
                lo, la = oracle.infer(m, xs[i].cpu().numpy())
                assert_equal(los[i].cpu().numpy(), lo, ("logits", s, i))
                assert_equal(las[i].cpu().numpy(), la, ("labels", s, i))
            g2.replay()
            torch.cuda.synchronize()
            lo, la = oracle.infer(m, xs[0].cpu().numpy())
            for i in range(2):
                assert_equal(los[i].cpu().numpy(), lo, ("reuse logits", s, i))
                assert_equal(las[i].cpu().numpy(), la, ("reuse labels", s, i))
        assert decisions(capfd) == []   # replays decide nothing: the graph holds its capture's decisions
        del g, g2
    finally:
        e.close()


def test_mode2_eager_launch_after_capture_keeps_its_wait(lib, oracle, capfd, monkeypatch):
    """eager A on stream S writes X; B is captured on S while A may still run; eager C on S reads X.  C compares itself with A,
    not with the captured B, and keeps its wait (before captured launches had their own record, C printed `independent`)."""
    torch = _torch()
    m, e = _overlap_engine(capfd, monkeypatch)
    drv = Driver()
    nc = m.n_classes
    n_a = 6400                                   # A's logits: 6400 x 10 x 4 bytes = 1000 images of 256 bytes for C
    n_c = n_a * nc * 4 // m.img_bytes
    s = torch.cuda.Stream()
    x_a, x_b = images(n_a, m.img_bytes, False, 80), images(n_a, m.img_bytes, False, 81)
    lo_a, la_a = torch.full((n_a, nc), SENTINEL, dtype=torch.int32, device="cuda"), torch.empty(n_a, dtype=torch.int32, device="cuda")
    lo_b, la_b = torch.empty((n_a, nc), dtype=torch.int32, device="cuda"), torch.empty(n_a, dtype=torch.int32, device="cuda")
    x_c = lo_a.view(torch.int8).view(n_c, m.img_bytes)
    lo_c, la_c = torch.empty((n_c, nc), dtype=torch.int32, device="cuda"), torch.empty(n_c, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    try:
        capfd.readouterr()
        st = s.cuda_stream
        e.infer_device(x_a, lo_a, la_a, stream=st)           # A
        drv.begin(s)
        e.infer_device(x_b, lo_b, la_b, stream=st)           # B, captured
        graph, exe = drv.end(s)
        e.infer_device(x_c, lo_c, la_c, stream=st)           # C reads A's logits
        s.synchronize()
        assert decisions(capfd) == ["wait", "wait (captured)", "wait"]
        want_a = oracle.infer(m, x_a.cpu().numpy())
        assert_equal(lo_a.cpu().numpy(), want_a[0], "A logits")
        lo, la = oracle.infer(m, x_c.cpu().numpy())
        assert_equal(lo_c.cpu().numpy(), lo, "C logits")
        assert_equal(la_c.cpu().numpy(), la, "C labels")
        drv.launch(exe, s)
        s.synchronize()
        assert_equal(la_b.cpu().numpy(), oracle.infer(m, x_b.cpu().numpy())[1], "B labels")
        drv.destroy(graph, exe)
    finally:
        e.close()


def test_captured_int8_launches_are_joined_by_a_programmatic_edge(engines, oracle):
    """two int8 launches captured back to back (mode 0): where the driver captures programmatic launches (CUDA 12.3 and later)
    the graph joins them with a programmatic edge, elsewhere with a plain one; the replay is bit-exact"""
    torch = _torch()
    m, e = engines("fc")
    drv = Driver()
    s = torch.cuda.Stream()
    x = images(N_MANY, m.img_bytes, False, 85)
    la = [torch.empty(N_MANY, dtype=torch.int32, device="cuda") for _ in range(2)]
    torch.cuda.synchronize()
    drv.begin(s)
    for t in la:
        e.infer_device(x, None, t, stream=s.cuda_stream)
    graph, exe = drv.end(s)
    try:
        assert drv.kernel_edges(graph) == [1 if drv.version() >= 12030 else 0]
        for t in la:
            t.fill_(SENTINEL)
        torch.cuda.synchronize()
        drv.launch(exe, s)
        s.synchronize()
        want = oracle.infer(m, x.cpu().numpy())[1]
        for i, t in enumerate(la):
            assert_equal(t.cpu().numpy(), want, ("labels", i))
    finally:
        drv.destroy(graph, exe)


# ---- host calls while another thread captures ---------------------------------------------------------------------------------

def test_host_calls_during_another_threads_global_capture(lib, engines, oracle):
    """thread 1 captures in global mode while thread 2 loops bnm_infer_batch (1 and 5 000 images), bnm_infer_topk,
    bnm_emulate_inference_quantized, bnm_infer_batch_device on an ordinary stream, the batched processfclayer and
    bnm_quantize_images, the reference-named processfclayer and ReLUNorm, and the host and device allocation entries: every call
    returns 0 with the oracle's (or the restatement's) results, and the capture ends valid with bit-exact replays"""
    torch = _torch()
    from bitnetmcu_b200 import engine as E
    m, e = engines("fc")
    L = m.layers[0]
    w = np.ascontiguousarray(L.weights)
    act = np.ascontiguousarray(images(300, L.n_in, False, 97).cpu().numpy())
    fc_want = np.stack([oracle.fclayer(a, w, L.bitperweight, L.n_in, L.n_out) for a in act])
    relu_want = oracle.relunorm(fc_want[0])
    xf = np.ascontiguousarray(images(700, m.img_bytes, True, 98).cpu().numpy())
    emul_want = emulate(m, xf)
    host = [np.ascontiguousarray(images(n, m.img_bytes, False, 90 + n).cpu().numpy()) for n in (1, 5000)]
    want = [oracle.infer(m, h) for h in host]
    d_x = images(N_MANY, m.img_bytes, False, 95)
    d_la = torch.empty(N_MANY, dtype=torch.int32, device="cuda")
    d_want = oracle.infer(m, d_x.cpu().numpy())[1]
    s2 = torch.cuda.Stream()
    g_x = images(N_MANY, m.img_bytes, False, 96)
    g_lo = torch.empty((N_MANY, m.n_classes), dtype=torch.int32, device="cuda")
    g_la = torch.empty(N_MANY, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    capturing, looped = threading.Event(), threading.Event()
    errors, rounds = [], 4

    def thread2():
        try:
            assert capturing.wait(60)
            for _ in range(rounds):
                for h, (lo, la) in zip(host, want):
                    got_lo, got_la = e.infer(h)
                    assert_equal(got_lo, lo, ("bnm_infer_batch logits", len(h)))
                    assert_equal(got_la, la, ("bnm_infer_batch labels", len(h)))
                cls, sc = e.topk(host[1], 5)
                wc, ws = _topk(want[1][0], 5)
                assert_equal(cls, wc, "bnm_infer_topk classes")
                assert_equal(sc, ws, "bnm_infer_topk scores")
                e.infer_device(d_x, None, d_la, stream=s2.cuda_stream)   # synchronised after the capture
                assert_equal(e.inference_quantized(xf), emul_want, "bnm_emulate_inference_quantized")
                assert_equal(E.processfclayer(act, w, L.bitperweight, L.n_in, L.n_out), fc_want, "bnm_processfclayer_batch")
                assert_equal(E.quantize_images(xf), scale_images(xf), "bnm_quantize_images")
                out = np.zeros(L.n_out, dtype=np.int32)
                lib.processfclayer(C.c_void_p(act[0].ctypes.data), C.c_void_p(w.ctypes.data), L.bitperweight, L.n_in, L.n_out,
                                   C.c_void_p(out.ctypes.data))
                assert_equal(out, fc_want[0], "processfclayer")
                o8 = np.zeros(L.n_out, dtype=np.int8)
                assert lib.ReLUNorm(C.c_void_p(out.ctypes.data), C.c_void_p(o8.ctypes.data), L.n_out) == relu_want[1]
                assert_equal(o8, relu_want[0], "ReLUNorm")
                p = C.c_void_p()
                assert lib.bnm_device_alloc(0, 1 << 20, C.byref(p)) == 0 and p.value
                lib.bnm_device_free(p)
                h = lib.bnm_host_alloc(1 << 20)
                assert h
                lib.bnm_host_free(h)
        except BaseException as ex:   # noqa: BLE001 - reported by the main thread
            errors.append(ex)
        finally:
            looped.set()

    t = threading.Thread(target=thread2)
    t.start()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):                    # capture_error_mode="global"
        e.infer_device(g_x, g_lo, g_la)
        capturing.set()
        assert looped.wait(600)
    t.join()
    assert not errors, errors
    s2.synchronize()
    assert_equal(d_la.cpu().numpy(), d_want, "bnm_infer_batch_device labels")
    for s in range(R):
        g_x.copy_(images(N_MANY, m.img_bytes, False, 100 + s))
        g_la.fill_(SENTINEL)
        g.replay()
        torch.cuda.synchronize()
        lo, la = oracle.infer(m, g_x.cpu().numpy())
        assert_equal(g_lo.cpu().numpy(), lo, ("replay logits", s))
        assert_equal(g_la.cpu().numpy(), la, ("replay labels", s))
    del g


# ---- scratch of two graphs; options after capture -----------------------------------------------------------------------------

def test_two_graphs_of_one_cnn_model_replayed_at_once(engines, oracle):
    """two graphs of one CNN model, each holding its own feature scratch, replayed at the same time on two streams"""
    torch = _torch()
    m, e = engines("cnn48")
    n = N_MANY
    ents = [make_entry("int8", m, e, n, oracle) for _ in range(2)]
    graphs = [graph_of(ent.call) for ent in ents]
    streams = [torch.cuda.Stream() for _ in range(2)]
    for r in range(R):
        seeds = [120 + 2 * r, 121 + 2 * r]
        for ent, s in zip(ents, seeds):
            ent.x.copy_(images(n, m.img_bytes, False, s))
            for o in ent.outs:
                o.fill_(SENTINEL)
        torch.cuda.synchronize()
        for g, st in zip(graphs, streams):
            with torch.cuda.stream(st):
                g.replay()
        torch.cuda.synchronize()
        for i, (ent, s) in enumerate(zip(ents, seeds)):
            lo, la = oracle.infer(m, ent.x.cpu().numpy())
            assert_equal(ent.outs[0].cpu().numpy(), la, ("graph", i, "labels", r))
            assert_equal(ent.outs[1].cpu().numpy(), lo, ("graph", i, "logits", r))
    del graphs


def test_graph_keeps_its_route_after_the_path_option_changes(lib, oracle, capfd, monkeypatch):
    """a top-k graph captured on the fused route still runs it after BNM_OPT_PATH = BNM_PATH_LAYERS (no route line at replay),
    while eager calls take the layered route; both give the same classes and scores"""
    torch = _torch()
    from bitnetmcu_b200 import _lib
    m = MODELS["fc"]()
    e, _ = verbose_engine(capfd, monkeypatch, lambda: engine(m))
    try:
        ent = make_entry("topk", m, e, N_MANY, oracle, k=5)
        capfd.readouterr()
        g = graph_of(ent.call)
        captured = [l for l in capfd.readouterr().err.splitlines() if "topk route" in l]
        assert len(captured) == 1 and "fc_topk_kernel" in captured[0], captured
        e.set_option(_lib.OPT_PATH, _lib.PATH_LAYERS)
        replays = run_calls(ent, g.replay, [130])
        assert [l for l in capfd.readouterr().err.splitlines() if "route" in l] == []
        eager = run_calls(ent, ent.call, [130])
        layered = [l for l in capfd.readouterr().err.splitlines() if "topk route" in l]
        assert len(layered) == 1 and "layer by layer" in layered[0], layered
        for a, b in zip(replays[0], eager[0]):
            assert_equal(a, b, "replay vs layered eager")
        del g
    finally:
        e.close()
