"""Stream order of the fused FC kernel's int8 launches against the kernels next to them (DESIGN.md 4.1, "Launch").

Every int8 C-engine launch is a programmatic dependent launch: its CTAs start as the kernel before it on the stream leaves
each SM, and the producer's grid-dependency wait is all that keeps its image loads, and through them its result stores,
behind that kernel.  A launch that fills the grid also triggers the next launch at its entry.  So two FC launches next to each
other on one stream, with no operation between them, are where a missing or misplaced wait would show: launch k+1 reading
what launch k writes (RAW), both writing the same outputs (WAW), launch k+1 writing what launch k still reads (WAR).  Mode 2
of BNM_OPT_LAUNCH_OVERLAP drops the wait unless the library sees a buffer of the launch before touched again; its decision is
printed on every launch under BNM_VERBOSE (`fused launch: wait` / `independent`) and asserted here for every pattern.

Every case runs on every int8 row of kChainKernels (its plan line checked), sized from this GPU's SM count so that each
launch fills the grid with at least two tiles per SM, and is compared bit for bit with the oracle.  Whether a race shows in
one run depends on timing: the decision lines and the SASS checks of test_launch_wait_sass.py are the deterministic guards,
these the end-to-end check."""
import ctypes as C
import functools
import zlib

import numpy as np
import pytest

from conftest import load_model
from restate import TILE, scale_images
from support import CHAIN_ROWS, cnn_model, engine, kernel_clone, kernel_copies_are_kernels, kernel_copy, lib, plan_line, \
    plan_ring, verbose_engine

pytestmark = pytest.mark.gpu

ROW_IDS = [r for r, _ in CHAIN_ROWS]
POISON = 0x5A5A5A5A            # int32 fill of a buffer a launch reads: a stale read gives different logits
LOGIT_SENTINEL, LABEL_SENTINEL = -0x3C3C3C3D, -7
PAIRS = 4                      # adjacent launch pairs per case


@functools.lru_cache(maxsize=None)
def _sm():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _n():
    """a launch that fills the grid with two tiles per SM and a ragged third round on some CTAs"""
    return 2 * _sm() * TILE + 77


def _images(n, img_bytes, seed):
    rng = np.random.default_rng(seed)
    x = rng.integers(-128, 127, size=(n, img_bytes), dtype=np.int8, endpoint=True)
    x[rng.integers(0, n, size=n // 16)] = 127
    x[rng.integers(0, n, size=n // 16)] = -128
    return x


@functools.lru_cache(maxsize=None)
def _model(row):
    return dict(CHAIN_ROWS)[row]()


@pytest.fixture(scope="module")
def batches(oracle):
    """row -> (model, [two batches of _n() images], [their oracle (logits, labels)]), computed once per row"""
    @functools.lru_cache(maxsize=None)
    def get(row):
        m = _model(row)
        xs = [_images(_n(), m.img_bytes, zlib.crc32(row.encode()) + k) for k in range(2)]
        return m, xs, [oracle.infer(m, x) for x in xs]
    return get


def _engine(capfd, monkeypatch, row, m):
    """the row's engine built with BNM_VERBOSE (its launches print their wait decision); the plan must name the row"""
    from bitnetmcu_b200 import _lib
    e, err = verbose_engine(capfd, monkeypatch, lambda: engine(m, _lib.PATH_TCGEN05))
    line = plan_line(err)
    assert line and e.active_path == _lib.PATH_TCGEN05, err
    assert plan_ring(line, "int8")[0] == row, line
    return e


def decisions(capfd):
    """the `fused launch:` decisions printed since the last call"""
    return [l.split("fused launch: ")[1] for l in capfd.readouterr().err.splitlines() if "fused launch: " in l]


def _eq(got, want, what):
    g = got.cpu().numpy()
    if want.dtype == np.uint32:
        g = g.astype(np.uint32)
    bad = np.flatnonzero((g != want).reshape(len(want), -1).any(axis=1))
    assert bad.size == 0, (what, f"{bad.size} of {len(want)} rows wrong, first {bad[:4].tolist()}, tiles {np.unique(bad // TILE)[:6].tolist()}")


def _gather(lib, e, img, log, lab, g, stream):
    """bnm_infer_batch_device_gather on `stream`, without waiting for it"""
    from bitnetmcu_b200 import _lib
    ptr = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None
    _lib.check(lib.bnm_infer_batch_device_gather(e.handle, ptr(img), img.shape[0], ptr(log), ptr(lab), C.byref(g),
                                                 C.c_void_p(stream.cuda_stream)), "bnm_infer_batch_device_gather")


def _dst(g, log, lab, off):
    g.n_logits_dst, g.n_labels_dst, g.row_offset = int(log is not None), int(lab is not None), off
    if log is not None:
        g.logits_dst[0] = log.data_ptr()
    if lab is not None:
        g.labels_dst[0] = lab.data_ptr()
    return g


# ---- RAW: launch k+1's images are launch k's logits -------------------------------------------------------------------------

@pytest.mark.parametrize("mode,at", [(0, "last round"), (1, "last round"), (2, "exact")])
@pytest.mark.parametrize("row", ROW_IDS)
def test_raw_images_are_the_previous_launchs_logits(lib, oracle, capfd, monkeypatch, row, mode, at):
    """launch k writes logits and labels of three full ring rounds of images into a poisoned buffer; launch k+1, right behind
    it, takes a 16-byte aligned slice of that buffer as its int8 images, 2 tiles per SM of them.  "last round": the slice
    starts at the logits of launch k's last ring round, so launch k+1's first tiles read the rows launch k writes last (the
    rest of the slice runs into the poison behind them); "exact" (mode 2): its images pointer is launch k's logits pointer,
    which the library must see and keep the wait for.  Expected: the oracle on the buffer's bytes after launch k."""
    import torch
    from bitnetmcu_b200 import _lib
    m = _model(row)
    C_, img = m.n_classes, m.img_bytes
    n1, n2 = 3 * _sm() * TILE, 2 * _sm() * TILE
    span = n2 * img
    off = 0 if at == "exact" else (n1 - _sm() * TILE) * 4 * C_
    words = max(n1 * C_, -(-(off + span) // 4))
    x1 = _images(n1, img, zlib.crc32(row.encode()) + 7)
    want1_lo, want1_la = oracle.infer(m, x1)
    after = np.full(words, POISON, dtype="<i4")
    after[:n1 * C_] = want1_lo.reshape(-1)
    want2_lo, want2_la = oracle.infer(m, after.view(np.int8)[off:off + span].reshape(n2, img))
    e = _engine(capfd, monkeypatch, row, m)
    e.set_option(_lib.OPT_LAUNCH_OVERLAP, mode)
    d_x1 = torch.from_numpy(x1).cuda()
    buf = torch.empty(words, dtype=torch.int32, device="cuda")
    lo1 = buf[:n1 * C_].view(n1, C_)
    la1 = torch.empty(n1, dtype=torch.int32, device="cuda")
    img2 = buf.view(torch.int8)[off:off + span].view(n2, img)
    assert img2.data_ptr() % 16 == 0 and (at != "exact" or img2.data_ptr() == lo1.data_ptr())
    lo2 = torch.empty((n2, C_), dtype=torch.int32, device="cuda")
    la2 = torch.empty(n2, dtype=torch.int32, device="cuda")
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    decisions(capfd)
    got = []
    with torch.cuda.stream(s):
        for _ in range(PAIRS):
            buf.fill_(POISON)
            e.infer_device(d_x1, lo1, la1)
            e.infer_device(img2, lo2, la2)
            got.append((kernel_clone(lo1), kernel_clone(la1), kernel_clone(lo2), kernel_clone(la2)))
        s.synchronize()
    assert decisions(capfd) == ["wait"] * 2 * PAIRS
    for k, (g1, l1, g2, l2) in enumerate(got):
        _eq(g1, want1_lo, (row, mode, k, "launch k logits"))
        _eq(l1, want1_la, (row, mode, k, "launch k labels"))
        _eq(g2, want2_lo, (row, mode, k, "launch k+1 logits (images = launch k's logits)"))
        _eq(l2, want2_la, (row, mode, k, "launch k+1 labels"))
    e.close()


# ---- WAW: adjacent launches, different images, the same outputs ---------------------------------------------------------------

@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("row", ROW_IDS)
def test_waw_last_launch_wins(lib, batches, capfd, monkeypatch, row, mode):
    """2 x PAIRS launches back to back, alternating two resident batches, all into one logits and one labels buffer:
    afterwards both hold exactly the last launch's rows.  In mode 2 the reused outputs must keep every wait."""
    import torch
    from bitnetmcu_b200 import _lib
    m, xs, wants = batches(row)
    n = _n()
    e = _engine(capfd, monkeypatch, row, m)
    e.set_option(_lib.OPT_LAUNCH_OVERLAP, mode)
    d_x = [torch.from_numpy(x).cuda() for x in xs]
    lo = torch.full((n, m.n_classes), LOGIT_SENTINEL, dtype=torch.int32, device="cuda")
    la = torch.full((n,), LABEL_SENTINEL, dtype=torch.int32, device="cuda")
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    decisions(capfd)
    with torch.cuda.stream(s):
        for k in range(2 * PAIRS):
            e.infer_device(d_x[k & 1], lo, la)
        s.synchronize()
    assert decisions(capfd) == ["wait"] * 2 * PAIRS
    _eq(lo, wants[1][0], (row, mode, "logits"))
    _eq(la, wants[1][1], (row, mode, "labels"))
    e.close()


# ---- WAR: launch k+1 writes its logits over the images launch k reads ------------------------------------------------------------

@pytest.mark.parametrize("mode,at", [(0, "tail"), (1, "tail"), (2, "exact")])
@pytest.mark.parametrize("row", ROW_IDS)
def test_war_next_logits_over_previous_images(lib, batches, capfd, monkeypatch, kernel_copies_are_kernels, row, mode, at):
    """launch k reads its images from a buffer whose tail (the rows it reads in its last ring round; "exact": its head, the
    same pointer) launch k+1, right behind it, overwrites with its logits.  A kernel restores the images before every pair.
    Launch k's outputs must equal the oracle on the original images, launch k+1's on its own."""
    import torch
    from bitnetmcu_b200 import _lib
    m, xs, wants = batches(row)
    n, C_ = _n(), m.n_classes
    e = _engine(capfd, monkeypatch, row, m)
    e.set_option(_lib.OPT_LAUNCH_OVERLAP, mode)
    src = torch.from_numpy(xs[0]).cuda()
    d_x2 = torch.from_numpy(xs[1]).cuda()
    buf = torch.empty_like(src)
    flat = buf.view(-1)
    span = n * C_ * 4
    off = 0 if at == "exact" else (flat.numel() - span) // 16 * 16
    lo2 = flat[off:off + span].view(torch.int32).view(n, C_)
    assert at != "exact" or lo2.data_ptr() == buf.data_ptr()
    lo1 = torch.empty((n, C_), dtype=torch.int32, device="cuda")
    la1 = torch.empty(n, dtype=torch.int32, device="cuda")
    la2 = torch.empty(n, dtype=torch.int32, device="cuda")
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    decisions(capfd)
    got = []
    with torch.cuda.stream(s):
        for _ in range(PAIRS):
            kernel_copy(buf, src)
            e.infer_device(buf, lo1, la1)
            e.infer_device(d_x2, lo2, la2)
            got.append((kernel_clone(lo1), kernel_clone(la1), kernel_clone(lo2), kernel_clone(la2)))
        s.synchronize()
    assert decisions(capfd) == ["wait"] * 2 * PAIRS
    for k, (g1, l1, g2, l2) in enumerate(got):
        _eq(g1, wants[0][0], (row, mode, k, "launch k logits (its images overwritten behind it)"))
        _eq(l1, wants[0][1], (row, mode, k, "launch k labels"))
        _eq(g2, wants[1][0], (row, mode, k, "launch k+1 logits"))
        _eq(l2, wants[1][1], (row, mode, k, "launch k+1 labels"))
    e.close()


# ---- mode 2: the result exchange's destinations ---------------------------------------------------------------------------------

@pytest.mark.parametrize("row", ROW_IDS)
def test_mode2_gather_destinations(lib, batches, capfd, monkeypatch, row):
    """double-buffered images, no own outputs, one logits and one labels destination.  At one row offset every launch writes
    the same rows: each keeps the wait and the last launch wins.  At two offsets whose rows do not overlap the launches are
    independent, and each range holds the rows of the last launch that wrote it."""
    import torch
    from bitnetmcu_b200 import _lib
    m, xs, wants = batches(row)
    n, C_ = _n(), m.n_classes
    e = _engine(capfd, monkeypatch, row, m)
    e.set_option(_lib.OPT_LAUNCH_OVERLAP, 2)
    d_x = [torch.from_numpy(x).cuda() for x in xs]
    dlo = torch.full((2 * n + 256, C_), LOGIT_SENTINEL, dtype=torch.int32, device="cuda")
    dla = torch.full((2 * n + 256,), LABEL_SENTINEL, dtype=torch.int32, device="cuda")
    g = _dst(_lib.BnmGather(), dlo, dla, 128)
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    decisions(capfd)
    with torch.cuda.stream(s):
        for k in range(2 * PAIRS):
            _gather(lib, e, d_x[k & 1], None, None, g, s)
        s.synchronize()
    assert decisions(capfd) == ["wait"] * 2 * PAIRS
    _eq(dlo[128:128 + n], wants[1][0], (row, "same offset: logits destination"))
    _eq(dla[128:128 + n], wants[1][1], (row, "same offset: labels destination"))
    assert (dlo[:128] == LOGIT_SENTINEL).all() and (dla[128 + n:] == LABEL_SENTINEL).all()
    # two offsets, rows [0, n) and [n + 256, 2 n + 256): batch 0 always to the first, batch 1 to the second
    dlo.fill_(LOGIT_SENTINEL)
    dla.fill_(LABEL_SENTINEL)
    gs = [_dst(_lib.BnmGather(), dlo, dla, 0), _dst(_lib.BnmGather(), dlo, dla, n + 256)]
    e.set_option(_lib.OPT_LAUNCH_OVERLAP, 2)
    torch.cuda.synchronize()
    decisions(capfd)
    with torch.cuda.stream(s):
        for k in range(2 * PAIRS):
            _gather(lib, e, d_x[k & 1], None, None, gs[k & 1], s)
        s.synchronize()
    assert decisions(capfd) == ["wait"] + ["independent"] * (2 * PAIRS - 1)
    for k, at in enumerate((0, n + 256)):
        _eq(dlo[at:at + n], wants[k][0], (row, "two offsets: logits", at))
        _eq(dla[at:at + n], wants[k][1], (row, "two offsets: labels", at))
    assert (dla[n:n + 256] == LABEL_SENTINEL).all()
    e.close()


# ---- mode 2: the decision for every pattern -------------------------------------------------------------------------------------

def test_mode2_decisions(lib, capfd, monkeypatch):
    """the wait decision of each int8 launch pattern in mode 2 (and that modes 0 and 1 always wait): independent only for a
    launch right behind another int8 launch on the same stream that touches none of its buffers, in any role"""
    import torch
    from bitnetmcu_b200 import _lib
    row = "<64,2,2,16,fixed>"
    m = _model(row)
    n = 1000
    e = _engine(capfd, monkeypatch, row, m)
    x = [torch.from_numpy(_images(n, m.img_bytes, k)).cuda() for k in range(2)]
    lo = [torch.empty((n, 10), dtype=torch.int32, device="cuda") for _ in range(2)]
    la = [torch.empty(n, dtype=torch.int32, device="cuda") for _ in range(2)]
    as_img = lambda t: t.view(torch.int8).reshape(-1)[:n * m.img_bytes].view(n, m.img_bytes)
    big = [torch.empty((n * m.img_bytes // 4,), dtype=torch.int32, device="cuda") for _ in range(2)]   # room for n images
    s, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    torch.cuda.synchronize()

    def run(mode, *launches):
        e.set_option(_lib.OPT_LAUNCH_OVERLAP, mode)
        decisions(capfd)
        for f in launches:
            f()
        torch.cuda.synchronize()
        return decisions(capfd)

    on = lambda img, l, b, st=s: lambda: e.infer_device(img, l, b, stream=st.cuda_stream)
    dbl = [on(x[0], lo[0], la[0]), on(x[1], lo[1], la[1])]
    for mode in (0, 1):
        assert run(mode, *dbl, *dbl) == ["wait"] * 4, mode
    # the first launch after the option is set waits; disjoint double-buffered launches are independent
    assert run(2, *dbl, *dbl) == ["wait", "independent", "independent", "independent"]
    # another stream
    assert run(2, dbl[0], on(x[1], lo[1], la[1], s2), on(x[0], lo[0], la[0], s2)) == ["wait", "wait", "independent"]
    # a launch of another form (top-k) in between
    cls = torch.empty((n, 1), dtype=torch.int32, device="cuda")
    topk = lambda: e.topk_device(x[1], 1, cls, stream=s.cuda_stream)
    assert run(2, dbl[0], topk, dbl[1]) == ["wait", "wait"]
    # labels-only launches: the absent logits are no shared buffer; a shared labels buffer is
    assert run(2, on(x[0], None, la[0]), on(x[1], None, la[1]), on(x[0], None, la[1])) == ["wait", "independent", "wait"]
    # the same images, logits or labels again
    assert run(2, dbl[0], on(x[0], lo[1], la[1]), on(x[1], lo[1], la[0]), on(x[0], lo[0], la[0]), on(x[1], lo[1], la[1])) == \
        ["wait", "wait", "wait", "wait", "independent"]
    # cross-role: images = the previous logits / labels; logits / labels = the previous images
    li = as_img(big[0])
    assert run(2, on(x[0], big[0][:n * 10].view(n, 10), la[0]), on(li, lo[1], la[1])) == ["wait", "wait"]
    assert run(2, on(x[0], lo[0], big[1][:n]), on(as_img(big[1]), lo[1], la[1])) == ["wait", "wait"]
    assert run(2, on(li, lo[0], la[0]), on(x[1], big[0][:n * 10].view(n, 10), la[1])) == ["wait", "wait"]
    assert run(2, on(li, lo[0], la[0]), on(x[1], lo[1], big[0][:n])) == ["wait", "wait"]
    # gather destinations: the same one at the same offset, another offset, a destination that is the previous images
    dst = torch.empty((3 * n, 10), dtype=torch.int32, device="cuda")
    dl = torch.empty(3 * n, dtype=torch.int32, device="cuda")
    ga = lambda img, g: lambda: _gather(lib, e, img, None, None, g, s)
    g0, g1 = _dst(_lib.BnmGather(), dst, dl, 0), _dst(_lib.BnmGather(), dst, dl, n)
    assert run(2, ga(x[0], g0), ga(x[1], g0), ga(x[0], g1), ga(x[1], g0)) == ["wait", "wait", "independent", "independent"]
    gl = _dst(_lib.BnmGather(), None, dl, 0)
    assert run(2, ga(x[0], gl), ga(x[1], _dst(_lib.BnmGather(), None, dl, 0))) == ["wait", "wait"]
    assert run(2, ga(x[0], gl), ga(x[1], _dst(_lib.BnmGather(), dst, None, 0))) == ["wait", "independent"]
    gi = _dst(_lib.BnmGather(), big[0][:n * 10].view(n, 10), None, 0)
    assert run(2, dbl[1], ga(x[0], gi), ga(li, gl)) == ["wait", "independent", "wait"]
    e.close()


# ---- mode 0: kernel producers and consumers next to every route ------------------------------------------------------------------

@pytest.mark.parametrize("row", ROW_IDS)
def test_mode0_kernel_neighbours_fc(lib, batches, capfd, monkeypatch, kernel_copies_are_kernels, row):
    """a kernel writes the images into the same buffer right before each launch, kernels read logits and labels right after"""
    import torch
    m, xs, wants = batches(row)
    n = _n()
    e = _engine(capfd, monkeypatch, row, m)
    src = [torch.from_numpy(x).cuda() for x in xs]
    d_x = torch.empty_like(src[0])
    lo = torch.empty((n, m.n_classes), dtype=torch.int32, device="cuda")
    la = torch.empty(n, dtype=torch.int32, device="cuda")
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    got = []
    with torch.cuda.stream(s):
        for k in range(2 * PAIRS):
            kernel_copy(d_x, src[k & 1])
            e.infer_device(d_x, lo, la)
            got.append((kernel_clone(lo), kernel_clone(la)))
        s.synchronize()
    for k, (gl, gb) in enumerate(got):
        _eq(gl, wants[k & 1][0], (row, k, "logits"))
        _eq(gb, wants[k & 1][1], (row, k, "labels"))
    e.close()


def test_mode0_kernel_neighbours_quantize_then_infer(lib, oracle, kernel_copies_are_kernels):
    """bnm_quantize_images_device writes the int8 images into one buffer right before each launch, at grid-filling size"""
    import torch
    from bitnetmcu_b200 import engine as E
    m = load_model("fc")
    n = _n()
    rng = np.random.default_rng(31)
    xs = [rng.normal(size=(n, 256)).astype(np.float32) for _ in range(2)]
    wants = [oracle.infer(m, scale_images(x)) for x in xs]
    e = engine(m)
    d_x = [torch.from_numpy(x).cuda() for x in xs]
    d_q = torch.empty((n, 256), dtype=torch.int8, device="cuda")
    lo = torch.empty((n, 10), dtype=torch.int32, device="cuda")
    la = torch.empty(n, dtype=torch.int32, device="cuda")
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    got = []
    with torch.cuda.stream(s):
        for k in range(2 * PAIRS):
            E.quantize_images_device(d_x[k & 1], d_q, stream=s.cuda_stream)
            e.infer_device(d_q, lo, la)
            got.append((kernel_clone(lo), kernel_clone(la)))
        s.synchronize()
    for k, (gl, gb) in enumerate(got):
        _eq(gl, wants[k & 1][0], (k, "logits"))
        _eq(gb, wants[k & 1][1], (k, "labels"))
    e.close()


def test_mode0_kernel_neighbours_cnn(lib, oracle, kernel_copies_are_kernels):
    """a CNN model: a kernel writes the images, the front-end kernel feeds the int8 form, kernels read the outputs"""
    import torch
    m = cnn_model(48, 10, seed=12)
    n = _n()
    xs = [_images(n, 256, 40 + k) for k in range(2)]
    wants = [oracle.infer(m, x) for x in xs]
    e = engine(m)
    src = [torch.from_numpy(x).cuda() for x in xs]
    d_x = torch.empty_like(src[0])
    lo = torch.empty((n, 10), dtype=torch.int32, device="cuda")
    la = torch.empty(n, dtype=torch.int32, device="cuda")
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    got = []
    with torch.cuda.stream(s):
        for k in range(2 * PAIRS):
            kernel_copy(d_x, src[k & 1])
            e.infer_device(d_x, lo, la)
            got.append((kernel_clone(lo), kernel_clone(la)))
        s.synchronize()
    for k, (gl, gb) in enumerate(got):
        _eq(gl, wants[k & 1][0], (k, "logits"))
        _eq(gb, wants[k & 1][1], (k, "labels"))
    e.close()


def test_mode0_kernel_neighbours_gather(lib, batches, kernel_copies_are_kernels):
    """a gather launch between a kernel that writes its images and kernels that read its own outputs and destinations"""
    import torch
    from bitnetmcu_b200 import _lib
    m, xs, wants = batches("<64,2,2,16,fixed>")
    n = _n()
    e = engine(m)
    src = [torch.from_numpy(x).cuda() for x in xs]
    d_x = torch.empty_like(src[0])
    lo = torch.empty((n, 10), dtype=torch.int32, device="cuda")
    la = torch.empty(n, dtype=torch.int32, device="cuda")
    dlo = torch.empty((n + 64, 10), dtype=torch.int32, device="cuda")
    dla = torch.empty(n + 64, dtype=torch.int32, device="cuda")
    g = _dst(_lib.BnmGather(), dlo, dla, 64)
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    got = []
    with torch.cuda.stream(s):
        for k in range(2 * PAIRS):
            kernel_copy(d_x, src[k & 1])
            _gather(lib, e, d_x, lo, la, g, s)
            got.append((kernel_clone(lo), kernel_clone(la), kernel_clone(dlo[64:]), kernel_clone(dla[64:])))
        s.synchronize()
    for k, outs in enumerate(got):
        for t, w, what in zip(outs, (wants[k & 1] * 2), ("logits", "labels", "logits destination", "labels destination")):
            _eq(t, w, (k, what))
    e.close()
