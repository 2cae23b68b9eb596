"""The fused FC kernels past their first trips round the tile ring (fc_wgmma.cu; DESIGN.md 4.1, "Synchronisation").

fc_chain_kernel and fc_emul_kernel are persistent.  CTA b of a grid of min(n_tiles, SMs) takes the 128-image tiles b, b + grid,
b + 2 grid, ...  Its local tile i goes to pipe i % pipes, and j = i / pipes is its place in that pipe: slot j % slots (two-slot
kernels: slot A the even j, slot B the odd ones), stage j % stages, ring round j / stages, phase parity round & 1.  A wrong phase
flip, empty-barrier wait or epilogue tile index shows only once a CTA has run more tiles than its pipe has stages, and every
launch starts again from stage 0, phase 0, so it takes one launch with enough tiles per CTA to get there.

CPU: the restatement of that schedule in restate.py (checked against the kernel's own running counters), and per ring shape a short sweep of
batch sizes whose coverage is checked.  GPU (tolerance 0): every kernel row, its ring shape read from the plan's BNM_VERBOSE line
and the SM count from the device, over its sweep -- one launch per batch size on a prefix of one device buffer -- against the
oracle (int8 and float input) or the NumPy restatement of the emulator."""
import zlib

import numpy as np
import pytest

from conftest import load_model
from restate import LEVEL_SHIFT, TILE, batch_size, emulate_fc, most_tiles_per_cta, ring_sweep, scale_images, sweep_gaps, \
    tile_schedule
from support import CHAIN_ROWS, Sweep, engine, lib, plan_line, plan_ring, random_fc, scattered_edge_images, verbose_engine

# ---- CPU -------------------------------------------------------------------------------------------------------------------

# (pipes, stages per pipe, slots) of the plans fc_chain_plan_create makes: the two-pipe rows, and one pipe of two to six stages
SHAPES = [(2, 3, 2), (1, 2, 1), (1, 3, 1), (1, 4, 1), (1, 5, 1), (1, 6, 1)]
SMS = [132, 114, 148, 7]


def _replay(n, sm, pipes, stages, slots):
    """the schedule from the kernel's own loops: my_tiles = the CTA's share; the producer's one ring position, advanced once
    every pipe has taken a tile; per pipe, the consumer's ring position advanced per tile, its slots taking the tiles in turn"""
    n_tiles = -(-n // TILE)
    grid = min(n_tiles, sm)
    out = {}

    def advance(stage, phase):
        stage += 1
        return (0, phase ^ 1) if stage == stages else (stage, phase)

    for b in range(grid):
        my_tiles = (n_tiles - b + grid - 1) // grid
        stage = phase = pipe = 0
        for i in range(my_tiles):
            out[b + i * grid] = [b, i, pipe, None, stage, phase]
            pipe += 1
            if pipe == pipes:
                pipe = 0
                stage, phase = advance(stage, phase)
        for p in range(pipes):
            stage = phase = x = 0
            for i in range(p, my_tiles, pipes):
                tile = out[b + i * grid]
                assert tile[2] == p and tile[4:] == [stage, phase], (n, b, i)   # producer and consumer agree
                tile[3] = x
                x = (x + 1) % slots
                stage, phase = advance(stage, phase)
    return out


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "%dx%d-slots%d" % s)
def test_schedule_matches_the_kernels_running_counters(shape):
    pipes, stages, slots = shape
    for sm in (7, 13):
        for n in [1, 127, 128, 129] + [batch_size(sm, t, r, tail) for t in range(1, 3 * stages * pipes + 3)
                                       for r, tail in ((1, 5), (sm, 0), (sm // 2, 127))]:
            s = tile_schedule(n, sm, pipes, stages, slots)
            ref = _replay(n, sm, pipes, stages, slots)
            got = np.stack([s.cta, s.local, s.pipe, s.slot, s.stage, s.phase], axis=1)
            assert got.tolist() == [ref[t] for t in range(len(ref))], (shape, sm, n)
            assert (s.phase == s.round % 2).all() and s.ragged == (len(ref) - 1 if n % TILE else -1)


@pytest.mark.parametrize("sm", SMS)
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "%dx%d-slots%d" % s)
def test_sweep_covers_three_ring_rounds(shape, sm):
    pipes, stages, slots = shape
    sizes = ring_sweep(sm, pipes, stages, slots)
    assert sizes == sorted(set(sizes)) and sizes[0] >= 1 and len(sizes) <= 12, sizes
    assert sizes[-1] < 350_000, sizes          # bounds the GPU test's images and oracle time
    assert most_tiles_per_cta(sizes, sm, *shape) >= pipes * (2 * stages + 1)
    assert sweep_gaps(sizes, sm, *shape) == [], (shape, sm, sizes)


def test_gaps_are_reported():
    """the coverage check itself: a sweep without its largest launch misses round 2, one without the odd-round ragged
    launches misses those tiles"""
    sm, shape = 132, (2, 3, 2)
    sizes = ring_sweep(sm, *shape)
    assert any(g.startswith("round position") for g in sweep_gaps(sizes[:-1], sm, *shape))
    assert len([g for g in sweep_gaps(sizes[:2] + sizes[-1:], sm, *shape) if g.startswith("ragged")]) == 4
    assert sweep_gaps(sizes[2:], sm, *shape) == ["a CTA with one tile", "fewer tiles than SMs", "n % 128 = 1", "n % 128 = 127"]


# ---- GPU -------------------------------------------------------------------------------------------------------------------

def _int8_rows():
    rows = [(row, row, make) for row, make in CHAIN_ROWS]
    # an odd class count on a one-pipe row: the logits go out as 32-bit stores, not 64-bit ones
    rows.append(("<256,1>", "<256,1>-37cls", lambda: random_fc(4, (256, 256, 37), 4)))
    return rows


def _plan(capfd, monkeypatch, model):
    """an engine on the fused path built with BNM_VERBOSE set, and its plan line"""
    from bitnetmcu_b200 import _lib
    e, err = verbose_engine(capfd, monkeypatch, lambda: engine(model, _lib.PATH_TCGEN05))
    line = plan_line(err)
    assert line and e.active_path == _lib.PATH_TCGEN05, err
    return e, line


def _ring(line, row, kind):
    """(pipes, stages, slots) of `kind` ("int8", "float" or "emul") from the plan line, which must name `row` for it"""
    got, ring = plan_ring(line, kind)
    assert got == row, line
    return ring


def _int8_images(n, img_bytes, seed):
    """uniform random rows with, scattered through the whole batch, rail rows (all -128, all 127, random -128 / 127 mixes) and
    MNIST-like rows (background -20, strokes up to 127)"""
    rng = np.random.default_rng(seed)
    x = rng.integers(-128, 127, size=(n, img_bytes), dtype=np.int8, endpoint=True)
    kind = rng.integers(0, 10, size=n)
    x[kind == 0] = -128
    x[kind == 1] = 127
    mix = np.flatnonzero(kind == 2)
    x[mix] = np.where(rng.integers(0, 2, size=(mix.size, img_bytes), dtype=np.int8) == 1, np.int8(127), np.int8(-128))
    mn = np.flatnonzero(kind >= 7)
    x[mn] = np.where(rng.integers(0, 5, size=(mn.size, img_bytes), dtype=np.int8) == 0,
                     rng.integers(64, 127, size=(mn.size, img_bytes), dtype=np.int8, endpoint=True), np.int8(-20))
    return x


LOGIT_SENTINEL, LABEL_SENTINEL = -0x5A5A5A5B, -7


@pytest.mark.gpu
@pytest.mark.parametrize("row,make", [(r, m) for r, _, m in _int8_rows()], ids=[i for _, i, _ in _int8_rows()])
def test_int8_row_past_two_ring_rounds(lib, oracle, capfd, monkeypatch, row, make):
    """bnm_infer_batch_device (one launch) at every size of the row's sweep, on prefixes of one image buffer; logits and labels
    bit for bit, nothing written past row n; then labels alone at the largest size"""
    import torch
    m = make()
    e, line = _plan(capfd, monkeypatch, m)
    sw = Sweep(f"{row} ({m.n_classes} classes)", _ring(line, row, "int8"))
    imgs = _int8_images(sw.sizes[-1], m.img_bytes, zlib.crc32(row.encode()) + m.n_classes)
    want_lo, want_la = oracle.infer(m, imgs)
    d_img = torch.from_numpy(imgs).cuda()
    for n in sw.sizes:
        d_lo = torch.full((n + TILE, m.n_classes), LOGIT_SENTINEL, dtype=torch.int32, device="cuda")
        d_la = torch.full((n + TILE,), LABEL_SENTINEL, dtype=torch.int32, device="cuda")
        e.infer_device(d_img[:n], d_lo[:n], d_la[:n])
        torch.cuda.synchronize()
        sw.check(n, d_lo, want_lo, LOGIT_SENTINEL, "logits")
        sw.check(n, d_la, want_la, LABEL_SENTINEL, "labels")
    d_la.fill_(LABEL_SENTINEL)
    e.infer_device(d_img, None, d_la[:n])
    torch.cuda.synchronize()
    sw.check(n, d_la, want_la, LABEL_SENTINEL, "labels (labels-only launch)")
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["fc", "rand_fp130_64"])
def test_float_row_past_two_ring_rounds(lib, oracle, capfd, monkeypatch, name):
    """bnm_infer_batch_device_f32 (<64,1,float>, the quantiser warps fill the ring) over the sweep of its own stage count;
    expected: the NumPy float32 scaling, then the oracle"""
    import torch
    m = load_model(name)
    e, line = _plan(capfd, monkeypatch, m)
    row = "<64,1,float>"
    sw = Sweep(f"{row} ({name})", _ring(line, row, "float"))
    x = scattered_edge_images(sw.sizes[-1], m.img_bytes, zlib.crc32(name.encode()))
    want_lo, want_la = oracle.infer(m, scale_images(x))
    d_x = torch.from_numpy(x).cuda()
    for n in sw.sizes:
        d_lo = torch.full((n + TILE, m.n_classes), LOGIT_SENTINEL, dtype=torch.int32, device="cuda")
        d_la = torch.full((n + TILE,), LABEL_SENTINEL, dtype=torch.int32, device="cuda")
        e.infer_device_f32(d_x[:n], d_lo[:n], d_la[:n])
        torch.cuda.synchronize()
        sw.check(n, d_lo, want_lo, LOGIT_SENTINEL, "logits")
        sw.check(n, d_la, want_la, LABEL_SENTINEL, "labels")
    d_la.fill_(LABEL_SENTINEL)
    e.infer_device_f32(d_x, None, d_la[:n])
    torch.cuda.synchronize()
    sw.check(n, d_la, want_la, LABEL_SENTINEL, "labels (labels-only launch)")
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name,logit_scale", [("fc", 0.5), ("8bit64", 1.0)])
def test_emulator_row_past_two_ring_rounds(lib, capfd, monkeypatch, name, logit_scale):
    """bnm_emulate_batch_device (<64,1,float,emul>) over the sweep of the float stage count; expected: the NumPy restatement of
    the emulator, float64 logits bit for bit, labels = np.argmax"""
    import torch
    from bitnetmcu_b200 import model as M
    m = load_model(name)
    last = [l for l in m.layers if l.kind == M.LAYER_FC][-1]
    assert 2.0 ** -LEVEL_SHIFT.get(last.bitperweight, 0) == logit_scale, name   # both logit scales of the kernel
    e, line = _plan(capfd, monkeypatch, m)
    row = "<64,1,float,emul>"
    sw = Sweep(f"{row} ({name})", _ring(line, row, "emul"))
    x = scattered_edge_images(sw.sizes[-1], m.img_bytes, zlib.crc32(name.encode()) + 1)
    want_lo = emulate_fc(m, x)
    want_la = np.argmax(want_lo, axis=1)
    d_x = torch.from_numpy(x).cuda()
    sentinel = -12345.5
    for n in sw.sizes:
        d_lo = torch.full((n + TILE, m.n_classes), sentinel, dtype=torch.float64, device="cuda")
        d_la = torch.full((n + TILE,), LABEL_SENTINEL, dtype=torch.int32, device="cuda")
        e.inference_quantized_device(d_x[:n], d_lo[:n], d_la[:n])
        torch.cuda.synchronize()
        sw.check(n, d_lo, want_lo, sentinel, "logits")
        sw.check(n, d_la, want_la, LABEL_SENTINEL, "labels")
    d_la.fill_(LABEL_SENTINEL)
    e.inference_quantized_device(d_x, None, d_la[:n])
    torch.cuda.synchronize()
    sw.check(n, d_la, want_la, LABEL_SENTINEL, "labels (labels-only launch)")
    e.close()
