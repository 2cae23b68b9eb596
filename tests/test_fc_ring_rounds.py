"""The fused FC kernels past their first trips round the tile ring (fc_wgmma.cu; DESIGN.md 4.1, "Synchronisation").

fc_chain_kernel and fc_emul_kernel are persistent.  CTA b of a grid of min(n_tiles, SMs) takes the 128-image tiles b, b + grid,
b + 2 grid, ...  Its local tile i goes to pipe i % pipes, and j = i / pipes is its place in that pipe: slot j % slots (two-slot
kernels: slot A the even j, slot B the odd ones), stage j % stages, ring round j / stages, phase parity round & 1.  A wrong phase
flip, empty-barrier wait or epilogue tile index shows only once a CTA has run more tiles than its pipe has stages, and every
launch starts again from stage 0, phase 0, so it takes one launch with enough tiles per CTA to get there.

CPU: a restatement of that schedule (checked against the kernel's own running counters), and per ring shape a short sweep of
batch sizes whose coverage is checked.  GPU (tolerance 0): every kernel row, its ring shape read from the plan's BNM_VERBOSE line
and the SM count from the device, over its sweep -- one launch per batch size on a prefix of one device buffer -- against the
oracle (int8 and float input) or the NumPy restatement of the emulator."""
import zlib
from typing import NamedTuple

import numpy as np
import pytest

from conftest import load_model

TILE = 128          # images per tile (kTileM)


# ---- the tile schedule, restated -------------------------------------------------------------------------------------------

class Schedule(NamedTuple):
    """One launch of n images; the per-tile arrays are indexed by global tile."""
    n: int
    grid: int
    cta: np.ndarray
    local: np.ndarray       # index among the CTA's tiles
    pipe: np.ndarray
    slot: np.ndarray        # 0 = slot A, 1 = slot B
    stage: np.ndarray       # stage inside the pipe
    phase: np.ndarray
    round: np.ndarray
    ragged: int             # the tile that holds fewer than 128 images, -1 when n is a multiple of 128
    per_pipe: np.ndarray    # [grid, pipes]: tiles of each CTA's pipe
    end_slot: np.ndarray    # [grid, pipes]: slot of the last of them (-1: the pipe has no tile)


def tile_schedule(n, sm, pipes, stages, slots):
    n_tiles = -(-n // TILE)
    grid = min(n_tiles, sm)
    t = np.arange(n_tiles)
    cta, local = t % grid, t // grid
    pipe, j = local % pipes, local // pipes
    rnd = j // stages
    per_pipe = np.zeros((grid, pipes), dtype=np.int64)
    np.add.at(per_pipe, (cta, pipe), 1)
    end_slot = np.where(per_pipe > 0, (per_pipe - 1) % slots, -1)
    return Schedule(n, grid, cta, local, pipe, j % slots, j % stages, rnd & 1, rnd, n_tiles - 1 if n % TILE else -1,
                    per_pipe, end_slot)


def top_tiles(pipes, stages, slots):
    """tiles per CTA that take every stage of every pipe (and so every slot that meets it) through rounds 0, 1 and 2: each phase
    parity of every stage is waited on at least twice, counting the full and the empty barrier.  That is at least
    pipes (2 stages + 1) + pipes slots whenever a pipe of two slots has three or more stages."""
    return 3 * stages * pipes


def _batch(sm, t, r, tail):
    """n for (t - 1) sm + r tiles, the last of them holding `tail` images (0: a full tile).  With r <= sm that last tile is
    local tile t - 1 of CTA r - 1."""
    return ((t - 1) * sm + r) * TILE - ((TILE - tail) if tail else 0)


def ring_sweep(sm, pipes, stages, slots):
    """ascending batch sizes that, launched one after the other, cover the ring: see sweep_gaps"""
    launches = [(1, max(1, sm // 2), 1),        # fewer tiles than SMs, one per CTA; n % 128 = 1
                (2, max(1, sm // 3), 127)]      # CTAs from r on hold one tile, the others two; n % 128 = 127
    k, ends = 0, pipes * slots
    for p in range(pipes):
        for x in range(slots):
            j = stages + (x - stages) % slots   # the first place of round 1 that slot x takes
            launches.append((j * pipes + p + 1, 1 + (sm - 1) * (k + 1) // (ends + 1), 40 + 23 * k))   # ragged last tile there
            k += 1
    launches.append((top_tiles(pipes, stages, slots), sm // 2 + 1, 0))   # rounds 0 to 2 everywhere; n % 128 = 0
    return sorted({_batch(sm, t, min(r, sm), tail) for t, r, tail in launches})


def sweep_gaps(sizes, sm, pipes, stages, slots):
    """what a sweep of launches leaves uncovered (empty: nothing):
      * every (pipe, slot, stage) the schedule puts in rounds 0, 1 and 2;
      * the ragged last tile on every (pipe, slot), in an odd round;
      * a CTA with one tile, and a launch with fewer tiles than SMs;
      * a CTA's pipe with an odd tile count (slot B idles at the end) and one with an even count (slot A idles);
      * n % 128 in {0, 1, 127}."""
    want = {(p, j % slots, j % stages, j // stages) for p in range(pipes) for j in range(3 * stages)}
    want_ragged = {(p, x) for p in range(pipes) for x in range(slots)}
    seen, ragged, misc = set(), set(), set()
    for n in sizes:
        s = tile_schedule(n, sm, pipes, stages, slots)
        seen |= set(zip(s.pipe.tolist(), s.slot.tolist(), s.stage.tolist(), s.round.tolist()))
        if s.ragged >= 0 and s.round[s.ragged] % 2:
            ragged.add((int(s.pipe[s.ragged]), int(s.slot[s.ragged])))
        if (s.per_pipe.sum(axis=1) == 1).any():
            misc.add("a CTA with one tile")
        if s.grid < sm:
            misc.add("fewer tiles than SMs")
        if ((s.per_pipe % 2 == 1) & (s.end_slot == 0)).any():
            misc.add("odd per-pipe count")
        if ((s.per_pipe % 2 == 0) & (s.per_pipe > 0) & (s.end_slot == slots - 1)).any():
            misc.add("even per-pipe count")
        misc.add(f"n % 128 = {n % TILE}")
    gaps = [f"round position {w}" for w in sorted(want - seen)]
    gaps += [f"ragged last tile on (pipe, slot) {w} in an odd round" for w in sorted(want_ragged - ragged)]
    gaps += [m for m in ("a CTA with one tile", "fewer tiles than SMs", "odd per-pipe count", "even per-pipe count",
                         "n % 128 = 0", "n % 128 = 1", "n % 128 = 127") if m not in misc]
    return gaps


def most_tiles_per_cta(sizes, sm, pipes, stages, slots):
    return max(int(tile_schedule(n, sm, pipes, stages, slots).local.max()) + 1 for n in sizes)


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
        for n in [1, 127, 128, 129] + [_batch(sm, t, r, tail) for t in range(1, 3 * stages * pipes + 3)
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

@pytest.fixture(scope="module")
def lib(built):
    from bitnetmcu_b200 import _lib
    l = _lib.load()
    assert l.bnm_device_count() > 0, "no CUDA device"
    return l


def _int8_rows():
    from test_labels_only import _ROWS, _random
    rows = [(row, row, make) for row, make in _ROWS]
    # an odd class count on a one-pipe row: the logits go out as 32-bit stores, not 64-bit ones
    rows.append(("<256,1>", "<256,1>-37cls", lambda: _random(4, (256, 256, 37), 4)))
    return rows


def _plan(capfd, monkeypatch, model):
    """an engine on the fused path built with BNM_VERBOSE set, and its plan line"""
    from bitnetmcu_b200 import _lib
    from bitnetmcu_b200.engine import Engine
    monkeypatch.setenv("BNM_VERBOSE", "1")
    capfd.readouterr()
    e = Engine(model, device=0, path=_lib.PATH_TCGEN05)
    lines = [l for l in capfd.readouterr().err.splitlines() if "fused FC plan" in l]
    monkeypatch.delenv("BNM_VERBOSE")
    assert lines and e.active_path == _lib.PATH_TCGEN05, lines
    return e, lines[-1]


def _ring(line, row, kind):
    """(pipes, stages, slots) of `kind` ("int8", "float" or "emul") from the plan line, which must name `row` for it"""
    import re
    if kind == "int8":
        assert re.search(r"fc_chain_kernel(<[^>]*>)", line).group(1) == row, line
        pipes, stages = map(int, re.search(r"(\d+) pipes x (\d+) stages", line).groups())
        fields = row[1:-1].split(",")
        assert int(fields[1]) == pipes, line
        return pipes, stages, int(fields[2]) if pipes == 2 else 1
    assert (f"float input {row}" if kind == "float" else f"emulator {row}") in line, line
    return 1, int(re.search(r"float input stages (\d+)", line).group(1)), 1


class _Sweep:
    """the sweep of one case on this GPU, and the tag every assertion message of the case carries"""

    def __init__(self, row, ring):
        import torch
        self.ring = ring
        self.sm = torch.cuda.get_device_properties(0).multi_processor_count
        self.sizes = ring_sweep(self.sm, *ring)
        self.top = most_tiles_per_cta(self.sizes, self.sm, *ring)
        self.tag = "%s: %d pipes x %d stages, %d slots, %d SMs, up to %d tiles per CTA" % ((row,) + ring + (self.sm, self.top))
        print(self.tag, "batch sizes", self.sizes)
        assert self.top >= ring[0] * (2 * ring[1] + 1), self.tag
        assert not sweep_gaps(self.sizes, self.sm, *ring), self.tag

    def where(self, n, rows):
        """(tile, CTA, local index, pipe, slot, stage, round) of the tiles that hold the given rows of launch n"""
        s = tile_schedule(n, self.sm, *self.ring)
        return [(int(t), int(s.cta[t]), int(s.local[t]), int(s.pipe[t]), "AB"[s.slot[t]], int(s.stage[t]), int(s.round[t]))
                for t in np.unique(np.asarray(rows) // TILE)[:6]]

    def check(self, n, got, want, sentinel, what):
        """rows :n of the (n + 128)-row device buffer `got` equal `want`; rows n: still hold the sentinel"""
        g = got.cpu().numpy()
        if what == "labels":
            g = g.astype(np.uint32) if want.dtype == np.uint32 else g.astype(np.int64)
        bad = np.flatnonzero((g[:n] != want[:n]).reshape(n, -1).any(axis=1))
        assert bad.size == 0, (self.tag, n, what, f"{bad.size} rows wrong, first {bad[:4].tolist()}",
                               "(tile, cta, local, pipe, slot, stage, round):", self.where(n, bad))
        assert (got[n:].cpu().numpy() == sentinel).all(), (self.tag, n, what, "written past row n")


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


def _float_images(n, elems, seed):
    """normal rows with, scattered through the whole batch, MNIST-normalised rows and rows at the edges of the input scaling:
    all zero (the 1e-5 floor), exact .5 ties after scaling, one huge pixel, constant negative rows"""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal(size=(n, elems), dtype=np.float32)
    kind = rng.integers(0, 10, size=n)
    mn = np.flatnonzero(kind >= 6)
    x[mn] = (rng.integers(0, 256, size=(mn.size, elems)) / 255.0 - 0.1307).astype(np.float32) / np.float32(0.3081)
    x[kind == 0] = 0.0
    x[kind == 1] = np.float32(0.5) / np.float32(127.0) * np.arange(elems, dtype=np.float32)
    x[kind == 2, 0] = np.float32(3e38)
    x[kind == 3] = -1.0
    return x


def _quantize(x):
    """the input scaling of the reference's caller in NumPy float32 (test_inference.py:140-141)"""
    scale = np.float32(127.0) / np.maximum(np.abs(x).max(axis=-1, keepdims=True), np.float32(1e-5))
    return np.round(x * scale).clip(-128, 127).astype(np.int8)


LOGIT_SENTINEL, LABEL_SENTINEL = -0x5A5A5A5B, -7


@pytest.mark.gpu
@pytest.mark.parametrize("row,make", [(r, m) for r, _, m in _int8_rows()], ids=[i for _, i, _ in _int8_rows()])
def test_int8_row_past_two_ring_rounds(lib, oracle, capfd, monkeypatch, row, make):
    """bnm_infer_batch_device (one launch) at every size of the row's sweep, on prefixes of one image buffer; logits and labels
    bit for bit, nothing written past row n; then labels alone at the largest size"""
    import torch
    m = make()
    e, line = _plan(capfd, monkeypatch, m)
    sw = _Sweep(f"{row} ({m.n_classes} classes)", _ring(line, row, "int8"))
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
    sw = _Sweep(f"{row} ({name})", _ring(line, row, "float"))
    x = _float_images(sw.sizes[-1], m.img_bytes, zlib.crc32(name.encode()))
    want_lo, want_la = oracle.infer(m, _quantize(x))
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
    from test_emulator_device import LEVEL_SHIFT, emulate_fc
    m = load_model(name)
    last = [l for l in m.layers if l.kind == M.LAYER_FC][-1]
    assert 2.0 ** -LEVEL_SHIFT.get(last.bitperweight, 0) == logit_scale, name   # both logit scales of the kernel
    e, line = _plan(capfd, monkeypatch, m)
    row = "<64,1,float,emul>"
    sw = _Sweep(f"{row} ({name})", _ring(line, row, "emul"))
    x = _float_images(sw.sizes[-1], m.img_bytes, zlib.crc32(name.encode()) + 1)
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
