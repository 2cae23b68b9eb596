"""NumPy restatements the tests compare the GPU against, one copy of each: the reference caller's input scaling, the reference
Python emulator's FC and CNN paths, the C engine's CNN front-end stages and conv3 input bound, and the fused FC kernels' tile
schedule.  Pure NumPy: no torch, no CUDA library."""
from typing import NamedTuple

import numpy as np

from bitnetmcu_b200 import model as M, pack as P

LEVEL_SHIFT = {2: 1, 4: 1}          # 2bitsym / 4bitsym levels are half the engine's integer weights (BitNetMCU.py:155-164)
TILE = 128                          # images per tile (kTileM)


# ---- the emulator ---------------------------------------------------------------------------------------------------------

def scale_images(x):
    """float32 images -> int8, test_inference.py:140-141 and BitNetMCU.py:435-436 in float32:
    round_half_even(x * 127 / max(max|x|, 1e-5)).clip(-128, 127), then .astype(np.int8).  A row with any NaN or infinity
    becomes the all-zero row: max and np.maximum carry a NaN into the scale, an infinity makes the scale 0 (inf * 0 is NaN, any
    finite pixel +-0), and each NaN product casts to 0 -- what .astype(np.int8) gives on x86-64 and AArch64, stated here so the
    restatement does not depend on the platform's cast."""
    x = np.asarray(x, dtype=np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        scale = np.float32(127.0) / np.maximum(np.abs(x).max(axis=-1, keepdims=True), np.float32(1e-5))
        y = np.round(x * scale).clip(-128, 127)
    return np.where(np.isnan(y), np.float32(0), y).astype(np.int8)


def bitlinear(model, act, nf4_extension=False):
    """the BitLinear layers (BitNetMCU.py:452-457, 527-530) on activations [n, k] -> float64 logits: per layer a float64
    product with the weight levels, a power-of-two rescale of every row to a maximum of at most 127 with round-half-even and
    ReLU, and no rescale after the last layer.  The levels are the engine's integer weights over the level scale: 4bit layers
    take their integers (the reference's +0.01 offset is not), NF4 layers zeros, or the extension's LUT with nf4_extension."""
    fc = [l for l in model.layers if l.kind == M.LAYER_FC]
    act = act.astype(np.float64)
    for i, l in enumerate(fc):
        # weight levels over the columns the previous layer delivers (Ternary pads n_in with zero trits)
        w = P.decode_int_weights(l, nf4_extension).astype(np.float64)[:, :act.shape[1]] / 2.0 ** LEVEL_SHIFT.get(l.bitperweight, 0)
        conv = act @ w.T
        if i + 1 == len(fc):
            return conv
        top = np.maximum(conv.max(axis=-1, keepdims=True), 1e-5)
        act = np.round(conv * np.exp2(np.floor(np.log2(127.0 / top)))).clip(0, 127)


def emulate_fc(model, x, nf4_extension=False):
    """float32 images [n, img_bytes] of an FC model -> the emulator's float64 logits [n, n_classes]"""
    return bitlinear(model, scale_images(x), nf4_extension)


def _conv_relu(a, w):
    """depthwise 3x3 (k_conv33relu's indices, no shift) + ReLU: a int64 [n, 1 or C, H, W], w int8 [C * 9] -> [n, C, H-2, W-2]"""
    n, _, h, wd = a.shape
    k = w.reshape(-1, 3, 3).astype(np.int64)
    out = np.zeros((n, k.shape[0], h - 2, wd - 2), dtype=np.int64)
    for dr in range(3):
        for dc in range(3):
            out += k[None, :, dr, dc, None, None] * a[:, :, dr:dr + h - 2, dc:dc + wd - 2]
    return np.maximum(out, 0)


def _renorm(v, rounding=np.round):
    """BitConv2d's renormalisation over each image's C*H*W outputs (float64); an all-zero image stays zero"""
    m = v.reshape(v.shape[0], -1).max(axis=1)
    scale = np.where(m > 0, 127.0 / np.maximum(m, 1), 0.0)[:, None, None, None]
    return rounding(v * scale).clip(0, 127).astype(np.int64)


def _pool(v):
    n, c, h, w = v.shape
    return v.reshape(n, c, h // 2, 2, w // 2, 2).max(axis=(3, 5))


def _conv_weights(model):
    return [l.weights for l in model.layers if l.kind == M.LAYER_CONV33]


def cnn_stages(model, x, rounding=np.round):
    """float32 images [n, 256] -> (conv1, conv2, conv3, features): the ReLU output of each convolution before its
    renormalisation (int64 [n, C, H, W]) and the int64 features [n, C*4], the (C, 2, 2) flatten.  rounding: the
    renormalisation's (np.round, half to even, is the emulator's)"""
    w1, w2, w3 = _conv_weights(model)
    c1 = _conv_relu(scale_images(x).astype(np.int64).reshape(-1, 1, 16, 16), w1)
    c2 = _conv_relu(_renorm(c1, rounding), w2)
    c3 = _conv_relu(_pool(_renorm(c2, rounding)), w3)
    f = _pool(_renorm(c3, rounding))
    return c1, c2, c3, f.reshape(f.shape[0], -1)


def cnn_features(model, x):
    """float32 images [n, 256] -> int64 features [n, C*4], the (C, 2, 2) flatten"""
    return cnn_stages(model, x)[3]


def emulate(model, x, block=512, nf4_extension=False):
    """float32 images -> the emulator's float64 logits, FC and CNN models; NF4 layers decoded as BNM_OPT_NF4_EXTENSION says"""
    if model.model_class == 0:
        return emulate_fc(model, x, nf4_extension)
    return np.concatenate([bitlinear(model, cnn_features(model, x[i:i + block]), nf4_extension) for i in range(0, len(x), block)])


# ---- the C engine's CNN front-end (dll.c:64-80) ------------------------------------------------------------------------------

def conv3_channel_bounds(model):
    """per channel, the largest pooled conv2 output (conv3's input) any int8 image can give, from the conv1 / conv2 weights:
    ((127 sum(w1 > 0) + 128 sum|w1 < 0|) >> 4) sum(w2 > 0) >> 4 -> int64 [C]"""
    w1, w2, _ = (w.astype(np.int64).reshape(-1, 9) for w in _conv_weights(model))
    b1 = (127 * np.where(w1 > 0, w1, 0).sum(axis=1) + 128 * np.where(w1 < 0, -w1, 0).sum(axis=1)) >> 4
    return (b1 * np.where(w2 > 0, w2, 0).sum(axis=1)) >> 4


def conv3_bound(model):
    """cnn_conv3_bound (generic_kernels.cu): the maximum of conv3_channel_bounds"""
    return int(conv3_channel_bounds(model).max())


def relunorm(v):
    """orc_ReLUNorm (inference.c:23-72) on rows int64 [n, k] without the argmax: shift = bit length of (max >> 7), then
    min(127, (x + rounding) >> shift) with rounding = (1 << shift) >> 1, negatives to 0"""
    m = v.max(axis=1)
    shift = np.array([int(t).bit_length() if t > 0 else 0 for t in m >> 7], dtype=np.int64)[:, None]
    return np.where(v < 0, 0, np.minimum(127, (v + ((1 << shift) >> 1)) >> shift))


class Frontend(NamedTuple):
    conv1: np.ndarray       # int64 [n, C, 14, 14]: processconv33ReLU(image, w1, 16, 4)
    conv2: np.ndarray       # [n, C, 6, 6]: processconv33ReLU(conv1, w2, 14, 4), pooled -- conv3's inputs
    conv3: np.ndarray       # [n, C, 2, 2]: processconv33ReLU(conv2, w3, 6, 4), pooled
    raw: np.ndarray         # [n, C*4]: the features before ReLUNorm, channel-major
    features: np.ndarray    # [n, C*4]: after ReLUNorm (dll.c:80)


def c_frontend(model, images):
    """the C engine's front-end (orc_processconv33ReLU / orc_processmaxpool22, bitnet_oracle.c) on int8 images [n, 256], int64
    throughout: conv = ReLU(sum) >> 4 with no rounding or clip"""
    w1, w2, w3 = _conv_weights(model)
    a = np.asarray(images, dtype=np.int8).astype(np.int64).reshape(-1, 1, 16, 16)
    c1 = _conv_relu(a, w1) >> 4
    c2 = _pool(_conv_relu(c1, w2) >> 4)
    c3 = _pool(_conv_relu(c2, w3) >> 4)
    raw = c3.reshape(c3.shape[0], -1)
    return Frontend(c1, c2, c3, raw, relunorm(raw))


# ---- the fused FC plan (fc_chain_plan_create, fc_wgmma.cu) ------------------------------------------------------------------
# The constants, each from the line of fc_wgmma.cu named beside it.  A wrong one shows on the GPU, where
# test_plan_shapes.test_plan_line compares the restated plan line with the library's.

SMEM_LIMIT = 227 * 1024 - 1024 - 1024          # :1192 an SM's 227 kB less the alignment slack and the static barriers
MAX_STAGES = 8                                  # :36 kMaxStages, ring stages over all pipes of a CTA
FLOAT_RING_BYTES = 8 * 2 * 4 * 256              # :1206 fring / element byte: kFloatQuantWarps (:38) x 2 slots x kFloatGroupRows (:40) x 256
FIXED_OUT_BYTES = 2 * 8 * (16 * 16 * 4 + 16 * 4)  # :334-336 kFixedOutBytes, the fixed-shape row's logits staging
MIN_SMEM = 116 * 1024                           # :1221 every form asks for more than half the SM: one CTA per SM
FIXED_SHAPE = dict(in_atoms=2, n_pad=[64, 64, 64, 16], k_steps=[8, 2, 2, 2], b_off=[0, 16384, 20480, 24576])   # :327-331
TWO_PIPE_ROWS = {"full": "fc_chain_kernel<64,2,2,64>", "last16": "fc_chain_kernel<64,2,2,16>",
                 "fixed": "fc_chain_kernel<64,2,2,16,fixed>"}                                                   # :1154-1158


class FormSpec(NamedTuple):
    in_bytes: int           # bytes per input element: 1 int8 rows, 4 float32, 2 float16 / bfloat16
    stage_cap: int          # stages per pipe at most
    rows: dict              # accumulator width -> kernel row name (the float-input forms: 64 only)


def _rows(fmt, widths=(64, 128, 192, 256)):
    return {n: fmt % n for n in widths}


FORMS = {   # :1124-1151 kForms, in FcForm order
    "int8": FormSpec(1, 6, _rows("fc_chain_kernel<%d,1>")),
    "float": FormSpec(4, 4, _rows("fc_chain_kernel<%d,1,float>", (64,))),
    "emul_float": FormSpec(4, 4, _rows("fc_emul_kernel<%d,1,float,emul>", (64,))),
    "emul_i8": FormSpec(1, 6, _rows("fc_emul_i8_kernel<%d,1,emul>")),
    "engines": FormSpec(4, 4, _rows("fc_engines_kernel<%d,1,float,engines>", (64,))),
    "topk": FormSpec(1, 6, _rows("fc_topk_kernel<%d,1,topk>")),
    "emul_topk": FormSpec(1, 6, _rows("fc_topk_kernel<%d,1,emul,topk>")),
    "float16": FormSpec(2, 4, _rows("fc_chain_h16_kernel<%d,1,16bit>", (64,))),
    "emul_float16": FormSpec(2, 4, _rows("fc_emul_h16_kernel<%d,1,16bit,emul>", (64,))),
    "engines16": FormSpec(2, 4, _rows("fc_engines_h16_kernel<%d,1,16bit,engines>", (64,))),
}
REFUSE_LAYERS = "fused path: 1..8 FC layers"
REFUSE_ROW = "fused path: input row must be a multiple of 16 bytes, <= 1024"
REFUSE_WIDE = "fused path: layer wider than 256 outputs"
REFUSE_SMEM = "fused path: weights do not fit in shared memory"


class Form(NamedTuple):
    row: str                # the kernel row's name
    stages: int             # per pipe
    smem: int               # dynamic shared memory of a launch


class Plan(NamedTuple):
    in_atoms: int           # the input row in 128-byte atoms
    n_pad: list             # per layer: outputs rounded up to 16
    k_steps: list           # per layer: K-steps of 32 in the weight image
    planes: list            # per layer: 2 where the layer holds a +128 weight (FP130), else 1
    b_off: list             # per layer: byte offset of its first plane in the weight image
    w_bytes: int            # the weight image, the zero tile behind the layers included
    max_n: int              # the accumulator width: 64, 128, 192 or 256
    pipes: int              # of the int8 C-engine form
    two_pipe_row: str       # "fixed", "last16" or "full" with two pipes, else ""
    float_fits: bool        # rows, classes and shared memory admit the float-input forms' rings
    forms: dict             # form name -> Form, for the forms the plan has
    logit_scale: float      # the emulator's logits: the last layer's accumulators times this

    @property
    def row(self):
        """the int8 C-engine form's row, its template arguments only ("<64,2,2,16>")"""
        return self.forms["int8"].row[self.forms["int8"].row.index("<"):]

    @property
    def float_forms(self):
        return "float" in self.forms


def _up(x, m):
    return -(-x // m) * m


def plan_of(model, nf4_extension=False):
    """fc_chain_plan_create's shape rules on an FC model (img_bytes-byte rows): the Plan, or the refusal message"""
    fc = model.fc_layers
    in_bytes = model.img_bytes
    if not 1 <= len(fc) <= 8:
        return REFUSE_LAYERS
    if in_bytes % 16 or in_bytes == 0 or in_bytes > 1024:
        return REFUSE_ROW
    n_pad = [_up(l.n_out, 16) for l in fc]
    k_pad = [_up(max(l.n_in, 1), 32) for l in fc]
    if max(n_pad) > 256:
        return REFUSE_WIDE
    in_atoms = -(-in_bytes // 128)
    stage = in_atoms * 16384
    # K of layer l > 0 stops at the previous layer's padded width: the activations past it are zero
    k_steps = [4 * in_atoms] + [_up(min(k_pad[l], n_pad[l - 1]), 32) // 32 for l in range(1, len(fc))]
    planes = [1 + int((P.decode_int_weights(l, nf4_extension) == 128).any()) for l in fc]
    sizes = [p * k * n * 32 for p, k, n in zip(planes, k_steps, n_pad)]
    b_off = [int(s) for s in np.cumsum([0] + sizes[:-1])]
    max_n = _up(max(n_pad), 64)
    w_bytes = sum(sizes) + max_n * 32
    w_fixed = _up(w_bytes, 128)
    if w_fixed + 2 * stage > SMEM_LIMIT:
        return REFUSE_SMEM
    pipes = 2 if max_n == 64 and (SMEM_LIMIT - w_fixed) // stage >= 4 else 1
    last16 = n_pad[-1] <= 16
    fixed = pipes == 2 and last16 and planes == [1] * len(fc) and \
        dict(in_atoms=in_atoms, n_pad=n_pad, k_steps=k_steps, b_off=b_off) == FIXED_SHAPE
    two_pipe_row = ("fixed" if fixed else "last16" if last16 else "full") if pipes == 2 else ""
    float_fits = in_bytes <= 256 and fc[-1].n_out <= 16 and w_fixed + 4 * FLOAT_RING_BYTES + 2 * stage <= SMEM_LIMIT
    forms = {}
    for name, s in FORMS.items():
        np_ = pipes if name == "int8" else 1
        row = TWO_PIPE_ROWS[two_pipe_row] if np_ == 2 else s.rows.get(max_n)
        if row is None or (s.in_bytes > 1 and not float_fits):
            continue
        extra = s.in_bytes * FLOAT_RING_BYTES if s.in_bytes > 1 else FIXED_OUT_BYTES if fixed and name == "int8" else 0
        stages = min(s.stage_cap, MAX_STAGES // np_, (SMEM_LIMIT - w_fixed - extra) // stage // np_)
        forms[name] = Form(row, stages, max(np_ * stages * stage + w_fixed + extra + 1024, MIN_SMEM))
    return Plan(in_atoms, n_pad, k_steps, planes, b_off, w_bytes, max_n, pipes, two_pipe_row, float_fits, forms,
                2.0 ** -LEVEL_SHIFT.get(fc[-1].bitperweight, 0))


def plan_lines(plan):
    """the two lines fc_chain_plan_create prints under BNM_VERBOSE (fc_wgmma.cu:1233-1246) for a Plan"""
    f = plan.forms
    i8 = f["int8"]
    fl = (f", float input {f['float'].row[f['float'].row.index('<'):]}, emulator {f['emul_float'].row[f['emul_float'].row.index('<'):]}"
          f", float input stages {f['float'].stages}") if plan.float_forms else ""
    return (f"bitnetmcu_b200: fused FC plan: {plan.max_n} accumulator columns, {plan.pipes} pipes x {i8.stages} stages, "
            f"{plan.w_bytes} weight bytes, {i8.smem} B smem, {i8.row}{fl}, int8 emulator {f['emul_i8'].row} x {f['emul_i8'].stages} stages",
            f"bitnetmcu_b200: fused FC top-k forms: {f['topk'].row} x {f['topk'].stages} stages, emulator {f['emul_topk'].row} x "
            f"{f['emul_topk'].stages} stages, {f['topk'].smem} B smem")


# ---- the fused FC kernels' tile schedule (tests/test_fc_ring_rounds.py) -----------------------------------------------------

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


def batch_size(sm, t, r, tail):
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
    return sorted({batch_size(sm, t, min(r, sm), tail) for t, r, tail in launches})


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
