"""The fused FC kernels' epilogue and hidden-layer rules at their edges (fc_wgmma.cu: the epilogue's argmax and row stores,
row_label, norm_coef, emul_coef; generic_kernels.cu behind BNM_PATH_LAYERS).

The contract: the label is the first maximum of the logits (strict '>' from -INT32_MAX, position 255; inference.c:32-37);
columns at or past n_classes take no part; rows of an even class count go out as 64-bit stores, odd ones as 32-bit stores; the
C engine's ReLUNorm (inference.c:41-67) and the emulator's rule (BitNetMCU.py:452-457) are exact at their shift, rounding and
clip boundaries.  Random models reach these edges only by chance, so the models here are built from integer weights whose
logits the test sets exactly:

* identity chains: layer 1 routes pixel perm[c] to unit c with weight 1, the hidden layers pass unit c on, the head is +-identity.
  A row maximum <= 127 has shift 0, so the logits are x[perm] (one layer) or +-relu(x[perm]) (deeper);
* one-layer 8bit and FP130 models on 768-byte rows, weights at -128 (8bit) or +128 (FP130's residual plane) and images at the
  rails: logits past 2^23;
* a layer 1 whose units are 127 S + 127 a + b (S: a gain block of pixels shared by some units, a and b: two private pixels),
  identity layers behind it: the logits are the hidden activations, and the pixels put each unit exactly on a boundary.

The crafted rows are few; a batch repeats them (row i holds pattern i % P, P odd), so every pattern lands on every row of a tile,
both rows of a thread, both warpgroup halves, and the sweep's largest launch (one ragged image short) puts them in every pipe,
slot, stage and ring round.

CPU: the fixtures hit what they are built for, and a NumPy restatement of the C rule equals the oracle's ReLUNorm.  GPU
(tolerance 0): every kernel row and entry point against the oracle (C engine) and restate.emulate_fc (emulator), each model's
row read from its BNM_VERBOSE lines."""
import itertools
import zlib

import numpy as np
import pytest

from restate import TILE, emulate_fc, scale_images
from support import N_MANY, Sweep, engine, gather_call, lib, plan_line, plan_ring, route, run_emulator, verbose_engine

# bitnetmcu_b200.model's encoding ids (checked in test_encoding_ids)
ENC_4BIT, ENC_8BIT, ENC_FP130, ENC_TERNARY = 12, 16, 20, 64
CHAIN_ENCS = [ENC_4BIT, ENC_TERNARY, ENC_8BIT]     # the deeper identity chains take these in turn: Ternary pads every K to 10s


# ---- builders --------------------------------------------------------------------------------------------------------------

def _fc(name, enc, w):
    from bitnetmcu_b200 import pack as P
    w = np.asarray(w, dtype=np.int64)
    if enc == ENC_TERNARY:
        return P.fc_layer_from_trits(name, w)
    return P.fc_layer_from_codes(name, enc, P.codes_from_int_weights(enc, w))


def _model(weights, img_bytes, enc=ENC_8BIT):
    from bitnetmcu_b200 import model as M
    m = M.Model(model_class=M.MODEL_FCMNIST, layers=[_fc(f"L{i + 1}", enc, w) for i, w in enumerate(weights)], img_bytes=img_bytes)
    m.validate()
    return m


def identity_chain(img_bytes, hidden, n_classes, sign, seed, enc=ENC_8BIT):
    """-> (model, perm): layer 1 routes pixel perm[c] to unit c, the hidden layers are identities, the head is sign x identity
    on the first n_classes units"""
    perm = np.random.default_rng(seed).permutation(img_bytes)
    outs, ws, n_in = list(hidden) + [n_classes], [], img_bytes
    k = np.arange(n_classes)
    for l, n_out in enumerate(outs):
        w = np.zeros((n_out, n_in), dtype=np.int64)
        w[k, perm[k] if l == 0 else k] = sign if l + 1 == len(outs) else 1
        ws.append(w)
        n_in = n_out
    return _model(ws, img_bytes, enc), perm


def _pairs(C):
    """every pair when C <= 16; else pairs in one thread (2q / 2q+1, c / c+8), across quad lanes, 16-column blocks and 64-column
    pieces, and the last columns"""
    if C <= 16:
        return list(itertools.combinations(range(C), 2))
    cand = [(0, 1), (2, 3), (6, 7), (12, 13), (0, 8), (3, 11), (7, 15), (16, 24), (0, 2), (1, 3), (1, 6), (4, 7), (5, 10), (15, 16),
            (7, 16), (0, 16), (16, 32), (31, 32), (17, 49), (63, 64), (0, 64), (5, 69), (62, 65), (64, 128), (127, 128), (0, 128),
            (100, 130), (128, 192), (191, 192), (0, 192), (130, 250), (200, 255), (0, C - 1), (C - 2, C - 1), (C // 2, C - 1)]
    return sorted({(i, j) for i, j in cand if i < j < C})


def argmax_rows(C, lo, hi, seed, anchor=False):
    """crafted logit rows for C classes, values in [lo, hi] -> (L int64 [P, C] with P odd, the planned maximum columns per row).
    Patterns: all equal; the maximum tied at pairs; three-way ties with the last column; a unique maximum at every column; v at j
    with v - 1 at i < j and the reverse; tops cycle through positive, zero and negative values where [lo, hi] allows (negative
    tops: all-negative rows).  anchor: every row holds a value of magnitude 127."""
    rng = np.random.default_rng(seed)
    tops = list(dict.fromkeys(t for t in (hi, hi - 1, (lo + hi) // 2, 1, 0, -1, lo + 1) if lo < t <= hi))
    rows, planned = [], []

    def add(vals, top):
        if top == lo and len(vals) < C:
            return
        r = rng.integers(lo, top, size=C) if top > lo else np.full(C, lo)
        for c, v in vals.items():
            r[c] = v
        if anchor and np.abs(r).max() != 127:
            free = [c for c in range(C) if c not in vals]
            if not free or lo > -127:
                return
            r[free[0]] = -127
        rows.append(r)
        planned.append(sorted(c for c, v in vals.items() if v == top))

    for t in tops + [lo, 127 if hi == 127 else lo, -127 if lo == -127 else hi]:
        add({c: t for c in range(C)}, t)
    pairs = _pairs(C)
    for k, (i, j) in enumerate(pairs):
        t = tops[k % len(tops)]
        add({i: t, j: t}, t)
        if t - 1 >= lo:
            add({j: t, i: t - 1}, t)
            add({i: t, j: t - 1}, t)
    if C >= 3:
        for k, (i, j) in enumerate(p for p in pairs if p[1] < C - 1):
            t = tops[k % len(tops)]
            add({i: t, j: t, C - 1: t}, t)
        add({C - 3: tops[0], C - 2: tops[0], C - 1: tops[0]}, tops[0])
    for c in range(C):
        t = tops[c % len(tops)]
        add({c: t}, t)
    if len(rows) % 2 == 0:
        rows.append(rows[0].copy())
        planned.append(planned[0])
    return np.stack(rows).astype(np.int64), planned


def argmax_images(L, perm, img_bytes, sign, seed):
    """int8 images whose pixel perm[c] holds sign * L[:, c] (the deep -I head gets -L), the other pixels random; pixel
    perm[C] (when there is one) is the 127 anchor of the float forms' scaling"""
    rng = np.random.default_rng(seed)
    C = L.shape[1]
    q = rng.integers(-127, 128, size=(L.shape[0], img_bytes))
    q[:, perm[:C]] = L * sign
    if C < img_bytes:
        q[:, perm[C]] = np.where(np.arange(L.shape[0]) % 2, 127, -127)
    assert np.abs(q).max() <= 127
    return q.astype(np.int8)


# (row, [(img_bytes, hidden widths)], class counts).  A one-layer 8bit model (logits = x[perm], values of both signs) and a
# deeper identity chain in 4bit, Ternary or 8bit (+I head on even class counts: logits >= 0, -I on odd ones: logits <= 0) per
# class count.  One layer on 768-byte rows has a fused plan up to 32 classes (two 96 kB stages and 24 K-steps x n_pad weight
# bytes); at 64 classes it runs layer by layer.
ARGMAX_ROWS = [
    ("<64,2,2,16>", [(256, ()), (256, (64, 64))], [1, 2, 3, 7, 8, 9, 15, 16]),
    ("<64,2,2,16,fixed>", [(256, (64, 64, 64))], [1, 2, 3, 7, 8, 9, 15, 16]),
    ("<64,2,2,64>", [(256, ()), (256, (64, 64))], [17, 31, 32, 33, 63, 64]),
    ("<64,1>", [(512, ()), (512, (64,)), (768, ())], [1, 10, 17, 64]),
    ("<128,1>", [(256, ()), (256, (128,))], [65, 127, 128]),
    ("<192,1>", [(256, ()), (256, (192,))], [129, 191, 192]),
    ("<256,1>", [(256, ()), (256, (256,))], [193, 255, 256]),
]
ARGMAX_CASES = [(row, shapes, C) for row, shapes, counts in ARGMAX_ROWS for C in counts]


def fused_768(C):
    return C <= 32


def argmax_case(shapes, C):
    """-> [(tag, model, perm, sign, L, planned, q)] for the class count C"""
    out = []
    for img_bytes, hidden in shapes:
        # the fixed row has no one-layer model: both heads there.  When every pixel holds a logit, the -I head's logits of -127
        # are the 127 anchor.
        signs = [1] if not hidden else ([1, -1] if len(hidden) == 3 else [1 if C % 2 == 0 and C < img_bytes else -1])
        for sign in signs:
            seed = zlib.crc32(repr((img_bytes, hidden, C, sign)).encode())
            enc = ENC_8BIT if not hidden else CHAIN_ENCS[(C + (sign < 0)) % len(CHAIN_ENCS)]
            m, perm = identity_chain(img_bytes, hidden, C, sign, seed, enc)
            lo, hi = (-127, 127) if not hidden else ((0, 127) if sign > 0 else (-127, 0))
            L, planned = argmax_rows(C, lo, hi, seed, anchor=C >= img_bytes)
            out.append(("-".join(map(str, (img_bytes,) + tuple(hidden) + (C,))) + f" x{sign:+d} enc {enc}", m, perm, sign, L, planned,
                        argmax_images(L, perm, img_bytes, sign, seed)))
    return out


def magnitude_model(enc, C, img_bytes):
    """one layer, weights of magnitude 128 in the first half of the classes and 64 in the second (so a row's logits lie on both
    sides of +-2^23, where a 32-bit key value << 8 wraps) -- -128 / -64 in 8bit, +128 / +64 in FP130, whose +128 takes the
    second weight plane -- but on pixels 0 and 1, where 8bit rows step by one (-128 + c, -128 + c // 2) and FP130 rows take
    -1 / -2 (pixel 0: odd columns -2; pixel 1: columns 3 and C - 1 -2)"""
    c = np.arange(C)
    w = np.repeat(np.where(c < (C + 1) // 2, 128, 64)[:, None], img_bytes, axis=1).astype(np.int64)
    if enc == ENC_8BIT:
        w = -w
        w[:, 0], w[:, 1] = -128 + c, -128 + c // 2
    else:
        w[:, 0], w[:, 1] = -1 - c % 2, np.where((c == 3) | (c == C - 1), -2, -1)
    return _model([w], img_bytes, enc)


def magnitude_images(img_bytes):
    """rails (-128 everywhere: 8bit logits up to 128 * 128 * img_bytes, FP130's most negative; 127 everywhere: the other way
    round) with pixels 0 and 1 at
    -128, -1, 0, 1, 127: ties and neighbours one apart at the top"""
    rows = []
    for base in (-128, 127):
        for x0, x1 in itertools.product((-128, -1, 0, 1, 127), repeat=2):
            r = np.full(img_bytes, base)
            r[0], r[1] = x0, x1
            rows.append(r)
    rows.append(rows[0])
    return np.stack(rows).astype(np.int8)


# ---- the hidden-layer rules at their boundaries ---------------------------------------------------------------------------

def c_rule(acc):
    """inference.c:41-67 on int64 rows: shift = bit length of (row max >> 7) (0 for a row max <= 0), then per element
    x < 0 -> 0, else min(127, (x + ((1 << shift) >> 1)) >> shift)"""
    acc = np.asarray(acc, dtype=np.int64)
    top = np.maximum(acc.max(axis=1), 0) >> 7
    shift = np.array([int(v).bit_length() for v in top], dtype=np.int64)[:, None]
    rnd = (np.int64(1) << shift) >> 1
    return np.where(acc < 0, 0, np.minimum(127, (acc + rnd) >> shift))


def c_shift(m):
    return (max(int(m), 0) >> 7).bit_length()


def emul_shift(m):
    """-e of the emulator's 2^e = 2^floor(log2(127 / m)), 0 when e >= 0"""
    return max(0, -int(np.floor(np.log2(127.0 / m)))) if m > 0 else 0


class Gain:
    """layer 1 of a boundary model: pixel 0 is the float forms' 127 anchor (weight 0); pixels 1..g the gain block (weight 127,
    taken by the gain units); then two private pixels per controlled unit (weights 127 and 1).  A controlled unit's accumulator is
    127 S [gain] + 127 a + b, every other unit's 0.  Identity layers behind it; `head` classes (default: all H units)."""

    def __init__(self, img_bytes, H, g, K, seed, tail=(), head=None):
        self.img_bytes, self.H, self.g = img_bytes, H, g
        rng = np.random.default_rng(seed)
        self.units = np.arange(H) if K == H else np.sort(rng.choice(H, K, replace=False))
        self.gain = np.arange(K) % 3 != 2
        assert 1 + g + 2 * K <= img_bytes
        w = np.zeros((H, img_bytes), dtype=np.int64)
        w[self.units[self.gain], 1:1 + g] = 127
        w[self.units, 1 + g + 2 * np.arange(K)] = 127
        w[self.units, 2 + g + 2 * np.arange(K)] = 1
        self.w1 = w
        self.head = head or H
        ws, n_in = [w], H
        for n_out in list(tail) + [self.head]:
            ws.append(np.eye(n_out, n_in, dtype=np.int64))
            n_in = n_out
        self.model = _model(ws, img_bytes)
        self.top = 127 * 127 * g + 127 * 127 + 127          # the largest accumulator a gain unit reaches

    def maxima(self):
        """the row maxima: both sides of every C shift boundary, 128 2^s - 1 and 128 2^s, and both sides of every emulator
        boundary, floor(127 2^-e) and one more"""
        ms = {v for s in range(16) for v in ((128 << s) - 1, 128 << s)}
        ms |= {v for e in range(-15, 7) for v in (int(np.floor(127 * 2.0 ** -e)), int(np.floor(127 * 2.0 ** -e)) + 1)}
        return sorted(m for m in ms if 0 < m <= self.top)

    def images(self, seed):
        """one row per (row maximum, controlled unit holding it); the other units at the boundaries of that row's shifts"""
        rng = np.random.default_rng(seed)
        K, small = len(self.units), 127 * 127 + 127
        rows = []
        for M in self.maxima():
            sh, es = c_shift(M), emul_shift(M)
            S = 0 if M <= small else min(127 * self.g, -(-(M - small) // 127))   # a gain unit reaches 127 S +- small
            must = [M - 1, 0, -1]
            for k in {sh, es} - {0}:
                h = 1 << (k - 1)
                top = ((M - 1) // h - 1) // 2                    # the largest t with (2t + 1) h < M
                must += [h, h - 1, 3 * h, 3 * h - 1, 255 * h, 255 * h - 1]
                must += [v for t in (top, top - 1) if t >= 0 for v in ((2 * t + 1) * h, (2 * t + 1) * h - 1)]
            must = [t for t in must if t < M]
            halves = [(2 * t + 1) << (k - 1) for k in {sh, es} - {0} for t in range(128)]
            for pos in range(K):
                if S and not self.gain[pos]:
                    continue                                     # this row's maximum needs the gain block
                tgt = np.zeros(K, dtype=np.int64)
                free = [k for k in rng.permutation(K) if k != pos]
                tgt[pos] = M
                for t in must:
                    for i, k in enumerate(free):
                        base = 127 * S if self.gain[k] else 0
                        if -small <= t - base <= small:
                            tgt[k] = t
                            free.pop(i)
                            break
                for k in free:
                    base = 127 * S if self.gain[k] else 0
                    opts = [t for t in halves if -small < t - base <= small and t < M] or [base]
                    t = opts[rng.integers(len(opts))] - rng.integers(0, 2)
                    tgt[k] = min(t, M - 1)
                rows.append(self._pixels(tgt, S))
        if len(rows) % 2 == 0:
            rows.append(rows[0])
        return np.stack(rows).astype(np.int8)

    def _pixels(self, tgt, S):
        r = np.zeros(self.img_bytes, dtype=np.int64)
        r[0] = 127
        r[1:1 + S // 127] = 127
        if S // 127 < self.g:
            r[1 + S // 127] = S % 127
        R = tgt - np.where(self.gain, 127 * S, 0)
        a = np.clip(np.rint(R / 127.0), -127, 127).astype(np.int64)
        b = R - 127 * a
        assert np.abs(b).max() <= 127, (tgt, S)
        K = len(self.units)
        r[1 + self.g + 2 * np.arange(K)] = a
        r[2 + self.g + 2 * np.arange(K)] = b
        return r

    def acc(self, q):
        return q.astype(np.int64) @ self.w1.T


# (tag, row of the int8 form, layout): the 64-wide hidden layer on 256-byte rows (shifts 0 to 13) and 512-byte rows (to 15),
# the 128-, 192- and 256-wide ones on 256-byte rows (0 to 12) with 96 controlled units among them; 16-class heads for the
# float-input rows
GAIN_CASES = [
    ("256-64", "<64,2,2,64>", dict(img_bytes=256, H=64, g=126, K=64)),
    ("512-64", "<64,1>", dict(img_bytes=512, H=64, g=383, K=64)),
    ("256-128", "<128,1>", dict(img_bytes=256, H=128, g=63, K=96)),
    ("256-192", "<192,1>", dict(img_bytes=256, H=192, g=63, K=96)),
    ("256-256", "<256,1>", dict(img_bytes=256, H=256, g=63, K=96)),
    ("256-64-64-16", "<64,2,2,16>", dict(img_bytes=256, H=64, g=126, K=64, tail=(64,), head=16)),
    ("256-64-64-64-16", "<64,2,2,16,fixed>", dict(img_bytes=256, H=64, g=126, K=64, tail=(64, 64), head=16)),
]


def gain_case(tag):
    _, row, kw = next(c for c in GAIN_CASES if c[0] == tag)
    seed = zlib.crc32(tag.encode())
    g = Gain(seed=seed, **kw)
    return row, g, g.images(seed)


# ---- CPU -------------------------------------------------------------------------------------------------------------------

def test_encoding_ids():
    from bitnetmcu_b200 import model as M
    assert (M.ENC_4BIT, M.ENC_8BIT, M.ENC_FP130, M.ENC_TERNARY) == (ENC_4BIT, ENC_8BIT, ENC_FP130, ENC_TERNARY)


@pytest.mark.parametrize("row,shapes,C", ARGMAX_CASES, ids=[f"{r}-{C}cls" for r, _, C in ARGMAX_CASES])
def test_argmax_fixtures(oracle, row, shapes, C):
    """the ties sit at the planned columns, the oracle's label is the smallest of them, its logits are the planned ones, and the
    float images scale to the int8 ones exactly"""
    cases = argmax_case(shapes, C)
    assert {m.layers[0].bitperweight for _, m, *_ in cases if len(m.layers) > 1} <= set(CHAIN_ENCS)
    for tag, m, perm, sign, L, planned, q in cases:
        assert L.shape[0] % 2 == 1 and L.shape[0] > C, tag
        for r in range(L.shape[0]):
            assert np.flatnonzero(L[r] == L[r].max()).tolist() == planned[r], (tag, r)
        assert list(range(C)) in planned and all([c] in planned for c in range(C)), tag
        if C >= 2:
            assert [0, C - 1] in planned and [C - 2, C - 1] in planned, tag
            assert all([i, j] in planned for i, j in _pairs(C)), tag
            assert any(len(p) == 3 and p[-1] == C - 1 for p in planned) == (C >= 3), tag
        lo, la = oracle.infer(m, q)
        assert np.array_equal(lo, L) and np.array_equal(la, [p[0] for p in planned]), tag
        assert np.array_equal(scale_images(q.astype(np.float32)), q), tag
        if L.min() < 0:
            assert (L.max(axis=1) < 0).any(), f"{tag}: no all-negative row"


def test_chain_encodings_cover_every_row():
    """4bit, Ternary (K padded to a multiple of 10) and 8bit identity chains, each on several rows"""
    seen = {}
    for row, shapes, C in ARGMAX_CASES:
        for _, m, *_ in argmax_case(shapes, C):
            if len(m.layers) > 1:
                seen.setdefault(m.layers[0].bitperweight, set()).add(row)
    assert set(seen) == set(CHAIN_ENCS) and all(len(rows) >= 3 for rows in seen.values()), seen


@pytest.mark.parametrize("enc", [ENC_8BIT, ENC_FP130])
def test_magnitude_fixtures(oracle, enc):
    """logits past 2^23 both ways, rows on both sides of +-2^23, ties and neighbours one apart at the top, 128 * 128 * 768
    exactly for 8bit, FP130's +128 (the residual plane)"""
    from bitnetmcu_b200 import pack as P
    m = magnitude_model(enc, 17, 768)
    assert (P.decode_int_weights(m.layers[0]) == 128).any() == (enc == ENC_FP130)
    lo, la = oracle.infer(m, magnitude_images(768))
    top = lo.max(axis=1)
    assert lo.max() > 1 << 23 and lo.min() < -(1 << 23)
    assert ((top >= 1 << 23) & (lo.min(axis=1) > 0) & (lo.min(axis=1) < 1 << 23)).any()    # a maximum past 2^23 over logits below
    assert ((top > -(1 << 23)) & (lo.min(axis=1) <= -(1 << 23))).any()    # a maximum above -2^23 over logits below it
    assert ((lo == top[:, None]).sum(axis=1) > 1)[top > 1 << 23].any()
    srt = np.sort(lo, axis=1)
    assert ((srt[:, -1] - srt[:, -2] == 1) & (top > 1 << 23)).any()
    if enc == ENC_8BIT:
        assert lo.max() == 128 * 128 * 768
        assert oracle.infer(magnitude_model(enc, 17, 1024), magnitude_images(1024))[0].max() == 1 << 24


@pytest.mark.parametrize("tag", [c[0] for c in GAIN_CASES])
def test_boundary_fixtures(oracle, tag):
    """every boundary the layout reaches is hit, the row maximum visits every 16-column block, quad lane, column pair half and
    64-column piece, the NumPy C rule equals the oracle's ReLUNorm, and the oracle's logits are the rule's activations"""
    row, g, q = gain_case(tag)
    acc = g.acc(q)
    assert np.array_equal(scale_images(q.astype(np.float32)), q)
    want = c_rule(acc)
    for i in range(0, acc.shape[0], 97):
        out, pos = oracle.relunorm(acc[i].astype(np.int32))
        assert np.array_equal(out, want[i]) and pos == int(np.argmax(acc[i])), (tag, i)
    lo, _ = oracle.infer(g.model, q)
    assert np.array_equal(lo, want[:, :g.head]), tag
    top, arg = acc.max(axis=1), acc.argmax(axis=1)
    reach = max(s for s in range(16) if (128 << s) <= g.top)
    assert reach == {256: 13 if g.H == 64 else 12, 512: 15}[g.img_bytes], (tag, reach)
    for s in range(reach + 1):
        assert {(128 << s) - 1, 128 << s} <= set(top.tolist()), (tag, s)
    for e in range(-15, 7):
        m = int(np.floor(127 * 2.0 ** -e))
        if m + 1 <= g.top:
            assert {m, m + 1} <= set(top.tolist()), (tag, e)
    sh = np.array([c_shift(v) for v in top])
    es = np.array([emul_shift(v) for v in top])
    for k in range(1, reach + 2):
        h = 1 << (k - 1)
        for rule, shifts in (("C", sh), ("emulator", es)):
            at = (shifts == k)[:, None]
            # (shift 16: the halves lie 2^15 apart, beyond the +-16 256 a unit's private pixels reach below a row maximum)
            for what, v in ((("half", acc), ("half - 1", acc + 1)) if k < 16 else ()):
                odd = (v > 0) & (v % h == 0) & ((v // h) % 2 == 1)      # v = (2t + 1) h
                t = (v // h - 1) // 2
                assert (odd & (t % 2 == 0) & at).any() and (odd & (t % 2 == 1) & at).any(), (tag, rule, what, k)
            if rule == "C" and k <= reach:
                assert ((acc == 255 * h) & at).any() and ((acc == 255 * h - 1) & at).any(), (tag, "clip", k)
    for k in range(reach + 2):
        assert ((acc == 0) & (sh == k)[:, None]).any() and ((acc == -1) & (sh == k)[:, None]).any(), (tag, "0 / -1", k)
    cols = g.units
    assert set(arg.tolist()) <= set(cols.tolist())
    for what, f in (("16-column block", lambda c: c // 16), ("quad lane", lambda c: c % 8 // 2), ("column of the pair", lambda c: c % 2),
                    ("block half", lambda c: c % 16 // 8), ("64-column piece", lambda c: c // 64)):
        assert set(f(arg[top > 127 * 127 + 127]).tolist()) == set(f(cols[g.gain]).tolist()) == set(f(np.arange(g.H)).tolist()), (tag, what)


def test_c_rule_restatement(oracle):
    """the NumPy C rule equals the oracle's ReLUNorm on random rows and on the edges: all negative, all zero, one huge value"""
    rng = np.random.default_rng(5)
    rows = [rng.integers(-(1 << 24), 1 << 24, size=64) >> rng.integers(0, 24) for _ in range(300)]
    rows += [np.full(64, -3), np.zeros(64, dtype=np.int64), np.r_[1 << 30, np.zeros(63, dtype=np.int64)]]
    for r in rows:
        out, _ = oracle.relunorm(r.astype(np.int32))
        assert np.array_equal(out, c_rule(r[None])[0]), r[:4]


# ---- GPU -------------------------------------------------------------------------------------------------------------------

class Batch:
    """P crafted rows on the device, repeated: row i of a batch is pattern i % P"""

    def __init__(self, q, want_lo, want_la, emu_lo):
        import torch
        self.P = q.shape[0]
        self.q = torch.from_numpy(q).cuda()
        self.x = self.q.float()
        self.want_lo = torch.from_numpy(want_lo.astype(np.int32)).cuda()
        self.want_la = torch.from_numpy(want_la.astype(np.int32)).cuda()
        self.emu_lo = torch.from_numpy(emu_lo).cuda()
        self.emu_la = torch.from_numpy(np.argmax(emu_lo, axis=1).astype(np.int32)).cuda()

    def idx(self, n):
        import torch
        return torch.arange(n, device="cuda") % self.P

    def check(self, sw, n, got, want, tag, what, sentinel=None):
        """rows :n of the device tensor got equal want[i % P]; rows n: (if any) hold the sentinel"""
        import torch
        w = want[self.idx(n)]
        bad = got[:n] != w.to(got.dtype)
        if bad.dim() > 1:
            bad = bad.any(dim=1)
        if bool(bad.any()):
            rows = torch.nonzero(bad).flatten().cpu().numpy()
            raise AssertionError((tag, n, what, f"{rows.size} rows wrong, first {rows[:4].tolist()}", "patterns",
                                  (rows[:4] % self.P).tolist(), "(tile, cta, local, pipe, slot, stage, round):",
                                  sw.where(n, rows) if sw else None))
        if sentinel is not None:
            assert bool((got[n:] == sentinel).all()), (tag, n, what, "written past row n")


SENT = -0x5A5A5A5B


def _launch_size(sw):
    n = sw.sizes[-1] - 51         # the sweep's largest launch (rounds 0 to 2 on every stage), its last tile ragged
    assert n % TILE and n > sw.sizes[-2], sw.sizes
    return n


def every_form(lib, capfd, monkeypatch, m, b, tag, int8_row):
    """every entry point of the model on the batch b: the int8 kernel row, float-input, emulator (float or int8 row) and two-engine
    forms on their sweeps' largest launches; host infer (logits + labels, labels only), gather (int32, u8) and BNM_PATH_LAYERS on
    N_MANY images -> the plan line"""
    import torch
    from bitnetmcu_b200 import _lib
    e, err = verbose_engine(capfd, monkeypatch, lambda: engine(m))
    line = plan_line(err)
    assert line and e.active_path == _lib.PATH_TCGEN05, (tag, err)
    row, ring = plan_ring(line, "int8")
    assert row == int8_row, (tag, line)
    C = m.n_classes
    small = m.img_bytes <= 256 and C <= 16 and int8_row.startswith("<64,")
    emul_row = "<64,1,float,emul>" if small else plan_ring(line, "emul_i8")[0]
    if small:
        assert plan_ring(line, "float")[0] == "<64,1,float>", (tag, line)
        assert route(err, "emulator") == f"fc_emul_kernel{emul_row}", (tag, err)
        assert route(err, "engines") == "fc_engines_kernel<64,1,float,engines>", (tag, err)
    else:
        assert "float input" not in line, (tag, line)
        assert route(err, "emulator") == f"k_quantize_images + fc_emul_i8_kernel{emul_row}", (tag, err)
        assert emul_row == f"<{ring_width(int8_row)},1,emul>", (tag, line)
    print(tag, line)

    # the int8 kernel row on a non-default stream
    sw = Sweep(f"{tag} {int8_row}", ring)
    n = _launch_size(sw)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        d_img = b.q[b.idx(n)]
        d_lo = torch.full((n + TILE, C), SENT, dtype=torch.int32, device="cuda")
        d_la = torch.full((n + TILE,), -7, dtype=torch.int32, device="cuda")
        e.infer_device(d_img, d_lo[:n], d_la[:n], stream=s.cuda_stream)
    s.synchronize()
    b.check(sw, n, d_lo, b.want_lo, tag, "logits", SENT)
    b.check(sw, n, d_la, b.want_la, tag, "labels", -7)
    d_la.fill_(-7)
    e.infer_device(d_img, None, d_la[:n])
    torch.cuda.synchronize()
    b.check(sw, n, d_la, b.want_la, tag, "labels (labels-only launch)", -7)
    del d_img, d_lo, d_la

    # the float-input row, the emulator
    if small:
        sw = Sweep(f"{tag} <64,1,float>", plan_ring(line, "float")[1])
        n = _launch_size(sw)
        d_x = b.x[b.idx(n)]
        d_lo = torch.full((n + TILE, C), SENT, dtype=torch.int32, device="cuda")
        d_la = torch.full((n + TILE,), -7, dtype=torch.int32, device="cuda")
        e.infer_device_f32(d_x, d_lo[:n], d_la[:n])
        torch.cuda.synchronize()
        b.check(sw, n, d_lo, b.want_lo, tag, "float-input logits", SENT)
        b.check(sw, n, d_la, b.want_la, tag, "float-input labels", -7)
        sw_e = Sweep(f"{tag} {emul_row}", plan_ring(line, "emul")[1])
    else:
        sw_e = Sweep(f"{tag} {emul_row}", plan_ring(line, "emul_i8")[1])
    n = _launch_size(sw_e)
    d_x = b.x[b.idx(n)]
    d_lo = torch.full((n + TILE, C), -12345.5, dtype=torch.float64, device="cuda")
    d_la = torch.full((n + TILE,), -7, dtype=torch.int32, device="cuda")
    e.inference_quantized_device(d_x, d_lo[:n], d_la[:n])
    torch.cuda.synchronize()
    b.check(sw_e, n, d_lo, b.emu_lo, tag, "emulator logits", -12345.5)
    b.check(sw_e, n, d_la, b.emu_la, tag, "emulator labels", -7)
    del d_x, d_lo, d_la

    # two engines in one call: both labels, counts against the oracle's and the restatement's labels
    n = N_MANY
    idx = b.idx(n)
    d_x = b.x[idx]
    truth = ((torch.arange(n, device="cuda") * 7) % (C + 1)).to(torch.int32)
    lc = torch.full((n,), -7, dtype=torch.int32, device="cuda")
    lp = torch.full((n,), -7, dtype=torch.int32, device="cuda")
    counts = torch.zeros(4, dtype=torch.int64, device="cuda")
    e.compare_engines_device(d_x, truth, lc, lp, counts)
    torch.cuda.synchronize()
    b.check(None, n, lc, b.want_la, tag, "engines: C labels")
    b.check(None, n, lp, b.emu_la, tag, "engines: emulator labels")
    wc, wp = b.want_la[idx], b.emu_la[idx]
    ok = truth < C
    want_counts = [n, int((ok & (wc == truth)).sum()), int((ok & (wp == truth)).sum()), int((wc != wp).sum())]
    assert counts.cpu().tolist() == want_counts, (tag, "engines: counts", counts.cpu().tolist(), want_counts)

    # host entry: logits and labels, labels only
    q = b.q[idx].cpu().numpy()
    lo, la = e.infer(q)
    b.check(None, n, torch.from_numpy(lo).cuda(), b.want_lo, tag, "host logits")
    b.check(None, n, torch.from_numpy(la.astype(np.int32)).cuda(), b.want_la, tag, "host labels")
    _, la = e.infer(q, want_logits=False)
    b.check(None, n, torch.from_numpy(la.astype(np.int32)).cuda(), b.want_la, tag, "host labels only")

    # gather: int32 logits and labels, u8 labels (n_classes <= 255; 256 classes are refused)
    off, d_img = 512, b.q[idx]
    dst_lo = torch.full((n + 640, C), SENT, dtype=torch.int32, device="cuda")
    dst_la = torch.full((n + 640,), -7, dtype=torch.int32, device="cuda")
    g = _lib.BnmGather()
    g.n_labels_dst, g.n_logits_dst, g.row_offset = 1, 1, off
    g.labels_dst[0], g.logits_dst[0] = dst_la.data_ptr(), dst_lo.data_ptr()
    _lib.check(gather_call(lib, e, d_img, None, None, g, torch.cuda.current_stream(0)), "gather")
    b.check(None, n, dst_lo[off:], b.want_lo, tag, "gather logits", SENT)
    b.check(None, n, dst_la[off:], b.want_la, tag, "gather labels", -7)
    assert bool((dst_lo[:off] == SENT).all()) and bool((dst_la[:off] == -7).all()), tag
    dst8 = torch.full((n + 640,), 201, dtype=torch.uint8, device="cuda")
    g8 = _lib.BnmGather()
    g8.n_labels_dst, g8.n_logits_dst, g8.row_offset, g8.labels_u8 = 1, 0, off, 1
    g8.labels_dst[0] = dst8.data_ptr()
    rc = gather_call(lib, e, d_img, None, None, g8, torch.cuda.current_stream(0))
    if C <= 255:
        _lib.check(rc, "gather u8")
        b.check(None, n, dst8[off:].to(torch.int32), b.want_la, tag, "gather u8 labels", 201)
        assert bool((dst8[:off] == 201).all()), tag
    else:
        assert rc != 0 and bool((dst8 == 201).all()), (tag, "u8 labels for 256 classes")

    # layer by layer: k_relunorm and k_emul_logits keep the same rules
    e.set_option(_lib.OPT_PATH, _lib.PATH_LAYERS)
    lo, la = e.infer(q)
    b.check(None, n, torch.from_numpy(lo).cuda(), b.want_lo, tag, "layers: logits")
    b.check(None, n, torch.from_numpy(la.astype(np.int32)).cuda(), b.want_la, tag, "layers: labels")
    elo, ela = run_emulator(e, d_x)
    b.check(None, n, torch.from_numpy(elo).cuda(), b.emu_lo, tag, "layers: emulator logits")
    b.check(None, n, torch.from_numpy(ela.astype(np.int32)).cuda(), b.emu_la, tag, "layers: emulator labels")
    e.close()
    return line


def ring_width(row):
    return int(row[1:].split(",")[0])


def layer_by_layer(capfd, monkeypatch, m, q, want_lo, want_la, emu, tag):
    """a model without a fused plan: BNM_VERBOSE names none and both routes run layer by layer; the host entry and the emulator
    on N_MANY images, row i holding pattern i % P"""
    import torch
    from bitnetmcu_b200 import _lib
    e, err = verbose_engine(capfd, monkeypatch, lambda: engine(m))
    assert plan_line(err) is None and e.active_path == _lib.PATH_LAYERS, (tag, err)
    assert route(err, "emulator") == "layer by layer", (tag, err)
    assert route(err, "engines") == "bnm_infer_batch_device_f32 + bnm_emulate_batch_device + k_engine_counts", (tag, err)
    idx = np.arange(N_MANY) % q.shape[0]
    lo, la = e.infer(q[idx])
    assert np.array_equal(lo, want_lo[idx]) and np.array_equal(la, want_la[idx]), tag
    elo, ela = run_emulator(e, torch.from_numpy(q[idx]).cuda().float())
    assert np.array_equal(elo, emu[idx]) and np.array_equal(ela, np.argmax(emu, axis=1)[idx]), tag
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("row,shapes,C", ARGMAX_CASES, ids=[f"{r}-{C}cls" for r, _, C in ARGMAX_CASES])
def test_argmax_on_every_form(lib, oracle, capfd, monkeypatch, row, shapes, C):
    """ties, near-ties, unique maxima and all-negative rows at every class count of the row, on every entry point"""
    for tag, m, perm, sign, L, planned, q in argmax_case(shapes, C):
        want_lo, want_la = oracle.infer(m, q)
        assert np.array_equal(want_lo, L), tag
        emu = emulate_fc(m, q.astype(np.float32))
        assert np.array_equal(np.argmax(emu, axis=1), want_la), tag      # scaling by 2^e keeps the order and the ties
        if m.img_bytes == 768 and not fused_768(C):
            layer_by_layer(capfd, monkeypatch, m, q, want_lo, want_la, emu, tag)
        else:
            every_form(lib, capfd, monkeypatch, m, Batch(q, want_lo, want_la, emu), tag, row)


@pytest.mark.gpu
@pytest.mark.parametrize("enc", [ENC_8BIT, ENC_FP130])
@pytest.mark.parametrize("C", [10, 17])
def test_logits_past_2_23(lib, oracle, capfd, monkeypatch, enc, C):
    """one layer on 768-byte rows (six 128-byte atoms, <64,1>): logits up to +-12 582 912, tied and one apart at the top.
    FP130's +128 takes a second weight plane (the plan's weight bytes show it); its two planes fit next to two 96 kB stages up to
    16 classes, so at 17 the FP130 model runs layer by layer."""
    m = magnitude_model(enc, C, 768)
    q = magnitude_images(768)
    want_lo, want_la = oracle.infer(m, q)
    emu = emulate_fc(m, q.astype(np.float32))
    assert np.abs(want_lo).max() > 1 << 23 and np.abs(emu).max() > 1 << 23
    tag = f"{enc}-768-{C}"
    if enc == ENC_FP130 and C > 16:
        layer_by_layer(capfd, monkeypatch, m, q, want_lo, want_la, emu, tag)
        return
    line = every_form(lib, capfd, monkeypatch, m, Batch(q, want_lo, want_la, emu), tag, "<64,1>")
    planes, n_pad = (2 if enc == ENC_FP130 else 1), (C + 15) // 16 * 16
    assert f" {planes * 24 * n_pad * 32 + 64 * 32} weight bytes" in line, (tag, planes, line)   # planes x K-steps x n_pad x 32 B + zeros


@pytest.mark.gpu
@pytest.mark.parametrize("img_bytes", [784, 1024])
def test_rows_past_six_atoms_run_layer_by_layer(lib, oracle, capfd, monkeypatch, img_bytes):
    """more than six 128-byte atoms per row leave no room for two ring stages: no fused plan, every entry layer by layer;
    1024-byte rows reach 128 * 128 * 1024 = 2^24"""
    m = magnitude_model(ENC_8BIT, 17, img_bytes)
    q = magnitude_images(img_bytes)
    want_lo, want_la = oracle.infer(m, q)
    if img_bytes == 1024:
        assert want_lo.max() == 1 << 24
    layer_by_layer(capfd, monkeypatch, m, q, want_lo, want_la, emulate_fc(m, q.astype(np.float32)), f"8bit-{img_bytes}-17")


@pytest.mark.gpu
@pytest.mark.parametrize("tag", [c[0] for c in GAIN_CASES])
def test_hidden_rules_at_their_boundaries(lib, oracle, capfd, monkeypatch, tag):
    """the row maximum on both sides of every shift boundary, other units at the rounding halves, the clip threshold, 0 and -1,
    the maximum in every block, quad lane and piece: the C rule against the oracle and the NumPy rule, the emulator's against
    the restatement, on every entry point the model has"""
    row, g, q = gain_case(tag)
    want_lo, want_la = oracle.infer(g.model, q)
    assert np.array_equal(want_lo, c_rule(g.acc(q))[:, :g.head]), tag
    emu = emulate_fc(g.model, q.astype(np.float32))
    every_form(lib, capfd, monkeypatch, g.model, Batch(q, want_lo, want_la, emu), tag, row)
