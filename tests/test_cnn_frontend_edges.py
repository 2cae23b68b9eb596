"""The CNN front-ends at their integer edges (DESIGN.md section 4.3).

* Packed conv3: k_cnn_frontend16_tc<true> runs conv3 on IDP.2A over unsigned 16-bit pairs when cnn_conv3_bound (the largest
  pooled conv2 output any int8 image can give) is at most 65535, otherwise <false> runs it on IMAD.  Crafted per-channel weight
  sums put the bound at exactly 65535 (packed) or 65536 (IMAD), through positive conv1 taps on all-127 images and negative ones
  on all-(-128) images (the 128 of the bound), and constant images spread conv3's inputs over [32768, 65535].  The route comes
  from the `cnn front-end:` line of BNM_VERBOSE.
* The features' ReLUNorm (dll.c:80): centre-tap channels make each feature a monotone function of the largest pixel of a 4 x 4
  block, so each image's feature maximum can be put on both sides of every shift boundary, with exact rounding ties below it
  and maxima that round up to 128 and clip to 127, the maximum in a channel that sits in another tile than most of its image.
* The emulator's renormalisations (BitNetMCU.py:459-526): conv maxima of 254 make the scale exactly 0.5, so odd sums land on
  exact .5 ties, where half to even and half up disagree when the floor is even; at each of the three renormalisations.
* More than 256 channels: the C engine refuses the model, the emulator runs it layer by layer.

CPU: the bound against the fixtures and random models, each crafted case against its target in the NumPy restatement of the
front-end stages (tests/restate.py), the SASS of both tensor-core instantiations.  GPU: every entry against the oracle and the
emulator restatement at tolerance 0.  The crafted models feed the features straight into the head, so one feature off by one
changes every logit."""
import ctypes as C
import re

import numpy as np
import pytest

from conftest import load_model
from restate import c_frontend, cnn_stages, conv3_bound, conv3_channel_bounds, emulate, scale_images
from support import cnn_model, engine, instructions, lib, route, run_emulator, run_emulator_layered, sass_functions, \
    verbose_engine

U16 = 65535
BNM_E_UNSUPPORTED = -3


def _split(total, rng):
    """nine non-negative int8 taps summing to total (<= 9 * 127), spread at random"""
    t = np.full(9, total // 9, dtype=np.int64)
    t[:total % 9] += 1
    for _ in range(40):
        i, j = rng.integers(0, 9, size=2)
        d = int(rng.integers(0, min(t[i], 127 - t[j]) + 1))
        t[i] -= d
        t[j] += d
    assert t.sum() == total and t.min() >= 0 and t.max() <= 127
    return rng.permutation(t)


# (sign of w1, sum |w1|, sum of w2): conv1 at its bound on all-127 (+) or all-(-128) (-) images, and conv2's pooled output then
# exactly at the bound: ((127 * 681 >> 4) * 194) >> 4 = 65535, ((127 * 546 >> 4) * 242) >> 4 = 65536,
# ((128 * 170 >> 4) * 771) >> 4 = 65535, ((128 * 128 >> 4) * 1024) >> 4 = 65536
EDGE = {"+65535": (1, 681, 194), "-65535": (-1, 170, 771), "+65536": (1, 546, 242), "-65536": (-1, 128, 1024)}


def _edge_weights(channels, kinds, seed):
    """conv weights [C, 9] x 3: channel c is EDGE[kinds[c]] or, for None, a channel of mixed signs whose bound stays below
    2^15; conv3 taps at -128 and 127 in every channel (large conv3 sums of both signs)"""
    rng = np.random.default_rng(seed)
    w1, w2, w3 = (np.zeros((channels, 9), dtype=np.int64) for _ in range(3))
    for c, kind in enumerate(kinds):
        if kind is None:
            w1[c] = _split(200, rng) * rng.choice([-1, 1], size=9)
            w2[c] = _split(120, rng) - _split(60, rng)
        else:
            sign, s1, s2 = EDGE[kind]
            w1[c] = sign * _split(s1, rng)
            w2[c] = _split(s2, rng)
        w3[c] = rng.integers(-128, 128, size=9)
        w3[c, rng.permutation(9)[:2]] = (-128, 127)
    return tuple(w.astype(np.int8) for w in (w1, w2, w3))


# (name, channels, the kinds that cycle through the channels, or a dict {channel: kind} over background channels, want bound)
EDGE_CASES = [
    ("packed-16", 16, ["+65535", "-65535", None], U16),
    ("packed-48", 48, ["+65535", None, "-65535", None], U16),
    ("packed-112", 112, ["-65535", "+65535", None, None, None], U16),
    ("packed-128", 128, ["+65535", "-65535", None, None], U16),
    ("imad-16", 16, ["+65536", "-65535", None], U16 + 1),
    ("imad-48", 48, ["-65536", "+65535", None], U16 + 1),
    ("imad-80-last", 80, {0: "+65535", 1: "-65535", 79: "+65536"}, U16 + 1),
    ("imad-128-last", 128, {5: "+65535", 64: "-65535", 127: "-65536"}, U16 + 1),
]


def _edge_model(case):
    name, channels, kinds, _ = case
    if isinstance(kinds, dict):
        kinds = [kinds.get(c) for c in range(channels)]
    else:
        kinds = [kinds[c % len(kinds)] for c in range(channels)]
    return cnn_model(channels, 10, seed=channels, w=_edge_weights(channels, kinds, seed=channels + len(name)), hidden=())


def _edge_base(seed):
    """constant images from 90 to 127 and from -90 to -128 (conv3 inputs over [32768, 65535] on the edge channels), the two
    rails, rail noise and uniform noise, then uniform images with a constant 127 or -128 square"""
    rng = np.random.default_rng(seed)
    base = [np.full(256, v) for v in list(range(90, 128)) + list(range(-128, -89))]
    base += [rng.choice([-128, 127], size=256) for _ in range(8)] + [rng.integers(-128, 128, size=256) for _ in range(8)]
    for v in (127, -128):
        for _ in range(8):
            x = rng.integers(-128, 128, size=(16, 16))
            y, z = rng.integers(0, 8, size=2)
            x[y:y + 9, z:z + 9] = v
            base.append(x.reshape(256))
    return np.array(base, dtype=np.int8)


def _edge_images(n, seed):
    """_edge_base repeated to n images"""
    base = _edge_base(seed)
    return base[np.arange(n) % len(base)]


def test_bound_of_the_fixtures_and_random_models():
    """the fixtures take the packed path, every random cnn_model the IMAD path"""
    want = {"cnn": 37349, "cnn_16": 37695, "cnn_16small": 47501, "cnn_32": 22406, "cnn_48": 24581, "cnn_letters": 21760}
    assert {k: conv3_bound(load_model(k)) for k in want} == want
    for channels in (16, 24, 48, 64, 128, 144, 256):
        for n_classes in (10, 37):
            assert conv3_bound(cnn_model(channels, n_classes, seed=channels + n_classes)) > U16


@pytest.mark.parametrize("case", EDGE_CASES, ids=[c[0] for c in EDGE_CASES])
def test_edge_cases_hit_their_bound(case):
    """the bound is the crafted one, and the images reach it: every channel at 65535 or 65536 gives exactly that pooled conv2
    output on the all-127 (positive conv1 taps) or all-(-128) image (negative ones), at least 30 images put conv3 inputs at or
    above 2^15, and every channel has conv3 taps at -128 and 127"""
    m = _edge_model(case)
    assert conv3_bound(m) == case[3]
    x = _edge_images(len(_edge_base(0)), seed=1)
    fe = c_frontend(m, x)
    assert fe.conv2.max() == case[3]
    assert (fe.conv2.reshape(len(x), -1).max(axis=1) >= 1 << 15).sum() >= 30
    w1, _, w3 = (l.weights.reshape(-1, 9) for l in m.conv_layers)
    bounds = conv3_channel_bounds(m)
    edge = np.flatnonzero(bounds >= U16)
    assert edge.size and bounds.max() == case[3]
    for c in edge:
        v = 127 if (w1[c] > 0).any() else -128
        i = np.flatnonzero((x == v).all(axis=1))[0]
        assert fe.conv2[i, c].max() == bounds[c], (case[0], v, c)
    assert (w3 == -128).any(axis=1).all() and (w3 == 127).any(axis=1).all()


def test_tc_frontend_sass(built):
    """conv3 on unsigned 16-bit pairs in <true> only, conv2 on signed 16-bit pairs in both (CUDA 12.9: 80 and 720)"""
    kernels = sass_functions()
    count = {}
    for packed in (True, False):
        name = f"_ZN3bnm19k_cnn_frontend16_tcILb{int(packed)}EEEvNS_11CnnTcParamsE"
        ins = instructions(kernels[name])
        count[packed] = (sum("IDP.2A.LO.U16.S8" in i for i in ins), sum("IDP.2A.LO.S16.S8" in i for i in ins))
    assert count[True][0] > 0 and count[False][0] == 0, count
    assert count[True][1] > 0 and count[False][1] > 0, count
    assert count[True][0] * 9 == count[True][1] and count[True][1] == count[False][1], count   # 80 : 720 today


def _front_line(err):
    lines = [l for l in err if "cnn front-end: " in l]
    assert len(lines) == 1, err
    bound, path = re.fullmatch(r".*cnn front-end: conv3 bound (\d+), conv3 on (IDP\.2A|IMAD)", lines[0]).groups()
    return int(bound), path


def _topk_want(logits, k):
    cls = np.argsort(-logits, kind="stable", axis=1)[:, :k]
    return cls, np.take_along_axis(logits, cls, axis=1)


def _all_entries(e, x, want, want_f32, tag):
    """bnm_infer_batch_device, bnm_infer_batch, bnm_infer_batch_device_f32 and bnm_infer_topk_device against the oracle"""
    import torch
    n = len(x)
    d_x = torch.from_numpy(x).cuda()
    lo = torch.full((n, 10), -7, dtype=torch.int32, device="cuda")
    la = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    e.infer_device(d_x, lo, la)
    torch.cuda.synchronize()
    got = lo.cpu().numpy()
    assert np.array_equal(got, want[0]), (tag, "device", np.argwhere(got != want[0])[:4])
    assert np.array_equal(la.cpu().numpy().astype(np.uint32), want[1]), (tag, "device labels")
    hl, hb = e.infer(x)
    assert np.array_equal(hl, want[0]) and np.array_equal(hb, want[1]), (tag, "host")
    d_f = torch.from_numpy(x.astype(np.float32)).cuda()
    e.infer_device_f32(d_f, lo, la)
    torch.cuda.synchronize()
    assert np.array_equal(lo.cpu().numpy(), want_f32[0]), (tag, "f32")
    assert np.array_equal(la.cpu().numpy().astype(np.uint32), want_f32[1]), (tag, "f32 labels")
    k = 10
    cls = torch.full((n, k), -1, dtype=torch.int32, device="cuda")
    sc = torch.full((n, k), -7, dtype=torch.int32, device="cuda")
    e.topk_device(d_x, k, cls, sc)
    torch.cuda.synchronize()
    wc, ws = _topk_want(want[0], k)
    assert np.array_equal(cls.cpu().numpy(), wc) and np.array_equal(sc.cpu().numpy(), ws), (tag, "topk")


@pytest.mark.gpu
@pytest.mark.parametrize("case", EDGE_CASES, ids=[c[0] for c in EDGE_CASES])
def test_packed_conv3_edge(lib, oracle, capfd, monkeypatch, case):
    """both front-ends, every entry, tolerance 0, batches around the group size and a few thousand; the verbose line names
    the bound and the path it selects"""
    from bitnetmcu_b200 import _lib
    m = _edge_model(case)
    e, err = verbose_engine(capfd, monkeypatch, lambda: engine(m))
    assert _front_line(err) == (conv3_bound(m), "IDP.2A" if case[3] <= U16 else "IMAD"), (case[0], err)
    e.close()
    group = 128 // np.gcd(m.channels, 128)
    for n in (group - 1 or 1, group + 1, 3001):
        x = _edge_images(n, seed=n)
        want = oracle.infer(m, x)
        want_f32 = oracle.infer(m, scale_images(x.astype(np.float32)))
        for fe in (_lib.CNN_AUTO, _lib.CNN_CUDA_CORES):
            e = engine(m, cnn_frontend=fe)
            _all_entries(e, x, want, want_f32, (case[0], n, fe))
            e.close()


@pytest.mark.gpu
def test_packed_conv3_many_groups_per_cta(lib, oracle):
    """one batch of several groups per CTA on both front-ends (C = 48: eight images a group, 20 000 images)"""
    from bitnetmcu_b200 import _lib
    m = _edge_model(EDGE_CASES[1])
    x = _edge_images(20000, seed=7)
    want = oracle.infer(m, x)
    for fe in (_lib.CNN_AUTO, _lib.CNN_CUDA_CORES):
        e = engine(m, cnn_frontend=fe)
        lo, la = e.infer(x)
        assert np.array_equal(lo, want[0]) and np.array_equal(la, want[1]), fe
        e.close()


# ---- the features' ReLUNorm ------------------------------------------------------------------------------------------------
# Channel c has centre taps g1, g2, g3 > 0 and nothing else, so feature (c, a, b) = h(g, v) with v the largest pixel of the 4 x 4
# block rows 4a + 4 .. 4a + 7, columns 4b + 4 .. 4b + 7, and h(g, v) = ((((g1 v) >> 4) g2 >> 4) g3) >> 4, monotone in v and in
# each gain.  Channel HI carries the largest gains in every position, so the image's maximum is h(g_HI, largest block pixel).

RN_C, HI = 48, 40      # at C = 48 image 2 of each group of eight holds channels 0..31 in one tile and 32..47 in the next
RN_TARGETS = [t for s in range(9) for t in ((128 << s) - 1, 128 << s)] + [((((127 * 127) >> 4) * 127 >> 4) * 127) >> 4]


def _h(g, v):
    g1, g2, g3 = (np.asarray(x, dtype=np.int64) for x in g)
    return ((((g1 * v) >> 4) * g2 >> 4) * g3) >> 4


def _shift(m):
    return int(m >> 7).bit_length()


def _hi_gains(t):
    """(g1, g2, g3, v): gains with h(g, v) = t, at the largest pixel v that has any, and there the largest g1, then g2"""
    g = np.arange(1, 128)
    for v in range(127, 0, -1):
        c2 = ((g[:, None] * v) >> 4) * g[None, :] >> 4                  # [g1, g2]
        g3 = -(-16 * t // np.maximum(c2, 1))
        ok = (c2 > 0) & (g3 <= 127) & ((c2 * g3) >> 4 == t)
        if ok.any():
            i, j = np.argwhere(ok)[-1]
            return int(g[i]), int(g[j]), int(g3[i, j]), v
    raise AssertionError(t)


def _relunorm_case(t, seed):
    """(conv weights, 8 images) whose feature maxima are all t, from channel HI; the other channels' gains at random below
    HI's, and the three other blocks' largest pixels chosen for the most exact rounding ties at the image's shift"""
    rng = np.random.default_rng(seed)
    g1, g2, g3, v = _hi_gains(t)
    gains = np.stack([rng.integers(1, g + 1, size=RN_C) for g in (g1, g2, g3)], axis=1)
    gains[HI] = (g1, g2, g3)
    w = [np.zeros((RN_C, 9), dtype=np.int8) for _ in range(3)]
    for k in range(3):
        w[k][:, 4] = gains[:, k]
    s = _shift(t)
    h = _h(gains.T[:, :, None], np.arange(v + 1)[None, :])                 # [channel, pixel]
    ties = ((h % (1 << s)) == (1 << s >> 1)).sum(axis=0) if s else np.zeros(v + 1, dtype=np.int64)
    best = np.argsort(-ties, kind="stable")
    imgs = []
    for i in range(8):
        x = rng.integers(-128, 128, size=(16, 16))
        blocks = [v, int(best[0])] + [int(best[1 + (i + 4 * k) % min(len(best) - 1, 11)]) for k in range(2)]
        order = rng.permutation(4)          # which block holds the maximum
        for b, top in zip(order, blocks):
            r, c = 4 + 4 * (b // 2), 4 + 4 * (b % 2)
            x[r:r + 4, c:c + 4] = rng.integers(0, top + 1, size=(4, 4))
            x[r + rng.integers(0, 4), c + rng.integers(0, 4)] = top
        imgs.append(x.reshape(256))
    return tuple(w), np.array(imgs, dtype=np.int8)


def _relunorm_model(t):
    w, x = _relunorm_case(t, seed=t)
    return cnn_model(RN_C, 10, seed=t % 1000, w=w, hidden=()), x


def test_relunorm_cases_hit_their_targets():
    """every image's raw feature maximum is its target, reached in channel HI; below each maximum of shift s >= 1 lie exact
    rounding ties; the 2^k - 1 maxima round up to 128 and clip to 127"""
    assert RN_TARGETS[-1] == 63507 and _shift(RN_TARGETS[-1]) == 9
    for t in RN_TARGETS:
        m, x = _relunorm_model(t)
        fe = c_frontend(m, x)
        raw = fe.raw.reshape(len(x), RN_C, 4)
        assert (raw.max(axis=(1, 2)) == t).all(), t
        assert (raw[:, HI].max(axis=1) == t).all(), t
        s = _shift(t)
        if s:
            ties = (raw % (1 << s) == (1 << s >> 1)) & (raw < t)
            assert ties.any(axis=(1, 2)).all(), (t, "no rounding tie")
        if t == (128 << s) - 1 and s:
            assert ((t + (1 << s >> 1)) >> s) == 128 and (fe.features.max(axis=1) == 127).all(), t


@pytest.mark.gpu
def test_relunorm_shift_boundaries(lib, oracle):
    """both front-ends against the oracle; each case's eight images in every position of a group of eight (C = 48), so the
    maximum's channel sits in another tile than most of its image for one of them"""
    from bitnetmcu_b200 import _lib
    for t in RN_TARGETS:
        m, x = _relunorm_model(t)
        x = np.concatenate([np.roll(x, k, axis=0) for k in range(8)] + [x[:3]])     # 67 images: a ragged last group
        want = oracle.infer(m, x)
        for fe in (_lib.CNN_AUTO, _lib.CNN_CUDA_CORES):
            e = engine(m, cnn_frontend=fe)
            lo, la = e.infer(x)
            assert np.array_equal(lo, want[0]) and np.array_equal(la, want[1]), (t, fe, np.argwhere(lo != want[0])[:4])
            e.close()


# ---- the emulator's renormalisation ties -----------------------------------------------------------------------------------
# Every conv layer has two taps of 1 side by side in its first row.  Pixel row 0 at 127 puts 254 into conv1 row 0; after each
# renormalisation (scale 127 / 254 = 0.5 exactly) that row is 127 again, so conv2 and conv3 peak at 254 as well, and every odd
# sum below is an exact .5 tie.  Float images of integers with largest magnitude 127 scale to themselves.

def _tie_model(channels=16):
    w = np.zeros((channels, 9), dtype=np.int8)
    w[:, :2] = 1
    return cnn_model(channels, 10, seed=254, w=(w, w, w), hidden=())


def _tie_images(m, n, seed):
    """n images of uniform pixels in [-127, 127] below a row of 127, those of 2n with a tie of even floor at every stage"""
    rng = np.random.default_rng(seed)
    x = rng.integers(-127, 128, size=(2 * n, 16, 16))
    x[:, 0, :] = 127
    x = x.reshape(2 * n, 256).astype(np.float32)
    keep = np.ones(2 * n, dtype=bool)
    for c in cnn_stages(m, x)[:3]:
        keep &= (c.reshape(2 * n, -1) % 4 == 1).any(axis=1)
    assert keep.sum() >= n
    return x[keep][:n]


def _half_up(v):
    return np.floor(v + 0.5)


def test_tie_images_hit_their_targets():
    """each renormalisation's maximum is 254 for every image and below it lie ties whose floor is even (s = 1 mod 4); half up
    instead of half to even changes the features of most images"""
    m = _tie_model()
    x = _tie_images(m, 600, seed=1)
    assert np.array_equal(scale_images(x), x.astype(np.int8))
    stages = cnn_stages(m, x)
    for k, c in enumerate(stages[:3]):
        c = c.reshape(len(x), -1)
        assert (c.max(axis=1) == 254).all(), k
        assert ((c % 4 == 1).sum(axis=1) > 0).all(), k
    changed = (cnn_stages(m, x, rounding=_half_up)[3] != stages[3]).any(axis=1)
    assert changed.mean() > 0.5, changed.mean()


@pytest.mark.gpu
def test_emulator_renormalisation_ties(lib, capfd, monkeypatch):
    """k_cnn_emul_frontend == the layered route == the restatement, tolerance 0"""
    m = _tie_model()
    x = _tie_images(m, 600, seed=1)
    e, err = verbose_engine(capfd, monkeypatch, lambda: engine(m))
    assert route(err, "emulator").startswith("k_cnn_emul_frontend + "), err
    want = emulate(m, x)
    lo, la = run_emulator(e, x)
    assert np.array_equal(lo, want), np.argwhere(lo != want)[:5]
    assert np.array_equal(la, np.argmax(want, axis=1))
    lo2, la2 = run_emulator_layered(e, x)
    assert np.array_equal(lo2, want) and np.array_equal(la2, la)
    e.close()


# ---- more than 256 channels ------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_more_than_256_channels(lib, capfd, monkeypatch):
    """the C engine has no front-end for 272 channels (BNM_E_UNSUPPORTED, naming the front-end); the emulator runs them layer
    by layer"""
    import torch
    m = cnn_model(272, 10, seed=272)
    x = _tie_images(_tie_model(), 40, seed=2) * np.float32(0.5)
    e, err = verbose_engine(capfd, monkeypatch, lambda: engine(m))
    assert route(err, "emulator") == "layer by layer", err
    d_x = torch.from_numpy(scale_images(x)).cuda()
    lo = torch.empty((len(x), 10), dtype=torch.int32, device="cuda")
    rc = lib.bnm_infer_batch_device(e.handle, C.c_void_p(d_x.data_ptr()), len(x), C.c_void_p(lo.data_ptr()), None, None)
    assert rc == BNM_E_UNSUPPORTED
    assert "CNN front-end: 272 channels" in lib.bnm_last_error().decode()
    got, _ = run_emulator(e, x)
    assert np.array_equal(got, emulate(m, x))
    e.close()
