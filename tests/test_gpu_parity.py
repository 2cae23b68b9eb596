"""GPU parity tests (run with -m gpu on an H100): the CUDA paths, called through the C ABI, against the oracle and
the committed golden vectors made by the unmodified reference.  Integer work: the bar is bit-exact."""
import ctypes as C
import json
import os
import zlib

import numpy as np
import pytest

from conftest import GOLDEN, load_model, model_names
from restate import scale_images
from support import N_MANY, engine, frontends, gather_call, kernel_clone, kernel_copies_are_kernels, kernel_copy, lib

pytestmark = pytest.mark.gpu


def _rand_images(n, seed=0):
    rng = np.random.default_rng(seed)
    imgs = rng.integers(-128, 128, size=(n, 256)).astype(np.int8)
    k = min(n, 64)
    imgs[:k] = np.clip(imgs[:k], -20, 127)        # MNIST-like: background ~ -20, strokes to 127
    if n > 200:
        imgs[64:80] = -128
        imgs[80:96] = 127
        imgs[96:112] = 0
        imgs[112:128, ::2] = 0
    return imgs


@pytest.mark.parametrize("path", ["layers", "tcgen05"])
@pytest.mark.parametrize("name", model_names())
def test_model_matches_golden_and_oracle(lib, oracle, golden, digits, name, path):
    from bitnetmcu_b200 import _lib
    model = load_model(name)
    n = 5000 + 37
    r = _rand_images(n, seed=len(name))
    oo, ol = oracle.infer(model, r)
    for fe in frontends(model):
        e = engine(model, _lib.PATH_LAYERS if path == "layers" else _lib.PATH_TCGEN05, cnn_frontend=fe)
        assert e.active_path == (_lib.PATH_LAYERS if path == "layers" else _lib.PATH_TCGEN05)
        imgs, _ = digits
        lo, la = e.infer(imgs)
        assert np.array_equal(lo, golden[name + "/digits_logits"]), f"digits logits differ from the reference (front-end {fe})"
        assert np.array_equal(la, golden[name + "/digits_labels"])
        xs = oracle.xorshift_images(256)
        lo, la = e.infer(xs)
        assert np.array_equal(lo, golden[name + "/xs_logits"]), f"front-end {fe}"
        assert np.array_equal(la, golden[name + "/xs_labels"])
        # ragged random batch (not a multiple of the 128-image tile), full compare with the oracle
        lo, la = e.infer(r)
        assert np.array_equal(lo, oo), f"front-end {fe}: {np.argwhere(lo != oo)[:5]}"
        assert np.array_equal(la, ol)
        e.close()


@pytest.mark.parametrize("n", [0, 1, 2, 127, 128, 129, 255, 257, 1000])
def test_edge_batch_sizes(lib, oracle, n):
    from bitnetmcu_b200 import _lib
    for name in ("fc", "cnn_48"):
        m = load_model(name)
        for path in (_lib.PATH_LAYERS, _lib.PATH_TCGEN05):
            for fe in frontends(m):
                e = engine(m, path, cnn_frontend=fe)
                imgs = _rand_images(n, seed=n)
                lo, la = e.infer(imgs)
                assert lo.shape == (n, m.n_classes)
                if n:
                    oo, ol = oracle.infer(m, imgs)
                    assert np.array_equal(lo, oo) and np.array_equal(la, ol), (name, path, fe)
                e.close()


def test_survey_kat_on_gpu(lib, oracle):
    """SURVEY.md 8c: CRC-32 of the first 1000x10 logits of the xorshift stream = fc621bad; label sums."""
    kat = json.load(open(os.path.join(GOLDEN, "kat.json")))
    e = engine(load_model("fc"))
    xs = oracle.xorshift_images(400000)
    lo, la = e.infer(xs)
    assert "%08x" % zlib.crc32(lo[:1000].astype("<i4").tobytes()) == kat["fc_xs_crc32_first1000"]
    assert int(la[:1000].sum()) == kat["fc_xs_sum_labels_1000"]
    assert int(la.sum()) == kat["fc_xs_sum_labels_400000"]
    e.close()
    e = engine(load_model("cnn"))
    _, la = e.infer(xs[:40000])
    assert int(la.sum()) == kat["cnn_xs_sum_labels_40000"]
    e.close()


def test_nf4_extension(lib, oracle):
    """id 36 decodes to zeros like the reference (inference.c:202) unless the documented LUT extension is on."""
    from bitnetmcu_b200 import _lib
    m = load_model("rand_nf4_64")
    imgs = _rand_images(777)
    for path in (_lib.PATH_LAYERS, _lib.PATH_TCGEN05):
        e = engine(m, path)
        lo, _ = e.infer(imgs)
        assert not lo.any()
        e.set_option(_lib.OPT_NF4_EXTENSION, 1)
        lo, la = e.infer(imgs)
        oo, ol = oracle.infer(m, imgs, nf4_extension=True)
        assert oo.any() and np.array_equal(lo, oo) and np.array_equal(la, ol)
        e.close()


@pytest.mark.parametrize("name", ["fc", "binary160", "cnn"])
def test_full_size_batch_properties(lib, oracle, name):
    """BASELINE.json sizes (2^20 images): full compare with the oracle where it is quick, plus size-independent
    properties: shard invariance (batch == concat of shards) and permutation equivariance."""
    from bitnetmcu_b200 import _lib
    m = load_model(name)
    n = 1 << 20
    rng = np.random.default_rng(5)
    imgs = rng.integers(-128, 128, size=(n, 256), dtype=np.int8)
    e = engine(m)
    lo, la = e.infer(imgs)
    # shards of uneven size reproduce the same rows
    cut = 333333
    l1, a1 = e.infer(imgs[:cut])
    l2, a2 = e.infer(imgs[cut:])
    assert np.array_equal(lo, np.concatenate([l1, l2])) and np.array_equal(la, np.concatenate([a1, a2]))
    # permutation equivariance on a slice
    perm = rng.permutation(1 << 16)
    lp, _ = e.infer(imgs[: 1 << 16][perm])
    assert np.array_equal(lp, lo[: 1 << 16][perm])
    # checksum of checksums against the oracle on the full batch (FC) or a 1/8 sample (CNN is slower on CPU)
    ns = n if m.model_class == 0 else n // 8
    oo, ol = oracle.infer(m, imgs[:ns])
    assert zlib.crc32(lo[:ns].tobytes()) == zlib.crc32(oo.tobytes())
    assert np.array_equal(la[:ns], ol)
    e.close()


def test_host_pipeline_chunks(lib, oracle):
    from bitnetmcu_b200 import _lib
    m = load_model("fc")
    imgs = _rand_images(10000, seed=3)
    oo, ol = oracle.infer(m, imgs)
    for chunk in (128, 1024, 4096):
        e = engine(m)
        e.set_option(_lib.OPT_CHUNK_IMAGES, chunk)
        lo, la = e.infer(imgs)
        assert np.array_equal(lo, oo) and np.array_equal(la, ol)
        lo2, none = e.infer(imgs, want_labels=False)
        assert none is None and np.array_equal(lo2, oo)
        e.close()


def test_device_api_torch(lib, oracle):
    import torch
    m = load_model("fc")
    imgs = _rand_images(3000, seed=4)
    oo, ol = oracle.infer(m, imgs)
    e = engine(m)
    d_img = torch.from_numpy(imgs).cuda()
    d_log = torch.empty((3000, 10), dtype=torch.int32, device="cuda")
    d_lab = torch.empty(3000, dtype=torch.int32, device="cuda")
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        e.infer_device(d_img, d_log, d_lab)
    s.synchronize()
    assert np.array_equal(d_log.cpu().numpy(), oo) and np.array_equal(d_lab.cpu().numpy().astype(np.uint32), ol)
    assert e.launch_count(3000) == 1
    e.close()


@pytest.mark.parametrize("mode,n", [(0, 148 * 128 * 7 + 77), (1, 148 * 128 * 7 + 77), (2, 148 * 128 * 7 + 77), (2, 1000)])
def test_launch_overlap_modes(lib, oracle, kernel_copies_are_kernels, mode, n):
    """BNM_OPT_LAUNCH_OVERLAP: back-to-back launches on one stream stay bit-exact.  Modes 0 and 1 (dependent launch + wait)
    with the SAME buffers reused by every launch, a producer kernel (kernel_copy, an elementwise kernel: a copy_ would be a
    memcpy, which a dependent launch never overlaps) writing the images right before each launch and a consumer kernel
    (kernel_clone) reading the outputs right after -- ordinary stream semantics must hold; mode 2 with double-buffered
    inputs and outputs, the promise it asks for."""
    import torch
    from bitnetmcu_b200 import _lib
    m = load_model("fc")
    # n: several tiles per SM + a ragged last tile; the small n does not fill the GPU -> no early trigger even in mode 2
    batches = [_rand_images(n, seed=20 + k) for k in range(4)]
    want = [oracle.infer(m, b) for b in batches]
    e = engine(m)
    e.set_option(_lib.OPT_LAUNCH_OVERLAP, mode)
    s = torch.cuda.Stream()
    src = [torch.from_numpy(b).cuda() for b in batches]
    nbuf = 2 if mode == 2 else 1
    d_img = [torch.empty_like(src[0]) for _ in range(nbuf)]
    d_log = [torch.empty((n, 10), dtype=torch.int32, device="cuda") for _ in range(nbuf)]
    d_lab = [torch.empty(n, dtype=torch.int32, device="cuda") for _ in range(nbuf)]
    got = []
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        if mode == 2:
            for rep in range(6):                    # inputs resident; consecutive launches use disjoint buffers
                for k in range(4):
                    e.infer_device(src[k], d_log[k & 1], d_lab[k & 1])
            # the last two launches wrote batches 2 and 3 into buffers 0 and 1
            s.synchronize()
            got = [(d_log[0].cpu().numpy(), d_lab[0].cpu().numpy()), (d_log[1].cpu().numpy(), d_lab[1].cpu().numpy())]
            ref = [want[2], want[3]]
        else:
            ref = []
            for k in range(4):                      # producer kernel -> our kernel -> consumer kernel, same buffers every time
                kernel_copy(d_img[0], src[k])
                e.infer_device(d_img[0], d_log[0], d_lab[0])
                got.append((kernel_clone(d_log[0]), kernel_clone(d_lab[0])))
                ref.append(want[k])
            s.synchronize()
            got = [(a.cpu().numpy(), b.cpu().numpy()) for a, b in got]
    for (gl, gb), (wl, wb) in zip(got, ref):
        assert np.array_equal(gl, wl) and np.array_equal(gb.astype(np.uint32), wb)
    e.close()


# ---- the four kernels one by one --------------------------------------------------------------------------------

@pytest.mark.parametrize("enc", [1, 2, 4, 12, 16, 20, 36, 64, 3])
def test_processfclayer_batch(lib, oracle, enc):
    from bitnetmcu_b200 import engine as E
    rng = np.random.default_rng(enc)
    for n_in, n_out in [(256, 64), (64, 10), (160, 160), (320, 7), (32, 1)]:
        if enc == 64:
            n_in = (n_in + 9) // 10 * 10
            w = rng.integers(0, 65536, size=n_out * n_in // 10, dtype=np.uint32).astype(np.uint16)
        else:
            w = rng.integers(0, 2 ** 32, size=n_out * n_in // 4 + 4, dtype=np.uint64).astype(np.uint32)
        act = rng.integers(-128, 128, size=(300, n_in)).astype(np.int8)
        got = E.processfclayer(act, w, enc, n_in, n_out)
        want = np.stack([oracle.fclayer(act[i], w, enc, n_in, n_out) for i in range(act.shape[0])])
        assert np.array_equal(got, want), (enc, n_in, n_out)


def test_relunorm_batch(lib, oracle):
    from bitnetmcu_b200 import engine as E
    cases = [([127, 128, 255, 256, -3], [32, 32, 64, 64, 0], 3), ([255, 254, 253, 127, 1], [127, 127, 127, 64, 1], 0),
             ([1000, 509, 510, -1, 1], [125, 64, 64, 0, 0], 0), ([-5, -1, -7], [0, 0, 0], 1)]
    for x, want, pos in cases:
        out, p = E.relunorm(np.array(x, dtype=np.int32))
        assert out[0].tolist() == want and int(p[0]) == pos
    out, p = E.relunorm(np.array([5, 9, 9, 2], dtype=np.int32))
    assert int(p[0]) == 1
    rng = np.random.default_rng(1)
    for n_in in (1, 10, 33, 64, 160, 256, 1000):
        for scale in (1, 100, 20000, 500000, 4000000, 2 ** 30):
            x = rng.integers(-scale, scale + 1, size=(200, n_in)).astype(np.int32)
            x[::7] = -np.abs(x[::7]) - 1
            x[5, n_in // 2] = scale
            out, p = E.relunorm(x)
            for i in range(0, 200, 3):
                o, q = oracle.relunorm(x[i])
                assert q == int(p[i]) and np.array_equal(o, out[i])


def test_conv_pool_batch(lib, oracle):
    from bitnetmcu_b200 import engine as E
    rng = np.random.default_rng(2)
    for xy in (16, 14, 6, 4, 3):
        act = rng.integers(-20000, 20000, size=(50, xy * xy)).astype(np.int32)
        w = rng.integers(-128, 128, size=(7, 9)).astype(np.int8)
        got = E.conv33relu(act, w, xy, 4)
        for i in range(50):
            assert np.array_equal(got[i], oracle.conv33relu(act[i], w[i % 7], xy, 4))
        if xy % 2 == 0:
            gp = E.maxpool22(act, xy)
            for i in range(50):
                assert np.array_equal(gp[i], oracle.maxpool22(act[i], xy))


def test_reference_named_symbols(lib, oracle):
    """The drop-in symbols keep the reference signatures (BitNetMCU_inference.h:15-60), host pointers, one item."""
    rng = np.random.default_rng(3)
    m = load_model("fc")
    L = m.layers[0]
    act = rng.integers(-128, 128, size=256).astype(np.int8)
    out = np.zeros(64, dtype=np.int32)
    w = np.ascontiguousarray(L.weights)
    lib.processfclayer(C.c_void_p(act.ctypes.data), C.c_void_p(w.ctypes.data), L.bitperweight, 256, 64, C.c_void_p(out.ctypes.data))
    assert np.array_equal(out, oracle.fclayer(act, w, L.bitperweight, 256, 64))
    inp = out.copy()
    o8 = np.zeros(64, dtype=np.int8)
    pos = lib.ReLUNorm(C.c_void_p(inp.ctypes.data), C.c_void_p(o8.ctypes.data), 64)
    want, wpos = oracle.relunorm(out)
    assert pos == wpos and np.array_equal(o8, want)
    assert lib.ReLUNorm(C.c_void_p(inp.ctypes.data), C.c_void_p(o8.ctypes.data), 0) == 255
    # in-place conv + pool with the returned end pointers (dll.c:71-76)
    buf = rng.integers(-128, 128, size=256).astype(np.int32)
    w9 = rng.integers(-128, 128, size=9).astype(np.int8)
    want = oracle.conv33relu(buf, w9, 16, 4)
    end = lib.processconv33ReLU(C.c_void_p(buf.ctypes.data), C.c_void_p(w9.ctypes.data), 16, 4, C.c_void_p(buf.ctypes.data))
    assert end == buf.ctypes.data + 196 * 4 and np.array_equal(buf[:196], want)
    wantp = oracle.maxpool22(buf[:196], 14)
    end = lib.processmaxpool22(C.c_void_p(buf.ctypes.data), 14, C.c_void_p(buf.ctypes.data))
    assert end == buf.ctypes.data + 49 * 4 and np.array_equal(buf[:49], wantp)


# ---- worst-case magnitudes (SURVEY.md section 7 "Bit-exact corner cases" and range bounds) ------------------------

def _extreme_images():
    rng = np.random.default_rng(123)
    imgs = np.empty((400, 256), dtype=np.int8)
    imgs[:100] = -128
    imgs[100:200] = 127
    imgs[200:300] = rng.choice(np.array([-128, 127], dtype=np.int8), size=(100, 256))
    imgs[300:] = rng.integers(-128, 128, size=(100, 256))
    return imgs


@pytest.mark.parametrize("enc_name", ["4bitsym", "8bit", "FP130", "Binary", "2bitsym"])
def test_extreme_weights_fc(lib, oracle, enc_name):
    """All weights at the largest magnitude of the encoding (both signs), images at the int8 rails: the accumulators hit
    256*128*15 = 491 520 (4bitsym) / 4.2 M (8bit, FP130 incl. the +128 residual plane); rows with max < 128 (shift 0) and
    all-negative rows occur too."""
    from bitnetmcu_b200 import _lib, model as M, pack as P
    from bitnetmcu_b200.engine import Engine
    enc = P.QUANT_IDS[enc_name]
    lut = P.INT_LUT[enc]
    hi, lo = int(np.argmax(lut)), int(np.argmin(lut))
    rng = np.random.default_rng(7)
    layers = []
    widths = (256, 64, 64, 64, 10)
    for i in range(4):
        codes = rng.choice(np.array([hi, lo], dtype=np.uint32), size=(widths[i + 1], widths[i]), p=[0.6, 0.4])
        if i == 1:
            codes[:8] = lo          # some all-negative rows
        layers.append(P.fc_layer_from_codes(f"L{i + 1}", enc, codes))
    m = M.Model(model_class=M.MODEL_FCMNIST, layers=layers)
    imgs = _extreme_images()
    want_logits, want_labels = oracle.infer(m, imgs)
    assert np.abs(want_logits).max() > 1000
    for path in (_lib.PATH_LAYERS, _lib.PATH_TCGEN05):
        e = Engine(m, path=path)
        lo_, la_ = e.infer(imgs)
        assert np.array_equal(lo_, want_logits) and np.array_equal(la_, want_labels), path
        e.close()


def test_extreme_weights_cnn(lib, oracle):
    """conv weights at -128 / 127 and images at the rails: conv1 reaches its bound 9*128*128>>4 = 9216 (int16 pairs for the
    dp2a conv2), conv2 663 552, conv3 up to 4.7e7 (SURVEY.md section 7)."""
    from bitnetmcu_b200 import model as M
    from bitnetmcu_b200.engine import Engine
    base = load_model("cnn_48")
    rng = np.random.default_rng(9)
    for l in base.layers:
        if l.kind == M.LAYER_CONV33:
            w = rng.choice(np.array([-128, 127], dtype=np.int8), size=l.weights.shape)
            w[:9] = -128
            w[9:18] = 127
            l.weights = w
    imgs = _extreme_images()
    want_logits, want_labels = oracle.infer(base, imgs)
    from bitnetmcu_b200 import _lib
    for fe in frontends(base):
        e = Engine(base)
        e.set_option(_lib.OPT_CNN_FRONTEND, fe)
        lo_, la_ = e.infer(imgs)
        assert np.array_equal(lo_, want_logits) and np.array_equal(la_, want_labels), fe
        e.close()


def test_quantize_images_matches_numpy(lib):
    """SURVEY.md 8f rank 3: the float -> int8 input scaling of test_inference.py:140-141, bit-identical to NumPy float32
    (tolerance 0: every step is one correctly rounded IEEE op; np.round = round half to even)."""
    from bitnetmcu_b200 import engine as E
    rng = np.random.default_rng(4)
    x = rng.normal(size=(3000, 256)).astype(np.float32)
    x[:50] = (rng.integers(0, 256, size=(50, 256)) / 255.0 - 0.1307).astype(np.float32) / np.float32(0.3081)   # MNIST-like normalisation
    x[50] = 0.0                                  # all-zero image: the 1e-5 floor
    x[51] = 1e-7
    x[52, :] = np.float32(0.5) / np.float32(127.0) * np.arange(256, dtype=np.float32)   # many exact .5 ties
    x[53] = -x[52]
    x[54, 0] = 3e38
    want = scale_images(x)
    got = E.quantize_images(x)
    assert got.dtype == np.int8 and np.array_equal(got, want)


def test_float_images_to_labels_on_device(lib, oracle):
    """float images -> bnm_quantize_images_device -> bnm_infer_batch_device on one stream, nothing touches the host in
    between; compared with the NumPy scaling (test_inference.py:140-141) followed by the oracle."""
    import torch
    from bitnetmcu_b200 import engine as E
    m = load_model("fc")
    rng = np.random.default_rng(9)
    x = rng.normal(size=(5000, 256)).astype(np.float32)
    q = scale_images(x)
    want_logits, want_labels = oracle.infer(m, q)
    e = engine(m)
    d_x = torch.from_numpy(x).cuda()
    d_q = torch.empty((5000, 256), dtype=torch.int8, device="cuda")
    d_log = torch.empty((5000, 10), dtype=torch.int32, device="cuda")
    d_lab = torch.empty(5000, dtype=torch.int32, device="cuda")
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        E.quantize_images_device(d_x, d_q)
        e.infer_device(d_q, d_log, d_lab)
    s.synchronize()
    assert np.array_equal(d_q.cpu().numpy(), q)
    assert np.array_equal(d_log.cpu().numpy(), want_logits) and np.array_equal(d_lab.cpu().numpy().astype(np.uint32), want_labels)
    e.close()


# ---- function-level parity on the tensor-core path (VERDICT r1 item 8) --------------------------------------------
# processfclayer (inference.c:88-208) through fc_chain_kernel itself: a one-layer model's logits ARE the layer's output.

_FUSED_SINGLE = [(256, 64), (64, 10), (160, 160), (320, 7), (32, 1), (256, 17), (256, 37), (128, 250), (768, 10)]


@pytest.mark.parametrize("enc", [1, 2, 4, 12, 16, 20, 64])
def test_processfclayer_on_tcgen05(lib, oracle, enc):
    """Single-layer models over the (n_in, n_out) grid incl. 320->7, 160->160, ternary-padded widths and n_out in {17, 37,
    250} (> 16 classes: the chunked logits/argmax epilogue), both kernels, against the oracle's processfclayer + ReLUNorm."""
    from bitnetmcu_b200 import _lib, model as M, pack as P
    from bitnetmcu_b200.engine import Engine
    rng = np.random.default_rng(100 + enc)
    for n_in, n_out in _FUSED_SINGLE:
        if enc == 1 and n_in % 32:
            continue
        m = P.random_fc_model(enc, (n_in, n_out), seed=enc * 1000 + n_in + n_out)
        m.img_bytes = n_in                      # ternary: the layer declares the padded width, the image keeps n_in bytes
        imgs = rng.integers(-128, 128, size=(777, n_in)).astype(np.int8)
        imgs[:16] = -128
        imgs[16:32] = 127
        want, want_lab = oracle.infer(m, imgs)
        L = m.layers[0]
        row = oracle.fclayer(np.pad(imgs[40], (0, L.n_in - n_in)), L.weights, enc, L.n_in, n_out)
        assert np.array_equal(want[40], row)
        for path in (_lib.PATH_TCGEN05, _lib.PATH_LAYERS):
            e = Engine(m, path=path)
            assert e.active_path == path
            lo, la = e.infer(imgs)
            assert np.array_equal(lo, want), (enc, n_in, n_out, path, np.argwhere(lo != want)[:4])
            assert np.array_equal(la, want_lab), (enc, n_in, n_out, path)
            e.close()


@pytest.mark.parametrize("enc", [2, 4, 12, 16, 20, 64, 1])
@pytest.mark.parametrize("widths", [(256, 96, 64, 37), (256, 160, 160, 17), (256, 48, 250), (256, 16, 16, 10), (64, 224, 32, 20),
                                    (256, 64, 64, 64, 64, 64, 64, 64, 10), (256, 160, 144, 10), (256, 256, 10), (128, 176, 176, 176, 7),
                                    (256, 96, 96, 10)])
def test_chains_on_tcgen05(lib, oracle, enc, widths):
    """Random-code chains with odd shapes on the fused path: register-A layers of every width class (16..256, 64-wide pieces plus
    16-wide tails), FP130 with +128 (residual plane) in EVERY layer, > 16 classes, the 8-layer maximum, all three accumulator
    widths and both pipe counts."""
    from bitnetmcu_b200 import _lib, pack as P
    from bitnetmcu_b200.engine import Engine
    if enc == 1 and any(w % 32 for w in widths[:-1]):
        widths = tuple((w + 31) // 32 * 32 for w in widths[:-1]) + (widths[-1],)
    if enc == 2 and any(w % 16 for w in widths[:-1]):
        pytest.skip("2bitsym rows need n_in % 16 == 0")
    m = P.random_fc_model(enc, widths, seed=enc + sum(widths))
    m.img_bytes = widths[0]
    rng = np.random.default_rng(sum(widths))
    n_img = 148 * 128 * 3 + 11 if widths in ((256, 160, 144, 10), (256, 96, 96, 10)) else 1500 + 11   # several tiles per CTA for the new forms
    imgs = rng.integers(-128, 128, size=(n_img, widths[0])).astype(np.int8)
    imgs[:50] = np.clip(imgs[:50], 0, 127)
    want, want_lab = oracle.infer(m, imgs)
    e = Engine(m, path=_lib.PATH_TCGEN05)
    lo, la = e.infer(imgs)
    assert np.array_equal(lo, want), (enc, widths, np.argwhere(lo != want)[:4])
    assert np.array_equal(la, want_lab)
    e.close()


def test_later_model_keeps_earlier_models_shared_memory(lib, oracle):
    """Creating a model must not lower the dynamic shared memory limit of a kernel another live model launches: FC 4bitsym-64's
    fused launch asks for more shared memory than Binary-160's."""
    from bitnetmcu_b200 import _lib
    fc = engine(load_model("fc"), _lib.PATH_TCGEN05)
    b160 = engine(load_model("binary160"), _lib.PATH_TCGEN05)
    imgs = _rand_images(5000 + 37, seed=3)
    lo, la = fc.infer(imgs)
    oo, ol = oracle.infer(load_model("fc"), imgs)
    assert np.array_equal(lo, oo) and np.array_equal(la, ol)
    b160.close()
    fc.close()


def test_launch_overlap_mode2_reused_buffers_keep_stream_order(lib, oracle, kernel_copies_are_kernels):
    """Mode 2 drops the grid-dependency wait only for launches whose buffers differ from the previous call's.  Reusing the
    SAME buffers with a producer kernel (kernel_copy) in front of every launch and a consumer kernel (kernel_clone) after it
    (the pattern mode 2 does not promise) must still be ordered: the library falls back to the wait when it sees a pointer
    of the previous launch again."""
    import torch
    from bitnetmcu_b200 import _lib
    m = load_model("fc")
    n = 148 * 128 * 5 + 3
    batches = [_rand_images(n, seed=40 + k) for k in range(4)]
    want = [oracle.infer(m, b) for b in batches]
    e = engine(m)
    e.set_option(_lib.OPT_LAUNCH_OVERLAP, 2)
    s = torch.cuda.Stream()
    src = [torch.from_numpy(b).cuda() for b in batches]
    d_img = torch.empty_like(src[0])
    d_log = torch.empty((n, 10), dtype=torch.int32, device="cuda")
    d_lab = torch.empty(n, dtype=torch.int32, device="cuda")
    got = []
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        for rep in range(3):
            for k in range(4):
                kernel_copy(d_img, src[k])
                e.infer_device(d_img, d_log, d_lab)
                if rep == 2:
                    got.append((kernel_clone(d_log), kernel_clone(d_lab)))
        s.synchronize()
    for (gl, gb), (wl, wb) in zip(got, want):
        assert np.array_equal(gl.cpu().numpy(), wl) and np.array_equal(gb.cpu().numpy().astype(np.uint32), wb)
    e.close()


@pytest.mark.parametrize("channels", [8, 16, 24, 32, 40, 48, 64, 80, 96, 100, 112, 128, 144, 200, 256])
def test_cnn_frontends_agree_for_every_channel_count(lib, oracle, channels):
    """Random conv weights for every channel count the tensor-core front-end takes (multiples of 16 up to 128: tiles that
    straddle images for C = 48 / 80 / 96, eight images per tile for C = 16) against the oracle, both front-end kernels, ragged
    batch sizes around the group size; and counts only the CUDA-core kernel runs: not a multiple of 16 (idle threads in its
    CTA of 256 / C images), and more than 128 (one image per CTA)."""
    from bitnetmcu_b200 import _lib, model as M, pack as P
    from bitnetmcu_b200.engine import Engine
    rng = np.random.default_rng(channels)
    layers = []
    for name, xy in (("L2", 16), ("L4", 14)):
        layers.append(M.Layer(kind=M.LAYER_CONV33, name=name, bitperweight=8, n_in=xy, n_out=channels, in_channels=1 if xy == 16 else channels,
                              groups=1 if xy == 16 else channels, weights=rng.integers(-128, 128, size=channels * 9).astype(np.int8)))
    layers.append(M.Layer(kind=M.LAYER_MAXPOOL22, name="L6", n_in=12, n_out=6))
    layers.append(M.Layer(kind=M.LAYER_CONV33, name="L7", bitperweight=8, n_in=6, n_out=channels, in_channels=channels, groups=channels,
                          weights=rng.integers(-128, 128, size=channels * 9).astype(np.int8)))
    layers.append(M.Layer(kind=M.LAYER_MAXPOOL22, name="L9", n_in=4, n_out=2))
    fc = P.random_fc_model(M.ENC_4BITSYM, (channels * 4, 64, 10), seed=channels)
    for i, l in enumerate(fc.layers):
        l.name = f"L{11 + 2 * i}"
        layers.append(l)
    m = M.Model(model_class=M.MODEL_CNNMNIST, layers=layers)
    m.validate()
    for n in (1, 7, 8, 9, 300, 4099):
        imgs = _rand_images(n, seed=n + channels)
        want, want_lab = oracle.infer(m, imgs)
        for fe in frontends(m):
            e = Engine(m)
            e.set_option(_lib.OPT_CNN_FRONTEND, fe)
            lo, la = e.infer(imgs)
            assert np.array_equal(lo, want) and np.array_equal(la, want_lab), (channels, n, fe, np.argwhere(lo != want)[:4])
            e.close()


# ---- emulation mode: QuantizedModel.inference_quantized on the GPU (SURVEY.md 8f rank 4) -----------------------------

@pytest.mark.parametrize("name", ["fc", "1k", "12k_FP130", "2bitsym96", "8bit64", "binary160", "ternary64", "cnn", "cnn_48", "cnn_16small"])
def test_inference_quantized_emulation_matches_reference_python(lib, name):
    """tests/golden/emulator.npz holds the logits of the reference's own Python emulator (BitNetMCU.py:420-535, run in the build
    container by tests/golden/make_emulator_golden.py) on 64 float32 images.  Every intermediate of the emulator is an exact
    dyadic rational for these encodings (and the conv renormalisation is one IEEE float64 multiply + rint), so the GPU restatement
    must reproduce the float64 logits exactly: tolerance 0."""
    from bitnetmcu_b200.engine import Engine
    g = np.load(os.path.join(GOLDEN, "emulator.npz"))
    e = Engine(load_model(name))
    got = e.inference_quantized(g["images"])
    want = g[name]
    assert got.shape == want.shape and got.dtype == np.float64
    assert np.array_equal(got, want), (name, np.argwhere(got != want)[:5], got[0][:4], want[0][:4])
    assert np.array_equal(np.argmax(got, axis=1), np.argmax(want, axis=1))
    e.close()


# ---- fused result exchange (SURVEY.md 8e): the epilogue stores rows into other buffers as well ---------------------------------

def _gather_case(lib, oracle, name, n, dst_device):
    """One engine on GPU 0; destination buffers on `dst_device` (0: plain second buffers; 1: peer memory over NVLink)."""
    import torch
    from bitnetmcu_b200 import _lib
    m = load_model(name)
    imgs = _rand_images(n, seed=77)
    want, want_lab = oracle.infer(m, imgs)
    e = engine(m, _lib.PATH_TCGEN05)
    if dst_device != 0:
        _lib.check(lib.bnm_enable_peer_access(0, dst_device), "bnm_enable_peer_access")
    C_ = m.n_classes
    rows, off = n + 640, 512            # destination holds more rows; this call's rows land at row_offset 512
    dst_log = [torch.full((rows, C_), -7, dtype=torch.int32, device=f"cuda:{dst_device}") for _ in range(2)]
    dst_lab = [torch.full((rows,), -7, dtype=torch.int32, device=f"cuda:{dst_device}") for _ in range(2)]
    d_img = torch.from_numpy(imgs).cuda(0)
    d_log = torch.empty((n, C_), dtype=torch.int32, device="cuda:0")
    d_lab = torch.empty(n, dtype=torch.int32, device="cuda:0")
    g = _lib.BnmGather()
    g.n_labels_dst, g.n_logits_dst, g.row_offset = 2, 2, off
    for k in range(2):
        g.labels_dst[k] = dst_lab[k].data_ptr()
        g.logits_dst[k] = dst_log[k].data_ptr()
    torch.cuda.synchronize()
    s = torch.cuda.current_stream(0)
    _lib.check(gather_call(lib, e, d_img, d_log, d_lab, g, s), "gather")
    assert np.array_equal(d_log.cpu().numpy(), want) and np.array_equal(d_lab.cpu().numpy().astype(np.uint32), want_lab)
    # one byte per label (bnm_gather.labels_u8)
    dst8 = torch.full((rows,), 201, dtype=torch.uint8, device=f"cuda:{dst_device}")
    g8 = _lib.BnmGather()
    g8.n_labels_dst, g8.n_logits_dst, g8.row_offset, g8.labels_u8 = 1, 0, off, 1
    g8.labels_dst[0] = dst8.data_ptr()
    _lib.check(gather_call(lib, e, d_img, d_log, d_lab, g8, s), "gather u8")
    g8h = dst8.cpu().numpy()
    assert np.array_equal(g8h[off:off + n], want_lab.astype(np.uint8)) and (g8h[:off] == 201).all() and (g8h[off + n:] == 201).all()
    for k in range(2):
        gl, gb = dst_log[k].cpu().numpy(), dst_lab[k].cpu().numpy()
        assert np.array_equal(gl[off:off + n], want), (name, n, dst_device, k)
        assert np.array_equal(gb[off:off + n].astype(np.uint32), want_lab)
        assert (gl[:off] == -7).all() and (gl[off + n:] == -7).all() and (gb[:off] == -7).all() and (gb[off + n:] == -7).all()   # nothing else touched
    e.close()


@pytest.mark.parametrize("name,n", [("fc", N_MANY), ("fc", 1000), ("cnn_letters", 3000), ("binary160", 5000), ("cnn_48", 2049)])
def test_fused_gather_epilogue_same_gpu(lib, oracle, name, n):
    """bnm_infer_batch_device_gather with destinations on the same GPU: full tiles take the staged bulk-store path (16-byte
    aligned rows), the ragged last tile and > 16 classes (cnn_letters: 37) the direct stores; rows outside the call stay untouched."""
    _gather_case(lib, oracle, name, n, 0)


def test_fused_gather_epilogue_peer_gpu(lib, oracle):
    """Same with the destinations in the memory of a second GPU (P2P over NVLink), when the box has one."""
    if lib.bnm_device_count() < 2:
        pytest.skip("needs two GPUs")
    _gather_case(lib, oracle, "fc", 148 * 128 * 3 + 5, 1)


# ---- float input fused into the FC kernel's load stage (SURVEY.md 8f rank 3) ----------------------------------------------------------

def _edge_row_images(n, elems, seed):
    rng = np.random.default_rng(seed)
    x = rng.normal(size=(n, elems)).astype(np.float32)
    k = min(n, 50)
    x[:k] = (rng.integers(0, 256, size=(k, elems)) / 255.0 - 0.1307).astype(np.float32) / np.float32(0.3081)   # MNIST-like normalisation
    if n > 60:
        x[50] = 0.0                                                                      # all-zero image: the 1e-5 floor
        x[51] = 1e-7
        x[52, :] = np.float32(0.5) / np.float32(127.0) * np.arange(elems, dtype=np.float32)   # many exact .5 ties
        x[53] = -x[52]
        x[54, 0] = 3e38
        x[55] = -1.0
    return x


@pytest.mark.parametrize("name,n", [("fc", N_MANY), ("fc", 1), ("fc", 129), ("ternary64", 5000), ("1k", 4097), ("binary160", 3000), ("cnn_48", 2500),
                                    ("binary160", (1 << 20) + 77)])
def test_float_input_fused_into_the_fc_kernel(lib, oracle, name, n):
    """bnm_infer_batch_device_f32: float32 images -> int32 logits in one kernel for FC models (four quantiser warps write the int8 A
    operand of layer 1 into shared memory, SWIZZLE_128B by hand), through the scaling kernel for CNN models and wider FC models,
    per pass of 2^20 images (Binary-160 at 2^20 + 77 crosses a pass); compared with the NumPy scaling of test_inference.py:140-141
    followed by the oracle.  Tolerance 0."""
    import torch
    m = load_model(name)
    x = _edge_row_images(n, m.img_bytes, seed=n)
    q = scale_images(x)
    want, want_lab = oracle.infer(m, q)
    e = engine(m)
    d_x = torch.from_numpy(x).cuda()
    d_log = torch.empty((n, m.n_classes), dtype=torch.int32, device="cuda")
    d_lab = torch.empty(n, dtype=torch.int32, device="cuda")
    for _ in range(2):                      # twice: the launch is repeatable (each one starts its ring at stage 0, phase 0)
        e.infer_device_f32(d_x, d_log, d_lab)
    torch.cuda.synchronize()
    got = d_log.cpu().numpy()
    assert np.array_equal(got, want), (name, n, np.argwhere(got != want)[:5])
    assert np.array_equal(d_lab.cpu().numpy().astype(np.uint32), want_lab)
    e.close()


def test_float_input_odd_row_widths(lib, oracle):
    """Rows narrower than 256 elements (160: the second 128-byte atom is half padding; 64, 32: one atom) through the fused float path."""
    import torch
    from bitnetmcu_b200 import _lib, pack as P
    from bitnetmcu_b200.engine import Engine
    for n_in, n_out in [(160, 160), (64, 10), (32, 1), (128, 16)]:
        m = P.random_fc_model(4, (n_in, 64, n_out), seed=n_in)
        m.img_bytes = n_in
        x = _edge_row_images(1777, n_in, seed=n_in)
        want, want_lab = oracle.infer(m, scale_images(x))
        e = Engine(m, path=_lib.PATH_TCGEN05)
        d_x = torch.from_numpy(x).cuda()
        d_log = torch.empty((1777, n_out), dtype=torch.int32, device="cuda")
        d_lab = torch.empty(1777, dtype=torch.int32, device="cuda")
        e.infer_device_f32(d_x, d_log, d_lab)
        torch.cuda.synchronize()
        assert np.array_equal(d_log.cpu().numpy(), want), (n_in, n_out)
        assert np.array_equal(d_lab.cpu().numpy().astype(np.uint32), want_lab)
        e.close()
