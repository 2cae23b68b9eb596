"""The emulator's fused routes beyond the float-input row (bnm_emulate_batch_device, emulate_device in capi.cu):

* FC models wider than 64 or with more than 16 classes: k_quantize_images, then fc_emul_i8_kernel<max_n> (int8 TMA input, one
  pipe, one slot, the last layer at full width, the emulator's hidden-layer rule and float64 logits);
* CNN models up to 128 channels: k_cnn_emul_frontend (input scaling, three convolutions with the per-image renormalisation, two
  pools; BitNetMCU.py:435-445, 459-526), then fc_emul_i8_kernel on its features.

CPU tests: a NumPy restatement of the emulator's CNN path against the reference emulator's own logits (the expectation of the
GPU tests), and the new kernels' SASS.  GPU tests (tolerance 0): fused == layered (BNM_PATH_LAYERS) == restatement."""
import os
import re
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, load_model

LEVEL_SHIFT = {2: 1, 4: 1}          # 2bitsym / 4bitsym levels are half the engine's integer weights (BitNetMCU.py:155-164)
CHUNK = 1 << 20                     # images per front-end / FC launch pair of the new routes


# ---- NumPy restatement of the emulator ------------------------------------------------------------------------------------

def _scale(x):
    """BitNetMCU.py:435-436 in float32: round_half_even(x * 127 / max(max|x|, 1e-5)).clip(-128, 127)"""
    x = np.asarray(x, dtype=np.float32)
    scale = np.float32(127.0) / np.maximum(np.abs(x).max(axis=-1, keepdims=True), np.float32(1e-5))
    return np.round(x * scale).clip(-128, 127).astype(np.int64)


def _fc(model, act):
    """the BitLinear layers (BitNetMCU.py:452-457, 527-530) on float64 activations [n, k] -> float64 logits"""
    from bitnetmcu_b200 import model as M, pack as P
    fc = [l for l in model.layers if l.kind == M.LAYER_FC]
    act = act.astype(np.float64)
    for i, l in enumerate(fc):
        w = P.decode_int_weights(l).astype(np.float64)[:, :act.shape[1]] / 2.0 ** LEVEL_SHIFT.get(l.bitperweight, 0)
        conv = act @ w.T
        if i + 1 == len(fc):
            return conv
        top = np.maximum(conv.max(axis=-1, keepdims=True), 1e-5)
        act = np.round(conv * np.exp2(np.floor(np.log2(127.0 / top)))).clip(0, 127)


def _conv_relu(a, w):
    """depthwise 3x3 (k_conv33relu's indices, no shift) + ReLU: a int64 [n, 1 or C, H, W], w int8 [C * 9] -> [n, C, H-2, W-2]"""
    n, _, h, wd = a.shape
    k = w.reshape(-1, 3, 3).astype(np.int64)
    out = np.zeros((n, k.shape[0], h - 2, wd - 2), dtype=np.int64)
    for dr in range(3):
        for dc in range(3):
            out += k[None, :, dr, dc, None, None] * a[:, :, dr:dr + h - 2, dc:dc + wd - 2]
    return np.maximum(out, 0)


def _renorm(v):
    """BitConv2d's renormalisation over each image's C*H*W outputs (float64); an all-zero image stays zero"""
    m = v.reshape(v.shape[0], -1).max(axis=1)
    scale = np.where(m > 0, 127.0 / np.maximum(m, 1), 0.0)[:, None, None, None]
    return np.round(v * scale).clip(0, 127).astype(np.int64)


def _pool(v):
    n, c, h, w = v.shape
    return v.reshape(n, c, h // 2, 2, w // 2, 2).max(axis=(3, 5))


def cnn_features(model, x):
    """float32 images [n, 256] -> int64 features [n, C*4], the (C, 2, 2) flatten"""
    from bitnetmcu_b200 import model as M
    w1, w2, w3 = [l.weights for l in model.layers if l.kind == M.LAYER_CONV33]
    a = _scale(x).reshape(-1, 1, 16, 16)
    a = _renorm(_conv_relu(a, w1))
    a = _pool(_renorm(_conv_relu(a, w2)))
    a = _pool(_renorm(_conv_relu(a, w3)))
    return a.reshape(a.shape[0], -1)


def emulate(model, x, block=512):
    """float32 images -> the emulator's float64 logits, FC and CNN models"""
    if model.model_class == 0:
        return _fc(model, _scale(x))
    return np.concatenate([_fc(model, cnn_features(model, x[i:i + block])) for i in range(0, len(x), block)])


def test_cnn_restatement_reproduces_reference_emulator():
    """tests/golden/emulator.npz holds the reference emulator's own logits"""
    g = np.load(os.path.join(GOLDEN, "emulator.npz"))
    for name in ("cnn", "cnn_48", "cnn_16small"):
        got = emulate(load_model(name), g["images"])
        assert got.dtype == np.float64 and np.array_equal(got, g[name]), (name, np.argwhere(got != g[name])[:5])


def test_new_kernels_sass(built):
    """four int8 emulator rows (IGMMA, no local memory) next to exactly one fc_emul_kernel and eight fc_chain_kernel
    instantiations, and a front-end kernel without local memory"""
    from bitnetmcu_b200 import _lib
    out = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    kernels = {k.split()[0]: k for k in re.split(r"\n\s*Function : ", out)[1:]}
    rows = sorted(k for k in kernels if k.startswith("_ZN3bnm17fc_emul_i8_kernel"))
    assert [re.search(r"ILi(\d+)E", k).group(1) for k in rows] == ["128", "192", "256", "64"], rows
    assert len([k for k in kernels if k.startswith("_ZN3bnm14fc_emul_kernel")]) == 1
    assert len([k for k in kernels if k.startswith("_ZN3bnm15fc_chain_kernel")]) == 8
    front = [k for k in kernels if k.startswith("_ZN3bnm19k_cnn_emul_frontend")]
    assert len(front) == 1
    for k in rows + front:
        ins = [i.strip() for i in re.findall(r"/\*[0-9a-f]{4,}\*/\s+([^;]*);", kernels[k])]
        assert len(ins) > 100, k
        assert not [i for i in ins if re.match(r"(@\S+\s+)?(LDL|STL)\b", i)], f"local memory in {k}"
        assert (k in front) != any(i.startswith("IGMMA") for i in ins), k


# ---- GPU ------------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def lib(built):
    from bitnetmcu_b200 import _lib
    l = _lib.load()
    assert l.bnm_device_count() > 0, "no CUDA device"
    return l


def _route(model, capfd, monkeypatch):
    """an engine built with BNM_VERBOSE set, and the emulator route line it prints"""
    from bitnetmcu_b200.engine import Engine
    monkeypatch.setenv("BNM_VERBOSE", "1")
    capfd.readouterr()
    e = Engine(model, device=0)
    lines = [l for l in capfd.readouterr().err.splitlines() if "emulator route:" in l]
    monkeypatch.delenv("BNM_VERBOSE")
    assert len(lines) == 1, lines
    return e, lines[0].split("emulator route: ")[1]


def _run(e, x, want_logits=True, want_labels=True, stream=None):
    """device call -> (logits, labels) as NumPy, None for what was not asked for; x NumPy or a CUDA tensor"""
    import torch
    d_x = x if isinstance(x, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).cuda()
    n = d_x.shape[0]
    lo = torch.full((n, e.n_classes), np.nan, dtype=torch.float64, device="cuda") if want_logits else None
    la = torch.full((n,), -1, dtype=torch.int32, device="cuda") if want_labels else None
    e.inference_quantized_device(d_x, lo, la, stream=stream)
    torch.cuda.synchronize()
    return (lo.cpu().numpy() if want_logits else None), (la.cpu().numpy().astype(np.int64) if want_labels else None)


def _layered(e, x):
    from bitnetmcu_b200 import _lib
    e.set_option(_lib.OPT_PATH, _lib.PATH_LAYERS)
    try:
        return _run(e, x)
    finally:
        e.set_option(_lib.OPT_PATH, _lib.PATH_AUTO)


def _check(e, x, want, tag):
    """default path == restatement (logits and np.argmax labels), and == the layered emulator"""
    lo, la = _run(e, x)
    assert np.array_equal(lo, want), (tag, np.argwhere(lo != want)[:5])
    assert np.array_equal(la, np.argmax(want, axis=1)), tag
    lo2, la2 = _layered(e, x)
    assert np.array_equal(lo2, lo) and np.array_equal(la2, la), tag


def _images(n, seed, elems=256):
    rng = np.random.default_rng(seed)
    x = rng.normal(size=(n, elems)).astype(np.float32)
    k = min(n, 40)
    x[:k] = (rng.integers(0, 256, size=(k, elems)) / 255.0 - 0.1307).astype(np.float32) / np.float32(0.3081)
    return x


GOLDEN_ROUTES = {
    "fc": "fc_emul_kernel<64,1,float,emul>", "1k": "fc_emul_kernel<64,1,float,emul>",
    "12k_FP130": "fc_emul_kernel<64,1,float,emul>", "8bit64": "fc_emul_kernel<64,1,float,emul>",
    "ternary64": "fc_emul_kernel<64,1,float,emul>",
    "binary160": "k_quantize_images + fc_emul_i8_kernel<192,1,emul>",
    "2bitsym96": "k_quantize_images + fc_emul_i8_kernel<128,1,emul>",
    "cnn": "k_cnn_emul_frontend + fc_emul_i8_kernel<128,1,emul>",
    "cnn_48": "k_cnn_emul_frontend + fc_emul_i8_kernel<128,1,emul>",
    "cnn_16small": "k_cnn_emul_frontend + fc_emul_i8_kernel<64,1,emul>",
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(GOLDEN_ROUTES))
def test_golden_models_on_default_route(lib, capfd, monkeypatch, name):
    """all ten emulator.npz models on the default path: the reference emulator's logits bit for bit, labels = np.argmax, and the
    route BNM_VERBOSE names"""
    g = np.load(os.path.join(GOLDEN, "emulator.npz"))
    e, route = _route(load_model(name), capfd, monkeypatch)
    assert route == GOLDEN_ROUTES[name], (name, route)
    _check(e, g["images"], g[name], name)
    e.close()


def _fc_models():
    from bitnetmcu_b200 import model as M, pack as P
    out = []
    for i, enc in enumerate((M.ENC_BINARY, M.ENC_2BITSYM, M.ENC_4BITSYM, M.ENC_4BIT, M.ENC_8BIT, M.ENC_FP130, M.ENC_TERNARY)):
        width = (96, 160, 192, 256)[i % 4]
        out.append((f"{M.ENC_NAMES[enc]}-{width}", P.random_fc_model(enc, (256, width, width, 10), seed=enc), (width + 63) // 64 * 64))
    for width in (96, 160, 192, 256):
        out.append((f"4bitsym-{width}-mixed", P.random_fc_model(M.ENC_4BITSYM, (256, width, 64, width, 12), seed=width), (width + 63) // 64 * 64))
    for cls in (17, 37, 47, 62):
        out.append((f"2bitsym-64-{cls}cls", P.random_fc_model(M.ENC_2BITSYM, (256, 64, 64, cls), seed=cls), 64))
    out.append(("fp130-64-37cls", P.random_fc_model(M.ENC_FP130, (256, 64, 37), seed=37), 64))
    out.append(("ternary-64-47cls", P.random_fc_model(M.ENC_TERNARY, (256, 64, 47), seed=47), 64))
    m = P.random_fc_model(M.ENC_4BITSYM, (784, 64, 10), seed=784)   # 784-byte rows: no fused plan, layer by layer
    m.img_bytes = 784
    out.append(("4bitsym-784in", m, None))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("idx", range(18))
def test_random_fc_models(lib, capfd, monkeypatch, idx):
    """every encoding (FP130's residual plane, Ternary's padded inputs) at widths 96 / 160 / 192 / 256, 17 / 37 / 47 / 62
    classes at 64 wide, 784-byte rows: fused == layered == restatement"""
    tag, m, row = _fc_models()[idx]
    x = _images(3001, seed=idx, elems=m.img_bytes)
    e, route = _route(m, capfd, monkeypatch)
    assert route == (f"k_quantize_images + fc_emul_i8_kernel<{row},1,emul>" if row else "layer by layer"), (tag, route)
    _check(e, x, emulate(m, x), tag)
    e.close()


def cnn_model(channels, n_classes, seed, w=(None, None, None)):
    """a random CNN model: conv weights uniform in [-128, 127] with +-127 taps in every layer (or the given weights), a 64-wide
    4bitsym hidden layer and an n_classes head"""
    from bitnetmcu_b200 import model as M, pack as P
    rng = np.random.default_rng(seed)

    def conv_w(i):
        if w[i] is not None:
            return np.asarray(w[i], dtype=np.int8).reshape(channels * 9)
        k = rng.integers(-128, 128, size=channels * 9).astype(np.int8)
        k[rng.integers(0, channels * 9, size=max(2, channels))] = 127
        k[rng.integers(0, channels * 9, size=max(2, channels))] = -127
        return k
    layers = [M.Layer(kind=M.LAYER_CONV33, name="L2", bitperweight=8, n_in=16, n_out=channels, in_channels=1, groups=1, weights=conv_w(0)),
              M.Layer(kind=M.LAYER_CONV33, name="L4", bitperweight=8, n_in=14, n_out=channels, in_channels=channels, groups=channels,
                      weights=conv_w(1)),
              M.Layer(kind=M.LAYER_MAXPOOL22, name="L6", n_in=12, n_out=6),
              M.Layer(kind=M.LAYER_CONV33, name="L7", bitperweight=8, n_in=6, n_out=channels, in_channels=channels, groups=channels,
                      weights=conv_w(2)),
              M.Layer(kind=M.LAYER_MAXPOOL22, name="L9", n_in=4, n_out=2)]
    fc = P.random_fc_model(M.ENC_4BITSYM, (channels * 4, 64, n_classes), seed=seed)
    for i, l in enumerate(fc.layers):
        l.name = f"L{11 + 2 * i}"
        layers.append(l)
    m = M.Model(model_class=M.MODEL_CNNMNIST, layers=layers)
    m.validate()
    return m


@pytest.mark.gpu
@pytest.mark.parametrize("channels", [16, 24, 48, 64, 128])
@pytest.mark.parametrize("n_classes", [10, 37])
def test_random_cnn_models(lib, capfd, monkeypatch, channels, n_classes):
    m = cnn_model(channels, n_classes, seed=channels + n_classes)
    x = _images(1500, seed=channels)
    e, route = _route(m, capfd, monkeypatch)
    assert route.startswith("k_cnn_emul_frontend + fc_emul_i8_kernel<64,"), route
    _check(e, x, emulate(m, x), (channels, n_classes))
    e.close()


@pytest.mark.gpu
def test_crafted_inputs(lib):
    """all-zero images; conv2 or conv3 outputs <= 0 everywhere (non-positive taps on non-negative inputs): a renormalisation
    whose maximum is 0 gives zeros, where NumPy would give nan"""
    from bitnetmcu_b200.engine import Engine
    x = _images(700, seed=5)
    x[:110] = 0.0
    x[100:110, 7] = np.float32(-3.0)          # one negative pixel, every other one zero
    rng = np.random.default_rng(3)
    neg = -rng.integers(0, 129, size=48 * 9)
    for w, what in (((None, None, None), "random"), ((None, neg, None), "conv2 <= 0"), ((None, None, neg), "conv3 <= 0")):
        m = cnn_model(48, 10, seed=4, w=w)
        want = emulate(m, x)
        if what != "random":
            assert not cnn_features(m, x).any(), what
        e = Engine(m, device=0)
        _check(e, x, want, what)
        e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["binary160", "cnn_48"])
@pytest.mark.parametrize("n", [1, 127, 128, 129, 148 * 128 * 2 + 77])
def test_batch_sizes(lib, name, n):
    """one image, one tile, ragged tiles, several tiles per CTA; twice in a row.  The restatement covers the first and the last
    1 000 images (the ragged tail), the layered emulator all of them."""
    from bitnetmcu_b200.engine import Engine
    m = load_model(name)
    x = _images(n, seed=n)
    idx = np.unique(np.r_[0:min(n, 1000), max(0, n - 1000):n])
    want = emulate(m, x[idx])
    e = Engine(m, device=0)
    for _ in range(2):
        lo, la = _run(e, x)
        assert np.array_equal(lo[idx], want) and np.array_equal(la[idx], np.argmax(want, axis=1)), (name, n)
    lo2, la2 = _layered(e, x)
    assert np.array_equal(lo2, lo) and np.array_equal(la2, la), (name, n)
    e.close()


def _device_images(n, seed):
    import torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn((n, 256), generator=g, device="cuda")


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["2bitsym96", "cnn_16small"])
def test_one_past_the_chunk(lib, name):
    """2^20 + 1 images: two chunks, the second of one image.  fused == layered for all of them, == restatement for the images
    around the chunk boundary"""
    from bitnetmcu_b200.engine import Engine
    m = load_model(name)
    d_x = _device_images(CHUNK + 1, seed=2)
    e = Engine(m, device=0)
    lo, la = _run(e, d_x)
    lo2, la2 = _layered(e, d_x)
    assert np.array_equal(lo, lo2) and np.array_equal(la, la2)
    import torch
    idx = np.r_[0:200, CHUNK - 200:CHUNK + 1]
    want = emulate(m, d_x[torch.as_tensor(idx, device="cuda")].cpu().numpy())
    assert np.array_equal(lo[idx], want) and np.array_equal(la[idx], np.argmax(want, axis=1))
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("width", [64, 128, 192, 256])
def test_ring_rounds(lib, capfd, monkeypatch, width):
    """enough tiles per CTA that every ring stage of the int8 emulator row serves at least three rounds: fused == layered,
    == restatement on the last tiles (the ones that ran in the latest rounds)"""
    import torch
    from bitnetmcu_b200 import model as M, pack as P
    m = P.random_fc_model(M.ENC_8BIT, (256, width, width, 17), seed=width)
    e, route = _route(m, capfd, monkeypatch)
    assert route == f"k_quantize_images + fc_emul_i8_kernel<{width},1,emul>", route
    max_stages = 6   # fc_chain_plan_create: the int8 emulator form has at most 6 stages
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    n = sms * 128 * (3 * max_stages + 1) + 77
    d_x = _device_images(n, seed=width)
    lo, la = _run(e, d_x)
    lo2, la2 = _layered(e, d_x)
    assert np.array_equal(lo, lo2) and np.array_equal(la, la2), width
    idx = np.r_[0:300, n - 2 * sms * 128:n]
    want = emulate(m, d_x[torch.as_tensor(idx, device="cuda")].cpu().numpy())
    assert np.array_equal(lo[idx], want) and np.array_equal(la[idx], np.argmax(want, axis=1)), width
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["2bitsym96", "cnn"])
def test_labels_only_and_logits_only(lib, name):
    from bitnetmcu_b200.engine import Engine
    m = load_model(name)
    x = _images(5000, seed=8)
    e = Engine(m, device=0)
    full, lab = _run(e, x)
    lo, la = _run(e, x, want_logits=False)
    assert lo is None and np.array_equal(la, lab)
    lo, la = _run(e, x, want_labels=False)
    assert la is None and np.array_equal(lo, full)
    assert np.array_equal(full, emulate(m, x))
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["binary160", "cnn_48"])
def test_non_default_stream_and_host_entry(lib, name):
    """images made on a side stream and the call on that stream, ordered by it alone; the host entry
    (bnm_emulate_inference_quantized, which runs the same routes per chunk) gives the same logits"""
    import torch
    from bitnetmcu_b200.engine import Engine
    m = load_model(name)
    n = 148 * 128 * 3 + 5
    x = _images(n, seed=3)
    e = Engine(m, device=0)
    h_x = torch.from_numpy(x).pin_memory()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        d_x = torch.empty((n, 256), dtype=torch.float32, device="cuda")
        d_x.copy_(h_x, non_blocking=True)
        d_x.mul_(1.0)
        lo = torch.empty((n, m.n_classes), dtype=torch.float64, device="cuda")
        la = torch.empty(n, dtype=torch.int32, device="cuda")
        e.inference_quantized_device(d_x, lo, la)
    s.synchronize()
    got, got_la = lo.cpu().numpy(), la.cpu().numpy()
    idx = np.r_[0:1000, n - 1000:n]
    want = emulate(m, x[idx])
    assert np.array_equal(got[idx], want) and np.array_equal(got_la[idx], np.argmax(want, axis=1))
    assert np.array_equal(got, _run(e, x)[0]) and np.array_equal(got_la, _run(e, x)[1])
    assert np.array_equal(e.inference_quantized(x), got)
    e.close()
