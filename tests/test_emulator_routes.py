"""The emulator's fused routes beyond the float-input row (bnm_emulate_batch_device, run_route in capi.cu):

* FC models wider than 64 or with more than 16 classes: k_quantize_images, then fc_emul_i8_kernel<max_n> (int8 TMA input, one
  pipe, one slot, the last layer at full width, the emulator's hidden-layer rule and float64 logits);
* CNN models up to 128 channels (beyond that: layer by layer): k_cnn_emul_frontend (input scaling, three convolutions with the per-image renormalisation, two
  pools; BitNetMCU.py:435-445, 459-526), then fc_emul_i8_kernel on its features.

CPU tests: a NumPy restatement of the emulator's CNN path against the reference emulator's own logits (the expectation of the
GPU tests), and the new kernels' SASS.  GPU tests (tolerance 0): fused == layered (BNM_PATH_LAYERS) == restatement."""
import os
import re

import numpy as np
import pytest

from conftest import GOLDEN, load_model
from restate import cnn_features, emulate
from support import N_MANY, cnn_model, crafted_cnn_case, engine, instructions, lib, local_memory, normal_images, route, \
    run_emulator, run_emulator_layered, sass_functions, verbose_engine

CHUNK = 1 << 20                     # images per front-end / FC launch pair of the new routes


def test_cnn_restatement_reproduces_reference_emulator():
    """tests/golden/emulator.npz holds the reference emulator's own logits"""
    g = np.load(os.path.join(GOLDEN, "emulator.npz"))
    for name in ("cnn", "cnn_48", "cnn_16small"):
        got = emulate(load_model(name), g["images"])
        assert got.dtype == np.float64 and np.array_equal(got, g[name]), (name, np.argwhere(got != g[name])[:5])


def test_new_kernels_sass(built):
    """four int8 emulator rows (IGMMA, no local memory) next to exactly one fc_emul_kernel and eight fc_chain_kernel
    instantiations, and a front-end kernel without local memory"""
    kernels = sass_functions()
    rows = sorted(k for k in kernels if k.startswith("_ZN3bnm17fc_emul_i8_kernel"))
    assert [re.search(r"ILi(\d+)E", k).group(1) for k in rows] == ["128", "192", "256", "64"], rows
    assert len([k for k in kernels if k.startswith("_ZN3bnm14fc_emul_kernel")]) == 1
    assert len([k for k in kernels if k.startswith("_ZN3bnm15fc_chain_kernel")]) == 8
    front = [k for k in kernels if k.startswith("_ZN3bnm19k_cnn_emul_frontend")]
    assert len(front) == 1
    for k in rows + front:
        ins = instructions(kernels[k])
        assert len(ins) > 100, k
        assert not local_memory(ins), f"local memory in {k}"
        assert (k in front) != any(i.startswith("IGMMA") for i in ins), k


# ---- GPU ------------------------------------------------------------------------------------------------------------------

def _check(e, x, want, tag):
    """default path == restatement (logits and np.argmax labels), and == the layered emulator"""
    lo, la = run_emulator(e, x)
    assert np.array_equal(lo, want), (tag, np.argwhere(lo != want)[:5])
    assert np.array_equal(la, np.argmax(want, axis=1)), tag
    lo2, la2 = run_emulator_layered(e, x)
    assert np.array_equal(lo2, lo) and np.array_equal(la2, la), tag


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
    e, err = verbose_engine(capfd, monkeypatch, lambda: engine(load_model(name)))
    assert route(err, "emulator") == GOLDEN_ROUTES[name], (name, err)
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
    x = normal_images(3001, seed=idx, elems=m.img_bytes)
    e, err = verbose_engine(capfd, monkeypatch, lambda: engine(m))
    assert route(err, "emulator") == (f"k_quantize_images + fc_emul_i8_kernel<{row},1,emul>" if row else "layer by layer"), (tag, err)
    _check(e, x, emulate(m, x), tag)
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("channels", [16, 24, 48, 64, 128, 144, 256])
@pytest.mark.parametrize("n_classes", [10, 37])
def test_random_cnn_models(lib, capfd, monkeypatch, channels, n_classes):
    """up to 128 channels k_cnn_emul_frontend, beyond that the layer-by-layer route"""
    m = cnn_model(channels, n_classes, seed=channels + n_classes)
    x = normal_images(1500, seed=channels)
    e, err = verbose_engine(capfd, monkeypatch, lambda: engine(m))
    if channels <= 128:
        assert route(err, "emulator").startswith("k_cnn_emul_frontend + fc_emul_i8_kernel<64,"), err
    else:
        assert route(err, "emulator") == "layer by layer", err
    _check(e, x, emulate(m, x), (channels, n_classes))
    e.close()


@pytest.mark.gpu
def test_crafted_inputs(lib):
    """all-zero images; conv2 or conv3 outputs <= 0 everywhere (non-positive taps on non-negative inputs): a renormalisation
    whose maximum is 0 gives zeros, where NumPy would give nan"""
    x, models = crafted_cnn_case()
    for m, what in models:
        want = emulate(m, x)
        if what != "random":
            assert not cnn_features(m, x).any(), what
        e = engine(m)
        _check(e, x, want, what)
        e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["binary160", "cnn_48"])
@pytest.mark.parametrize("n", [1, 127, 128, 129, N_MANY])
def test_batch_sizes(lib, name, n):
    """one image, one tile, ragged tiles, several tiles per CTA; twice in a row.  The restatement covers the first and the last
    1 000 images (the ragged tail), the layered emulator all of them."""
    m = load_model(name)
    x = normal_images(n, seed=n)
    idx = np.unique(np.r_[0:min(n, 1000), max(0, n - 1000):n])
    want = emulate(m, x[idx])
    e = engine(m)
    for _ in range(2):
        lo, la = run_emulator(e, x)
        assert np.array_equal(lo[idx], want) and np.array_equal(la[idx], np.argmax(want, axis=1)), (name, n)
    lo2, la2 = run_emulator_layered(e, x)
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
    m = load_model(name)
    d_x = _device_images(CHUNK + 1, seed=2)
    e = engine(m)
    lo, la = run_emulator(e, d_x)
    lo2, la2 = run_emulator_layered(e, d_x)
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
    e, err = verbose_engine(capfd, monkeypatch, lambda: engine(m))
    assert route(err, "emulator") == f"k_quantize_images + fc_emul_i8_kernel<{width},1,emul>", err
    max_stages = 6   # fc_chain_plan_create: the int8 emulator form has at most 6 stages
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    n = sms * 128 * (3 * max_stages + 1) + 77
    d_x = _device_images(n, seed=width)
    lo, la = run_emulator(e, d_x)
    lo2, la2 = run_emulator_layered(e, d_x)
    assert np.array_equal(lo, lo2) and np.array_equal(la, la2), width
    idx = np.r_[0:300, n - 2 * sms * 128:n]
    want = emulate(m, d_x[torch.as_tensor(idx, device="cuda")].cpu().numpy())
    assert np.array_equal(lo[idx], want) and np.array_equal(la[idx], np.argmax(want, axis=1)), width
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["2bitsym96", "cnn"])
def test_labels_only_and_logits_only(lib, name):
    m = load_model(name)
    x = normal_images(5000, seed=8)
    e = engine(m)
    full, lab = run_emulator(e, x)
    lo, la = run_emulator(e, x, want_logits=False)
    assert lo is None and np.array_equal(la, lab)
    lo, la = run_emulator(e, x, want_labels=False)
    assert la is None and np.array_equal(lo, full)
    assert np.array_equal(full, emulate(m, x))
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["binary160", "cnn_48"])
def test_non_default_stream_and_host_entry(lib, name):
    """images made on a side stream and the call on that stream, ordered by it alone; the host entry
    (bnm_emulate_inference_quantized, which runs the same routes per chunk) gives the same logits"""
    import torch
    m = load_model(name)
    n = 148 * 128 * 3 + 5
    x = normal_images(n, seed=3)
    e = engine(m)
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
    assert np.array_equal(got, run_emulator(e, x)[0]) and np.array_equal(got_la, run_emulator(e, x)[1])
    assert np.array_equal(e.inference_quantized(x), got)
    e.close()
