"""Labels-only inference (GPU, H100): every batched entry takes a NULL logits buffer and then produces the labels alone.
The labels must equal the oracle's on every path, every CNN front-end and every instantiation of the fused FC kernel."""
import ctypes as C
import re

import numpy as np
import pytest

from conftest import load_model, model_names
from restate import scale_images
from support import CHAIN_ROWS, N_MANY, build_c_shim, engine, frontends, kernel_clone, kernel_copies_are_kernels, lib, plan_line, \
    verbose_engine

pytestmark = pytest.mark.gpu


def _images(n, img_bytes=256, seed=0):
    rng = np.random.default_rng(seed)
    imgs = rng.integers(-128, 128, size=(n, img_bytes)).astype(np.int8)
    imgs[: min(n, 64)] = np.clip(imgs[: min(n, 64)], -20, 127)   # MNIST-like rows: background ~ -20, strokes to 127
    return imgs


@pytest.mark.parametrize("path", ["layers", "tcgen05"])
@pytest.mark.parametrize("name", model_names())
def test_golden_models_labels_only(lib, oracle, name, path):
    """Every fixture model, both paths, every CNN front-end: a ragged batch (not a multiple of the 128-image tile)."""
    from bitnetmcu_b200 import _lib
    m = load_model(name)
    imgs = _images(5037, seed=len(name))
    _, want = oracle.infer(m, imgs)
    p = _lib.PATH_LAYERS if path == "layers" else _lib.PATH_TCGEN05
    for fe in frontends(m):
        e = engine(m, p, fe)
        assert e.active_path == p
        lo, la = e.infer(imgs, want_logits=False)
        assert lo is None and np.array_equal(la, want), (name, path, fe)
        e.close()


@pytest.mark.parametrize("n", [0, 1, 127, 128, 129, 1000])
def test_edge_batch_sizes_labels_only(lib, oracle, n):
    from bitnetmcu_b200 import _lib
    imgs = _images(n, seed=n)
    for name in ("fc", "cnn_48"):
        m = load_model(name)
        want = oracle.infer(m, imgs)[1] if n else np.empty(0, dtype=np.uint32)
        for path in (_lib.PATH_LAYERS, _lib.PATH_TCGEN05):
            for fe in frontends(m):
                e = engine(m, path, fe)
                lo, la = e.infer(imgs, want_logits=False)
                assert lo is None and la.shape == (n,) and np.array_equal(la, want), (name, path, fe)
                e.close()


@pytest.mark.parametrize("row", [r for r, _ in CHAIN_ROWS])
def test_every_chain_kernel_row_labels_only(lib, oracle, capfd, monkeypatch, row):
    from bitnetmcu_b200 import _lib
    m = dict(CHAIN_ROWS)[row]()
    e, err = verbose_engine(capfd, monkeypatch, lambda: engine(m, _lib.PATH_TCGEN05))
    plan = plan_line(err)
    assert plan and re.search(r"fc_chain_kernel(<[^>]*>)", plan).group(1) == row, err
    n = N_MANY
    imgs = _images(n, m.img_bytes, seed=len(row))
    _, want = oracle.infer(m, imgs)
    lo, la = e.infer(imgs, want_logits=False)
    assert lo is None and np.array_equal(la, want), row
    e.close()


def test_float_input_row_labels_only(lib, oracle, capfd, monkeypatch):
    """the fused float-input row (<64,1,float>) through bnm_infer_batch_device_f32 with NULL logits"""
    from bitnetmcu_b200 import _lib
    m = load_model("fc")
    e, err = verbose_engine(capfd, monkeypatch, lambda: engine(m, _lib.PATH_TCGEN05))
    assert any("float input <64,1,float>" in l for l in err)
    _float_case(e, m, oracle, N_MANY)
    e.close()


def _float_case(e, m, oracle, n):
    import torch
    rng = np.random.default_rng(n)
    x = rng.normal(size=(n, m.img_bytes)).astype(np.float32)
    _, want = oracle.infer(m, scale_images(x))
    d_x = torch.from_numpy(x).cuda()
    d_lab = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    for _ in range(2):                      # twice: the launch is repeatable (each one starts its ring at stage 0, phase 0)
        e.infer_device_f32(d_x, None, d_lab)
    torch.cuda.synchronize()
    assert np.array_equal(d_lab.cpu().numpy().astype(np.uint32), want)


@pytest.mark.parametrize("name", ["fc", "binary160"])
def test_float_input_labels_only(lib, oracle, name):
    """fc: the fused float kernel; binary160 (192 columns): the scaling kernel into scratch, then the int8 entry"""
    m = load_model(name)
    e = engine(m)
    _float_case(e, m, oracle, 3001)
    e.close()


@pytest.mark.parametrize("name", ["fc", "cnn_48"])
def test_device_labels_only_on_torch_stream(lib, oracle, name):
    import torch
    m = load_model(name)
    imgs = _images(3000, seed=4)
    _, want = oracle.infer(m, imgs)
    e = engine(m)
    d_img = torch.from_numpy(imgs).cuda()
    d_lab = torch.full((3000,), -1, dtype=torch.int32, device="cuda")
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        e.infer_device(d_img, None, d_lab)
    s.synchronize()
    assert np.array_equal(d_lab.cpu().numpy().astype(np.uint32), want)
    e.close()


@pytest.mark.parametrize("name", ["fc", "cnn"])
def test_host_pipeline_labels_only(lib, oracle, name):
    """bnm_infer_batch with NULL logits: the chunked three-stream pipeline at several chunk sizes and the small-batch path"""
    from bitnetmcu_b200 import _lib
    m = load_model(name)
    imgs = _images(10000, seed=3)
    _, want = oracle.infer(m, imgs)
    for chunk in (128, 1024, 4096):
        e = engine(m)
        e.set_option(_lib.OPT_CHUNK_IMAGES, chunk)
        lo, la = e.infer(imgs, want_logits=False)
        assert lo is None and np.array_equal(la, want), chunk
        e.close()
    e = engine(m)
    for n in (1, 777, 1024):               # n <= 1024: staged through the small-batch buffers
        lo, la = e.infer(imgs[:n], want_logits=False)
        assert lo is None and np.array_equal(la, want[:n]), n
    lo, la = e.infer(imgs[:777])           # and a call with logits after labels-only ones
    assert np.array_equal(la, want[:777]) and np.array_equal(lo, oracle.infer(m, imgs[:777])[0])
    e.close()


@pytest.mark.parametrize("mode", [1, 2])
def test_launch_overlap_labels_only(lib, oracle, kernel_copies_are_kernels, mode):
    """BNM_OPT_LAUNCH_OVERLAP with NULL logits: back-to-back launches on one stream, images and labels double-buffered, stay
    bit-exact.  Then one labels buffer reused by every launch (resident images, a consumer kernel -- kernel_clone, not a
    memcpy -- reading it right after each): the library must see the reuse and keep the launches ordered, whatever the
    absent logits."""
    import torch
    from bitnetmcu_b200 import _lib
    m = load_model("fc")
    n = 148 * 128 * 7 + 77                  # fills the GPU: launches trigger early
    batches = [_images(n, seed=60 + k) for k in range(4)]
    want = [oracle.infer(m, b)[1] for b in batches]
    e = engine(m)
    e.set_option(_lib.OPT_LAUNCH_OVERLAP, mode)
    src = [torch.from_numpy(b).cuda() for b in batches]     # resident inputs: consecutive launches never share a buffer
    d_lab = [torch.full((n,), -1, dtype=torch.int32, device="cuda") for _ in range(2)]
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        for rep in range(6):
            for k in range(4):
                e.infer_device(src[k], None, d_lab[k & 1])
        s.synchronize()
        # the last two launches wrote batches 2 and 3 into label buffers 0 and 1
        got = [d_lab[0].cpu().numpy(), d_lab[1].cpu().numpy()]
        assert np.array_equal(got[0].astype(np.uint32), want[2]) and np.array_equal(got[1].astype(np.uint32), want[3])
        one = torch.full((n,), -1, dtype=torch.int32, device="cuda")
        seen = []
        for rep in range(3):
            for k in range(4):
                e.infer_device(src[k], None, one)
                seen.append(kernel_clone(one))
        s.synchronize()
    for i, t in enumerate(seen):
        assert np.array_equal(t.cpu().numpy().astype(np.uint32), want[i % 4]), i
    e.close()


def test_gather_labels_only(lib, oracle):
    """single-GPU result exchange with NULL logits: local labels plus a labels destination, then the destination alone"""
    import torch
    from bitnetmcu_b200 import _lib
    m = load_model("fc")
    n, rows, off = N_MANY, N_MANY + 640, 512
    imgs = _images(n, seed=77)
    _, want = oracle.infer(m, imgs)
    e = engine(m, _lib.PATH_TCGEN05)
    d_img = torch.from_numpy(imgs).cuda()
    d_lab = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    dst = [torch.full((rows,), -7, dtype=torch.int32, device="cuda") for _ in range(2)]
    s = torch.cuda.current_stream()
    for k, local in enumerate((d_lab, None)):
        g = _lib.BnmGather()
        g.n_labels_dst, g.n_logits_dst, g.row_offset = 1, 0, off
        g.labels_dst[0] = dst[k].data_ptr()
        lab_ptr = C.c_void_p(local.data_ptr()) if local is not None else None
        _lib.check(lib.bnm_infer_batch_device_gather(e.handle, C.c_void_p(d_img.data_ptr()), n, None, lab_ptr, C.byref(g),
                                                     C.c_void_p(s.cuda_stream)), "gather")
    s.synchronize()
    assert np.array_equal(d_lab.cpu().numpy().astype(np.uint32), want)
    for k in range(2):
        h = dst[k].cpu().numpy()
        assert np.array_equal(h[off:off + n].astype(np.uint32), want) and (h[:off] == -7).all() and (h[off + n:] == -7).all(), k
    e.close()


def test_no_output_is_an_error(lib):
    """every entry needs at least one output; the emulation entry keeps its logits mandatory"""
    import torch
    from bitnetmcu_b200 import _lib
    e = engine(load_model("fc"))
    imgs = _images(300)
    d_img = torch.from_numpy(imgs).cuda()
    d_x = torch.zeros((300, 256), dtype=torch.float32, device="cuda")
    h = e.handle
    assert lib.bnm_infer_batch(h, C.c_void_p(imgs.ctypes.data), 300, None, None) == -1
    assert b"no output" in lib.bnm_last_error()
    assert lib.bnm_infer_batch_device(h, C.c_void_p(d_img.data_ptr()), 300, None, None, None) == -1
    assert lib.bnm_infer_batch_device_f32(h, C.c_void_p(d_x.data_ptr()), 300, None, None, None) == -1
    g = _lib.BnmGather()                    # a gather with no destinations is no output either
    assert lib.bnm_infer_batch_device_gather(h, C.c_void_p(d_img.data_ptr()), 300, None, None, C.byref(g), None) == -1
    x = np.zeros((300, 256), dtype=np.float32)
    assert lib.bnm_emulate_inference_quantized(h, C.c_void_p(x.ctypes.data), 300, None) == -1
    with pytest.raises(ValueError):
        e.infer(imgs, want_labels=False, want_logits=False)
    torch.cuda.synchronize()
    e.close()


@pytest.mark.parametrize("name", ["fc", "cnn"])
def test_c_shim_inference_batch_labels_only(built, oracle, tmp_path, name):
    """InferenceBatch(images, n, NULL, labels) through the gcc-built plain-C shim"""
    dll, _, d = build_c_shim(str(tmp_path), name)
    lib = C.CDLL(dll)
    lib.InferenceBatch.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
    lib.InferenceBatch.restype = C.c_int
    imgs = np.ascontiguousarray(np.concatenate([d["images"], _images(2000, seed=5)]))
    _, want = oracle.infer(load_model(name), imgs)
    labels = np.full(len(imgs), 255, dtype=np.uint32)
    assert lib.InferenceBatch(imgs.ctypes.data, len(imgs), None, labels.ctypes.data) == 0
    assert np.array_equal(labels, want) and np.array_equal(labels[:10], d["labels"])
    assert lib.InferenceBatch(imgs.ctypes.data, 1, None, None) != 0
