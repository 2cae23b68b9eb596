"""float16 and bfloat16 images on the float device entries (include/bitnetmcu_b200.h section 11).

Every 16-bit entry is defined as its float32 sibling on the images widened to float32, so every GPU case here runs both on the
same images and compares every output with tolerance 0: logits, labels, top-k classes and scores, counts, and the int8 rows of
bnm_quantize_images_device_f16.  The cases cover the one-kernel FC forms (fc_chain_h16_kernel and its emulator and two-engine
siblings), the 16-bit scaling kernel ahead of every other route, both formats, the sizes around a tile and past the first trip
round the tile ring, and the values at the edges of the scaling (subnormals, the 1e-5 floor, ties, infinities, NaN)."""
import ctypes as C

import numpy as np
import pytest

from conftest import load_model
from restate import TILE, scale_images
from support import instructions, lib, local_memory, random_fc, sass_functions, verbose_engine  # noqa: F401 (lib: fixture)

FORMATS = ["float16", "bfloat16"]
BNM_E_ARG, BNM_E_NODEV = -1, -2


def _model(name):
    from bitnetmcu_b200 import model as M
    made = {
        "fc37": lambda: random_fc(4, (256, 64, 64, 37), 2),           # 37 classes: no float-input form
        "rows160": lambda: random_fc(4, (160, 64, 64, 10), 4),        # rows narrower than 256 elements, one-kernel forms
        "rows64": lambda: random_fc(4, (64, 64, 10), 5),
        "rows32": lambda: random_fc(4, (32, 64, 10), 6),
        "ternary-130": lambda: random_fc(M.ENC_TERNARY, (130, 64, 10), 7),   # 130-element rows: no fused plan, layer by layer
    }
    return made[name]() if name in made else load_model(name)


# model -> the kernel that reads its 16-bit rows in bnm_infer_batch_device_f16 on the default path
MODELS = {
    "fc": "fc_chain_h16_kernel", "ternary64": "fc_chain_h16_kernel", "rows160": "fc_chain_h16_kernel",
    "rows64": "fc_chain_h16_kernel", "rows32": "fc_chain_h16_kernel",
    "fc37": "k_quantize_images", "2bitsym96": "k_quantize_images", "binary160": "k_quantize_images",
    "ternary-130": "k_quantize_images", "12k_FP130": "fc_chain_h16_kernel", "cnn_16small": "k_quantize_images", "cnn_48": "k_quantize_images",
}


# ---- CPU ----------------------------------------------------------------------------------------------------------------------

def widen(bits, fmt):
    """the kernels' exact widening of 16-bit patterns (uint16) to float32, restated with integer arithmetic: bfloat16 is the top
    half of a float32; float16 moves its exponent and mantissa into float32's, normalising subnormals"""
    b = np.asarray(bits, dtype=np.uint32)
    if fmt == "bfloat16":
        return (b << 16).view(np.float32)
    sign, exp, man = (b >> 15) << 31, (b >> 10) & 0x1F, b & 0x3FF
    out = np.where(exp == 0x1F, (0xFF << 23) | (man << 13), ((exp + 112) << 23) | (man << 13))   # inf / NaN, normal
    sub = man.astype(np.float64) * 2.0 ** -24                                                   # subnormal and zero: exact
    out = np.where(exp == 0, sub.astype(np.float32).view(np.uint32), out)
    return (out | sign).astype(np.uint32).view(np.float32)


def test_widening_restatement_matches_numpy():
    """all 65 536 patterns of each format: float16 as NumPy widens np.float16 to float32, bfloat16 as the top 16 bits of the
    float32 it was cut from (NaN: any NaN)"""
    bits = np.arange(1 << 16, dtype=np.uint32).astype(np.uint16)
    want = bits.view(np.float16).astype(np.float32)
    got = widen(bits, "float16")
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan) and np.array_equal(got[~nan].view(np.uint32), want[~nan].view(np.uint32))
    f = np.random.default_rng(0).uniform(-3e38, 3e38, 4096).astype(np.float32)
    top = (f.view(np.uint32) >> 16).astype(np.uint16)
    assert np.array_equal(widen(top, "bfloat16").view(np.uint32), f.view(np.uint32) & 0xFFFF0000)


@pytest.mark.parametrize("fmt", FORMATS)
def test_scaling_restatement_on_widened_rows(fmt):
    """the 16-bit scaling restated (widen, then restate.scale_images) on the edge rows equals the float32 scaling of the
    images a torch caller passes today, ``images.float()`` (all-zero rows, subnormals, the 1e-5 floor, 65504, ties, infinities,
    NaN: the rows holding either scale to zeros)"""
    import torch
    rows = _edge_rows(256, fmt)
    bits = _bits(rows, fmt)
    x = widen(bits, fmt)
    caller = torch.from_numpy(rows).to(getattr(torch, fmt)).float().numpy()
    with np.errstate(invalid="ignore", over="ignore"):
        q = scale_images(x)
        assert np.array_equal(q, scale_images(caller))
        if fmt == "float16":
            assert np.array_equal(q, scale_images(bits.view(np.float16).astype(np.float32)))
    assert not q[0].any()                                   # an all-zero row scales to zeros
    assert not q[5:9].any()                                 # so does every row holding an infinity or a NaN
    assert q[[1, 2, 3, 9, 11]].any(axis=1).all()            # the finite rows around them do not
    assert np.array_equal(q[4], np.round(rows[4]).clip(-128, 127).astype(np.int8))   # scale 1: ties to even


def test_entries_fail_without_device(built):
    from bitnetmcu_b200 import _lib
    l = _lib.load()
    if l.bnm_device_count() > 0:
        pytest.skip("a CUDA device is present")
    x = np.zeros((4, 256), dtype=np.uint16)
    o = np.zeros(64, dtype=np.int64)
    p, q = C.c_void_p(x.ctypes.data), C.c_void_p(o.ctypes.data)
    assert l.bnm_quantize_images_device_f16(p, 1, 4, 256, q, None) == BNM_E_NODEV
    assert b"no CUDA device" in l.bnm_last_error()
    for rc in (l.bnm_infer_batch_device_f16(None, p, 1, 4, q, q, None), l.bnm_emulate_batch_device_f16(None, p, 1, 4, q, q, None),
               l.bnm_compare_engines_device_f16(None, p, 1, 4, None, q, q, q, None),
               l.bnm_infer_topk_device_f16(None, p, 1, 4, 1, q, q, None), l.bnm_emulate_topk_device_f16(None, p, 2, 4, 1, q, q, None)):
        assert rc != 0
    from bitnetmcu_b200.engine import Engine
    with pytest.raises(_lib.BnmError):
        Engine(load_model("fc"))


def test_new_kernels_have_no_local_memory(built):
    """the three 16-bit float-input kernels and both 16-bit scaling kernels exist once each and keep everything in registers"""
    kernels = sass_functions()
    for key in ("_ZN3bnm19fc_chain_h16_kernel", "_ZN3bnm18fc_emul_h16_kernel", "_ZN3bnm21fc_engines_h16_kernel",
                "_ZN3bnm17k_quantize_imagesILNS_10HalfFormatE1E", "_ZN3bnm17k_quantize_imagesILNS_10HalfFormatE2E"):
        funcs = [k for k in kernels if k.startswith(key)]
        assert len(funcs) == 1, (key, funcs)
        assert not local_memory(instructions(kernels[funcs[0]])), funcs[0]


# ---- images -------------------------------------------------------------------------------------------------------------------

def _edge_rows(d, fmt):
    """float32 rows [12, d] at the edges of the 16-bit scaling; every value representable (or saturating) in fmt"""
    rng = np.random.default_rng(11)
    r = np.zeros((12, d), dtype=np.float32)
    r[1] = rng.uniform(-6e-5, 6e-5, d)                        # float16 subnormals (and bfloat16's small normals)
    r[2, ::3], r[2, 1::3], r[2, 2::3] = 65504.0, -0.0, 0.0    # float16's largest value and both zeros
    r[3] = rng.uniform(-1e-5, 1e-5, d)                         # maximum near the 1e-5 floor, a float16 subnormal
    r[4] = rng.integers(-127, 127, d) + 0.5                    # max 127: scale 1, every product an exact .5 tie
    r[4, 0] = 127.0
    r[5] = rng.standard_normal(d)
    r[5, 7] = np.inf
    r[6] = rng.standard_normal(d)
    r[6, 3] = -np.inf
    r[7] = rng.standard_normal(d)
    r[7, 5] = np.nan
    r[8, 0], r[8, 1], r[8, 2:] = np.nan, np.inf, 1.0
    if fmt == "bfloat16":
        r[9] = rng.uniform(-3e38, 3e38, d)                     # near bfloat16's (and float32's) largest finite values
        r[10] = rng.uniform(-1e-38, 1e-38, d)                  # below 1e-38: float32 subnormals
    else:
        r[9] = rng.uniform(-65504, 65504, d)
        r[10] = rng.uniform(-1e-7, 1e-7, d)                    # the smallest float16 subnormals and zero
    r[11] = rng.standard_normal(d) * 1e3
    return r


def _bits(rows, fmt):
    """float32 rows -> the uint16 patterns of their fmt values (torch's round to nearest even)"""
    import torch
    t = torch.from_numpy(np.ascontiguousarray(rows)).to(getattr(torch, fmt))
    return t.view(torch.int16).numpy().view(np.uint16)


def images(n, d, fmt, seed):
    """n rows of fmt images on the device: the edge rows, then rows of random scale, repeating"""
    import torch
    rng = np.random.default_rng(seed)
    base = np.concatenate([_edge_rows(d, fmt), (rng.standard_normal((501, d)) * 10.0 ** rng.uniform(-4, 4, (501, 1))).astype(np.float32)])
    x = torch.from_numpy(base).to(getattr(torch, fmt)).cuda()
    return x[torch.arange(n, device="cuda") % x.shape[0]].contiguous()


# ---- GPU: every entry against its float32 sibling ------------------------------------------------------------------------------

def _eq(a, b, what):
    assert a.shape == b.shape and bool((a == b).all()), (what, int((a != b).sum()))


def _entries(e, x, tag):
    """every 16-bit entry of engine e on images x against its float32 sibling on x.float(), each output combination"""
    import torch
    from bitnetmcu_b200 import engine as E
    n, Cn, xf = x.shape[0], e.n_classes, x.float()
    dev = dict(device="cuda")

    def pair(fn, specs):
        got, want = [[None if s is None else torch.full(s[0], s[2], dtype=s[1], **dev) for s in specs] for _ in range(2)]
        fn(x, *got)
        fn(xf, *want)
        for g, w, k in zip(got, want, range(len(specs))):
            if g is not None:
                _eq(g, w, (tag, fn.__name__, k))
        return got

    lo, la = ((n, Cn), torch.int32, -7), ((n,), torch.int32, -7)
    flo = ((n, Cn), torch.float64, -7.0)
    for outs in ((lo, la), (None, la), (lo, None)):
        pair(e.infer_device_f32, outs)
    for outs in ((flo, la), (None, la), (flo, None)):
        pair(e.inference_quantized_device, outs)
    truth = torch.from_numpy(np.arange(n, dtype=np.int32) % Cn).cuda()
    for t in (truth, None):
        counts = [torch.zeros(4, dtype=torch.int64, **dev) for _ in range(2)]
        labs = [[torch.full((n,), -7, dtype=torch.int32, **dev) for _ in range(2)] for _ in range(2)]
        for _ in range(2):   # counts add up over two calls
            e.compare_engines_device(x, t, labs[0][0], labs[0][1], counts[0])
            e.compare_engines_device(xf, t, labs[1][0], labs[1][1], counts[1])
        _eq(counts[0], counts[1], (tag, "counts", t is None))
        _eq(labs[0][0], labs[1][0], (tag, "labels_c"))
        _eq(labs[0][1], labs[1][1], (tag, "labels_py"))
        assert int(counts[0][0]) == 2 * n
    kmax = min(Cn, 16)
    for k in sorted({1, min(5, kmax), kmax}):
        for scores in (True, False):
            pair(lambda im, c, s: e.topk_device_f32(im, k, c, s), [((n, k), torch.int32, -7), ((n, k), torch.int32, -7) if scores else None])
            pair(lambda im, c, s: e.emulate_topk_device(im, k, c, s), [((n, k), torch.int32, -7), ((n, k), torch.float64, -7.0) if scores else None])
    q = [torch.full(x.shape, 99, dtype=torch.int8, **dev) for _ in range(2)]
    E.quantize_images_device(x, q[0])
    E.quantize_images_device(xf, q[1])
    torch.cuda.synchronize()
    _eq(q[0], q[1], (tag, "quantize"))


def _ring_n():
    """past the first trip round every float-input form's ring: five tiles per CTA plus a ragged tile"""
    import torch
    return 5 * torch.cuda.get_device_properties(0).multi_processor_count * TILE + 77


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("name", list(MODELS))
def test_entries_equal_float32_sibling(lib, fmt, name):
    from bitnetmcu_b200.engine import Engine
    m = _model(name)
    e = Engine(m, device=0)
    for n in (0, 1, 127, 128, 129, 1000, _ring_n()):
        _entries(e, images(n, m.img_bytes, fmt, n), (name, fmt, n))
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("name", ["fc", "binary160", "cnn_48"])
def test_layer_path_forced(lib, fmt, name):
    from bitnetmcu_b200 import _lib
    from bitnetmcu_b200.engine import Engine
    m = _model(name)
    e = Engine(m, device=0, path=_lib.PATH_LAYERS)
    for n in (1, 129, 3000):
        _entries(e, images(n, m.img_bytes, fmt, n), (name, "layers", fmt, n))
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", FORMATS)
def test_cnn_front_ends(lib, fmt):
    """CNN-16small and CNN-48 on both C-engine front-ends; the emulator's runs k_cnn_emul_frontend_i8 on the scaled rows"""
    import torch
    from bitnetmcu_b200 import _lib
    from support import engine, frontends
    for name in ("cnn_16small", "cnn_48"):
        m = _model(name)
        for fe in frontends(m):
            e = engine(m, cnn_frontend=fe)
            x = images(5000, 256, fmt, 3)
            got = [torch.empty(5000, dtype=torch.int32, device="cuda") for _ in range(2)]
            e.infer_device_f32(x, None, got[0])
            e.infer_device_f32(x.float(), None, got[1])
            _eq(got[0], got[1], (name, fe, fmt))
            e.close()
    assert _lib.CNN_TENSOR_CORES in frontends(_model("cnn_48"))


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", FORMATS)
def test_scaling_route_past_a_pass(lib, fmt):
    """Binary-160 (scaling kernel, then the int8 form) on 2^20 + 77 images: the second pass of the scaling route starts at row 2^20"""
    import torch
    from bitnetmcu_b200.engine import Engine
    m = _model("binary160")
    e = Engine(m, device=0)
    n = (1 << 20) + 77
    x = images(n, 256, fmt, 9)
    got = [torch.empty((n, 10), dtype=torch.int32, device="cuda") for _ in range(2)]
    lab = [torch.empty(n, dtype=torch.int32, device="cuda") for _ in range(2)]
    e.infer_device_f32(x, got[0], lab[0])
    e.infer_device_f32(x.float(), got[1], lab[1])
    _eq(got[0], got[1], "logits")
    _eq(lab[0], lab[1], "labels")
    py = [torch.empty(n, dtype=torch.int32, device="cuda") for _ in range(2)]
    e.inference_quantized_device(x, None, py[0])
    e.inference_quantized_device(x.float(), None, py[1])
    _eq(py[0], py[1], "emulator labels")
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["fc", "binary160", "cnn_48"])
def test_kernels_of_each_route(lib, name):
    """the kernels a 16-bit call runs: the 16-bit float-input forms on a one-kernel model, the 16-bit scaling kernel elsewhere,
    and no float32 kernel of the sibling.  torch.profiler records in a process of its own, in that process's only profiler
    session: a later session in the same process can miss activities (tests/support.py, _kernel_copy_profile)."""
    import json
    import os
    import subprocess
    import sys
    from conftest import ROOT
    script = f"""
import json, sys
sys.path[:0] = [{ROOT!r}, {os.path.join(ROOT, "tests")!r}]
import torch
from torch.profiler import ProfilerActivity, profile
from bitnetmcu_b200.engine import Engine
from test_half_input import _model, images
e = Engine(_model({name!r}), device=0)
x = images(4096, 256, "bfloat16", 1)
la = torch.empty(4096, dtype=torch.int32, device="cuda")
calls = [lambda: e.infer_device_f32(x, None, la), lambda: e.inference_quantized_device(x, None, la),
         lambda: e.compare_engines_device(x, None, la)]
for call in calls:
    call()
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
    for call in calls:
        call()
    torch.cuda.synchronize()
print(json.dumps([ev.name for ev in prof.events() if ev.device_type == torch.autograd.DeviceType.CUDA]))
e.close()
"""
    run = subprocess.run([sys.executable, "-c", script], capture_output=True, text=True, cwd=ROOT, timeout=300)
    assert run.returncode == 0, run.stderr[-3000:]
    names = json.loads(run.stdout.strip().splitlines()[-1])
    want = ["fc_chain_h16_kernel", "fc_emul_h16_kernel", "fc_engines_h16_kernel"] if name == "fc" else ["HalfFormat)2>"]
    for kernel in want:
        assert any(kernel in k for k in names), (name, kernel, names)
    float32 = ("fc_chain_kernel<64, 1, true", "fc_emul_kernel(", "fc_engines_kernel(", "k_quantize_images(float", "k_cnn_emul_frontend(")
    assert not any(f in k for f in float32 for k in names), names


@pytest.mark.gpu
def test_topk_route_lines(lib, capfd, monkeypatch):
    """BNM_VERBOSE names the 16-bit scaling kernel in the top-k route lines"""
    import torch
    from bitnetmcu_b200.engine import Engine
    e, _ = verbose_engine(capfd, monkeypatch, lambda: Engine(_model("fc"), device=0))
    c = torch.empty((256, 5), dtype=torch.int32, device="cuda")
    e.topk_device_f32(images(256, 256, "float16", 0), 5, c)
    e.emulate_topk_device(images(256, 256, "bfloat16", 0), 5, c)
    torch.cuda.synchronize()
    err = capfd.readouterr().err
    assert "topk route: bnm_infer_topk_device_f16: k_quantize_images<float16> + fc_topk_kernel<64,1,topk>" in err, err
    assert "topk route: bnm_emulate_topk_device_f16: k_quantize_images<bfloat16> + fc_topk_kernel<64,1,emul,topk>" in err, err
    e.close()


@pytest.mark.gpu
def test_bad_arguments(lib):
    """a misaligned image pointer and a format other than 1 or 2 return BNM_E_ARG on every entry"""
    import torch
    from bitnetmcu_b200.engine import Engine
    e = Engine(_model("fc"), device=0)
    x = images(130, 256, "float16", 0)
    bufs = [torch.empty(130 * 16, dtype=torch.float64, device="cuda") for _ in range(3)]
    o, o2, o3 = (C.c_void_p(b.data_ptr()) for b in bufs)
    h = e.handle
    good, odd = C.c_void_p(x.data_ptr()), C.c_void_p(x.data_ptr() + 2)
    calls = {
        "infer": lambda p, f: lib.bnm_infer_batch_device_f16(h, p, f, 128, o, o2, None),
        "emulate": lambda p, f: lib.bnm_emulate_batch_device_f16(h, p, f, 128, o, o2, None),
        "compare": lambda p, f: lib.bnm_compare_engines_device_f16(h, p, f, 128, None, o, o2, o3, None),
        "topk": lambda p, f: lib.bnm_infer_topk_device_f16(h, p, f, 128, 5, o, o2, None),
        "emulate_topk": lambda p, f: lib.bnm_emulate_topk_device_f16(h, p, f, 128, 5, o, o2, None),
    }
    for what, call in calls.items():
        assert call(good, 1) == 0 and call(good, 2) == 0, what
        assert call(odd, 1) == BNM_E_ARG and b"aligned" in lib.bnm_last_error(), what
        for f in (0, 3, -1):
            assert call(good, f) == BNM_E_ARG and b"format" in lib.bnm_last_error(), (what, f)
    assert lib.bnm_quantize_images_device_f16(good, 3, 128, 256, o, None) == BNM_E_ARG
    assert lib.bnm_quantize_images_device_f16(good, 0, 0, 256, o, None) == BNM_E_ARG   # whatever n
    assert lib.bnm_infer_topk_device_f16(h, good, 1, 128, 11, o, o, None) == BNM_E_ARG   # k past n_classes
    torch.cuda.synchronize()
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("name", ["fc", "binary160"])
def test_graph_replay_equals_eager(lib, fmt, name):
    """each 16-bit entry captured with torch.cuda.graph: a replay on new images equals the eager call on them"""
    import torch
    from bitnetmcu_b200 import engine as E
    from bitnetmcu_b200.engine import Engine
    m = _model(name)
    e = Engine(m, device=0)
    n, Cn = 3000, m.n_classes
    x = images(n, 256, fmt, 1)
    z = lambda s, d: torch.zeros(s, dtype=d, device="cuda")
    lo, la, flo, cl, sc, fsc, q, cnt = (z((n, Cn), torch.int32), z(n, torch.int32), z((n, Cn), torch.float64), z((n, 5), torch.int32),
                                        z((n, 5), torch.int32), z((n, 5), torch.float64), z((n, 256), torch.int8), z(4, torch.int64))
    calls = [lambda: e.infer_device_f32(x, lo, la), lambda: e.inference_quantized_device(x, flo, la),
             lambda: e.compare_engines_device(x, None, la, None, cnt), lambda: e.topk_device_f32(x, 5, cl, sc),
             lambda: e.emulate_topk_device(x, 5, cl, fsc), lambda: E.quantize_images_device(x, q)]
    outs = [(lo, la), (flo, la), (la, cnt), (cl, sc), (cl, fsc), (q,)]
    s = torch.cuda.Stream()
    for call, o in zip(calls, outs):
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            call()   # warm-up outside the capture
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            call()
        x.copy_(images(n, 256, fmt, 2))
        for t in o:
            t.zero_()
        g.replay()
        torch.cuda.synchronize()
        got = [t.clone() for t in o]
        for t in o:
            t.zero_()
        call()
        torch.cuda.synchronize()
        for a, b in zip(got, o):
            _eq(a, b, (name, fmt, "graph"))
        del g
    e.close()


@pytest.mark.gpu
def test_launch_overlap_wait_after_16bit_call(lib, capfd, monkeypatch):
    """mode 2: an int8 launch right after a 16-bit one-kernel call keeps its wait, like one after a float32 call; two int8
    launches on disjoint buffers stay independent"""
    import torch
    from bitnetmcu_b200 import _lib
    from bitnetmcu_b200.engine import Engine
    e, _ = verbose_engine(capfd, monkeypatch, lambda: Engine(_model("fc"), device=0))
    n = 4096
    q = [torch.randint(-128, 128, (n, 256), dtype=torch.int8, device="cuda") for _ in range(3)]
    la = [torch.empty(n, dtype=torch.int32, device="cuda") for _ in range(4)]
    for fmt in FORMATS:
        x = images(n, 256, fmt, 4)
        e.set_option(_lib.OPT_LAUNCH_OVERLAP, 2)   # the first launch after it waits
        torch.cuda.synchronize()
        capfd.readouterr()
        s = torch.cuda.current_stream().cuda_stream
        e.infer_device(q[0], None, la[0], stream=s)
        e.infer_device(q[1], None, la[1], stream=s)
        e.infer_device_f32(x, None, la[2], stream=s)
        e.infer_device(q[2], None, la[3], stream=s)
        torch.cuda.synchronize()
        got = [l.split("fused launch: ")[1] for l in capfd.readouterr().err.splitlines() if "fused launch: " in l]
        assert got == ["wait", "independent", "wait"], (fmt, got)
    e.close()
