"""Plumbing more than one test module uses: the library fixture, engine factories, the BNM_VERBOSE lines, the library's SASS
dumped once, the ring sweep on this GPU, and the models, inputs and device calls that several modules feed.

Test modules import the fixture by name (`from support import lib`): pytest finds fixtures in a module's globals."""
import functools
import gc
import os
import re
import subprocess
import time
from typing import Callable, NamedTuple, Optional, Tuple

import numpy as np
import pytest

from conftest import GOLDEN, ROOT, load_model
from restate import TILE, most_tiles_per_cta, ring_sweep, sweep_gaps, tile_schedule

N_MANY = 148 * 128 * 2 + 77          # several tiles per CTA, a ragged last tile


@pytest.fixture(scope="module")
def lib(built):
    from bitnetmcu_b200 import _lib
    l = _lib.load()
    assert l.bnm_device_count() > 0, "no CUDA device"
    return l


# ---- engines ---------------------------------------------------------------------------------------------------------------

def engine(model, path=0, cnn_frontend=None):
    from bitnetmcu_b200 import _lib
    from bitnetmcu_b200.engine import Engine
    e = Engine(model, device=0, path=path)
    if cnn_frontend is not None:
        e.set_option(_lib.OPT_CNN_FRONTEND, cnn_frontend)
    return e


def frontends(model):
    """CNN models run once per front-end kernel (BNM_OPT_CNN_FRONTEND): CUDA cores and conv1-on-wgmma, which takes multiples of
    16 channels up to 128; FC models once."""
    from bitnetmcu_b200 import _lib
    if model.model_class != 1:
        return [None]
    tc = model.channels % 16 == 0 and model.channels <= 128
    return [_lib.CNN_CUDA_CORES, _lib.CNN_TENSOR_CORES] if tc else [_lib.CNN_CUDA_CORES]


def verbose_engine(capfd, monkeypatch, make):
    """the engine make() builds with BNM_VERBOSE set, and the lines it printed to stderr"""
    monkeypatch.setenv("BNM_VERBOSE", "1")
    capfd.readouterr()
    e = make()
    err = capfd.readouterr().err.splitlines()
    monkeypatch.delenv("BNM_VERBOSE")
    return e, err


def plan_line(err):
    """the last `fused FC plan` line, None when there is none"""
    plan = [l for l in err if "fused FC plan" in l]
    return plan[-1] if plan else None


def plan_ring(line, kind):
    """(row, (pipes, stages, slots)) of one form of a `fused FC plan` line: kind "int8" (fc_chain_kernel), "float" (the
    float-input row), "emul" (the float-input emulator row) or "emul_i8" (fc_emul_i8_kernel).  The slots are the third field
    of a two-pipe row's name <kN,pipes,slots,...>; a one-pipe row runs one."""
    if kind == "int8":
        row = re.search(r"fc_chain_kernel(<[^>]*>)", line).group(1)
        pipes, stages = map(int, re.search(r"(\d+) pipes x (\d+) stages", line).groups())
        fields = row[1:-1].split(",")
        assert int(fields[1]) == pipes, line
        return row, (pipes, stages, int(fields[2]) if pipes == 2 else 1)
    if kind == "emul_i8":
        row, stages = re.search(r"int8 emulator fc_emul_i8_kernel(<[^>]*>) x (\d+) stages", line).groups()
        return row, (1, int(stages), 1)
    row = re.search(r"float input (<[^>]*>)" if kind == "float" else r"emulator (<[^>]*>)", line).group(1)
    return row, (1, int(re.search(r"float input stages (\d+)", line).group(1)), 1)


def route(err, what):
    """the route of the one `<what> route:` line ("emulator" or "engines")"""
    lines = [l for l in err if f"{what} route: " in l]
    assert len(lines) == 1, lines
    return lines[0].split(f"{what} route: ")[1]


# ---- the library's SASS -----------------------------------------------------------------------------------------------------

@functools.lru_cache(maxsize=None)
def sass():
    """the SASS of the whole library, dumped once per session; take the `built` fixture before the first call"""
    from bitnetmcu_b200 import _lib
    return subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout


@functools.lru_cache(maxsize=None)
def sass_functions():
    """{mangled name: SASS text} of every function in the library"""
    return {k.split()[0]: k for k in re.split(r"\n\s*Function : ", sass())[1:]}


def instructions(text):
    return [i.strip() for i in re.findall(r"/\*[0-9a-f]{4,}\*/\s+([^;]*);", text)]


def local_memory(ins):
    """the instructions that load or store local memory"""
    return [i for i in ins if re.match(r"(@\S+\s+)?(LDL|STL)\b", i)]


# ---- the ring sweep on this GPU ---------------------------------------------------------------------------------------------

class Sweep:
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


# ---- models ------------------------------------------------------------------------------------------------------------------

def random_fc(enc, widths, seed):
    """a random FC model whose images are widths[0] bytes"""
    from bitnetmcu_b200 import pack as P
    m = P.random_fc_model(enc, widths, seed=seed)
    m.img_bytes = widths[0]
    return m


def with_plus128(codes, l):
    """FP130 codes with +128 (code 7) in every third row: row o at column (5 o + l) % n_in"""
    c = codes.copy()
    o = np.arange(0, c.shape[0], 3)
    c[o, (5 * o + l) % c.shape[1]] = 7
    return c


def fp130_codes(rng, n_out, n_in):
    """random FP130 codes without +128; -128 (code 15) stays, it fits an int8 plane"""
    c = rng.integers(0, 16, size=(n_out, n_in), dtype=np.uint32)
    c[c == 7] = 15
    return c


def chain(img_bytes, layers, seed):
    """a random FC model of img_bytes-byte rows; layers: (encoding, outputs), or (FP130, outputs, True) for +128 weights"""
    from bitnetmcu_b200 import model as M, pack as P
    rng = np.random.default_rng(seed)
    out, n_in = [], img_bytes
    for i, (enc, n_out, *plus) in enumerate(layers):
        name = f"L{i + 1}"
        if enc == M.ENC_TERNARY:
            out.append(P.fc_layer_from_trits(name, rng.integers(-1, 2, size=(n_out, n_in))))
        else:
            codes = fp130_codes(rng, n_out, n_in) if enc == M.ENC_FP130 else \
                rng.integers(0, 1 << P.CODE_BITS[enc], size=(n_out, n_in), dtype=np.uint32)
            out.append(P.fc_layer_from_codes(name, enc, with_plus128(codes, i) if plus else codes))
        n_in = n_out
    m = M.Model(model_class=M.MODEL_FCMNIST, layers=out, img_bytes=img_bytes)
    m.validate()
    return m


# every row of kChainKernels (fc_wgmma.cu), with a model that selects it (checked against the plan's BNM_VERBOSE line)
CHAIN_ROWS = [
    ("<64,1>", lambda: random_fc(4, (512, 64, 64, 10), 1)),           # 512-byte rows: room for three 64 kB stages, one pipe
    ("<64,2,2,64>", lambda: random_fc(4, (256, 64, 64, 37), 2)),      # 37 classes: the last layer is wider than 16
    ("<64,2,2,16>", lambda: load_model("1k")),                        # 16-wide layers, three of them: not the fixed class
    ("<64,2,2,16,fixed>", lambda: load_model("fc")),
    ("<128,1>", lambda: load_model("2bitsym96")),
    ("<192,1>", lambda: load_model("binary160")),
    ("<256,1>", lambda: random_fc(4, (256, 256, 10), 3)),
]


def cnn_model(channels, n_classes, seed, w=(None, None, None), hidden=(64,)):
    """a random CNN model: conv weights uniform in [-128, 127] with +-127 taps in every layer (or the given weights), 4bitsym
    hidden layers of the given widths (default one, 64 wide; none: the features feed the head directly) and an n_classes head"""
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
    fc = P.random_fc_model(M.ENC_4BITSYM, (channels * 4,) + tuple(hidden) + (n_classes,), seed=seed)
    for i, l in enumerate(fc.layers):
        l.name = f"L{11 + 2 * i}"
        layers.append(l)
    m = M.Model(model_class=M.MODEL_CNNMNIST, layers=layers)
    m.validate()
    return m


# ---- inputs -------------------------------------------------------------------------------------------------------------------

def int8_images(n, d, seed):
    """n int8 rows of d bytes: rows at the int8 rails, all zero, one value, then random rows"""
    rng = np.random.default_rng(seed)
    q = rng.integers(-128, 128, size=(n, d)).astype(np.int8)
    rails = [np.full(d, 127), np.full(d, -128), np.zeros(d), np.where(np.arange(d) % 2, -128, 127),
             np.where(rng.random(d) < 0.5, 127, -128), np.full(d, 1)]
    q[:len(rails)] = np.stack(rails)
    return q


def normal_images(n, seed, elems=256):
    """normal float32 rows, the first 40 of them MNIST-normalised"""
    rng = np.random.default_rng(seed)
    x = rng.normal(size=(n, elems)).astype(np.float32)
    k = min(n, 40)
    x[:k] = (rng.integers(0, 256, size=(k, elems)) / 255.0 - 0.1307).astype(np.float32) / np.float32(0.3081)
    return x


def scattered_edge_images(n, elems, seed):
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


def quantized_model_list(m, nf4_extension=False):
    """the reference emulator's layer list for model m (tests/golden/make_emulator_golden.py): weight levels = the integer
    weights over the encoding's level scale (NF4: zeros, or the extension's LUT with nf4_extension), Ternary's zero pad columns
    dropped"""
    from bitnetmcu_b200 import model as M, pack as P
    from restate import LEVEL_SHIFT
    out, width = [], m.img_bytes if m.model_class == 0 else m.channels * 4
    for l in m.layers:
        if l.kind == M.LAYER_FC:
            w = P.decode_int_weights(l, nf4_extension).astype(np.float64)[:, :width] / 2.0 ** LEVEL_SHIFT.get(l.bitperweight, 0)
            width = l.n_out
            out.append({"layer_type": "BitLinear", "incoming_weights": l.n_in, "outgoing_weights": l.n_out,
                        "quantized_weights": w.tolist(), "WScale": "PerTensor", "bpw": 0, "quantization_type": M.ENC_NAMES[l.bitperweight]})
        elif l.kind == M.LAYER_CONV33:
            first = l.n_in == 16
            out.append({"layer_type": "BitConv2d", "in_channels": 1 if first else l.n_out, "out_channels": l.n_out, "kernel_size": (3, 3),
                        "stride": 1, "padding": 0, "groups": 1 if first else l.n_out, "quantized_weights": l.weights.astype(np.float64).tolist(),
                        "incoming_x": 0, "incoming_y": 0, "outgoing_x": 0, "outgoing_y": 0, "bpw": 8, "quantization_type": "8bit"})
        else:
            out.append({"layer_type": "MaxPool2d", "kernel_size": 2, "stride": 2})
    return out


def crafted_cnn_case():
    """images: all zero, and one negative pixel among zeros, then normal rows; models: a random CNN and two whose conv2 or
    conv3 taps are all <= 0 (no positive output on non-negative inputs).  -> (images, [(model, what)])"""
    x = normal_images(700, seed=5)
    x[:110] = 0.0
    x[100:110, 7] = np.float32(-3.0)
    rng = np.random.default_rng(3)
    neg = -rng.integers(0, 129, size=48 * 9)
    return x, [(cnn_model(48, 10, seed=4, w=w), what)
               for w, what in (((None, None, None), "random"), ((None, neg, None), "conv2 <= 0"), ((None, None, neg), "conv3 <= 0"))]


# ---- device calls -------------------------------------------------------------------------------------------------------------

def run_emulator(e, x, want_logits=True, want_labels=True, stream=None):
    """the emulator's device entry -> (logits, labels) as NumPy, None for what was not asked for; x NumPy or a CUDA tensor"""
    import torch
    d_x = x if isinstance(x, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).cuda()
    n = d_x.shape[0]
    lo = torch.full((n, e.n_classes), np.nan, dtype=torch.float64, device="cuda") if want_logits else None
    la = torch.full((n,), -1, dtype=torch.int32, device="cuda") if want_labels else None
    e.inference_quantized_device(d_x, lo, la, stream=stream)
    torch.cuda.synchronize()
    return (lo.cpu().numpy() if want_logits else None), (la.cpu().numpy().astype(np.int64) if want_labels else None)


def run_emulator_layered(e, x):
    """run_emulator on the layer-by-layer route (BNM_PATH_LAYERS), then back to the default path"""
    from bitnetmcu_b200 import _lib
    e.set_option(_lib.OPT_PATH, _lib.PATH_LAYERS)
    try:
        return run_emulator(e, x)
    finally:
        e.set_option(_lib.OPT_PATH, _lib.PATH_AUTO)


def gather_call(lib, e, d_img, d_log, d_lab, g, stream):
    """bnm_infer_batch_device_gather of the engine on GPU 0 (images d_img, own outputs d_log / d_lab, either None, and the
    destinations of the BnmGather g) on `stream`, then waits for the stream -> the entry's return code"""
    import ctypes as Ct
    import torch
    ptr = lambda t: Ct.c_void_p(t.data_ptr()) if t is not None else None
    with torch.cuda.device(0):
        rc = lib.bnm_infer_batch_device_gather(e.handle, ptr(d_img), d_img.shape[0], ptr(d_log), ptr(d_lab), Ct.byref(g),
                                               Ct.c_void_p(stream.cuda_stream))
        stream.synchronize()
    return rc


# ---- device checks of one case's rows ------------------------------------------------------------------------------------
# d: the case on the device -- d.name, d.C (classes), d.idx(n) (the rows of a batch of n) and d.check(n, got, want, sentinel,
# what), which compares rows :n of an (n + 128)-row buffer with want[d.idx(n)] and the rows past n with the sentinel.

def to_device(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def out(shape, dtype, sentinel):
    """a device buffer of shape with 128 rows more, all sentinel"""
    import torch
    return torch.full((shape[0] + 128,) + tuple(shape[1:]), sentinel, dtype=dtype, device="cuda")


def top_k(logits, k):
    """the k best classes of each row and their scores: a stable sort, highest first, ties to the lower class"""
    cls = np.argsort(-logits, axis=1, kind="stable")[:, :k]
    return cls.astype(np.int32), np.take_along_axis(logits, cls, axis=1)



def c_float(e, d, n, x, want_lo, want_la, what):
    """the C engine's float entry (float32 or 16-bit rows x): logits and labels, then labels alone"""
    import torch
    lo, la = out((n, d.C), torch.int32, -5), out((n,), torch.int32, -7)
    e.infer_device_f32(x, lo[:n], la[:n])
    torch.cuda.synchronize()
    d.check(n, lo, want_lo, -5, f"{what} logits")
    d.check(n, la, want_la, -7, f"{what} labels")
    la.fill_(-7)
    e.infer_device_f32(x, None, la[:n])
    torch.cuda.synchronize()
    d.check(n, la, want_la, -7, f"{what} labels only")


def emulator(e, d, n, x, want_lo, want_la, what):
    """the emulator's entry: float64 logits and labels"""
    import torch
    lo, la = out((n, d.C), torch.float64, -12345.5), out((n,), torch.int32, -7)
    e.inference_quantized_device(x, lo[:n], la[:n])
    torch.cuda.synchronize()
    d.check(n, lo, want_lo, -12345.5, f"{what} emulator logits")
    d.check(n, la, want_la, -7, f"{what} emulator labels")


def both_engines(e, d, n, x, want_la, want_py_la, what):
    """bnm_compare_engines_device: the C labels, the emulator's labels where it is exact, and the counts"""
    import torch
    truth = ((torch.arange(n, device="cuda") * 7) % (d.C + 1)).to(torch.int32)
    lc, lp = out((n,), torch.int32, -7), out((n,), torch.int32, -7)
    counts = torch.zeros(4, dtype=torch.int64, device="cuda")
    e.compare_engines_device(x, truth, lc[:n], lp[:n], counts)
    torch.cuda.synchronize()
    d.check(n, lc, want_la, -7, f"{what} engines: C labels")
    wc = want_la[d.idx(n)]
    got = counts.cpu().tolist()
    assert got[:2] == [n, int((wc == truth).sum())], (d.name, n, what, "engines: counts", got)
    if want_py_la is not None:
        d.check(n, lp, want_py_la, -7, f"{what} engines: emulator labels")
        wp = want_py_la[d.idx(n)]
        assert got[2:] == [int((wp == truth).sum()), int((wc != wp).sum())], (d.name, n, what, "engines: counts", got)


# ---- kernel neighbours of a launch -------------------------------------------------------------------------------------------
# A dependent launch relaxes the ordering between two kernels only: after a cudaMemcpyAsync, which is what ATen makes of
# Tensor.copy_ and Tensor.clone on contiguous tensors of one dtype, the fused FC launch runs fully serialised and its
# grid-dependency wait is never put to the test.  Tests that place a producer or consumer next to a launch use these.

def kernel_copy(dst, src):
    """dst <- src (same dtype, an integer type) by an elementwise CUDA kernel, never a memory copy"""
    import torch
    torch.bitwise_xor(src, 0, out=dst)
    return dst


def kernel_clone(src):
    """a new tensor equal to src (an integer type), written by an elementwise CUDA kernel"""
    import torch
    return torch.bitwise_xor(src, 0)


@functools.lru_cache(maxsize=None)
def _kernel_copy_profile():
    """the CUDA activities torch.profiler records for one kernel_copy and one kernel_clone, and whether both copied.  Once per
    process: a later profiler session in the same process can miss activities."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    src = torch.arange(-128, 128, dtype=torch.int32, device="cuda").to(torch.int8).repeat(64)
    dst = torch.full_like(src, 5)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        kernel_copy(dst, src)
        out = kernel_clone(dst)
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    return names, bool(torch.equal(dst, src) and torch.equal(out, src))


@pytest.fixture(scope="session")
def kernel_copies_are_kernels(built):
    """kernel_copy and kernel_clone record a CUDA kernel each and no memcpy (torch.profiler); fails if torch ever turns them
    into copies"""
    names, copied = _kernel_copy_profile()
    assert not [n for n in names if "memcpy" in n.lower() or "memset" in n.lower()], names
    assert len([n for n in names if "BitwiseXor" in n]) == 2, names
    assert copied
    return True


# ---- the plain-C host side ----------------------------------------------------------------------------------------------------

def _write_test_data_header(path, images, labels):
    with open(path, "w") as f:
        for i in range(images.shape[0]):
            f.write(f"int8_t input_data_{i}[256] = {{" + ", ".join(str(int(v)) for v in images[i]) + "};\n")
            f.write(f"uint8_t label_{i} = {int(labels[i])};\n")


def build_c_shim(tmp, name):
    """gcc-build host/'s DLL shim and MNIST test program for a fixture model in tmp -> (dll, exe, digits.npz)"""
    from bitnetmcu_b200 import _lib
    from bitnetmcu_b200.pack import write_header
    m = load_model(name)
    # Model.load names the layers as the reference's dll.c expects: FC L1..L4 / CNN L2..L15 (dll.c:48-121)
    want = ["L2", "L4", "L6", "L7", "L9", "L11", "L13", "L15"] if m.model_class == 1 else ["L1", "L2", "L3", "L4"]
    assert [l.name for l in m.layers] == want[:len(m.layers)]
    write_header(m, os.path.join(tmp, "BitNetMCU_model.h"))
    d = np.load(os.path.join(GOLDEN, "digits.npz"))
    _write_test_data_header(os.path.join(tmp, "BitNetMCU_MNIST_test_data.h"), d["images"], d["labels"])
    libdir = os.path.dirname(_lib.LIB_PATH)
    common = ["-I" + tmp, "-I" + os.path.join(ROOT, "include"), "-L" + libdir, "-lbitnetmcu_b200", "-Wl,-rpath," + libdir]
    dll = os.path.join(tmp, "Bitnet_inf.dll")
    exe = os.path.join(tmp, "mnist_test")
    subprocess.run(["gcc", "-fPIC", "-shared", "-D_DLL", "-o", dll, os.path.join(ROOT, "host", "bitnetmcu_b200_dll.c")] + common, check=True)
    subprocess.run(["gcc", "-o", exe, os.path.join(ROOT, "host", "bitnetmcu_b200_test.c"), os.path.join(ROOT, "host", "bitnetmcu_b200_dll.c")] + common,
                   check=True)
    return dll, exe, d


# ---- batches past 2^31 and 2^32 bytes ------------------------------------------------------------------------------------------
# A large batch is periodic: U unique rows (an odd prime), row i of the batch unique row i mod U, built on the device by
# index_select, so nothing of GB size crosses the host.  Its expected result is the same entry on the U unique rows, pinned to the
# oracle or to restate, then tiled and compared on the device, in slices.  A 32-bit product anywhere in an offset would displace a
# read or a write by 2^31 or 2^32 bytes, which with U odd lands on another unique row: check_wrapped_offsets shows, on the CPU, that
# the expected result there differs for most rows.  Every output buffer holds a sentinel, checked past row n.

U = 8191                        # unique rows of a batch, an odd prime
P = 89                          # period of a window-scan page in both directions, an odd prime
SPARE = 128                     # sentinel rows past n in every output buffer
SLICE_BYTES = 256 << 20         # bytes of a row slice the device builds or compares at a time
GiB = 1 << 30
SENTINEL_I32, SENTINEL_F64, SENTINEL_I8 = -0x3C3C3C3D, -7.25e300, -0x3D   # fill of every output buffer
WRAPS = (1 << 31, 1 << 32)      # the byte displacements of a wrapped 32-bit offset


def row_uid(rows):
    """the unique row of batch rows (NumPy or torch integers)"""
    return rows % U


class Spec(NamedTuple):
    kind: str                     # the entry's key in its module's expected()
    name: str                     # the model
    n: int                        # images or windows
    in_bytes: Optional[int]       # bytes per input row (None: the window scan, whose pages stay small)
    outputs: Tuple[str, ...]      # what the call writes
    uid: Callable = row_uid
    planes: int = 1               # window scan: pages in the stack


def _differ(a, b):
    return (a != b).reshape(len(a), -1).any(axis=1)


def check_wrapped_offsets(case, s, res):
    """for every read and write of case s whose offsets pass a wrap W (2^31 or 2^32 bytes), the result a read or write displaced
    by W would give differs from the expected one (res: {output: NumPy [unique, ...]}) for most rows: reads of input row
    a - W / in_bytes, and the bytes a wrapped write of row a would put over the rows there, on every output of the call"""
    checked = 0
    for w in WRAPS:
        if s.in_bytes and s.n * s.in_bytes > w:
            assert w % s.in_bytes == 0
            d = w // s.in_bytes
            a = np.arange(d, min(s.n, d + U))
            diff = np.zeros(a.size, dtype=bool)
            for o in s.outputs:
                diff |= _differ(res[o][s.uid(a)], res[o][s.uid(a - d)])
            assert diff.mean() > 0.5, (case, "input", w, d, diff.mean())
            checked += 1
        for o in s.outputs:
            e = np.ascontiguousarray(res[o])
            rb = e[0].nbytes
            if s.n * rb <= w:
                continue
            b = e.view(np.uint8).reshape(e.shape[0], rb)
            a = np.arange(-(-w // rb), min(s.n, -(-w // rb) + U))
            pos = (a * rb - w)[:, None] + np.arange(rb)
            under = b[s.uid(pos // rb), pos % rb]          # what the rows there hold
            diff = _differ(b[s.uid(a)], under)
            assert diff.mean() > 0.5, (case, o, w, diff.mean())
            checked += 1
    assert checked, (case, "no offset of this case passes 2^31 bytes")
    assert s.in_bytes is None or (s.n - 77) & (s.n - 78) == 0, (case, "n is not 77 past a power of two")


def _free():
    import torch
    gc.collect()
    torch.cuda.empty_cache()
    return torch.cuda.mem_get_info()[0]


class Case:
    """one case: its need checked against the free device memory (skip with the figure); on exit its engines closed and its
    peak device memory (torch's tensors, and what the library held, as the device sees it) and wall time printed"""

    def __init__(self, what, n, need):
        self.what, self.n, self.need = what, n, need
        self.engines = []

    def engine(self, make):
        self.engines.append(make())
        return self.engines[-1]

    def __enter__(self):
        import torch
        free = _free()
        if free < self.need:
            pytest.skip(f"{self.what}: needs {self.need / GiB:.1f} GiB of device memory, {free / GiB:.1f} GiB free")
        torch.cuda.reset_peak_memory_stats()
        self.free0, self.reserved0 = free, torch.cuda.memory_reserved()
        self.t0 = time.perf_counter()
        return self

    def __exit__(self, *exc):
        import torch
        torch.cuda.synchronize()
        # the library's scratch pools keep their high-water mark until the engine closes
        held = (self.free0 - torch.cuda.mem_get_info()[0]) - (torch.cuda.memory_reserved() - self.reserved0)
        for e in self.engines:
            e.close()
        if exc[0] is None:
            peak = torch.cuda.max_memory_reserved() - self.reserved0 + held
            print(f"large batch: {self.what}: n = {self.n}, peak device memory {peak / GiB:.2f} GiB, "
                  f"wall {time.perf_counter() - self.t0:.2f} s")
        _free()
        return False


def _dtype(a):
    import torch
    return {np.dtype(np.float64): torch.float64, np.dtype(np.int8): torch.int8}.get(a.dtype, torch.int32)


def slices(t, n):
    """(start, end) of row slices of about SLICE_BYTES of tensor t, up to row n"""
    step = max(1, SLICE_BYTES // (t[0].numel() * t.element_size()))
    return [(s, min(n, s + step)) for s in range(0, n, step)]


def _on_device(unique):
    """unique rows (NumPy, or a torch tensor for the 16-bit formats NumPy lacks) on the device"""
    import torch
    u = unique if isinstance(unique, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(unique))
    return u.cuda()


def periodic(unique, n):
    """the CUDA batch [n, ...] whose row i is unique row i mod U, built slice by slice with index_select"""
    import torch
    u = _on_device(unique)
    out = torch.empty((n,) + tuple(u.shape[1:]), dtype=u.dtype, device="cuda")
    for s, e in slices(out, n):
        torch.index_select(u, 0, row_uid(torch.arange(s, e, device="cuda")), out=out[s:e])
    return out


def _sentinel(dtype):
    import torch
    return {torch.float64: SENTINEL_F64, torch.int8: SENTINEL_I8}.get(dtype, SENTINEL_I32)


def outputs(res, names, n):
    """{output: CUDA tensor [n + SPARE, ...] filled with the sentinel}, shaped like the expected rows"""
    import torch
    return {o: torch.full((n + SPARE,) + res[o].shape[1:], _sentinel(_dtype(res[o])), dtype=_dtype(res[o]), device="cuda")
            for o in names}


def views(outs, n, lead=None):
    """rows :n of every output buffer (reshaped to lead + row shape when given)"""
    return {o: (t[:n] if lead is None else t[:n].reshape(lead + tuple(t.shape[1:]))) for o, t in outs.items()}


def want_on_device(got, res, what):
    """the small call's outputs (CUDA, rows :U') equal the expected NumPy rows: -> them as CUDA tensors"""
    out = {}
    for o, t in got.items():
        w = res[o]
        g = t[:w.shape[0]].cpu().numpy()
        bad = np.flatnonzero(_differ(g.astype(w.dtype) if w.dtype == np.uint32 else g, w))
        assert bad.size == 0, (what, o, "small call", f"{bad.size} unique rows differ from the reference, first {bad[:6].tolist()}")
        out[o] = t[:w.shape[0]].clone()
    return out


def check_tiled(got, want, n, uid, what):
    """rows :n of got equal want[uid(row)], compared on the device in slices; rows n: still hold the sentinel"""
    import torch
    for o, t in got.items():
        w = want[o]
        for s, e in slices(t, n):
            bad = (t[s:e] != w.index_select(0, uid(torch.arange(s, e, device="cuda")))).reshape(e - s, -1).any(dim=1)
            if bool(bad.any()):
                rows = (torch.nonzero(bad)[:6, 0] + s).tolist()
                raise AssertionError((what, o, f"{int(bad.sum())} rows of {s}..{e} wrong, first {rows}",
                                      f"byte offsets {[r * t[0].numel() * t.element_size() for r in rows]}"))
        assert bool((t[n:] == _sentinel(t.dtype)).all()), (what, o, "written past row n")


def check_input(x, unique, what):
    """the periodic batch x still holds its rows"""
    import torch
    u = _on_device(unique)
    for s, e in slices(x, x.shape[0]):
        assert torch.equal(x[s:e], u.index_select(0, row_uid(torch.arange(s, e, device="cuda")))), (what, "input changed", s)


def need(s, res, extra=0):
    """device bytes of a case: the batch, the outputs with their sentinel rows, and 1 GiB for a comparison slice, the unique rows'
    results and the library's scratch and planes"""
    per_row = sum(res[o][0].nbytes for o in s.outputs)
    return s.n * (s.in_bytes or 0) + (s.n + SPARE) * per_row + GiB + extra
