"""The argument rules of every batched inference entry of the C ABI (GPU, H100), pinned entry by entry: a null model or null images,
every output NULL at n > 0 and at n == 0, k out of range for the top-k entries, each buffer 4 bytes off its allocation at n > 0
and at n == 0, truth without counts, and a gather with too many destinations or misaligned logits destinations.  Each case
checks the return code and, for an error, a fragment of bnm_last_error().  The entries do not share every rule: the two-engine
entry refuses a call without outputs even at n == 0, the top-k entries check k and their buffers' alignment whatever n, labels
and truth are never alignment-checked, and host buffers never are."""
import ctypes as C

import pytest

from conftest import load_model
from support import engine, lib

pytestmark = pytest.mark.gpu

N, K, ARG = 64, 3, -1

# entry: (device or host buffers, arguments after the model, in order: each a buffer, "n", "k" or "stream"; the outputs)
ENTRIES = {
    "bnm_infer_batch_device": ("dev", ["images:i8", "n", "logits:lo32", "labels:lab", "stream"], ["logits", "labels"]),
    "bnm_infer_batch_device_gather": ("dev", ["images:i8", "n", "logits:lo32", "labels:lab", "gather", "stream"], ["logits", "labels"]),
    "bnm_infer_batch_device_f32": ("dev", ["images:f32", "n", "logits:lo32", "labels:lab", "stream"], ["logits", "labels"]),
    "bnm_emulate_batch_device": ("dev", ["images:f32", "n", "logits:lo64", "labels:lab", "stream"], ["logits", "labels"]),
    "bnm_compare_engines_device": ("dev", ["images:f32", "n", "truth:lab2", "labels_c:lab", "labels_py:lab3", "counts:cnt", "stream"],
                                   ["labels_c", "labels_py", "counts"]),
    "bnm_infer_topk_device": ("dev", ["images:i8", "n", "k", "classes:cls", "scores:sc32", "stream"], ["classes", "scores"]),
    "bnm_infer_topk_device_f32": ("dev", ["images:f32", "n", "k", "classes:cls", "scores:sc32", "stream"], ["classes", "scores"]),
    "bnm_emulate_topk_device": ("dev", ["images:f32", "n", "k", "classes:cls", "scores:sc64", "stream"], ["classes", "scores"]),
    "bnm_infer_batch": ("host", ["images:i8", "n", "logits:lo32", "labels:lab"], ["logits", "labels"]),
    "bnm_infer_topk": ("host", ["images:i8", "n", "k", "classes:cls", "scores:sc32"], ["classes", "scores"]),
    "bnm_emulate_inference_quantized": ("host", ["images:f32", "n", "logits:lo64"], ["logits"]),
}

IMAGES16 = (ARG, "image buffer must be 16-byte aligned")
LOGITS8 = (ARG, "logits buffer must be 8-byte aligned")
# what each buffer 4 bytes off its allocation gives at n > 0 (buffers not listed: 0)
MISALIGNED = {
    "bnm_infer_batch_device": {"images": IMAGES16, "logits": LOGITS8},
    "bnm_infer_batch_device_gather": {"images": IMAGES16, "logits": LOGITS8},
    "bnm_infer_batch_device_f32": {"images": IMAGES16, "logits": LOGITS8},
    "bnm_emulate_batch_device": {"images": IMAGES16, "logits": LOGITS8},
    "bnm_compare_engines_device": {"images": IMAGES16, "counts": (ARG, "counts must be 8-byte aligned")},
    "bnm_infer_topk_device": {"images": IMAGES16},
    "bnm_infer_topk_device_f32": {"images": IMAGES16},
    "bnm_emulate_topk_device": {"images": IMAGES16, "scores": (ARG, "scores buffer must be 8-byte aligned")},
}
# what a call with every output NULL gives at n > 0 and at n == 0 (entries not listed: "no output" at n > 0 only)
NO_OUTPUT = {
    "bnm_compare_engines_device": ((ARG, "no output"), (ARG, "no output")),
    "bnm_infer_topk_device": ((ARG, "null argument"), (0, None)),
    "bnm_infer_topk_device_f32": ((ARG, "null argument"), (0, None)),
    "bnm_emulate_topk_device": ((ARG, "null argument"), (0, None)),
    "bnm_infer_topk": ((ARG, "null argument"), (0, None)),
    "bnm_emulate_inference_quantized": ((ARG, "null argument"), (0, None)),
}


@pytest.fixture(scope="module")
def setup(lib):
    import torch
    e = engine(load_model("fc"))          # 10 classes, fused path
    rows, c = N + 4, e.n_classes
    dev = {"i8": torch.zeros((rows, 256), dtype=torch.int8, device="cuda"),
           "f32": torch.ones((rows, 256), dtype=torch.float32, device="cuda"),
           "lo32": torch.zeros((rows, c), dtype=torch.int32, device="cuda"),
           "lo64": torch.zeros((rows, c), dtype=torch.float64, device="cuda"),
           "lab": torch.zeros(rows, dtype=torch.int32, device="cuda"),
           "lab2": torch.zeros(rows, dtype=torch.int32, device="cuda"),
           "lab3": torch.zeros(rows, dtype=torch.int32, device="cuda"),
           "cls": torch.zeros((rows, 16), dtype=torch.int32, device="cuda"),     # room for k = n_classes
           "sc32": torch.zeros((rows, 16), dtype=torch.int32, device="cuda"),
           "sc64": torch.zeros((rows, 16), dtype=torch.float64, device="cuda"),
           "cnt": torch.zeros(8, dtype=torch.int64, device="cuda")}
    host = {key: t.cpu().numpy() for key, t in dev.items()}
    yield e, {"dev": {key: (t, t.data_ptr()) for key, t in dev.items()}, "host": {key: (a, a.ctypes.data) for key, a in host.items()}}
    torch.cuda.synchronize()
    e.close()


def call(lib, setup, name, model=True, n=N, k=K, null=(), off=(), gather=None):
    """entry `name` on valid arguments but for: no model, n images, k, the arguments in `null` NULL, the ones in `off` 4 bytes
    past their allocations, and the gather spec -> (return code, bnm_last_error())"""
    e, bufs = setup
    where, args, _ = ENTRIES[name]
    vals = [e.handle if model else None]
    for a in args:
        arg, _, key = a.partition(":")
        if key:
            vals.append(None if arg in null else C.c_void_p(bufs[where][key][1] + (4 if arg in off else 0)))
        else:
            vals.append({"n": n, "k": k, "stream": None, "gather": None if gather is None else C.byref(gather)}[arg])
    rc = getattr(lib, name)(*vals)
    return rc, lib.bnm_last_error().decode()


def expect(got, want, what):
    rc, err = got
    assert rc == want[0], (what, rc, err)
    if want[1] is not None:
        assert want[1] in err, (what, err)


@pytest.mark.parametrize("name", sorted(ENTRIES))
def test_entry_argument_matrix(lib, setup, name):
    import torch
    where, args, outputs = ENTRIES[name]
    buffers = [a.partition(":")[0] for a in args if ":" in a]
    topk = "k" in args
    expect(call(lib, setup, name, model=False), (ARG, "null argument"), "null model")
    expect(call(lib, setup, name, null=("images",)), (ARG, "null argument"), "null images")
    expect(call(lib, setup, name, null=("images",), n=0), (0, None), "null images, n == 0")
    at_n, at_0 = NO_OUTPUT.get(name, ((ARG, "no output"), (0, None)))
    none = outputs + ["truth"]            # truth goes with counts (test_truth_without_counts)
    expect(call(lib, setup, name, null=none), at_n, "every output NULL")
    expect(call(lib, setup, name, null=none, n=0), at_0, "every output NULL, n == 0")
    if topk:
        for k in (0, 11, 17):   # n_classes = 10, at most 16
            expect(call(lib, setup, name, k=k), (ARG, "k = "), ("k", k))
        expect(call(lib, setup, name, k=0, n=0), (ARG, "k = "), "k = 0, n == 0")
        expect(call(lib, setup, name, k=10), (0, None), "k = n_classes")
    for b in buffers:
        want = MISALIGNED.get(name, {}).get(b, (0, None))
        expect(call(lib, setup, name, off=(b,)), want, ("4 bytes off", b))
        expect(call(lib, setup, name, off=(b,), n=0), want if where == "dev" and topk else (0, None), ("4 bytes off, n == 0", b))
    expect(call(lib, setup, name), (0, None), "valid")
    expect(call(lib, setup, name, n=0), (0, None), "valid, n == 0")
    torch.cuda.synchronize()


def test_truth_without_counts(lib, setup):
    for n in (N, 0):
        expect(call(lib, setup, "bnm_compare_engines_device", null=("counts",), n=n), (ARG, "truth without counts"), ("n", n))
    expect(call(lib, setup, "bnm_compare_engines_device", null=("truth",)), (0, None), "counts without truth")


def test_gather_destinations(lib, setup):
    import torch
    from bitnetmcu_b200 import _lib
    _, bufs = setup
    lab, lo = bufs["dev"]["lab2"][1], bufs["dev"]["lo32"][1]
    name = "bnm_infer_batch_device_gather"
    g = _lib.BnmGather()
    expect(call(lib, setup, name, null=("logits", "labels"), gather=g), (ARG, "no output"), "no destinations")
    expect(call(lib, setup, name, null=("logits", "labels"), gather=g, n=0), (0, None), "no destinations, n == 0")
    g.n_labels_dst = _lib.MAX_GATHER_DST + 1
    for d in range(_lib.MAX_GATHER_DST):
        g.labels_dst[d] = lab
    expect(call(lib, setup, name, gather=g), (ARG, "gather destinations"), "too many label destinations")
    g = _lib.BnmGather()
    g.n_logits_dst = _lib.MAX_GATHER_DST + 1
    expect(call(lib, setup, name, gather=g), (ARG, "gather destinations"), "too many logits destinations")
    g = _lib.BnmGather()
    g.n_logits_dst, g.logits_dst[0] = 1, lo + 4
    expect(call(lib, setup, name, gather=g), (ARG, "gather logits buffers must be 8-byte aligned"), "misaligned logits destination")
    expect(call(lib, setup, name, gather=g, n=0), (ARG, "gather logits buffers must be 8-byte aligned"), "misaligned, n == 0")
    g = _lib.BnmGather()
    g.n_labels_dst, g.labels_dst[0] = 1, lab
    expect(call(lib, setup, name, null=("logits", "labels"), gather=g), (0, None), "one label destination alone")
    torch.cuda.synchronize()
