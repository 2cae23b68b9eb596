"""The plain-C host side (host/*.c): compiles against any exported BitNetMCU_model.h with gcc and, on a GPU, reproduces
the reference's stdout for BASELINE.json config #1 (BitNetMCU_MNIST_test.c + 10 digits) and its ctypes protocol."""
import ctypes as C
import subprocess

import numpy as np
import pytest

from support import build_c_shim


@pytest.mark.parametrize("name", ["fc", "cnn", "1k"])
def test_shim_compiles_and_exports_inference(built, tmp_path, name):
    dll, exe, _ = build_c_shim(str(tmp_path), name)
    out = subprocess.run(["nm", "-D", "--defined-only", dll], capture_output=True, text=True, check=True).stdout
    for sym in ("Inference", "InferenceBatch", "BitMnistInference"):
        assert f" T {sym}" in out


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["fc", "cnn"])
def test_shim_reproduces_reference_stdout(built, tmp_path, name):
    dll, exe, d = build_c_shim(str(tmp_path), name)
    out = subprocess.run([exe], capture_output=True, text=True, check=True, timeout=120).stdout
    want = "".join(f"label: {int(l)} predicted: {int(l)}\n" for l in d["labels"])   # reference: 10/10 for both shipped models
    assert out == want
    # the ctypes protocol of test_inference.py:134-150
    lib = C.CDLL(dll)
    lib.Inference.argtypes = [C.POINTER(C.c_int8)]
    lib.Inference.restype = C.c_uint32
    for i in range(10):
        img = np.ascontiguousarray(d["images"][i])
        assert lib.Inference(img.ctypes.data_as(C.POINTER(C.c_int8))) == int(d["labels"][i])
