"""CPU-side checks of the boundary: the C-ABI library builds, loads without a GPU and exports every symbol that
include/bitnetmcu_b200.h declares; compute entries fail loudly (never fall back) when no CUDA device exists."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from conftest import ROOT, load_model
from support import sass


def _declared():
    text = open(os.path.join(ROOT, "include", "bitnetmcu_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"BNM_API\s+[\w\s\*]+?\b(\w+)\s*\(", text)))


def test_library_exports_every_declared_symbol(built):
    from bitnetmcu_b200 import _lib
    lib = _lib.load()
    declared = _declared()
    assert len(declared) >= 24
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in include/bitnetmcu_b200.h but not exported"
    assert sorted(_lib.EXPORTED) == declared
    out = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    exported = {l.split()[-1] for l in out.splitlines() if " T " in l}
    assert exported == set(declared), "library exports exactly the declared C ABI"
    assert lib.bnm_version() == 100


def test_library_contains_hopper_sass(built):
    """wgmma s8 / TMA / bulk copies show up as IGMMA / UTMALDG / UBLKCP in the sm_90a SASS."""
    text = sass()
    assert "sm_90a" in text
    for mnemonic in ("IGMMA", "WARPGROUP.ARRIVE", "UTMALDG", "UBLKCP", "VIADDMNMX", "VIMNMX3", "IDP.4A"):
        assert mnemonic in text, mnemonic


def test_no_cpu_fallback_without_gpu(built):
    from bitnetmcu_b200 import _lib
    lib = _lib.load()
    if lib.bnm_device_count() > 0:
        pytest.skip("a CUDA device is present")
    blob = load_model("fc").to_blob()
    h = C.c_void_p()
    rc = lib.bnm_model_load_blob(blob, len(blob), 0, C.byref(h))
    assert rc != 0 and not h.value and b"no CUDA device" in lib.bnm_last_error()
    x = np.zeros(8, dtype=np.int32)
    o = np.zeros(8, dtype=np.int8)
    assert lib.bnm_relunorm_batch(C.c_void_p(x.ctypes.data), C.c_void_p(o.ctypes.data), None, 8, 1) != 0
    from bitnetmcu_b200.engine import Engine
    with pytest.raises(_lib.BnmError):
        Engine(load_model("fc"))


def test_product_does_not_touch_the_oracle():
    """Only tests/, __graft_entry__.smoke() and bench.py may use oracle/ (as the checker)."""
    bad = []
    for base in ("bitnetmcu_b200", "include", "host"):
        for dirpath, _, files in os.walk(os.path.join(ROOT, base)):
            for f in files:
                if f.endswith((".py", ".cu", ".cuh", ".h", ".c", ".cpp")):
                    text = open(os.path.join(dirpath, f), errors="replace").read()
                    if re.search(r"\boracle\b|bitnet_oracle|libbnm_oracle|_ref/", text):
                        bad.append(os.path.join(dirpath, f))
    assert not bad, bad
