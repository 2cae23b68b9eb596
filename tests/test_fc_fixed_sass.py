"""CPU-side checks of the fixed-shape fused FC kernel (fc_chain_kernel<64, 2, int8, 2, 16, kFixed>, the FC 4bitsym-64 class):
its sm_90a SASS issues layer 1 as one unrolled run of wgmma, ReLUNorm without predicates, and its consumer warpgroups divide
nothing per tile."""
import re

import pytest

from support import instructions, sass_functions

FIXED = "_ZN3bnm15fc_chain_kernelILi64ELi2ELb0ELi2ELi16ELb1EEEv14CUtensorMap_stNS_11ChainParamsE"


@pytest.fixture(scope="module")
def fixed_sass(built):
    ins = instructions(sass_functions().get(FIXED, ""))
    assert len(ins) > 100, "fixed-shape instantiation missing from the library"
    return ins


def _consumer(ins):
    """the consumer warpgroups' code: from the register increase to the producer's decrease"""
    lo = next(k for k, i in enumerate(ins) if i.startswith("USETMAXREG.TRY_ALLOC"))
    hi = next(k for k, i in enumerate(ins) if i.startswith("USETMAXREG.DEALLOC"))
    assert lo < hi
    return ins[lo:hi]


def test_layer1_is_one_unrolled_igmma_run(fixed_sass):
    """8 x m64n64k32 (two SW128 atoms x four K-steps), the first one without accumulate, with no branch, warpgroup arrive or
    other MMA between them"""
    runs, cur = [], None
    for i in fixed_sass:
        if i.startswith("IGMMA.64x64x32"):
            if "!UPT" in i:
                cur = [i]
            elif cur is not None:
                cur.append(i)
            if cur is not None and len(cur) == 8:
                runs.append(cur)
                cur = None
        elif cur is not None and ("BRA" in i or "WARPGROUP" in i or "GMMA" in i or "EXIT" in i):
            cur = None
    ss = [r for r in runs if "gdesc" in r[0] and not re.search(r"IGMMA\S*\s+R\d+,\s+R\d+", r[0])]
    assert len(ss) >= 2, f"no contiguous layer-1 IGMMA run: {runs}"


def test_relunorm_unpredicated(fixed_sass):
    vimnmx3 = [i for i in _consumer(fixed_sass) if "VIMNMX3" in i]
    assert vimnmx3
    assert not [i for i in vimnmx3 if i.startswith("@")], "predicated VIMNMX3 in the fixed-shape ReLUNorm"


def test_consumer_has_no_division(fixed_sass):
    """the ring position advances by counters, not by a division by the stage count per tile"""
    assert not [i for i in _consumer(fixed_sass) if "MUFU.RCP" in i]


def test_every_instantiation_divides_once(built):
    """every role of every fc_chain_kernel instantiation advances its ring position by counters: the one unsigned integer
    division left (I2F.U32.RP starts its sequence) is the entry code's count of the CTA's tiles"""
    chain = {name: text for name, text in sass_functions().items() if name.startswith("_ZN3bnm15fc_chain_kernel")}
    assert FIXED in chain and len(chain) == 8, sorted(chain)
    for name, sass in chain.items():
        assert sass.count("I2F.U32.RP") == 1, name
