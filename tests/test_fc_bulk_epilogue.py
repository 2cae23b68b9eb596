"""The fixed-shape FC kernel's bulk-copy epilogue (fc_chain_kernel<64,2,2,16,fixed>, FC 4bitsym-64): every consumer warp stages
its 16 rows of logits and labels in shared memory and writes each block to HBM with one bulk async copy; the last tile's
partial block moves its 16-byte multiple that way and the rest with word stores.  Launches whose logits or labels are not
16-byte aligned take the plan's general 16-wide row instead.  CPU: the SASS of the fixed row.  GPU: bit-exact against the
oracle at every batch-size edge, with and without labels or logits, into buffers at 16-byte and 8-byte aligned offsets, and
nothing written past row n."""
import re

import numpy as np
import pytest

from conftest import load_model
from support import engine, instructions, lib, plan_line, sass_functions, verbose_engine  # noqa: F401

FIXED = "_ZN3bnm15fc_chain_kernelILi64ELi2ELb0ELi2ELi16ELb1EEEv14CUtensorMap_stNS_11ChainParamsE"
SENTINEL = -0x2BAD


def _consumer(ins):
    lo = next(k for k, i in enumerate(ins) if i.startswith("USETMAXREG.TRY_ALLOC"))
    hi = next(k for k, i in enumerate(ins) if i.startswith("USETMAXREG.DEALLOC"))
    return ins[lo:hi]


def test_fixed_epilogue_stores_by_bulk_copy(built):
    """the consumer code copies logits and labels out with UBLKCP and has no 64-bit global stores of logits"""
    ins = _consumer(instructions(sass_functions().get(FIXED, "")))
    assert [i for i in ins if "UBLKCP" in i], "no bulk copy in the fixed-shape consumer code"
    assert not [i for i in ins if re.match(r"(@\S+\s+)?STG\.E\.64\b", i)], "64-bit global stores left in the fixed-shape epilogue"


@pytest.fixture(scope="module")
def fc(lib, oracle):
    from bitnetmcu_b200 import _lib
    m = load_model("fc")
    e = engine(m, _lib.PATH_TCGEN05)
    yield m, e
    e.close()


@pytest.mark.gpu
def test_plan_takes_fixed_row(lib, capfd, monkeypatch):
    """FC 4bitsym-64 runs the fixed-shape row; its staging buffers leave two stages per pipe"""
    from bitnetmcu_b200 import _lib
    e, err = verbose_engine(capfd, monkeypatch, lambda: engine(load_model("fc"), _lib.PATH_TCGEN05))
    e.close()
    plan = plan_line(err)
    assert plan and "fc_chain_kernel<64,2,2,16,fixed>" in plan and "2 pipes x 2 stages" in plan, err


def _run(fc, oracle, n, logits_off, labels_off, with_logits=True, with_labels=True, seed=0):
    """n images into logits / labels views that start logits_off / labels_off 4-byte elements into their allocations"""
    import torch
    m, e = fc
    rng = np.random.default_rng(seed + n)
    imgs = rng.integers(-128, 128, size=(n, e.img_bytes)).astype(np.int8)
    want_lo, want_la = oracle.infer(m, imgs)
    c = e.n_classes
    lo_buf = torch.full(((n + 16) * c + logits_off,), SENTINEL, dtype=torch.int32, device="cuda")
    la_buf = torch.full((n + 16 + labels_off,), SENTINEL, dtype=torch.int32, device="cuda")
    lo = lo_buf[logits_off:logits_off + n * c].view(n, c) if with_logits else None
    la = la_buf[labels_off:labels_off + n] if with_labels else None
    e.infer_device(torch.from_numpy(imgs).cuda(), lo, la)
    torch.cuda.synchronize()
    got_lo, got_la = lo_buf.cpu().numpy(), la_buf.cpu().numpy()
    tag = (n, logits_off * 4, labels_off * 4, with_logits, with_labels)
    if with_logits:
        g = got_lo[logits_off:logits_off + n * c].reshape(n, c)
        bad = np.flatnonzero((g != want_lo).any(axis=1))
        assert bad.size == 0, (tag, "logits rows wrong", bad[:8].tolist())
    assert (got_lo[:logits_off] == SENTINEL).all() and (got_lo[logits_off + (n * c if with_logits else 0):] == SENTINEL).all(), \
        (tag, "logits written outside rows :n")
    if with_labels:
        bad = np.flatnonzero(got_la[labels_off:labels_off + n].astype(np.uint32) != want_la)
        assert bad.size == 0, (tag, "labels wrong", bad[:8].tolist())
    assert (got_la[:labels_off] == SENTINEL).all() and (got_la[labels_off + (n if with_labels else 0):] == SENTINEL).all(), \
        (tag, "labels written outside rows :n")


# 1001 and 1000: the last warp block holds 9 / 8 rows; 132 x 128 x 5 + 23 several tiles per CTA (every warp reuses its buffer)
SIZES = [1, 15, 16, 17, 127, 128, 129, 1000, 1001, 132 * 128 * 5 + 23]


@pytest.mark.gpu
@pytest.mark.parametrize("n", SIZES)
def test_fixed_row_batch_edges(fc, oracle, n):
    _run(fc, oracle, n, 0, 0)
    _run(fc, oracle, n, 0, 0, with_labels=False)
    _run(fc, oracle, n, 0, 0, with_logits=False)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [17, 1001, 132 * 128 * 5 + 23])
def test_fixed_row_16_byte_offsets(fc, oracle, n):
    """logits and labels 16 bytes into their allocations: 16-byte aligned, not aligned to a warp's 640-byte block"""
    _run(fc, oracle, n, 4, 4)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [17, 1001, 132 * 128 * 5 + 23])
@pytest.mark.parametrize("offs", [(2, 0), (0, 2), (2, 2)])
def test_8_byte_aligned_buffers_take_general_row(fc, oracle, n, offs):
    """logits or labels 8 bytes into their allocations: no bulk copy can write them, the general row does"""
    _run(fc, oracle, n, *offs)
