"""The tile-ring rule behind the fused FC kernel's barriers, checked on a discrete-event model with arbitrary latencies: no parity
wait may pass before its tile has landed, and every tile completes.  CPU only.

The rule: a shape with `slots` tile slots on `stages` ring stages needs at least slots / gcd(slots, stages) barriers per stage (the
latest same-stage tile that is certain to have landed when the waiter reaches tile j is that many ring rounds back).  In fc_wgmma.cu
every consumer warpgroup waits for every tile of its pipe in order -- in the model's terms one slot per pipe -- so one "full"
barrier per stage suffices for any stage count.  The model covers this rule only: it does not replay the kernel's two consumer
warpgroups per tile, its eight-arrival "empty" barrier or the producer's tile-order refill across two pipes.
"""
import re
from math import gcd
from pathlib import Path

import pytest

from ring_protocol_sim import Violation, simulate

# (waiters, slots per waiter, ring stages of a pipe): every stage count a ring can have (kMaxStages = 8); plans use two to six
SHIPPED = [(1, 1, stages) for stages in range(1, 9)]
FAST_CHAIN = dict(mma=(0.01, 0.05), epi=(0.01, 0.08), load_lat=(0.3, 4.0), slow_load=(0.05, 20.0))   # tiny model, slow loads


def kernel_full_bars():
    src = (Path(__file__).resolve().parents[1] / "bitnetmcu_b200" / "csrc" / "fc_wgmma.cu").read_text()
    decl = re.search(r"uint64_t bar_full\[([^\]]+)\](\[[^\]]+\])?", src)
    assert decl.group(1) == "kMaxStages" and decl.group(2) is None   # one barrier per stage
    return 1


@pytest.mark.parametrize("shape", SHIPPED)
def test_shipped_shapes_are_safe_with_the_kernels_barrier_count(shape):
    n_wg, slots, stages = shape
    bars = kernel_full_bars()
    assert bars >= n_wg * slots // gcd(n_wg * slots, stages)
    for seed in range(60):
        simulate(n_wg, slots, stages, full_bars=bars, seed=seed)
        simulate(n_wg, slots, stages, full_bars=bars, seed=seed, **FAST_CHAIN)


def test_two_barriers_per_stage_are_only_safe_while_slots_do_not_outnumber_stages():
    # slots <= stages: the wait for tile i + 2 stages comes after its slot's previous tile, whose load was requested after tile i landed
    for seed in range(60):
        simulate(3, 2, 6, full_bars=2, seed=seed, **FAST_CHAIN)
    # the development shape that trapped on the GPU (eight slots on six stages, tiny model, overlapped launches = slow loads)
    failures = 0
    for seed in range(60):
        try:
            simulate(4, 2, 6, full_bars=2, seed=seed, **FAST_CHAIN)
        except Violation:
            failures += 1
    assert failures > 0
    # ... and what the gather launches and the shared-memory-activation form would have risked with a very late load
    with pytest.raises(Violation):
        for seed in range(400):
            simulate(3, 1, 2, full_bars=2, seed=seed, **FAST_CHAIN)


def test_barriers_needed_is_slots_over_gcd():
    slow = dict(FAST_CHAIN, slow_load=(0.05, 40.0))
    for n_wg, slots, stages in [(3, 2, 5), (4, 1, 5), (3, 2, 4), (4, 2, 7), (4, 2, 6), (3, 2, 3)]:
        need = n_wg * slots // gcd(n_wg * slots, stages)
        for seed in range(40):   # enough barriers: never a violation
            simulate(n_wg, slots, stages, full_bars=need, seed=seed, n_tiles=90, **slow)
        if need > 1:             # too few: the adversarial latencies find it
            with pytest.raises(Violation):
                for seed in range(300):
                    simulate(n_wg, slots, stages, full_bars=max(1, need // 2), seed=seed, n_tiles=90, **slow)
