"""Discrete-event model of a per-CTA image-tile ring protocol (the general form of bitnetmcu_b200/csrc/fc_wgmma.cu's ring): the ring with
its "tile landed" mbarriers, the per-slot MMA / ready hand-off between a warpgroup's issuer warp and its epilogue warps, and the
refill of a stage by the warp that sees the tile's layer-1 MMAs complete.

TEST INFRASTRUCTURE: it exists to check one property the hardware will not check for us.  `mbarrier.try_wait.parity(P)` succeeds
when the barrier's CURRENT phase has parity != P -- so a wait that starts before the barrier's previous phase has completed
returns at once, on data that has not landed.  The kernel spreads the ring rounds of a stage over `full_bars` barriers
(round u -> barrier u % full_bars, parity (u / full_bars) & 1); the model asserts that no "tile landed" wait ever passes before
its tile has landed, for arbitrary load latencies and step durations, and that every tile completes (no deadlock).
"""
import heapq
import random


class Violation(Exception):
    pass


def simulate(n_wg, slots, n_stages, full_bars, n_tiles=60, n_layers=4, seed=0, load_lat=(0.3, 3.0), slow_load=(0.02, 25.0),
             mma=(0.05, 0.4), epi=(0.05, 1.2)):
    """One CTA processing n_tiles tiles.  Durations are drawn uniformly from the given ranges (us); with probability slow_load[0]
    a load takes slow_load[1] us more.  Raises Violation on an early pass of a "tile landed" wait or on a deadlock."""
    rng = random.Random(seed)
    n_virt = n_wg * slots
    now = [0.0]
    events = []   # (time, seq, fn)
    seq = [0]

    def at(t, fn):
        seq[0] += 1
        heapq.heappush(events, (t, seq[0], fn))

    completed = [[0] * n_stages for _ in range(full_bars)]   # completed phases per barrier
    landed = [False] * n_tiles
    mma_done = {}     # (tile, layer) -> True
    ready = {}        # (tile, layer): epilogue of that layer finished (operand written / accumulator drained)
    finished = [False] * n_tiles

    def issue_load(i):
        lat = rng.uniform(*load_lat) + (slow_load[1] if rng.random() < slow_load[0] else 0.0)

        def land():
            landed[i] = True
            completed[(i // n_stages) % full_bars][i % n_stages] += 1
        at(now[0] + lat, land)

    def landed_wait_passes(i):
        u = i // n_stages
        parity = (u // full_bars) & 1
        return (completed[u % full_bars][i % n_stages] & 1) != parity

    # processes as generators yielding predicates ("resume when this holds") or ("sleep", dt)
    def issuer(g):
        for r in range((n_tiles + n_virt - 1) // n_virt):
            for l in range(n_layers):
                for q in range(slots):
                    i = r * n_virt + g * slots + q
                    if i >= n_tiles:
                        continue
                    if r != 0 or l != 0:   # previous epilogue step of this slot
                        prev = (i, l - 1) if l > 0 else (i - n_virt, n_layers - 1)
                        yield lambda prev=prev: ready.get(prev, False)
                    if l == 0:
                        yield lambda i=i: landed_wait_passes(i)
                        if not landed[i]:
                            raise Violation(f"tile {i}: 'landed' wait passed before the load completed "
                                            f"(slots {n_virt}, stages {n_stages}, barriers per stage {full_bars})")
                    d = rng.uniform(*mma)
                    at(now[0] + d, lambda key=(i, l): mma_done.__setitem__(key, True))

    def epilogue(g):
        for r in range((n_tiles + n_virt - 1) // n_virt):
            for l in range(n_layers):
                for q in range(slots):
                    i = r * n_virt + g * slots + q
                    if i >= n_tiles:
                        continue
                    yield lambda key=(i, l): mma_done.get(key, False)
                    if l == 0 and i + n_stages < n_tiles:
                        issue_load(i + n_stages)   # the stage is free: refill it
                    yield ("sleep", rng.uniform(*epi))
                    ready[(i, l)] = True
                    if l == n_layers - 1:
                        finished[i] = True

    procs = [issuer(g) for g in range(n_wg)] + [epilogue(g) for g in range(n_wg)]
    waiting = {}   # proc -> predicate
    for i in range(min(n_stages, n_tiles)):
        issue_load(i)

    def step(p):
        """run process p until it blocks; returns False when it has ended"""
        while True:
            try:
                w = next(p)
            except StopIteration:
                waiting.pop(p, None)
                return False
            if isinstance(w, tuple):   # sleep
                waiting[p] = None
                at(now[0] + w[1], lambda p=p: wake(p))
                return True
            if w():
                continue
            waiting[p] = w
            return True

    def wake(p):
        waiting.pop(p, None)
        step(p)

    alive = set()
    for p in procs:
        if step(p):
            alive.add(p)
    while True:
        progressed = True
        while progressed:   # re-evaluate blocked predicates until a fixed point
            progressed = False
            for p, w in list(waiting.items()):
                if w is not None and w():
                    waiting.pop(p)
                    step(p)
                    progressed = True
        if not events:
            break
        t, _, fn = heapq.heappop(events)
        now[0] = t
        fn()
    if not all(finished):
        raise Violation(f"deadlock: {sum(finished)} of {n_tiles} tiles finished (slots {n_virt}, stages {n_stages}, "
                        f"barriers per stage {full_bars})")
    return now[0]
