"""CPU-side checks of where the fused FC kernels' grid-dependency wait sits in their sm_90a SASS (DESIGN.md 4.1, "Launch").

Every int8 C-engine launch is a programmatic dependent launch: its CTAs may start while the kernel before it on the stream is
still running, and only the producer's `griddepcontrol.wait` (SASS `ACQBULK`) keeps the image loads, and through them every
result store, behind that kernel.  What may run ahead of the wait is the prologue: barrier init, `setmaxnreg`, the bulk copy of
the weight image (`UBLKCP`, weights written at model build) and, in the fixed-shape kernel, the L2 prefetch of its first tiles
(`UTMAPF`).  `griddepcontrol.launch_dependents` is `PREEXIT`.

ptxas lays the consumer warpgroups' code out before the producer's, so "before the wait" cannot be read off the addresses.  The
checks walk the control-flow graph of the SASS instead: an edge from every instruction to the next one (none after an
unpredicated BRA, EXIT, RET or trap: ptxas places the bounded waits' trap code right in front of the producer's) and from
every branch or call to its target.  The wait is the one `ACQBULK`, reached either
unpredicated or through the branch right in front of it that skips exactly it -- the `wait_prior_grid` flag, clear only for
launches the caller declared independent (mode 2); the walk follows the wait, not that branch.  Then:

* "before the wait" is every instruction on a path from the entry to the `ACQBULK`: the producer lane's prologue;
* "behind the wait" is what every path from the entry reaches only through it (the `ACQBULK` dominates it).

Every tensor load of images (`UTMALDG`) must lie behind the wait, and nothing before it may store, reduce or atomically
update memory other than shared memory.  The consumers' stores are ordered by data instead: they store a tile only after its
full barrier completed, which takes the tensor loads behind the wait.  The float-input kernels' quantiser warps wait before
their first bulk copy of float rows; before their wait no global load or bulk copy may appear."""
import re

import pytest

from support import sass_functions

INT8_TMA = re.compile(r"_ZN3bnm(15fc_chain_kernelILi\d+ELi\d+ELb0E|17fc_emul_i8_kernel|14fc_topk_kernel)")
FLOAT_IN = re.compile(r"_ZN3bnm(15fc_chain_kernelILi\d+ELi\d+ELb1E|14fc_emul_kernel|17fc_engines_kernel)")
FIXED = "_ZN3bnm15fc_chain_kernelILi64ELi2ELb0ELi2ELi16ELb1EEEv14CUtensorMap_stNS_11ChainParamsE"

STORE = re.compile(r"^(STG|ST|RED|REDG|ATOM|ATOMG|UTMASTG|UTMAREDG|UBLKRED)\b")
GLOBAL_LOAD = re.compile(r"^(LDG|LD|UBLKCP|UTMALDG)\b")


def _opcode(ins):
    return re.sub(r"^@!?U?P\w+\s+", "", ins).split()[0]


def _parse(text):
    """[(address, instruction)] of one function"""
    return [(int(a, 16), i.strip()) for a, i in re.findall(r"/\*([0-9a-f]{4,})\*/\s+([^;]*);", text)]


class Cfg:
    """the control-flow graph of one function's SASS, by instruction index"""

    def __init__(self, ins):
        self.ins = ins
        at = {a: k for k, (a, _) in enumerate(ins)}
        self.succ = []
        for k, (_, i) in enumerate(ins):
            op, pred = _opcode(i), i.startswith("@")
            assert not op.startswith(("BRX", "JMX")), f"indirect branch, the walk cannot follow it: {i}"
            s = []
            if op.startswith(("BRA", "CALL", "JMP")):
                tgt = re.search(r"0x([0-9a-f]+)\s*$", i)
                assert tgt and int(tgt.group(1), 16) in at, i
                s.append(at[int(tgt.group(1), 16)])
            ends = op.startswith(("BRA", "JMP", "EXIT", "RET", "BPT.TRAP")) and not pred and not op.startswith("BRA.DIV")
            if not ends and k + 1 < len(ins):
                s.append(k + 1)
            self.succ.append(s)

    def reach(self, start, stop=None, succ=None):
        """instructions reachable from `start` without passing through `stop` (stop itself is included when reached)"""
        succ = succ or self.succ
        seen, todo = {start}, [start]
        while todo:
            k = todo.pop()
            if k == stop:
                continue
            for n in succ[k]:
                if n not in seen:
                    seen.add(n)
                    todo.append(n)
        return seen


def wait_split(text):
    """(instructions before the wait, instructions behind it, all instructions) of one kernel's SASS"""
    ins = _parse(text)
    assert len(ins) > 100, "function missing from the library"
    g = Cfg(ins)
    acq = [k for k, (_, i) in enumerate(ins) if _opcode(i) == "ACQBULK"]
    assert len(acq) == 1, f"{len(acq)} grid-dependency waits (ACQBULK), want exactly one"
    w = acq[0]
    # the branch that skips the wait when it is not wanted: right in front of it, to the instruction right after it.  Any
    # other path around the wait stays in the graph, and what it reaches is not behind the wait.
    succ = [list(s) for s in g.succ]
    if _opcode(ins[w - 1][1]).startswith("BRA") and w + 1 in succ[w - 1]:
        succ[w - 1] = [w]
    before = {k for k in g.reach(0, w, succ) if w in g.reach(k, w, succ)} - {w}
    unwaited = g.reach(0, w, succ) - {w}
    behind = set(range(len(ins))) - unwaited
    return [ins[k][1] for k in sorted(before)], [ins[k][1] for k in sorted(behind)], [i for _, i in ins]


def _kernels(pattern):
    got = {n: t for n, t in sass_functions().items() if pattern.match(n)}
    assert got, pattern.pattern
    return got


@pytest.fixture(scope="module")
def int8_kernels(built):
    k = _kernels(INT8_TMA)
    # the seven int8 rows of fc_chain_kernel, four fc_emul_i8_kernel<kN> and eight fc_topk_kernel<kN, kEmul>
    assert FIXED in k and len(k) == 7 + 4 + 8, sorted(k)
    return k


@pytest.fixture(scope="module")
def float_kernels(built):
    k = _kernels(FLOAT_IN)
    assert len(k) == 3, sorted(k)   # <64,1,float>, fc_emul_kernel, fc_engines_kernel
    return k


def test_int8_image_loads_lie_behind_the_one_wait(int8_kernels):
    """one ACQBULK; every UTMALDG only through it; before it the weight copy, the fixed-shape kernel's L2 prefetch, the early
    trigger, and no store, reduction or atomic"""
    for name, text in int8_kernels.items():
        before, behind, ins = wait_split(text)
        loads = [i for i in ins if _opcode(i).startswith("UTMALDG")]
        assert loads and all(i in behind for i in loads), (name, "a tensor load of images can run before the wait")
        assert not [i for i in before if GLOBAL_LOAD.match(_opcode(i)) and not _opcode(i).startswith("UBLKCP")], name
        assert [i for i in before if _opcode(i).startswith("UBLKCP")], (name, "the weight copy no longer runs ahead of the wait")
        prefetch = [i for i in ins if _opcode(i).startswith("UTMAPF")]
        if name == FIXED:
            assert prefetch and all(i in before for i in prefetch), (name, "the L2 prefetch of the first tiles")
        else:
            assert not prefetch, name
        assert not [i for i in before if STORE.match(_opcode(i))], (name, "a store ahead of the wait")
        assert sum(_opcode(i) == "PREEXIT" for i in ins) == 1 and [i for i in before if _opcode(i) == "PREEXIT"], \
            (name, "launch_dependents: once, ahead of the wait")


def test_float_quantiser_loads_lie_behind_its_wait(float_kernels):
    """the float-input rows: one ACQBULK, in the quantiser warps; no global load, bulk copy or store before it, and the bulk
    copies of float rows behind it"""
    for name, text in float_kernels.items():
        before, behind, ins = wait_split(text)
        assert not [i for i in before if GLOBAL_LOAD.match(_opcode(i)) or STORE.match(_opcode(i))], (name, before)
        assert not [i for i in ins if _opcode(i).startswith(("UTMALDG", "UTMAPF"))], name
        assert [i for i in behind if _opcode(i).startswith("UBLKCP")], (name, "no float-row bulk copy behind the wait")


def test_the_walk_sees_a_load_moved_ahead():
    """the analysis itself, on a hand-made function shaped like the producer branch: a load that moves in front of the wait,
    a second path around it and a deleted wait all fail"""
    good = """
        /*0000*/ ISETP.NE.AND P0, PT, RZ, UR4, PT ;
        /*0010*/ @P1 BRA 0x90 ;
        /*0020*/ UBLKCP.S.G [UR12], [UR10], UR7 ;
        /*0030*/ UTMAPF.L2.2D [UR10], [UR12] ;
        /*0040*/ @!P0 BRA 0x60 ;
        /*0050*/ ACQBULK ;
        /*0060*/ UTMALDG.2D [UR8], [UR18], desc[UR20] ;
        /*0070*/ @P2 BRA 0x60 ;
        /*0080*/ EXIT ;
        /*0090*/ STG.E [R2.64], R4 ;
        /*00a0*/ EXIT ;
    """ + "".join(f"        /*{0xb0 + 16 * k:04x}*/ NOP ;\n" for k in range(100))
    before, behind, _ = wait_split(good)
    assert before == ["ISETP.NE.AND P0, PT, RZ, UR4, PT", "@P1 BRA 0x90", "UBLKCP.S.G [UR12], [UR10], UR7",
                      "UTMAPF.L2.2D [UR10], [UR12]", "@!P0 BRA 0x60"]
    assert "UTMALDG.2D [UR8], [UR18], desc[UR20]" in behind and "STG.E [R2.64], R4" not in behind
    moved = good.replace("UTMAPF.L2.2D [UR10], [UR12]", "UTMALDG.2D [UR8], [UR18], desc[UR20]")
    before, _, _ = wait_split(moved)
    assert "UTMALDG.2D [UR8], [UR18], desc[UR20]" in before
    _, behind, _ = wait_split(good.replace("@P1 BRA 0x90", "@P1 BRA 0x60"))
    assert "UTMALDG.2D [UR8], [UR18], desc[UR20]" not in behind
    with pytest.raises(AssertionError, match="0 grid-dependency waits"):
        wait_split(good.replace("ACQBULK", "NOP"))
