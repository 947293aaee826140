"""CPU test of the tensor-core kernel's SASS: the consumers' step loop holds no global load.

A step's MMA record reaches the consumers through shared memory, on the barrier that delivers the step's operands. A
global load inside the step loop puts a round trip to L2 between two steps' MMAs: ptxas moves a loaded record to uniform
registers as soon as it is requested, so the warp waits there however far ahead the load was meant to run.

The step loop is found by its shape, not by its place in the code: it is the smallest loop (backward branch and its
target) that holds every HGMMA and the last wait on a barrier before the first HGMMA, which is the consumers' wait for
the step's operands. The loop around it is the item loop, whose head and epilogue may load from global memory."""
import re

import compiled


def test_no_global_load_in_the_step_loop():
    funcs = compiled.sass("tc_bsgemm2_kernel")
    assert len(funcs) >= 20, "too few tc_bsgemm2_kernel instantiations in the SASS: %d" % len(funcs)
    for name, lines in funcs.items():
        ins = compiled.instructions(lines)
        mma = [a for a, t in ins if "HGMMA" in t]
        waits = [a for a, t in ins if "SYNCS.PHASECHK" in t and a < min(mma)]
        assert mma and waits, name
        operand_wait = max(waits)
        loops = []
        for a, t in ins:
            m = re.search(r"\bBRA\S*\s+(?:\S+,\s*)?0x([0-9a-f]+)", t)
            if m and int(m.group(1), 16) <= operand_wait and a >= max(mma):
                loops.append((a - int(m.group(1), 16), int(m.group(1), 16), a))
        assert len(loops) >= 2, (name, "expected the step loop inside the item loop", loops)
        _, lo, hi = min(loops)
        loads = ["%04x %s" % (a, t) for a, t in ins if lo <= a <= hi and re.search(r"\bLDG\b|\bLDG\.", t)]
        assert not loads, (name, "global load between 0x%x and 0x%x, the consumers' step loop" % (lo, hi), loads)
