"""CPU test of the tensor-core kernel's SASS: a round issues only its real ops, and still as one wgmma group.

With 2 or 4 accumulator slots and 64-channel ops the consumers branch on a round's active set to a straight-line variant
that issues the MMAs of those accumulators alone (`tc2_mma_round`). Every variant must end one hardware wgmma group with
its last HGMMA (`gsb0`) and no earlier one, and the `wgmma.wait_group 1` after the round must follow before any other
MMA is issued. Otherwise the round's wait drains the tensor pipe: a guard predicate per MMA, for one, makes ptxas branch
around each HGMMA and close a group at every one. The 1- and 8-slot and the narrow instantiations keep the fixed round
and are held to the same group rule."""
import re

import compiled

_BRANCH = re.compile(r"\bBR[AX]\b|\bBRA\.|\bEXIT\b|\bRET\b")
_WAIT1 = "WARPGROUP.DEPBAR.LE gsb0, 0x1"


def _blocks(ins):
    """Straight-line runs of HGMMAs: split at every branch, warpgroup arrive and wgmma wait."""
    blocks, cur = [], []
    for a, t in ins:
        if "HGMMA" in t:
            cur.append((a, t))
        elif _BRANCH.search(t) or "WARPGROUP" in t:
            if cur:
                blocks.append(cur)
            cur = []
    if cur:
        blocks.append(cur)
    return blocks


def _next_wgmma_event(ins, start):
    """From the instruction after address `start`, follow fall-through and unconditional branches to the first
    instruction that issues or waits for MMAs."""
    at = {a: i for i, (a, _) in enumerate(ins)}
    i, seen = at[start] + 1, set()
    while i < len(ins) and i not in seen:
        seen.add(i)
        a, t = ins[i]
        if "HGMMA" in t or "WARPGROUP" in t:
            return t
        m = re.match(r"BRA\s+(?:`\()?0x([0-9a-f]+)", t)           # unconditional branch (no predicate)
        if m:
            i = at[int(m.group(1), 16)]
            continue
        i += 1
    return None


def test_each_round_variant_is_one_wgmma_group():
    funcs = compiled.sass("tc_bsgemm2_kernel")
    assert len(funcs) >= 20, "too few tc_bsgemm2_kernel instantiations in the SASS: %d" % len(funcs)
    for name, lines in funcs.items():
        n, maxb, ksub, _, _ = compiled.tc_template(name)
        ins = compiled.instructions(lines)
        blocks = _blocks(ins)
        assert blocks, name
        for b in blocks:
            closing = [t for _, t in b if "gsb0" in t]
            assert closing == [b[-1][1]], (name, "an HGMMA other than the last of its variant ends a wgmma group",
                                           ["%04x %s" % x for x in b])
            assert _WAIT1 in (_next_wgmma_event(ins, b[-1][0]) or ""), (name, "variant at 0x%x not followed by "
                                                                          "wait_group 1" % b[0][0])
        if 1 < maxb <= 4 and ksub == 4:
            # one variant per non-empty set of accumulators: 2^MAXB - 1 of them, each accumulator in half of the sets
            assert len(blocks) == 2 ** maxb - 1, (name, len(blocks))
            assert sum(len(b) for b in blocks) == ksub * maxb * 2 ** (maxb - 1), (name, [len(b) for b in blocks])
            waits = [t for _, t in ins if _WAIT1 in t]
            assert 1 <= len(waits) <= len(blocks), (name, len(waits))
