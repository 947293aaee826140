"""CPU test of the tensor-core kernel's SASS: the item epilogue does not wait for global memory.

The epilogue runs after the item's last MMA has retired, while the tensor pipe idles. What it reads besides the
accumulators - ReLU mask words, bias, image and weight pairs - is requested before it is needed, at the item's head or
one row of an accumulator ahead, so that its round trip to L2 overlaps MMAs or other epilogue work.

- TMA-store epilogues: no global load between the wait for the item's MMAs (WARPGROUP.DEPBAR.LE gsb0, 0x0) and the
  item's last TMA store. Each store is preceded by fence.proxy.async (MEMBAR.ALL.CTA), which waits for every load the
  warp has in flight, so a load there would be waited for at once.
- Final (last-layer forward) epilogues: every global load after that wait is followed by a store before its result is
  first read: the pairs of the next accumulator are in flight while the current one's outputs are written. The
  weighted CelebA kind (N = 48) is the exception: it has no registers for a second set of pairs."""
import re

import compiled

EPI_FINAL = {8, 9, 10, 11}
EPI_FINAL_TANH3_W = 11


def _regs(op):
    return {int(r) for r in re.findall(r"\bR(\d+)\b", op)}


def _ldg_dest(text):
    m = re.match(r"(?:@!?U?P\d+\s+)?LDG\S*\s+R(\d+),", text)
    if not m:
        return set()
    width = re.search(r"LDG\S*\.(64|128)\b", text)
    n = {None: 1, "64": 2, "128": 4}[width.group(1) if width else None]
    return set(range(int(m.group(1)), int(m.group(1)) + n))


def _sources(text):
    body = re.sub(r"^@!?U?P\w+\s+", "", text)
    parts = body.split(None, 1)
    if len(parts) < 2:
        return set()
    mnem, ops = parts
    ops = [o.strip() for o in ops.split(",")]
    if re.match(r"(STG|STS|ST|RED|ATOM)\b", mnem):
        return set().union(*(_regs(o) for o in ops))
    return set().union(*(_regs(o) for o in ops[1:])) if len(ops) > 1 else set()


def _is_ldg(text):
    return re.search(r"(^|\s)LDG\b|(^|\s)LDG\.", text) is not None


def tma_epilogue_loads(ins):
    """Global loads between each wait for all MMAs and the last TMA store after it."""
    bad = []
    stores = [a for a, t in ins if "UTMASTG" in t]
    for d in (a for a, t in ins if "WARPGROUP.DEPBAR.LE gsb0, 0x0" in t):
        after = [s for s in stores if s > d]
        assert after, "no TMA store after the wait at 0x%x" % d
        hi = max(after)
        bad += ["%04x %s" % (a, t) for a, t in ins if d < a <= hi and _is_ldg(t)]
    return bad


def final_loads_used_before_a_store(ins):
    """Global loads after the wait for all MMAs whose result is read before any store issues."""
    bad = []
    d = min(a for a, t in ins if "WARPGROUP.DEPBAR.LE gsb0, 0x0" in t)
    # the consumers' item loop ends at the first branch back to before the wait (the producer's code follows)
    back = []
    for a, t in ins:
        m = re.search(r"\bBRA\S*\s+(?:\S+,\s*)?0x([0-9a-f]+)", t)
        if m and a > d > int(m.group(1), 16):
            back.append(a)
    assert back, "no item loop around the wait at 0x%x" % d
    hi = min(back)
    for i, (a, t) in enumerate(ins):
        if not d < a <= hi or not _is_ldg(t):
            continue
        dest = _ldg_dest(t)
        for b, u in ins[i + 1:]:
            if compiled.is_stg(u):
                break
            if dest & _sources(u):
                bad.append("%04x %s  (read at %04x by %s)" % (a, t, b, u))
                break
            if dest and _ldg_dest(u) >= dest:      # overwritten by another load before any read
                break
    return bad


def test_epilogue_does_not_wait_for_global_memory():
    funcs = compiled.sass("tc_bsgemm2_kernel")
    assert len(funcs) >= 20, "too few tc_bsgemm2_kernel instantiations in the SASS: %d" % len(funcs)
    n_tma = n_final = 0
    for name, lines in funcs.items():
        n, maxb, ksub, epi, out_bytes = compiled.tc_template(name)
        ins = compiled.instructions(lines)
        if out_bytes == 2 and n >= 64 and epi not in EPI_FINAL:
            n_tma += 1
            bad = tma_epilogue_loads(ins)
            assert not bad, (name, "global load in the TMA-store epilogue", bad)
        elif epi in EPI_FINAL and not (epi == EPI_FINAL_TANH3_W and n > 32):
            n_final += 1
            bad = final_loads_used_before_a_store(ins)
            assert not bad, (name, "an epilogue load is waited for before the previous row's stores", bad)
    assert n_tma >= 15 and n_final >= 5, (n_tma, n_final)
