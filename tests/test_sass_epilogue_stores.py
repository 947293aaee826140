"""CPU test of the tensor-core kernel's SASS: how the TMA-store epilogues write their output.

Every 64-column unit of an fp16 output is staged in shared memory and written by a TMA store, after a
fence.proxy.async (MEMBAR.ALL.CTA) that orders the staging writes before the store's reads.

- No global store between the wait for the item's MMAs (WARPGROUP.DEPBAR.LE gsb0, 0x0) and the item's last fence: the
  ReLU kinds hold their mask words in registers and store them after the item's last TMA store, so that no fence has a
  global store of the same item ahead of it.
- The staging buffer is written with stmatrix (STSM, four 8x8 matrices per instruction), not with scalar STS."""
import re

import compiled

EPI_FINAL = {8, 9, 10, 11}


def _mnem(text):
    return re.sub(r"^@!?U?P\w+\s+", "", text).split()[0]


def epilogue_spans(ins):
    """(wait, last fence, last TMA store) of each wait for all MMAs."""
    spans = []
    stores = [a for a, t in ins if "UTMASTG" in t]
    for d in (a for a, t in ins if "WARPGROUP.DEPBAR.LE gsb0, 0x0" in t):
        after = [s for s in stores if s > d]
        assert after, "no TMA store after the wait at 0x%x" % d
        hi = max(after)
        fences = [a for a, t in ins if d < a < hi and _mnem(t) == "MEMBAR.ALL.CTA"]
        assert fences, "no fence before the TMA stores after the wait at 0x%x" % d
        spans.append((d, max(fences), hi))
    return spans


def test_tma_epilogue_stores():
    funcs = compiled.sass("tc_bsgemm2_kernel")
    n_tma = 0
    for name, lines in funcs.items():
        n, maxb, ksub, epi, out_bytes = compiled.tc_template(name)
        if not (out_bytes == 2 and n >= 64 and epi not in EPI_FINAL):
            continue
        n_tma += 1
        ins = compiled.instructions(lines)
        for d, fence, hi in epilogue_spans(ins):
            stg = ["%04x %s" % (a, t) for a, t in ins if d < a < fence and compiled.is_stg(t)]
            assert not stg, (name, "global store ahead of the item's last fence.proxy.async", stg)
            ops = [_mnem(t) for a, t in ins if d < a <= hi]
            assert any(o.startswith("STSM") for o in ops), (name, "the staging buffer is not written with stmatrix")
            sts = [o for o in ops if o == "STS" or o.startswith("STS.")]
            assert not sts, (name, "scalar shared-memory stores in the epilogue", sts)
    assert n_tma >= 15, n_tma
