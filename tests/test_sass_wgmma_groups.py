"""CPU test of the tensor-core kernel's SASS: its wgmma waits count the MMA groups that the hardware tracks.

ptxas ends a hardware wgmma group in every iteration of the run-time round loop. A commit that does not directly follow
an MMA therefore becomes an empty HGMMA (destination RZ). When that happens, the `wgmma.wait_group 1` after it waits for
every real MMA, and the tensor pipe drains at every step boundary."""
import re

import compiled


def test_every_wgmma_group_holds_mmas():
    funcs = compiled.sass("tc_bsgemm2_kernel")
    assert len(funcs) >= 20, "too few tc_bsgemm2_kernel instantiations in the SASS: %d" % len(funcs)
    for name, lines in funcs.items():
        empty = [l.strip() for l in lines if re.search(r"\bHGMMA\.\S+ RZ,", l)]
        assert not empty, (name, empty)
        assert any("WARPGROUP.DEPBAR.LE gsb0, 0x1" in l for l in lines), name
