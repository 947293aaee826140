"""CPU test of the tensor-core kernel's SASS: its wgmma waits count the MMA groups that the hardware tracks.

ptxas ends a hardware wgmma group in every iteration of the run-time round loop. A commit that does not directly follow
an MMA therefore becomes an empty HGMMA (destination RZ). When that happens, the `wgmma.wait_group 1` after it waits for
every real MMA, and the tensor pipe drains at every step boundary."""
import os
import re
import shutil
import subprocess

import pytest


def _sass(tmp_path):
    from defensegan_b200 import _native
    nvcc = shutil.which(os.environ.get("NVCC", "nvcc"))
    if nvcc is None:
        pytest.skip("nvcc not found")
    cuobjdump = shutil.which("cuobjdump") or os.path.join(os.path.dirname(nvcc), "cuobjdump")
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not found")
    flags = [f for f in _native.NVCC_FLAGS if f not in ("-shared", "-Xcompiler", "-fPIC")]
    cubin = str(tmp_path / "dgan_api.cubin")
    res = subprocess.run([nvcc] + flags + ["-cubin", os.path.join(_native.CSRC_DIR, "dgan_api.cu"), "-o", cubin],
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert res.returncode == 0, res.stdout[-4000:]
    res = subprocess.run([cuobjdump, "-sass", cubin], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert res.returncode == 0, res.stdout[-4000:]
    funcs, name = {}, None
    for line in res.stdout.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1)
            funcs[name] = []
        elif name is not None:
            funcs[name].append(line)
    return {k: v for k, v in funcs.items() if "tc_bsgemm2_kernel" in k}


def test_every_wgmma_group_holds_mmas(tmp_path):
    funcs = _sass(tmp_path)
    assert len(funcs) >= 20, "too few tc_bsgemm2_kernel instantiations in the SASS: %d" % len(funcs)
    for name, lines in funcs.items():
        empty = [l.strip() for l in lines if re.search(r"\bHGMMA\.\S+ RZ,", l)]
        assert not empty, (name, empty)
        assert any("WARPGROUP.DEPBAR.LE gsb0, 0x1" in l for l in lines), name
