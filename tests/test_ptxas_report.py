"""CPU test of what the compiler made of the tensor-core kernel: every tc_bsgemm2_kernel instantiation issues its wgmma
without compiler-inserted serialisation (ptxas C7520) and keeps accumulators and epilogue in registers (no spills)."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _ptxas_report(tmp_path):
    from defensegan_b200 import _native
    nvcc = shutil.which(os.environ.get("NVCC", "nvcc"))
    if nvcc is None:
        pytest.skip("nvcc not found")
    flags = [f for f in _native.NVCC_FLAGS if f not in ("-shared", "-Xcompiler", "-fPIC")]
    cmd = [nvcc] + flags + ["-cubin", "-Xptxas", "-v", os.path.join(_native.CSRC_DIR, "dgan_api.cu"),
                            "-o", str(tmp_path / "dgan_api.cubin")]
    res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert res.returncode == 0, res.stdout[-4000:]
    return res.stdout


def test_tensor_core_kernels_are_not_serialised_and_do_not_spill(tmp_path):
    log = _ptxas_report(tmp_path)
    serialised = [l for l in log.splitlines() if "C7520" in l and "tc_bsgemm2_kernel" in l]
    assert not serialised, serialised
    spills, fn = {}, None
    for line in log.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            fn = m.group(1)
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and fn is not None and "tc_bsgemm2_kernel" in fn:
            spills[fn] = (int(m.group(1)), int(m.group(2)))
            fn = None
    assert len(spills) >= 20, "ptxas reported too few tc_bsgemm2_kernel instantiations: %d" % len(spills)
    bad = {k: v for k, v in spills.items() if v != (0, 0)}
    assert not bad, bad
