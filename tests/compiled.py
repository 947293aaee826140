"""What the compiler made of the library: one `nvcc -cubin -Xptxas -v` compile of dgan_api.cu per test session, with the
flags of the library build, and one `cuobjdump -sass` of the result.  The CPU tests of ptxas's resource report and of
the SASS read it from here.  Skips when nvcc or cuobjdump is missing."""
import atexit
import functools
import os
import re
import shutil
import subprocess
import tempfile

import pytest


def _tool(name):
    path = shutil.which(name) or os.path.join(os.path.dirname(_nvcc()), name)
    if not os.path.exists(path):
        pytest.skip("%s not found" % name)
    return path


@functools.lru_cache(maxsize=None)
def _nvcc():
    nvcc = shutil.which(os.environ.get("NVCC", "nvcc"))
    if nvcc is None:
        pytest.skip("nvcc not found")
    return nvcc


@functools.lru_cache(maxsize=None)
def _compile():
    """(cubin path, ptxas log).  The cubin lives in a temporary directory removed at exit."""
    from defensegan_b200 import _native
    tmp = tempfile.mkdtemp(prefix="dgan_cubin_")
    atexit.register(shutil.rmtree, tmp, True)
    cubin = os.path.join(tmp, "dgan_api.cubin")
    flags = [f for f in _native.NVCC_FLAGS if f not in ("-shared", "-Xcompiler", "-fPIC")]
    res = subprocess.run([_nvcc()] + flags + ["-cubin", "-Xptxas", "-v", os.path.join(_native.CSRC_DIR, "dgan_api.cu"),
                          "-o", cubin], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert res.returncode == 0, res.stdout[-4000:]
    return cubin, res.stdout


def ptxas_log():
    return _compile()[1]


@functools.lru_cache(maxsize=None)
def resources():
    """{mangled function: (stack frame, spill store, spill load) bytes} from ptxas's report."""
    out, fn = {}, None
    for line in ptxas_log().splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            fn = m.group(1)
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and fn is not None:
            out[fn] = tuple(int(v) for v in m.groups())
            fn = None
    return out


@functools.lru_cache(maxsize=None)
def _sass_all():
    cubin = _compile()[0]
    res = subprocess.run([_tool("cuobjdump"), "-sass", cubin], stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                         text=True)
    assert res.returncode == 0, res.stdout[-4000:]
    funcs, name = {}, None
    for line in res.stdout.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1)
            funcs[name] = []
        elif name is not None:
            funcs[name].append(line)
    return funcs


def sass(kernel=""):
    """{mangled function: SASS lines} of the functions whose name contains `kernel`."""
    return {k: v for k, v in _sass_all().items() if kernel in k}


def demangle(names):
    """The demangled form of each mangled name, in order."""
    res = subprocess.run([_tool("cu++filt")], input="\n".join(names), stdout=subprocess.PIPE, text=True, check=True)
    return res.stdout.split("\n")[:len(names)]


def instructions(lines):
    """[(address, instruction text)] of a function's SASS lines."""
    out = []
    for line in lines:
        m = re.search(r"/\*([0-9a-f]{4,})\*/\s+(.*?);", line)
        if m:
            out.append((int(m.group(1), 16), m.group(2).strip()))
    return out


def tc_template(name):
    """(N, slots per round, k16 per op, epilogue, output bytes) of a mangled tc_bsgemm2_kernel instantiation."""
    m = re.search(r"tc_bsgemm2_kernelILi(\d+)ELi(\d+)ELi(\d+)ELi(\d+)E(6__half|f)", name)
    assert m, name
    n, maxb, ksub, epi, t = m.groups()
    return int(n), int(maxb), int(ksub), int(epi), 2 if t == "6__half" else 4


def is_stg(text):
    return re.search(r"(^|\s)STG\b|(^|\s)STG\.", text) is not None
