"""CPU tests of the C ABI that include/defensegan_b200.h declares: the C prototype of every entry point, frozen in one
table that a C99 compiler checks against the header; the ctypes argtypes and restype that the binding declares for each
of them; and the size and field offsets of every struct the binding mirrors."""
import ctypes
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STRUCTS = ["dgan_desc", "dgan_rec_params", "dgan_prune_point", "dgan_adam_params", "dgan_conv_op", "dgan_sparse_dev"]

# The C type of every entry point, as "return type (parameter types)".  A parameter keeps its name where the ctypes rule
# depends on it.
SIGNATURES = {
    "dgan_abi_version": "int (void)",
    "dgan_last_error": "const char* (void)",
    "dgan_num_weights": "int (const dgan_desc*)",
    "dgan_create": "int (dgan_handle*, const dgan_desc*, const float* const*, int, void*)",
    "dgan_destroy": "int (dgan_handle)",
    "dgan_workspace_bytes": "size_t (dgan_handle, int, int)",
    "dgan_reconstruct": "int (dgan_handle, const dgan_rec_params*, const float*, const float*, float*, float*, "
                        "int32_t*, void*, size_t, void*)",
    "dgan_sample_z0": "int (dgan_handle, uint64_t, uint64_t, int, float*, void*)",
    "dgan_forward": "int (dgan_handle, const float*, int, float*, void*, size_t, void*)",
    "dgan_loss_grad": "int (dgan_handle, const float*, int, int, const float*, float*, float*, float*, void*, size_t, "
                      "void*)",
    "dgan_vjp": "int (dgan_handle, const float*, int, const float*, float*, float*, void*, size_t, void*)",
    "dgan_jvp": "int (dgan_handle, const float*, int, const float*, float*, float*, void*, size_t, void*)",
    "dgan_last_launch_count": "int64_t (dgan_handle)",
    "dgan_last_enqueue_count": "int64_t (dgan_handle)",
    "dgan_macs_per_row": "int64_t (dgan_handle)",
    "dgan_profile_enable": "int (dgan_handle, int)",
    "dgan_profile_num_kinds": "int (dgan_handle)",
    "dgan_profile_kind_name": "const char* (dgan_handle, int)",
    "dgan_profile_read": "int (dgan_handle, int, double*, int64_t*, double*)",
    "dgan_workspace_bytes_weighted": "size_t (dgan_handle, int, int)",
    "dgan_reconstruct_weighted": "int (dgan_handle, const dgan_rec_params*, const float*, const float*, const float*, "
                                 "float*, float*, int32_t*, void*, size_t, void*)",
    "dgan_loss_grad_weighted": "int (dgan_handle, const float*, const float*, int, int, const float*, float*, float*, "
                               "float*, void*, size_t, void*)",
    "dgan_workspace_bytes_measured": "size_t (dgan_handle, int, int, int)",
    "dgan_reconstruct_measured": "int (dgan_handle, const dgan_rec_params*, const float*, int, const float*, "
                                 "const float*, float*, float*, int32_t*, void*, size_t, void*)",
    "dgan_loss_grad_measured": "int (dgan_handle, const float*, int, const float*, int, int, const float*, float*, "
                               "float*, float*, void*, size_t, void*)",
    "dgan_workspace_bytes_measured_csr": "size_t (dgan_handle, int, int, int, int)",
    "dgan_reconstruct_measured_csr": "int (dgan_handle, const dgan_rec_params*, const int32_t*, const int32_t*, "
                                     "const float*, int, int, const float*, const float*, float*, float*, int32_t*, "
                                     "void*, size_t, void*)",
    "dgan_loss_grad_measured_csr": "int (dgan_handle, const int32_t*, const int32_t*, const float*, int, int, "
                                   "const float*, int, int, const float*, float*, float*, float*, void*, size_t, "
                                   "void*)",
    "dgan_workspace_bytes_pruned": "size_t (dgan_handle, int, int, const dgan_prune_point*, int, int)",
    "dgan_reconstruct_pruned": "int (dgan_handle, const dgan_rec_params*, const dgan_prune_point*, int, const float*, "
                               "const float*, const float*, float*, float*, int32_t*, void*, size_t, void*)",
    "dgan_workspace_bytes_measured_pruned": "size_t (dgan_handle, int, int, int, int, const dgan_prune_point*, int)",
    "dgan_reconstruct_measured_pruned": "int (dgan_handle, const dgan_rec_params*, const dgan_prune_point*, int, "
                                        "const float*, int, const float*, const float*, float*, float*, int32_t*, "
                                        "void*, size_t, void*)",
    "dgan_reconstruct_measured_csr_pruned": "int (dgan_handle, const dgan_rec_params*, const dgan_prune_point*, int, "
                                            "const int32_t*, const int32_t*, const float*, int, int, const float*, "
                                            "const float*, float*, float*, int32_t*, void*, size_t, void*)",
    "dgan_workspace_bytes_adam": "size_t (dgan_handle, int, int, int, const dgan_prune_point*, int)",
    "dgan_workspace_bytes_measured_adam": "size_t (dgan_handle, int, int, int, int, const dgan_prune_point*, int)",
    "dgan_reconstruct_adam": "int (dgan_handle, const dgan_rec_params*, const dgan_adam_params*, "
                             "const dgan_prune_point*, int, const float*, const float*, const float*, float*, float*, "
                             "int32_t*, void*, size_t, void*)",
    "dgan_reconstruct_measured_adam": "int (dgan_handle, const dgan_rec_params*, const dgan_adam_params*, "
                                      "const dgan_prune_point*, int, const float*, int, const float*, const float*, "
                                      "float*, float*, int32_t*, void*, size_t, void*)",
    "dgan_reconstruct_measured_csr_adam": "int (dgan_handle, const dgan_rec_params*, const dgan_adam_params*, "
                                          "const dgan_prune_point*, int, const int32_t*, const int32_t*, "
                                          "const float*, int, int, const float*, const float*, float*, float*, "
                                          "int32_t*, void*, size_t, void*)",
    "dgan_reconstruct_huber": "int (dgan_handle, const dgan_rec_params*, const dgan_adam_params*, float, "
                              "const dgan_prune_point*, int, const float*, const float*, const float*, float*, "
                              "float*, int32_t*, void*, size_t, void*)",
    "dgan_reconstruct_measured_huber": "int (dgan_handle, const dgan_rec_params*, const dgan_adam_params*, float, "
                                       "const dgan_prune_point*, int, const float*, int, const float*, const float*, "
                                       "float*, float*, int32_t*, void*, size_t, void*)",
    "dgan_reconstruct_measured_csr_huber": "int (dgan_handle, const dgan_rec_params*, const dgan_adam_params*, float, "
                                           "const dgan_prune_point*, int, const int32_t*, const int32_t*, "
                                           "const float*, int, int, const float*, const float*, float*, float*, "
                                           "int32_t*, void*, size_t, void*)",
    "dgan_loss_grad_huber": "int (dgan_handle, float, const float*, const float*, int, int, const float*, float*, "
                            "float*, float*, void*, size_t, void*)",
    "dgan_loss_grad_measured_huber": "int (dgan_handle, float, const float*, int, const float*, int, int, "
                                     "const float*, float*, float*, float*, void*, size_t, void*)",
    "dgan_loss_grad_measured_csr_huber": "int (dgan_handle, float, const int32_t*, const int32_t*, const float*, int, "
                                         "int, const float*, int, int, const float*, float*, float*, float*, void*, "
                                         "size_t, void*)",
    "dgan_conv_op_m": "int (dgan_handle, const dgan_conv_op*)",
    "dgan_workspace_bytes_measured_conv": "size_t (dgan_handle, int, int, const dgan_conv_op*, "
                                          "const dgan_prune_point*, int, int)",
    "dgan_reconstruct_measured_conv": "int (dgan_handle, const dgan_rec_params*, const dgan_adam_params*, "
                                      "const float* huber_delta, const dgan_prune_point*, int, const dgan_conv_op*, "
                                      "const float*, const float*, const float*, float*, float*, int32_t*, void*, "
                                      "size_t, void*)",
    "dgan_loss_grad_measured_conv": "int (dgan_handle, const float* huber_delta, const dgan_conv_op*, const float*, "
                                    "const float*, int, int, const float*, float*, float*, float*, void*, size_t, "
                                    "void*)",
    "dgan_reconstruct_prior": "int (dgan_handle, const dgan_rec_params*, const dgan_adam_params*, "
                              "const float* huber_delta, float, const dgan_prune_point*, int, const float*, "
                              "const float*, const float*, float*, float*, int32_t*, void*, size_t, void*)",
    "dgan_reconstruct_measured_prior": "int (dgan_handle, const dgan_rec_params*, const dgan_adam_params*, "
                                       "const float* huber_delta, float, const dgan_prune_point*, int, const float*, "
                                       "int, const float*, const float*, float*, float*, int32_t*, void*, size_t, "
                                       "void*)",
    "dgan_reconstruct_measured_csr_prior": "int (dgan_handle, const dgan_rec_params*, const dgan_adam_params*, "
                                           "const float* huber_delta, float, const dgan_prune_point*, int, "
                                           "const int32_t*, const int32_t*, const float*, int, int, const float*, "
                                           "const float*, float*, float*, int32_t*, void*, size_t, void*)",
    "dgan_reconstruct_measured_conv_prior": "int (dgan_handle, const dgan_rec_params*, const dgan_adam_params*, "
                                            "const float* huber_delta, float, const dgan_prune_point*, int, "
                                            "const dgan_conv_op*, const float*, const float*, const float*, float*, "
                                            "float*, int32_t*, void*, size_t, void*)",
    "dgan_workspace_bytes_sparse_dev": "size_t (dgan_handle, int, int, int, int, const dgan_prune_point*, int)",
    "dgan_workspace_bytes_measured_sparse_dev": "size_t (dgan_handle, int, int, int, int, const dgan_conv_op*, int, "
                                                "const dgan_prune_point*, int)",
    "dgan_reconstruct_sparse_dev": "int (dgan_handle, const dgan_rec_params*, const dgan_adam_params*, "
                                   "const float* huber_delta, const float* z_prior, const dgan_prune_point*, int, "
                                   "const dgan_sparse_dev*, float*, const float*, const float*, const float*, float*, "
                                   "float*, int32_t*, void*, size_t, void*)",
    "dgan_reconstruct_measured_sparse_dev": "int (dgan_handle, const dgan_rec_params*, const dgan_adam_params*, "
                                            "const float* huber_delta, const float* z_prior, const dgan_prune_point*, "
                                            "int, const dgan_sparse_dev*, float*, const float*, int, const float*, "
                                            "const float*, float*, float*, int32_t*, void*, size_t, void*)",
    "dgan_reconstruct_measured_csr_sparse_dev": "int (dgan_handle, const dgan_rec_params*, const dgan_adam_params*, "
                                                "const float* huber_delta, const float* z_prior, "
                                                "const dgan_prune_point*, int, const dgan_sparse_dev*, float*, "
                                                "const int32_t*, const int32_t*, const float*, int, int, "
                                                "const float*, const float*, float*, float*, int32_t*, void*, size_t, "
                                                "void*)",
    "dgan_reconstruct_measured_conv_sparse_dev": "int (dgan_handle, const dgan_rec_params*, const dgan_adam_params*, "
                                                 "const float* huber_delta, const float* z_prior, "
                                                 "const dgan_prune_point*, int, const dgan_sparse_dev*, float*, "
                                                 "const dgan_conv_op*, const float*, const float*, const float*, "
                                                 "float*, float*, int32_t*, void*, size_t, void*)",
}


def _ctypes_rules():
    """C type -> the ctypes type the binding declares for it.  Every other pointer is a c_void_p."""
    from defensegan_b200 import _native
    P = ctypes.POINTER
    rules = {"int": ctypes.c_int, "size_t": ctypes.c_size_t, "float": ctypes.c_float, "uint64_t": ctypes.c_uint64,
             "int64_t": ctypes.c_int64, "dgan_handle": ctypes.c_void_p, "const char*": ctypes.c_char_p,
             # nullable scalars: NULL leaves the option off
             "const float* huber_delta": P(ctypes.c_float), "const float* z_prior": P(ctypes.c_float),
             # dgan_create's handle out-parameter and weight-pointer array
             "dgan_handle*": P(ctypes.c_void_p), "const float* const*": P(ctypes.c_void_p),
             # dgan_profile_read's outputs
             "double*": P(ctypes.c_double), "int64_t*": P(ctypes.c_int64)}
    rules.update({"const %s*" % s: P(getattr(_native, s)) for s in STRUCTS})
    return rules


def _split(signature):
    ret, params = signature.split(" (", 1)
    params = params[:-1]
    return ret, [] if params == "void" else params.split(", ")


def test_binding_declares_every_entry_as_the_header_does():
    from defensegan_b200 import _native
    lib = _native.load_library()
    assert sorted(SIGNATURES) == sorted(_native.ABI_SYMBOLS)
    rules = _ctypes_rules()

    def ctype(c):
        return rules.get(c, ctypes.c_void_p) if "*" in c else rules[c]

    header = open(os.path.join(ROOT, "include", "defensegan_b200.h")).read()
    header = re.sub(r"/\*.*?\*/|//[^\n]*", "", header, flags=re.S)
    for sym, signature in SIGNATURES.items():
        ret, params = _split(signature)
        # a parameter the table names (its ctypes rule depends on the name) has that name in the header too
        declared = re.search(r"\b%s\s*\(([^)]*)\)" % sym, header).group(1)
        for p in params:
            if re.fullmatch(r".*\*\s*\w+", p):
                assert re.search(r"\*\s*%s\s*(,|$)" % p.rsplit(None, 1)[1], declared), (sym, p)
        fn = getattr(lib, sym)
        assert fn.restype == ctype(ret), (sym, fn.restype)
        assert list(fn.argtypes) == [ctype(p) for p in params], sym


def test_header_is_c99_with_these_signatures_and_struct_layouts_match_ctypes(tmp_path):
    """The header compiles as C (gcc -std=c99 -pedantic, no C++ or CUDA types) and gives every entry the table's type; a
    C caller linked against the library sees the structs with the binding's size and field offsets, the ABI version,
    the weight count and an error reported through dgan_last_error()."""
    from defensegan_b200 import _native
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("no gcc")
    lines = ["#include <stdio.h>", "#include <stddef.h>", '#include "defensegan_b200.h"']
    for sym, signature in SIGNATURES.items():
        ret, params = _split(signature)
        lines.append("%s (*p_%s)(%s) = %s;" % (ret, sym, ", ".join(params) or "void", sym))
    lines.append("int main(void) {")
    for st in STRUCTS:
        lines.append('  printf("%s %%zu", sizeof(%s));' % (st, st))
        for f, _ in getattr(_native, st)._fields_:
            lines.append('  printf(" %%zu", offsetof(%s, %s));' % (st, f))
        lines.append('  printf("\\n");')
    lines += ["  dgan_desc d = {DGAN_ABI_VERSION, DGAN_ARCH_CELEBA, 128, 64, 0, 1};",
              '  printf("abi %d %d %d\\n", DGAN_ABI_VERSION, dgan_abi_version(), dgan_num_weights(&d));',
              '  printf("err %d %s\\n", dgan_create(NULL, &d, NULL, 0, NULL), dgan_last_error());', "  return 0;", "}"]
    src = tmp_path / "abi.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "abi"
    libdir = os.path.dirname(_native.build_library())
    res = subprocess.run([gcc, "-std=c99", "-pedantic", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src),
                          "-o", str(exe), "-L", libdir, "-l:" + _native.LIB_NAME, "-Wl,-rpath," + libdir],
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert res.returncode == 0, res.stdout
    out = subprocess.run([str(exe)], stdout=subprocess.PIPE, text=True, check=True).stdout.splitlines()
    assert len(out) == len(STRUCTS) + 2, out
    for line in out[:len(STRUCTS)]:
        tok = line.split()
        cls = getattr(_native, tok[0])
        assert int(tok[1]) == ctypes.sizeof(cls), tok[0]
        assert [int(t) for t in tok[2:]] == [getattr(cls, f).offset for f, _ in cls._fields_], tok[0]
    abi, err = out[-2].split(), out[-1].split()
    assert abi[0] == "abi" and [int(t) for t in abi[1:]] == [_native.ABI_VERSION, _native.ABI_VERSION, 10]
    assert err[0] == "err" and int(err[1]) < 0 and len(err) > 2          # status code + message
