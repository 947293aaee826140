"""CPU test of ptxas's resource report for every kernel of the library: which kernels exist and how many instantiations
each has, and that none needs more stack or spills more than the table allows.  A kernel that spills, or that gets a
stack frame (a local array indexed at run time, a call that is not inlined), reads and writes local memory on every
use; the tensor-core kernel would also stall its MMAs.  ptxas must not serialise the tensor-core kernel's wgmma (C7520)
either."""
import glob
import os
import re

import compiled

# name: (instantiations, {template arguments: allowed (stack frame, spill store, spill load) bytes}).  Every
# instantiation not listed is allowed (0, 0, 0).
KERNELS = {
    "adam_kernel": (1, {}),
    "adam_prior_kernel": (1, {}),
    "bn_apply_bwd_kernel": (2, {}),
    "bn_apply_fwd_kernel": (2, {}),
    "bn_apply_jvp_kernel": (2, {}),
    "bn_reduce_kernel": (8, {}),
    "bsgemm_f32_kernel": (4, {}),
    "conv_stage_kernel": (1, {}),
    "cotangent_kernel": (4, {}),
    "cotangent_rowmax_kernel": (3, {}),
    "cotangent_scale_kernel": (1, {}),
    "csr_fill_transpose_kernel": (1, {}),
    "csr_scan_kernel": (1, {}),
    "csr_stage_entries_kernel": (1, {}),
    "csr_stage_rows_kernel": (1, {}),
    "csr_validate_kernel": (1, {}),
    "final_bwd_kernel": (2, {}),
    # fp32 CelebA last-layer forwards: three channels of 5x5 taps per output pixel in registers
    "final_fwd_huber_kernel": (4, {"<float,3,1,true>": (24, 24, 32)}),
    "final_fwd_loss_kernel": (8, {"<float,3,1,true>": (32, 44, 56), "<float,3,2,false>": (32, 40, 44)}),
    "init_z_kernel": (1, {"": (32, 0, 0)}),
    "loss_finish_kernel": (1, {}),
    "loss_finish_prior_kernel": (1, {}),
    "measured_conv_adjoint_kernel": (1, {}),
    "measured_conv_huber_kernel": (1, {}),
    "measured_conv_kernel": (1, {}),
    "measured_csr_huber_kernel": (1, {}),
    "measured_csr_kernel": (2, {}),
    "measured_gemm_huber_kernel": (2, {}),
    "measured_gemm_kernel": (4, {}),
    "momentum_kernel": (1, {}),
    "momentum_prior_kernel": (1, {}),
    "momentum_rows_kernel": (1, {}),
    "momentum_rows_prior_kernel": (1, {}),
    "pad_copy_kernel": (1, {}),
    "prior_term_kernel": (1, {}),
    "prune_gather_adam_kernel": (1, {}),
    "prune_gather_kernel": (1, {}),
    "prune_idx_kernel": (1, {}),
    "prune_select_kernel": (1, {}),
    "scale_copy_kernel": (1, {}),
    "sdev_gather_kernel": (1, {}),
    "sdev_image_resid_kernel": (4, {}),
    "sdev_select_kernel": (1, {}),
    "sdev_term_kernel": (1, {}),
    "sdev_update_kernel": (1, {}),
    "select_kernel": (1, {}),
    "tangent_in_kernel": (1, {}),
    "tangent_out_kernel": (4, {}),
    # the 48-wide fp16 last-layer forwards (CelebA) keep a 16-byte frame, but spill nothing
    "tc_bsgemm2_kernel": (39, {"<48,4,4,%d,__half>" % epi: (16, 0, 0) for epi in (9, 11, 13, 15)}),
    "tc_convert_kernel": (1, {}),
    "tc_final_tiles_kernel": (1, {}),
    "tc_linear_bwd_tiles_kernel": (1, {}),
    "transpose_tiles_kernel": (1, {}),
}
# A Huber instantiation spills no more than its squared-error twin.
SPILLS_NO_MORE_THAN = {"final_fwd_huber_kernel<float,3,1,true>": "final_fwd_loss_kernel<float,3,1,true>"}
# Huber last-layer epilogues of the tensor-core kernel (EPI_FINAL_*_H / _WH)
TC_HUBER_EPILOGUES, TC_HUBER_INSTANTIATIONS = (12, 13, 14, 15), 6


def _short(demangled):
    """`name<template arguments>` of a demangled kernel, e.g. final_fwd_loss_kernel<float,3,1,true>."""
    d = re.sub(r"^void ", "", demangled).replace("dgan::", "")
    depth = 0
    for i, c in enumerate(d):
        depth += (c == "<") - (c == ">")
        if c == "(" and depth == 0:
            d = d[:i]
            break
    return d.replace("(int)", "").replace("(bool)1", "true").replace("(bool)0", "false").replace(" ", "")


def _report():
    """{name<template arguments>: (stack, spill store, spill load)} and {same: mangled name}."""
    res = compiled.resources()
    mangled = sorted(res)
    short = [_short(d) for d in compiled.demangle(mangled)]
    return {s: res[m] for s, m in zip(short, mangled)}, dict(zip(short, mangled))


def test_the_table_names_every_kernel_in_the_sources():
    from defensegan_b200 import _native
    names = set()
    for path in glob.glob(os.path.join(_native.CSRC_DIR, "*.cu*")):
        names |= set(re.findall(r"__global__\s+void\s+(?:__\w+__\([^)]*\)\s+)*(\w+)\s*\(", open(path).read()))
    assert names == set(KERNELS), (sorted(names - set(KERNELS)), sorted(set(KERNELS) - names))


def test_every_kernel_stays_within_its_stack_and_spill_allowance():
    report, mangled = _report()
    counts = {}
    for inst in report:
        counts[inst.split("<")[0]] = counts.get(inst.split("<")[0], 0) + 1
    assert counts == {k: n for k, (n, _) in KERNELS.items()}
    for name, (_, allowed) in KERNELS.items():
        assert all(name + args in report for args in allowed), (name, sorted(allowed))
    over = {}
    for inst, used in report.items():
        name = inst.split("<")[0]
        allowed = KERNELS[name][1].get(inst[len(name):], (0, 0, 0))
        if any(u > a for u, a in zip(used, allowed)):
            over[inst] = (used, allowed)
    assert not over, over
    for inst, twin in SPILLS_NO_MORE_THAN.items():
        assert report[inst][1] <= report[twin][1] and report[inst][2] <= report[twin][2], (inst, report[inst], twin,
                                                                                           report[twin])
    tc = [m for m in mangled.values() if "tc_bsgemm2_kernel" in m]
    assert len(tc) >= 20, len(tc)
    assert sum(compiled.tc_template(m)[3] in TC_HUBER_EPILOGUES for m in tc) == TC_HUBER_INSTANTIATIONS


def test_tensor_core_kernel_is_not_serialised():
    serialised = [l for l in compiled.ptxas_log().splitlines() if "C7520" in l and "tc_bsgemm2_kernel" in l]
    assert not serialised, serialised
