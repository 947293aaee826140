"""ctypes binding of the C-ABI in include/defensegan_b200.h.

PyTorch is used only for device memory and streams.  There is no CPU fallback: if the shared
library is missing or no sm_90 GPU is present, every compute entry point raises.
"""
from __future__ import annotations

import ctypes
import os
import subprocess
import sys
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch
import torch.autograd.forward_ad as fwAD
from torch.autograd.function import once_differentiable

from .operators import ConvOperator

_PKG_DIR = os.path.dirname(os.path.abspath(__file__))
LIB_NAME = "libdefensegan_b200.so"
LIB_PATH = os.environ.get("DGAN_LIB", os.path.join(_PKG_DIR, LIB_NAME))   # DGAN_LIB: A/B-test another build
CSRC_DIR = os.path.join(_PKG_DIR, "csrc")
INCLUDE_DIR = os.path.join(os.path.dirname(_PKG_DIR), "include")

ARCH_IDS = {"mnist": 0, "f-mnist": 0, "fmnist": 0, "celeba": 1}
PRECISIONS = {"fp32": 0, "fp16": 1}

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "-shared",
]

# Every symbol include/defensegan_b200.h declares.
ABI_SYMBOLS = [
    "dgan_abi_version", "dgan_last_error", "dgan_num_weights", "dgan_create", "dgan_destroy",
    "dgan_workspace_bytes", "dgan_reconstruct", "dgan_sample_z0", "dgan_forward", "dgan_loss_grad", "dgan_vjp", "dgan_jvp",
    "dgan_last_launch_count", "dgan_last_enqueue_count", "dgan_macs_per_row", "dgan_profile_enable", "dgan_profile_num_kinds",
    "dgan_profile_kind_name", "dgan_profile_read",
    "dgan_workspace_bytes_weighted", "dgan_reconstruct_weighted", "dgan_loss_grad_weighted",
    "dgan_workspace_bytes_measured", "dgan_reconstruct_measured", "dgan_loss_grad_measured",
    "dgan_workspace_bytes_measured_csr", "dgan_reconstruct_measured_csr", "dgan_loss_grad_measured_csr",
    "dgan_workspace_bytes_pruned", "dgan_reconstruct_pruned",
    "dgan_workspace_bytes_measured_pruned", "dgan_reconstruct_measured_pruned", "dgan_reconstruct_measured_csr_pruned",
    "dgan_workspace_bytes_adam", "dgan_workspace_bytes_measured_adam", "dgan_reconstruct_adam", "dgan_reconstruct_measured_adam",
    "dgan_reconstruct_measured_csr_adam",
    "dgan_reconstruct_huber", "dgan_reconstruct_measured_huber", "dgan_reconstruct_measured_csr_huber",
    "dgan_loss_grad_huber", "dgan_loss_grad_measured_huber", "dgan_loss_grad_measured_csr_huber",
    "dgan_conv_op_m", "dgan_workspace_bytes_measured_conv", "dgan_reconstruct_measured_conv", "dgan_loss_grad_measured_conv",
    "dgan_reconstruct_prior", "dgan_reconstruct_measured_prior", "dgan_reconstruct_measured_csr_prior",
    "dgan_reconstruct_measured_conv_prior",
    "dgan_workspace_bytes_sparse_dev", "dgan_workspace_bytes_measured_sparse_dev", "dgan_reconstruct_sparse_dev",
    "dgan_reconstruct_measured_sparse_dev", "dgan_reconstruct_measured_csr_sparse_dev",
    "dgan_reconstruct_measured_conv_sparse_dev",
]


class dgan_desc(ctypes.Structure):
    _fields_ = [("abi_version", ctypes.c_int32), ("arch", ctypes.c_int32), ("latent_dim", ctypes.c_int32),
                ("net_dim", ctypes.c_int32), ("use_bn", ctypes.c_int32), ("precision", ctypes.c_int32)]


class dgan_rec_params(ctypes.Structure):
    _fields_ = [("batch", ctypes.c_int32), ("rec_rr", ctypes.c_int32), ("rec_iters", ctypes.c_int32),
                ("rec_lr", ctypes.c_float), ("momentum", ctypes.c_float), ("decay_lr", ctypes.c_int32),
                ("seed", ctypes.c_uint64), ("z_row_offset", ctypes.c_uint64)]


class dgan_prune_point(ctypes.Structure):
    _fields_ = [("iter", ctypes.c_int32), ("keep", ctypes.c_int32)]


class dgan_adam_params(ctypes.Structure):
    _fields_ = [("beta1", ctypes.c_float), ("beta2", ctypes.c_float), ("eps", ctypes.c_float)]


class dgan_conv_op(ctypes.Structure):
    _fields_ = [("kh", ctypes.c_int32), ("kw", ctypes.c_int32), ("pad_h", ctypes.c_int32), ("pad_w", ctypes.c_int32),
                ("stride", ctypes.c_int32)]


class dgan_sparse_dev(ctypes.Structure):
    _fields_ = [("l1", ctypes.c_float), ("step", ctypes.c_float)]


ABI_VERSION = 2


def check_adam_params(adam):
    """Adam's (beta1, beta2, eps) as a tuple of floats, after the rules of dgan_reconstruct_adam: 0 <= beta1 < 1,
    0 <= beta2 < 1 and a finite eps > 0 (as fp32, the type the library reads).  A ValueError names the bad value."""
    try:
        vals = tuple(adam)
    except TypeError:
        raise ValueError("adam is a (beta1, beta2, eps) triple, got %r" % (adam,)) from None
    if len(vals) != 3:
        raise ValueError("adam is a (beta1, beta2, eps) triple, got %r" % (adam,))
    out = []
    for name, v in zip(("beta1", "beta2", "eps"), vals):
        if isinstance(v, bool) or not isinstance(v, (int, float, np.integer, np.floating)):
            raise ValueError("adam %s = %r is not a number" % (name, v))
        out.append(float(np.float32(v)))
    b1, b2, eps = out
    if not 0.0 <= b1 < 1.0:
        raise ValueError("adam beta1 = %r must be in [0, 1)" % (vals[0],))
    if not 0.0 <= b2 < 1.0:
        raise ValueError("adam beta2 = %r must be in [0, 1)" % (vals[1],))
    if not (np.isfinite(eps) and eps > 0.0):
        raise ValueError("adam eps = %r must be finite and > 0" % (vals[2],))
    return b1, b2, eps


def check_huber_delta(huber_delta):
    """The Huber loss's delta as a float, after the rule of dgan_reconstruct_huber: > 0 as fp32 (the type the library
    reads), +inf allowed.  A ValueError names the bad value (NaN, 0, a negative or a non-number)."""
    if isinstance(huber_delta, bool) or not isinstance(huber_delta, (int, float, np.integer, np.floating)):
        raise ValueError("huber_delta = %r is not a number" % (huber_delta,))
    try:
        with np.errstate(over="ignore"):   # beyond fp32's range: +-inf, as the library would read it
            d = float(np.float32(huber_delta))
    except OverflowError:                  # an int beyond a double's range
        d = float("inf") if huber_delta > 0 else float("-inf")
    if not d > 0.0:
        raise ValueError("huber_delta = %r must be > 0 (+inf allowed)" % (huber_delta,))
    return d


def check_z_prior(z_prior):
    """The latent prior's weight lambda as a float, after the rule of dgan_reconstruct_prior: as fp32 (the type the
    library reads) finite and >= 0, with 2 lambda finite in fp32.  A ValueError names the bad value (NaN, an infinity, a
    negative value, one whose double overflows fp32, or a non-number)."""
    if isinstance(z_prior, bool) or not isinstance(z_prior, (int, float, np.integer, np.floating)):
        raise ValueError("z_prior = %r is not a number" % (z_prior,))
    try:
        with np.errstate(over="ignore"):   # beyond fp32's range: +-inf, as the library would read it
            lam = np.float32(z_prior)
    except OverflowError:                  # an int beyond a double's range
        lam = np.float32(np.inf)
    with np.errstate(over="ignore"):
        two = lam * np.float32(2.0)
    if not (np.isfinite(lam) and lam >= 0.0 and np.isfinite(two)):
        raise ValueError("z_prior = %r must be finite and >= 0, with 2 z_prior finite in fp32" % (z_prior,))
    return float(lam)


def check_sparse_dev(sparse_dev, n: Optional[int] = None):
    """Sparse deviations' (l1, step) as a tuple of floats, after the rules of dgan_reconstruct_sparse_dev: both as fp32
    (the type the library reads) finite and >= 0; with n (H*W*C for the image loss, m for a measured one) also
    eta = step n / 2 and tau = eta l1, in double, finite in fp32.  A ValueError names the bad value."""
    try:
        vals = tuple(sparse_dev)
    except TypeError:
        raise ValueError("sparse_dev is an (l1, step) pair, got %r" % (sparse_dev,)) from None
    if len(vals) != 2:
        raise ValueError("sparse_dev is an (l1, step) pair, got %r" % (sparse_dev,))
    out = []
    for name, v in zip(("l1", "step"), vals):
        if isinstance(v, bool) or not isinstance(v, (int, float, np.integer, np.floating)):
            raise ValueError("sparse_dev %s = %r is not a number" % (name, v))
        try:
            with np.errstate(over="ignore"):   # beyond fp32's range: +-inf, as the library would read it
                f = float(np.float32(v))
        except OverflowError:                  # an int beyond a double's range
            f = float("inf")
        if not (np.isfinite(f) and f >= 0.0):
            raise ValueError("sparse_dev %s = %r must be finite and >= 0" % (name, v))
        out.append(f)
    l1, step = out
    if n is not None:
        eta = step * float(n) / 2.0
        with np.errstate(over="ignore"):
            if not np.isfinite(np.float32(eta)):
                raise ValueError("sparse_dev step = %r: eta = step * n / 2 = %r overflows fp32" % (vals[1], eta))
            if not np.isfinite(np.float32(eta * l1)):
                raise ValueError("sparse_dev l1 = %r: tau = eta * l1 = %r overflows fp32" % (vals[0], eta * l1))
    return l1, step


def check_prune_schedule(prune, rec_rr: int, rec_iters: int):
    """A restart-pruning schedule as a list of (iter, keep) int pairs, after the rules of dgan_reconstruct_pruned:
    1 <= iter_1 < iter_2 < ... <= rec_iters - 1 and rec_rr >= keep_1 >= keep_2 >= ... >= 1.  A ValueError names the
    first bad point."""
    try:
        points = [tuple(p) for p in prune]
    except TypeError:
        raise ValueError("a prune schedule is a sequence of (iter, keep) pairs, got %r" % (prune,)) from None
    if not points:
        raise ValueError("a prune schedule needs at least one (iter, keep) point")
    out = []
    prev_it, prev_keep = 0, int(rec_rr)
    for k, p in enumerate(points):
        if len(p) != 2 or not all(isinstance(v, (int, np.integer)) and not isinstance(v, bool) for v in p):
            raise ValueError("prune point %d %r: expected a pair of integers (iter, keep)" % (k, p))
        it, keep = int(p[0]), int(p[1])
        bad = None
        if it <= prev_it:
            bad = "iter must be >= 1" if k == 0 else "iter must exceed the previous point's (%d)" % prev_it
        elif it > rec_iters - 1:
            bad = "iter must be <= rec_iters - 1 = %d" % (rec_iters - 1)
        elif keep < 1:
            bad = "keep must be >= 1"
        elif keep > prev_keep:
            bad = ("keep must be <= rec_rr = %d" % rec_rr) if k == 0 else \
                "keep must not exceed the previous point's (%d)" % prev_keep
        if bad is not None:
            raise ValueError("prune point %d (iter %d, keep %d): %s" % (k, it, keep, bad))
        out.append((it, keep))
        prev_it, prev_keep = it, keep
    return out


def _compile(out_path: str, extra_flags: List[str], verbose: bool, force: bool) -> str:
    """nvcc csrc/dgan_api.cu -> out_path unless out_path is up to date: it exists, no source is newer, and it was built
    with the same command (recorded in out_path + ".cmd", so a library built with other flags - another GPU
    architecture, say - is rebuilt)."""
    srcs = [os.path.join(CSRC_DIR, f) for f in sorted(os.listdir(CSRC_DIR))]
    srcs.append(os.path.join(INCLUDE_DIR, "defensegan_b200.h"))
    cmd = [os.environ.get("NVCC", "nvcc")] + NVCC_FLAGS + extra_flags + [os.path.join(CSRC_DIR, "dgan_api.cu"), "-o", out_path]
    stamp = out_path + ".cmd"
    if not force and os.path.exists(out_path) and os.path.exists(stamp):
        with open(stamp) as f:
            same_cmd = f.read() == " ".join(cmd)
        lib_m = os.path.getmtime(out_path)
        if same_cmd and all(os.path.getmtime(s) <= lib_m for s in srcs):
            return out_path
    if verbose:
        print(" ".join(cmd), file=sys.stderr)
    res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + res.stdout)
    with open(stamp, "w") as f:
        f.write(" ".join(cmd))
    return out_path


def build_library(force: bool = False, verbose: bool = False) -> str:
    """Compile csrc/ for sm_90a with nvcc into the in-tree shared library (cross-compiles
    without a GPU).  Rebuilds when any source is newer than the library or the compile command changed."""
    return _compile(LIB_PATH, [], verbose, force)


PROBE_LIB_PATH = os.path.join(_PKG_DIR, "libdefensegan_b200_probe.so")


def build_probe_library(force: bool = False) -> str:
    """The same sources with -DDGAN_PROBE: per-CTA clock / %globaltimer counters in the tensor-core kernels and
    dgan_debug_probe_read().  Measurement aid only (tools/probe_step.py, the `timeline` pass of bench.py run it in a
    process of its own through DGAN_LIB); the product library carries none of it."""
    return _compile(PROBE_LIB_PATH, ["-DDGAN_PROBE"], False, force)


_lib = None


def load_library() -> ctypes.CDLL:
    """dlopen the in-tree library and declare the signatures of the header."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            "%s not found: run `python -c 'import __graft_entry__ as g; g.build()'` (or "
            "defensegan_b200._native.build_library()) first. There is no CPU fallback." % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH)
    lib.dgan_abi_version.restype = ctypes.c_int
    if lib.dgan_abi_version() != ABI_VERSION:
        raise RuntimeError("%s has ABI version %d, this binding needs %d: rebuild it (__graft_entry__.build())"
                           % (LIB_PATH, lib.dgan_abi_version(), ABI_VERSION))
    vp, i32, u64, f32, sz = ctypes.c_void_p, ctypes.c_int, ctypes.c_uint64, ctypes.c_float, ctypes.c_size_t
    lib.dgan_abi_version.restype = i32
    lib.dgan_abi_version.argtypes = []
    lib.dgan_last_error.restype = ctypes.c_char_p
    lib.dgan_last_error.argtypes = []
    lib.dgan_num_weights.restype = i32
    lib.dgan_num_weights.argtypes = [ctypes.POINTER(dgan_desc)]
    lib.dgan_create.restype = i32
    lib.dgan_create.argtypes = [ctypes.POINTER(vp), ctypes.POINTER(dgan_desc), ctypes.POINTER(vp), i32, vp]
    lib.dgan_destroy.restype = i32
    lib.dgan_destroy.argtypes = [vp]
    lib.dgan_workspace_bytes.restype = sz
    lib.dgan_workspace_bytes.argtypes = [vp, i32, i32]
    lib.dgan_reconstruct.restype = i32
    lib.dgan_reconstruct.argtypes = [vp, ctypes.POINTER(dgan_rec_params), vp, vp, vp, vp, vp, vp, sz, vp]
    lib.dgan_workspace_bytes_weighted.restype = sz
    lib.dgan_workspace_bytes_weighted.argtypes = [vp, i32, i32]
    lib.dgan_reconstruct_weighted.restype = i32
    lib.dgan_reconstruct_weighted.argtypes = [vp, ctypes.POINTER(dgan_rec_params), vp, vp, vp, vp, vp, vp, vp, sz, vp]
    lib.dgan_loss_grad_weighted.restype = i32
    lib.dgan_loss_grad_weighted.argtypes = [vp, vp, vp, i32, i32, vp, vp, vp, vp, vp, sz, vp]
    lib.dgan_workspace_bytes_measured.restype = sz
    lib.dgan_workspace_bytes_measured.argtypes = [vp, i32, i32, i32]
    lib.dgan_reconstruct_measured.restype = i32
    lib.dgan_reconstruct_measured.argtypes = [vp, ctypes.POINTER(dgan_rec_params), vp, i32, vp, vp, vp, vp, vp, vp, sz, vp]
    lib.dgan_loss_grad_measured.restype = i32
    lib.dgan_loss_grad_measured.argtypes = [vp, vp, i32, vp, i32, i32, vp, vp, vp, vp, vp, sz, vp]
    lib.dgan_workspace_bytes_measured_csr.restype = sz
    lib.dgan_workspace_bytes_measured_csr.argtypes = [vp, i32, i32, i32, i32]
    lib.dgan_reconstruct_measured_csr.restype = i32
    lib.dgan_reconstruct_measured_csr.argtypes = [vp, ctypes.POINTER(dgan_rec_params), vp, vp, vp, i32, i32, vp, vp, vp, vp,
                                                  vp, vp, sz, vp]
    lib.dgan_loss_grad_measured_csr.restype = i32
    lib.dgan_loss_grad_measured_csr.argtypes = [vp, vp, vp, vp, i32, i32, vp, i32, i32, vp, vp, vp, vp, vp, sz, vp]
    lib.dgan_workspace_bytes_pruned.restype = sz
    lib.dgan_workspace_bytes_pruned.argtypes = [vp, i32, i32, ctypes.POINTER(dgan_prune_point), i32, i32]
    lib.dgan_reconstruct_pruned.restype = i32
    lib.dgan_reconstruct_pruned.argtypes = [vp, ctypes.POINTER(dgan_rec_params), ctypes.POINTER(dgan_prune_point), i32, vp,
                                            vp, vp, vp, vp, vp, vp, sz, vp]
    lib.dgan_workspace_bytes_measured_pruned.restype = sz
    lib.dgan_workspace_bytes_measured_pruned.argtypes = [vp, i32, i32, i32, i32, ctypes.POINTER(dgan_prune_point), i32]
    lib.dgan_reconstruct_measured_pruned.restype = i32
    lib.dgan_reconstruct_measured_pruned.argtypes = [vp, ctypes.POINTER(dgan_rec_params), ctypes.POINTER(dgan_prune_point), i32,
                                                     vp, i32, vp, vp, vp, vp, vp, vp, sz, vp]
    lib.dgan_reconstruct_measured_csr_pruned.restype = i32
    lib.dgan_reconstruct_measured_csr_pruned.argtypes = [vp, ctypes.POINTER(dgan_rec_params), ctypes.POINTER(dgan_prune_point),
                                                         i32, vp, vp, vp, i32, i32, vp, vp, vp, vp, vp, vp, sz, vp]
    pp, ap = ctypes.POINTER(dgan_prune_point), ctypes.POINTER(dgan_adam_params)
    lib.dgan_workspace_bytes_adam.restype = sz
    lib.dgan_workspace_bytes_adam.argtypes = [vp, i32, i32, i32, pp, i32]
    lib.dgan_workspace_bytes_measured_adam.restype = sz
    lib.dgan_workspace_bytes_measured_adam.argtypes = [vp, i32, i32, i32, i32, pp, i32]
    lib.dgan_reconstruct_adam.restype = i32
    lib.dgan_reconstruct_adam.argtypes = [vp, ctypes.POINTER(dgan_rec_params), ap, pp, i32, vp, vp, vp, vp, vp, vp, vp, sz, vp]
    lib.dgan_reconstruct_measured_adam.restype = i32
    lib.dgan_reconstruct_measured_adam.argtypes = [vp, ctypes.POINTER(dgan_rec_params), ap, pp, i32, vp, i32, vp, vp, vp, vp,
                                                   vp, vp, sz, vp]
    lib.dgan_reconstruct_measured_csr_adam.restype = i32
    lib.dgan_reconstruct_measured_csr_adam.argtypes = [vp, ctypes.POINTER(dgan_rec_params), ap, pp, i32, vp, vp, vp, i32, i32,
                                                       vp, vp, vp, vp, vp, vp, sz, vp]
    f32 = ctypes.c_float
    lib.dgan_reconstruct_huber.restype = i32
    lib.dgan_reconstruct_huber.argtypes = [vp, ctypes.POINTER(dgan_rec_params), ap, f32, pp, i32, vp, vp, vp, vp, vp, vp, vp,
                                           sz, vp]
    lib.dgan_reconstruct_measured_huber.restype = i32
    lib.dgan_reconstruct_measured_huber.argtypes = [vp, ctypes.POINTER(dgan_rec_params), ap, f32, pp, i32, vp, i32, vp, vp,
                                                    vp, vp, vp, vp, sz, vp]
    lib.dgan_reconstruct_measured_csr_huber.restype = i32
    lib.dgan_reconstruct_measured_csr_huber.argtypes = [vp, ctypes.POINTER(dgan_rec_params), ap, f32, pp, i32, vp, vp, vp,
                                                        i32, i32, vp, vp, vp, vp, vp, vp, sz, vp]
    lib.dgan_loss_grad_huber.restype = i32
    lib.dgan_loss_grad_huber.argtypes = [vp, f32, vp, vp, i32, i32, vp, vp, vp, vp, vp, sz, vp]
    lib.dgan_loss_grad_measured_huber.restype = i32
    lib.dgan_loss_grad_measured_huber.argtypes = [vp, f32, vp, i32, vp, i32, i32, vp, vp, vp, vp, vp, sz, vp]
    lib.dgan_loss_grad_measured_csr_huber.restype = i32
    lib.dgan_loss_grad_measured_csr_huber.argtypes = [vp, f32, vp, vp, vp, i32, i32, vp, i32, i32, vp, vp, vp, vp, vp, sz, vp]
    lib.dgan_sample_z0.restype = i32
    cp, fp = ctypes.POINTER(dgan_conv_op), ctypes.POINTER(ctypes.c_float)
    lib.dgan_conv_op_m.restype = i32
    lib.dgan_conv_op_m.argtypes = [vp, cp]
    lib.dgan_workspace_bytes_measured_conv.restype = sz
    lib.dgan_workspace_bytes_measured_conv.argtypes = [vp, i32, i32, cp, pp, i32, i32]
    lib.dgan_reconstruct_measured_conv.restype = i32
    lib.dgan_reconstruct_measured_conv.argtypes = [vp, ctypes.POINTER(dgan_rec_params), ap, fp, pp, i32, cp, vp, vp, vp, vp,
                                                   vp, vp, vp, sz, vp]
    lib.dgan_loss_grad_measured_conv.restype = i32
    lib.dgan_loss_grad_measured_conv.argtypes = [vp, fp, cp, vp, vp, i32, i32, vp, vp, vp, vp, vp, sz, vp]
    rp = ctypes.POINTER(dgan_rec_params)
    lib.dgan_reconstruct_prior.restype = i32
    lib.dgan_reconstruct_prior.argtypes = [vp, rp, ap, fp, f32, pp, i32, vp, vp, vp, vp, vp, vp, vp, sz, vp]
    lib.dgan_reconstruct_measured_prior.restype = i32
    lib.dgan_reconstruct_measured_prior.argtypes = [vp, rp, ap, fp, f32, pp, i32, vp, i32, vp, vp, vp, vp, vp, vp, sz, vp]
    lib.dgan_reconstruct_measured_csr_prior.restype = i32
    lib.dgan_reconstruct_measured_csr_prior.argtypes = [vp, rp, ap, fp, f32, pp, i32, vp, vp, vp, i32, i32, vp, vp, vp, vp,
                                                        vp, vp, sz, vp]
    lib.dgan_reconstruct_measured_conv_prior.restype = i32
    lib.dgan_reconstruct_measured_conv_prior.argtypes = [vp, rp, ap, fp, f32, pp, i32, cp, vp, vp, vp, vp, vp, vp, vp, sz,
                                                         vp]
    sdp = ctypes.POINTER(dgan_sparse_dev)
    lib.dgan_workspace_bytes_sparse_dev.restype = sz
    lib.dgan_workspace_bytes_sparse_dev.argtypes = [vp, i32, i32, i32, i32, pp, i32]
    lib.dgan_workspace_bytes_measured_sparse_dev.restype = sz
    lib.dgan_workspace_bytes_measured_sparse_dev.argtypes = [vp, i32, i32, i32, i32, cp, i32, pp, i32]
    lib.dgan_reconstruct_sparse_dev.restype = i32
    lib.dgan_reconstruct_sparse_dev.argtypes = [vp, rp, ap, fp, fp, pp, i32, sdp, vp, vp, vp, vp, vp, vp, vp, vp, sz, vp]
    lib.dgan_reconstruct_measured_sparse_dev.restype = i32
    lib.dgan_reconstruct_measured_sparse_dev.argtypes = [vp, rp, ap, fp, fp, pp, i32, sdp, vp, vp, i32, vp, vp, vp, vp, vp,
                                                         vp, sz, vp]
    lib.dgan_reconstruct_measured_csr_sparse_dev.restype = i32
    lib.dgan_reconstruct_measured_csr_sparse_dev.argtypes = [vp, rp, ap, fp, fp, pp, i32, sdp, vp, vp, vp, vp, i32, i32, vp,
                                                             vp, vp, vp, vp, vp, sz, vp]
    lib.dgan_reconstruct_measured_conv_sparse_dev.restype = i32
    lib.dgan_reconstruct_measured_conv_sparse_dev.argtypes = [vp, rp, ap, fp, fp, pp, i32, sdp, vp, cp, vp, vp, vp, vp, vp,
                                                              vp, vp, sz, vp]
    lib.dgan_sample_z0.argtypes = [vp, u64, u64, i32, vp, vp]
    lib.dgan_forward.restype = i32
    lib.dgan_forward.argtypes = [vp, vp, i32, vp, vp, sz, vp]
    lib.dgan_loss_grad.restype = i32
    lib.dgan_loss_grad.argtypes = [vp, vp, i32, i32, vp, vp, vp, vp, vp, sz, vp]
    lib.dgan_vjp.restype = i32
    lib.dgan_vjp.argtypes = [vp, vp, i32, vp, vp, vp, vp, sz, vp]
    lib.dgan_jvp.restype = i32
    lib.dgan_jvp.argtypes = [vp, vp, i32, vp, vp, vp, vp, sz, vp]
    lib.dgan_last_launch_count.restype = ctypes.c_int64
    lib.dgan_last_launch_count.argtypes = [vp]
    lib.dgan_last_enqueue_count.restype = ctypes.c_int64
    lib.dgan_last_enqueue_count.argtypes = [vp]
    lib.dgan_macs_per_row.restype = ctypes.c_int64
    lib.dgan_macs_per_row.argtypes = [vp]
    lib.dgan_profile_enable.restype = i32
    lib.dgan_profile_enable.argtypes = [vp, i32]
    lib.dgan_profile_num_kinds.restype = i32
    lib.dgan_profile_num_kinds.argtypes = [vp]
    lib.dgan_profile_kind_name.restype = ctypes.c_char_p
    lib.dgan_profile_kind_name.argtypes = [vp, i32]
    lib.dgan_profile_read.restype = i32
    lib.dgan_profile_read.argtypes = [vp, i32, ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_int64),
                                      ctypes.POINTER(ctypes.c_double)]
    _lib = lib
    return lib


def _check(lib, rc: int, what: str):
    if rc != 0:
        msg = lib.dgan_last_error()
        raise RuntimeError("%s failed (status %d): %s" % (what, rc, msg.decode() if msg else "?"))


def _ptr(t: Optional[torch.Tensor]):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


def _byref_or_none(obj):
    """ctypes.byref(obj) for a nullable pointer argument, None (NULL) for None."""
    return ctypes.byref(obj) if obj is not None else None


def _require_cuda_f32(t: torch.Tensor, name: str) -> torch.Tensor:
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise RuntimeError("%s must be a CUDA tensor (there is no CPU path)" % name)
    if t.dtype != torch.float32:
        t = t.to(torch.float32)
    return t.contiguous()


def _require_cuda_i32(t: torch.Tensor, name: str) -> torch.Tensor:
    """A CUDA index tensor as contiguous int32; int64 indices must fit."""
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise RuntimeError("%s must be a CUDA tensor (there is no CPU path)" % name)
    if t.dtype != torch.int32:
        t = t.to(torch.int32)
    return t.contiguous()


INT32_MAX = 2 ** 31 - 1


def _require_aligned_out(rec: torch.Tensor) -> None:
    """The reconstruct entries store rec 16 bytes at a time: a view that starts elsewhere (out=buf[1:]) is refused."""
    if rec.data_ptr() % 16 != 0:
        raise ValueError("out must be 16-byte aligned: its data starts %d bytes past a 16-byte boundary"
                         % (rec.data_ptr() % 16))


def _float_ref(v: Optional[float]):
    """A nullable const float* argument: NULL for None."""
    return _byref_or_none(None if v is None else ctypes.c_float(v))


_ENTRY_OF_KIND = {"image": "", "dense": "_measured", "csr": "_measured_csr", "conv": "_measured_conv"}


def _route(kind: str, operands=(), m: int = 0, nnz: int = -1, conv: Optional[dgan_conv_op] = None, weighted: bool = False,
           sched=None, ap: Optional[dgan_adam_params] = None, delta: Optional[float] = None, lam: Optional[float] = None,
           sd: Optional[dgan_sparse_dev] = None, dev: Optional[torch.Tensor] = None):
    """The sizer and the C entry of a projection with checked options, for an operator kind "image" (operands: the
    images and the weights, or NULL), "dense" (a, m, y), "csr" (row_ptr, col_idx, val, m, nnz, y) or "conv" (op, k, y):
    (sizer, its arguments after (handle, batch, rec_rr), entry, its arguments between dgan_rec_params and z0).  The
    entry follows sparse_dev > z_prior > huber_delta > adam > prune > weighted / plain.  Huber and the prior run on
    their counterpart's workspace, so the sizer follows sparse_dev > conv > adam > prune > the operator's own."""
    measured = kind != "image"
    n_points = len(sched) if sched is not None else 0
    if sd is not None and measured:
        sizer = ("dgan_workspace_bytes_measured_sparse_dev",
                 (int(m), int(nnz), _byref_or_none(conv), int(ap is not None), sched, n_points))
    elif sd is not None:
        sizer = ("dgan_workspace_bytes_sparse_dev", (int(weighted), int(ap is not None), sched, n_points))
    elif kind == "conv":
        sizer = ("dgan_workspace_bytes_measured_conv", (ctypes.byref(conv), sched, n_points, int(ap is not None)))
    elif ap is not None and measured:
        sizer = ("dgan_workspace_bytes_measured_adam", (int(m), int(nnz), sched, n_points))
    elif ap is not None:
        sizer = ("dgan_workspace_bytes_adam", (int(weighted), sched, n_points))
    elif sched is not None and measured:
        sizer = ("dgan_workspace_bytes_measured_pruned", (int(m), int(nnz), sched, n_points))
    elif sched is not None:
        sizer = ("dgan_workspace_bytes_pruned", (sched, n_points, int(weighted)))
    elif kind == "csr":
        sizer = ("dgan_workspace_bytes_measured_csr", (int(m), int(nnz)))
    elif kind == "dense":
        sizer = ("dgan_workspace_bytes_measured", (int(m),))
    else:
        sizer = ("dgan_workspace_bytes_weighted" if weighted else "dgan_workspace_bytes", ())
    entry = "dgan_reconstruct" + _ENTRY_OF_KIND[kind]
    operands = tuple(operands)
    if sd is not None:
        options = (_byref_or_none(ap), _float_ref(delta), _float_ref(lam), sched, n_points, ctypes.byref(sd), _ptr(dev))
        entry += "_sparse_dev"
    elif lam is not None:
        options = (_byref_or_none(ap), _float_ref(delta), lam, sched, n_points)
        entry += "_prior"
    elif kind == "conv":
        options = (_byref_or_none(ap), _float_ref(delta), sched, n_points)
    elif delta is not None:
        options = (_byref_or_none(ap), delta, sched, n_points)
        entry += "_huber"
    elif ap is not None:
        options = (ctypes.byref(ap), sched, n_points)
        entry += "_adam"
    elif sched is not None:
        options = (sched, n_points)
        entry += "_pruned"
    else:
        options = ()
        if weighted:
            entry += "_weighted"
        elif not measured:
            operands = operands[:1]              # dgan_reconstruct takes no weights
    return sizer + (entry, options + operands)


class NativeGenerator:
    """Owns one dgan_handle (the generator's re-laid-out weights on one GPU)."""

    def __init__(self, arch: str, weights: Sequence[torch.Tensor], latent_dim: int = 128, net_dim: int = 64,
                 use_bn: bool = False, precision: str = "fp32", device: Optional[torch.device] = None):
        if not torch.cuda.is_available():
            raise RuntimeError("defensegan_b200 needs a CUDA (sm_90) device; there is no CPU fallback")
        if arch not in ARCH_IDS:
            raise ValueError("unknown arch %r" % (arch,))
        if precision not in PRECISIONS:
            raise ValueError("precision must be one of %s" % sorted(PRECISIONS))
        self.lib = load_library()
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.arch, self.precision = arch, precision
        self.latent_dim, self.net_dim = int(latent_dim), int(net_dim)
        self.use_bn = bool(use_bn)
        self.image_dim = (64, 64, 3) if ARCH_IDS[arch] == 1 else (28, 28, 1)
        self.hwc = self.image_dim[0] * self.image_dim[1] * self.image_dim[2]
        self._handle = ctypes.c_void_p(0)
        self._ws = None
        desc = dgan_desc(ABI_VERSION, ARCH_IDS[arch], self.latent_dim, self.net_dim, int(bool(use_bn)), PRECISIONS[precision])
        with torch.cuda.device(self.device):
            # the handle copies the weights (on `stream`): they only have to outlive those copies
            ws = [_require_cuda_f32(w.to(self.device), "weight") for w in weights]
            n_expected = self.lib.dgan_num_weights(ctypes.byref(desc))
            if len(ws) != n_expected:
                raise ValueError("expected %d weight tensors, got %d" % (n_expected, len(ws)))
            arr = (ctypes.c_void_p * len(ws))(*[w.data_ptr() for w in ws])
            stream = torch.cuda.current_stream(self.device)
            h = ctypes.c_void_p(0)
            _check(self.lib, self.lib.dgan_create(ctypes.byref(h), ctypes.byref(desc), arr, len(ws),
                                                  ctypes.c_void_p(stream.cuda_stream)), "dgan_create")
            self._handle = h
            stream.synchronize()
            del ws

    def close(self):
        if getattr(self, "_handle", None) is not None and self._handle.value:
            torch.cuda.synchronize(self.device)
            self.lib.dgan_destroy(self._handle)
            self._handle = ctypes.c_void_p(0)

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- helpers -------------------------------------------------------------------------
    def _workspace(self, batch: int, rec_rr: int, weighted: bool = False, m: int = 0, nnz: int = -1, sched=None,
                   adam: bool = False, conv: Optional[dgan_conv_op] = None, sdev: bool = False):
        """The workspace of a call with these options, sized by the sizer _route picks: (1024-byte aligned pointer,
        bytes)."""
        kind = "conv" if conv is not None else "csr" if m > 0 and nnz >= 0 else "dense" if m > 0 else "image"
        sizer, args = _route(kind, (), m, nnz, conv, weighted, sched, dgan_adam_params() if adam else None,
                             sd=dgan_sparse_dev() if sdev else None)[:2]
        return self._workspace_of(sizer, args, batch, rec_rr)

    def _workspace_of(self, sizer: str, args, batch: int, rec_rr: int):
        need = int(getattr(self.lib, sizer)(self._handle, batch, rec_rr, *args))
        if need == 0:
            raise RuntimeError("dgan_workspace_bytes returned 0 (invalid batch / rec_rr)")
        if self._ws is None or self._ws.numel() < need + 1024:
            if self._ws is not None:
                # earlier calls (possibly on other streams) may still use the old block: let them finish before the
                # caching allocator can hand it to somebody else
                torch.cuda.synchronize(self.device)
            self._ws = None
            self._ws = torch.empty(need + 1024, dtype=torch.uint8, device=self.device)
        base = self._ws.data_ptr()
        aligned = (base + 1023) // 1024 * 1024
        return ctypes.c_void_p(aligned), need

    @property
    def macs_per_row(self) -> int:
        return int(self.lib.dgan_macs_per_row(self._handle))

    @property
    def last_launch_count(self) -> int:
        return int(self.lib.dgan_last_launch_count(self._handle))

    @property
    def last_enqueue_count(self) -> int:
        """Stream operations the host issued for the last reconstruct (the L-step loop is one CUDA-graph launch)."""
        return int(self.lib.dgan_last_enqueue_count(self._handle))

    def profile_enable(self, on: bool) -> None:
        _check(self.lib, self.lib.dgan_profile_enable(self._handle, int(bool(on))), "dgan_profile_enable")

    def profile_read(self):
        """[{name, ms, launches, flops_per_launch}] for the launches recorded since profile_enable(True)."""
        nk = int(self.lib.dgan_profile_num_kinds(self._handle))
        ms = (ctypes.c_double * nk)()
        cnt = (ctypes.c_int64 * nk)()
        fl = (ctypes.c_double * nk)()
        _check(self.lib, self.lib.dgan_profile_read(self._handle, nk, ms, cnt, fl), "dgan_profile_read")
        return [dict(name=self.lib.dgan_profile_kind_name(self._handle, k).decode(), ms=float(ms[k]),
                     launches=int(cnt[k]), flops_per_launch=float(fl[k])) for k in range(nk)]

    # -- entry points ----------------------------------------------------------------------
    def reconstruct(self, images: torch.Tensor, rec_rr: int, rec_iters: int, rec_lr: float = 10.0,
                    z_init_val: Optional[torch.Tensor] = None, seed: int = 0, momentum: float = 0.7,
                    decay_lr: bool = False, out: Optional[torch.Tensor] = None, return_aux: bool = False,
                    z_row_offset: int = 0, pixel_weights: Optional[torch.Tensor] = None,
                    prune: Optional[Sequence[Sequence[int]]] = None, adam: Optional[Sequence[float]] = None,
                    huber_delta: Optional[float] = None, z_prior: Optional[float] = None, sparse_dev=None,
                    deviation_out: Optional[torch.Tensor] = None):
        """pixel_weights ([B,H,W,C], finite, in [0, 1]; the values are not checked here - DefenseGANBase.reconstruct does):
        the projection minimises the weighted loss (1/HWC) sum_p w_p (G(z)_p - x_p)^2 instead
        (dgan_reconstruct_weighted).
        prune (a sequence of (iter, keep) pairs, see check_prune_schedule): from iteration iter on, each image keeps only
        its `keep` restarts of lowest loss at iteration iter - 1 (dgan_reconstruct_pruned); idx is the chosen restart's
        original index.  None runs every restart to the end.
        adam ((beta1, beta2, eps), see check_adam_params): update z with Adam instead of momentum (dgan_reconstruct_adam,
        with or without pixel_weights and prune); momentum is then ignored, and rec_lr is Adam's step in z units, so the
        momentum path's values do not carry over.  None runs the momentum update.
        huber_delta (> 0, +inf allowed; see check_huber_delta): the Huber data term instead of the squared error
        (dgan_reconstruct_huber, with any of pixel_weights, prune and adam): residuals beyond delta count linearly, so a
        few badly wrong pixels pull the fit less.  With momentum the gradient of clipped residuals shrinks with delta, so
        rec_lr has to grow as delta falls; Adam is invariant to that scale.  None runs the squared error, through exactly
        the entry and arguments it always did.
        z_prior (lambda >= 0, see check_z_prior): each restart minimises J = D + lambda ||z||^2, a Gaussian prior on z that
        keeps it where the generator was trained (dgan_reconstruct_prior, with any of pixel_weights, prune, adam and
        huber_delta).  D keeps its 1/HWC normaliser, so lambda is relative to the mean loss: the lambda of a formulation on
        the unnormalised sum does not carry over.  The returned loss is J, the restart is J's arg-min and prune ranks by
        J.  0.0 runs the prior entry and gives the bits of the call without it; None runs the call without the prior,
        through exactly the entry and arguments it always did.
        sparse_dev ((l1, step), see check_sparse_dev): fit G(z) + nu with an l1 penalty on a per-pixel deviation nu
        (Sparse-Gen; dgan_reconstruct_sparse_dev, with any of pixel_weights, prune, adam, huber_delta and z_prior): a few
        pixels G cannot produce (occluders, dead pixels, impulse noise) go into nu instead of dragging z.  The returned
        image stays G(z) of the chosen restart, the returned loss is J = D(G(z) + nu) [+ lambda ||z||^2] + l1 ||nu||_1;
        deviation_out (a [B,H,W,C] float32 CUDA tensor, 16-byte aligned) receives that restart's nu.  step = 1 with the
        squared error is the exact minimiser over nu per step, which treats residuals beyond l1 * H*W*C / 2 as
        deviations.  None runs the call without deviations, through exactly the entry and arguments it always did."""
        x = _require_cuda_f32(images, "images")
        batch = x.shape[0]
        if x.numel() != batch * self.hwc:
            raise ValueError("images must be [B,%d,%d,%d]" % self.image_dim)
        if rec_rr <= 0 or rec_iters <= 0 or batch <= 0:
            raise ValueError("batch, rec_rr and rec_iters must be positive")
        pw = self._pixel_weights(pixel_weights, batch)
        rec, loss, idx = self._project("image", (_ptr(x), _ptr(pw)), batch, self.hwc, rec_rr, rec_iters, rec_lr, z_init_val,
                                       seed, momentum, decay_lr, out, z_row_offset, prune, adam, huber_delta, z_prior,
                                       sparse_dev, deviation_out, weighted=pw is not None)
        rec = rec.view(images.shape) if out is None else rec
        if return_aux:
            return rec, loss, idx
        return rec

    def _project(self, kind: str, operands, batch: int, m: int, rec_rr: int, rec_iters: int, rec_lr: float, z_init_val,
                 seed: int, momentum: float, decay_lr: bool, out, z_row_offset: int, prune, adam, huber_delta, z_prior,
                 sparse_dev, deviation_out, weighted: bool = False, nnz: int = -1, conv: Optional[dgan_conv_op] = None):
        """reconstruct and reconstruct_measured after their operator's checks: the options checked, then the call _route
        picks for the operator kind and its C arguments `operands` (m: the measurements, H*W*C for images).  Returns
        (rec [B*H*W*C], loss, idx)."""
        sched = self._schedule(prune, rec_rr, rec_iters)
        ap = self._adam(adam)
        delta = None if huber_delta is None else check_huber_delta(huber_delta)
        lam = None if z_prior is None else check_z_prior(z_prior)
        sd, dev = self._sparse_dev(sparse_dev, deviation_out, batch, m)
        z0 = None
        if z_init_val is not None:
            z0 = _require_cuda_f32(z_init_val, "z_init_val")
            if z0.numel() != batch * rec_rr * self.latent_dim:
                raise ValueError("z_init_val must be [B*rec_rr, latent_dim]")
        with torch.cuda.device(self.device):
            rec = out if out is not None else torch.empty((batch,) + self.image_dim, dtype=torch.float32, device=self.device)
            if not (rec.is_cuda and rec.dtype == torch.float32 and rec.is_contiguous() and rec.numel() == batch * self.hwc):
                raise ValueError("out must be a contiguous CUDA float32 tensor " +
                                 ("shaped like images" if kind == "image" else
                                  "of B*%d*%d*%d elements" % self.image_dim))
            _require_aligned_out(rec)
            loss = torch.empty(batch, dtype=torch.float32, device=self.device)
            idx = torch.empty(batch, dtype=torch.int32, device=self.device)
            sizer, sizer_args, entry, args = _route(kind, operands, m, nnz, conv, weighted, sched, ap, delta, lam, sd, dev)
            ws, need = self._workspace_of(sizer, sizer_args, batch, rec_rr)
            stream = torch.cuda.current_stream(self.device).cuda_stream
            prm = dgan_rec_params(batch, int(rec_rr), int(rec_iters), float(rec_lr), float(momentum), int(bool(decay_lr)),
                                  seed & (2 ** 64 - 1), int(z_row_offset))
            rc = getattr(self.lib, entry)(self._handle, ctypes.byref(prm), *args, _ptr(z0), _ptr(rec), _ptr(loss),
                                          _ptr(idx), ws, need, ctypes.c_void_p(stream))
            _check(self.lib, rc, entry)
        return rec, loss, idx

    def _schedule(self, prune, rec_rr: int, rec_iters: int):
        """A prune schedule as the dgan_prune_point array of the pruned entries (None stays None), checked with
        check_prune_schedule and refused with use_bn."""
        if prune is None:
            return None
        if self.use_bn:
            raise ValueError("restart pruning is not supported with use_bn: the batch statistics couple the rows")
        points = check_prune_schedule(prune, int(rec_rr), int(rec_iters))
        return (dgan_prune_point * len(points))(*[dgan_prune_point(it, keep) for it, keep in points])

    def _sparse_dev(self, sparse_dev, deviation_out, batch: int, n: int):
        """(dgan_sparse_dev or None, deviation_out or None) for the sparse-deviation entries: sparse_dev checked with
        check_sparse_dev for n values per row (H*W*C, or the measured m); deviation_out, which needs sparse_dev, a
        contiguous CUDA float32 tensor of batch * H*W*C elements, 16-byte aligned."""
        if sparse_dev is None:
            if deviation_out is not None:
                raise ValueError("deviation_out needs sparse_dev: without deviations there is nothing to return")
            return None, None
        sd = dgan_sparse_dev(*check_sparse_dev(sparse_dev, n))
        if deviation_out is not None:
            d = deviation_out
            if not (isinstance(d, torch.Tensor) and d.is_cuda and d.dtype == torch.float32 and d.is_contiguous() and
                    d.numel() == batch * self.hwc):
                raise ValueError("deviation_out must be a contiguous CUDA float32 tensor of B*%d*%d*%d elements"
                                 % self.image_dim)
            if d.data_ptr() % 16 != 0:
                raise ValueError("deviation_out must be 16-byte aligned: its data starts %d bytes past a 16-byte boundary"
                                 % (d.data_ptr() % 16))
        return sd, deviation_out

    @staticmethod
    def _adam(adam):
        """Adam's parameters as the dgan_adam_params of the Adam entries (None stays None), checked with
        check_adam_params."""
        if adam is None:
            return None
        return dgan_adam_params(*check_adam_params(adam))

    def _measured(self, measurements: torch.Tensor, operator: torch.Tensor):
        """(y, A, batch, m): the measurements as a contiguous CUDA float32 [batch, m] tensor and the operator as [m, H*W*C]
        (shapes only; the values are not checked here - DefenseGANBase.reconstruct_measured does)."""
        a = _require_cuda_f32(operator, "operator")
        y = _require_cuda_f32(measurements, "measurements")
        if a.dim() != 2 or a.shape[1] != self.hwc or not 1 <= a.shape[0] <= self.hwc:
            raise ValueError("operator must be [m, %d] with 1 <= m <= %d, got %s" % (self.hwc, self.hwc, tuple(a.shape)))
        m = a.shape[0]
        if y.dim() != 2 or y.shape[1] != m or y.shape[0] <= 0:
            raise ValueError("measurements must be [B, %d] (the operator's m), got %s" % (m, tuple(y.shape)))
        return y, a, y.shape[0], m

    def _measured_csr(self, measurements: torch.Tensor, operator: torch.Tensor):
        """(y, (row_ptr, col_idx, val, nnz), batch, m) for a torch sparse CSR operator [m, H*W*C]: the indices as int32
        (an nnz int32 cannot hold is refused), the values as float32, all contiguous on the GPU (shapes only; the
        contents are not checked here - DefenseGANBase.reconstruct_measured does, and the library stages an invalid
        CSR as the empty operator with NaN measurements)."""
        if operator.dim() != 2 or operator.dense_dim() != 0:
            raise ValueError("operator must be a 2-D, non-batched, non-hybrid CSR tensor, got %d dims (%d dense)"
                             % (operator.dim(), operator.dense_dim()))
        if operator.shape[1] != self.hwc or not 1 <= operator.shape[0] <= self.hwc:
            raise ValueError("operator must be [m, %d] with 1 <= m <= %d, got %s"
                             % (self.hwc, self.hwc, tuple(operator.shape)))
        m = operator.shape[0]
        crow, col, val = operator.crow_indices(), operator.col_indices(), operator.values()
        nnz = int(col.numel())
        if nnz > INT32_MAX:
            raise ValueError("operator has %d non-zeros; at most %d are supported (int32 indices)" % (nnz, INT32_MAX))
        y = _require_cuda_f32(measurements, "measurements")
        if y.dim() != 2 or y.shape[1] != m or y.shape[0] <= 0:
            raise ValueError("measurements must be [B, %d] (the operator's m), got %s" % (m, tuple(y.shape)))
        csr = (_require_cuda_i32(crow, "operator.crow_indices()"), _require_cuda_i32(col, "operator.col_indices()"),
               _require_cuda_f32(val, "operator.values()"), nnz)
        return y, csr, y.shape[0], m

    def _measured_conv(self, measurements: torch.Tensor, operator):
        """(y, kernels, op, batch, m) for a ConvOperator: the measurements as a contiguous CUDA float32 [batch, m] tensor,
        the kernels broadcast to [batch, kh, kw] on the GPU and the geometry as a dgan_conv_op (shapes only; the values
        are not checked here - DefenseGANBase.reconstruct_measured does)."""
        m = operator.num_measurements(self.image_dim)
        y = _require_cuda_f32(measurements, "measurements")
        if y.dim() != 2 or y.shape[1] != m or y.shape[0] <= 0:
            raise ValueError("measurements must be [B, %d] (the operator's m), got %s" % (m, tuple(y.shape)))
        batch = y.shape[0]
        k = _require_cuda_f32(operator.kernels(batch, y.device), "operator kernels")
        kh, kw = operator.kernel_size
        op = dgan_conv_op(kh, kw, operator.padding[0], operator.padding[1], operator.stride)
        return y, k, op, batch, m

    def reconstruct_measured(self, measurements: torch.Tensor, operator: torch.Tensor, rec_rr: int, rec_iters: int,
                             rec_lr: float = 10.0, z_init_val: Optional[torch.Tensor] = None, seed: int = 0,
                             momentum: float = 0.7, decay_lr: bool = False, out: Optional[torch.Tensor] = None,
                             return_aux: bool = False, z_row_offset: int = 0,
                             prune: Optional[Sequence[Sequence[int]]] = None, adam: Optional[Sequence[float]] = None,
                             huber_delta: Optional[float] = None, z_prior: Optional[float] = None, sparse_dev=None,
                             deviation_out: Optional[torch.Tensor] = None):
        """The projection of reconstruct fitted to linear measurements (dgan_reconstruct_measured): measurements y
        [B, m] of images through operator A [m, H*W*C] (NHWC pixel order, 1 <= m <= H*W*C, shared by every image and
        restart).  Each restart minimises (1/m) ||A G(z) - y_i||^2; the R restarts of image i share y_i.  Returns G(z) of
        the arg-min restart as [B, H, W, C] (with return_aux also the minimum measured loss [B] and the restart [B]).
        A torch sparse CSR operator (operator.layout == torch.sparse_csr, columns strictly ascending within each row)
        runs dgan_reconstruct_measured_csr: the same semantics, at a cost set by its non-zeros.
        prune (a sequence of (iter, keep) pairs, see check_prune_schedule): restart pruning as in reconstruct, ranked by
        the measured loss (dgan_reconstruct_measured_pruned, or dgan_reconstruct_measured_csr_pruned for a CSR operator).
        None runs every restart to the end.
        adam ((beta1, beta2, eps)): the Adam update of reconstruct (dgan_reconstruct_measured_adam, or
        dgan_reconstruct_measured_csr_adam for a CSR operator), with or without prune.
        huber_delta: the Huber loss of reconstruct on the measurement residuals, (1/m) sum_j rho_delta(r_j)
        (dgan_reconstruct_measured_huber, or dgan_reconstruct_measured_csr_huber for a CSR operator), with any of prune
        and adam.  None runs the squared error as before.
        A defensegan_b200.operators.ConvOperator runs dgan_reconstruct_measured_conv: a convolution with one kernel per
        image (a shared kernel is passed as B copies), applied as a stencil, with any of prune, adam and huber_delta.
        z_prior: the latent prior of reconstruct, J = D + lambda ||z||^2 with D the measured loss and its 1/m normaliser
        (dgan_reconstruct_measured[_csr / _conv]_prior, with any of prune, adam and huber_delta); the lambda of a
        formulation on the unnormalised ||A G(z) - y||^2 is m times this one.  None runs the call without the prior as
        before.
        sparse_dev, deviation_out: the sparse deviations of reconstruct, fitting A (G(z) + nu) to y with D's 1/m
        normaliser (dgan_reconstruct_measured[_csr / _conv]_sparse_dev, with any of prune, adam, huber_delta and z_prior);
        nu lives in pixel space.  None runs the call without deviations as before."""
        nnz, conv = -1, None
        if isinstance(operator, ConvOperator):
            y, k, conv, batch, m = self._measured_conv(measurements, operator)
            kind, operands = "conv", (ctypes.byref(conv), _ptr(k), _ptr(y))
        elif operator.layout == torch.sparse_csr:
            y, (rp, ci, val, nnz), batch, m = self._measured_csr(measurements, operator)
            kind, operands = "csr", (_ptr(rp), _ptr(ci), _ptr(val), m, nnz, _ptr(y))
        else:
            y, a, batch, m = self._measured(measurements, operator)
            kind, operands = "dense", (_ptr(a), m, _ptr(y))
        if rec_rr <= 0 or rec_iters <= 0:
            raise ValueError("rec_rr and rec_iters must be positive")
        rec, loss, idx = self._project(kind, operands, batch, m, rec_rr, rec_iters, rec_lr, z_init_val, seed, momentum,
                                       decay_lr, out, z_row_offset, prune, adam, huber_delta, z_prior, sparse_dev,
                                       deviation_out, nnz=nnz, conv=conv)
        if return_aux:
            return rec, loss, idx
        return rec

    def loss_grad_measured(self, measurements: torch.Tensor, operator: torch.Tensor, z: torch.Tensor, rec_rr: int,
                           huber_delta: Optional[float] = None):
        """(G(z), per-row measured loss, d(sum loss)/dz) at z [B*rec_rr, latent] for measurements [B, m] through operator
        [m, H*W*C]: one evaluation of reconstruct_measured's loop body (dgan_loss_grad_measured, or
        dgan_loss_grad_measured_csr for a torch sparse CSR operator).  huber_delta: with the Huber loss of
        reconstruct_measured (dgan_loss_grad_measured[_csr]_huber); None: the squared error.  A ConvOperator runs
        dgan_loss_grad_measured_conv."""
        if isinstance(operator, ConvOperator):
            y, k, conv, batch, m = self._measured_conv(measurements, operator)
            return self._loss_grad("conv", (ctypes.byref(conv), _ptr(k), _ptr(y)), batch, z, rec_rr, huber_delta,
                                   conv=conv)
        if operator.layout == torch.sparse_csr:
            y, (rp, ci, val, nnz), batch, m = self._measured_csr(measurements, operator)
            return self._loss_grad("csr", (_ptr(rp), _ptr(ci), _ptr(val), m, nnz, _ptr(y)), batch, z, rec_rr, huber_delta,
                                   m=m, nnz=nnz)
        y, a, batch, m = self._measured(measurements, operator)
        return self._loss_grad("dense", (_ptr(a), m, _ptr(y)), batch, z, rec_rr, huber_delta, m=m)

    def _loss_grad(self, kind: str, operands, batch: int, z: torch.Tensor, rec_rr: int, huber_delta, pixel_weights=None,
                   m: int = 0, nnz: int = -1, conv: Optional[dgan_conv_op] = None):
        """loss_grad and loss_grad_measured after their operator's checks: (G(z), per-row loss, d(sum loss)/dz) from
        dgan_loss_grad[_weighted / _huber] for images (operands: the images; pixel_weights are checked here) or
        dgan_loss_grad_measured[_csr / _conv][_huber] (operands as _route's)."""
        zc = _require_cuda_f32(z, "z")
        n = batch * rec_rr
        if zc.shape[0] != n:
            raise ValueError("z must have batch*rec_rr rows")
        pw = self._pixel_weights(pixel_weights, batch)
        delta = None if huber_delta is None else check_huber_delta(huber_delta)
        if kind == "image":
            operands = (operands[0], _ptr(pw))
        entry = "dgan_loss_grad" + _ENTRY_OF_KIND[kind]
        if kind == "conv":
            operands = (_float_ref(delta),) + operands
        elif delta is not None:
            entry, operands = entry + "_huber", (delta,) + operands
        elif pw is not None:
            entry += "_weighted"
        elif kind == "image":
            operands = operands[:1]                  # dgan_loss_grad takes no weights
        with torch.cuda.device(self.device):
            g = torch.empty((n,) + self.image_dim, dtype=torch.float32, device=self.device)
            loss = torch.empty(n, dtype=torch.float32, device=self.device)
            grad = torch.empty(n, self.latent_dim, dtype=torch.float32, device=self.device)
            ws, need = self._workspace_of(*_route(kind, m=m, nnz=nnz, conv=conv, weighted=pw is not None)[:2], batch,
                                          rec_rr)
            stream = torch.cuda.current_stream(self.device).cuda_stream
            _check(self.lib, getattr(self.lib, entry)(self._handle, *operands, batch, rec_rr, _ptr(zc), _ptr(g),
                                                      _ptr(loss), _ptr(grad), ws, need, ctypes.c_void_p(stream)), entry)
        return g, loss, grad

    def sample_z0(self, n_rows: int, seed: int, z_row_offset: int = 0) -> torch.Tensor:
        """Rows [z_row_offset, z_row_offset + n_rows) of the N(0, 1/latent_dim) Philox stream `seed` - the z0 that
        reconstruct(..., z_init_val=None, seed=seed) starts from (reference models/gan.py:370-377)."""
        with torch.cuda.device(self.device):
            z = torch.empty(int(n_rows), self.latent_dim, dtype=torch.float32, device=self.device)
            stream = torch.cuda.current_stream(self.device).cuda_stream
            _check(self.lib, self.lib.dgan_sample_z0(self._handle, ctypes.c_uint64(seed & (2 ** 64 - 1)),
                                                     ctypes.c_uint64(int(z_row_offset)), int(n_rows), _ptr(z),
                                                     ctypes.c_void_p(stream)), "dgan_sample_z0")
        return z

    def forward(self, z: torch.Tensor) -> torch.Tensor:
        zc = _require_cuda_f32(z, "z")
        n = zc.shape[0]
        with torch.cuda.device(self.device):
            y = torch.empty((n,) + self.image_dim, dtype=torch.float32, device=self.device)
            ws, need = self._workspace(n, 1)
            stream = torch.cuda.current_stream(self.device).cuda_stream
            _check(self.lib, self.lib.dgan_forward(self._handle, _ptr(zc), n, _ptr(y), ws, need, ctypes.c_void_p(stream)),
                   "dgan_forward")
        return y

    def _pixel_weights(self, pixel_weights: Optional[torch.Tensor], batch: int) -> Optional[torch.Tensor]:
        """The weights as a contiguous CUDA float32 [batch, H, W, C] tensor (None stays None)."""
        if pixel_weights is None:
            return None
        pw = _require_cuda_f32(pixel_weights, "pixel_weights")
        if pw.numel() != batch * self.hwc or pw.shape[0] != batch:
            raise ValueError("pixel_weights must be [B,%d,%d,%d] like the images" % self.image_dim)
        return pw

    def loss_grad(self, images: torch.Tensor, z: torch.Tensor, rec_rr: int, pixel_weights: Optional[torch.Tensor] = None,
                  huber_delta: Optional[float] = None):
        """(G(z), per-row loss, d(sum loss)/dz) at z [batch*rec_rr, latent]; with pixel_weights [B,H,W,C] the loss is the
        weighted one of reconstruct (dgan_loss_grad_weighted); with huber_delta the Huber loss of reconstruct, weighted or
        not (dgan_loss_grad_huber)."""
        x = _require_cuda_f32(images, "images")
        return self._loss_grad("image", (_ptr(x),), x.shape[0], z, rec_rr, huber_delta, pixel_weights)

    def vjp(self, z: torch.Tensor, dy: torch.Tensor, want_y: bool = False):
        """Vector-Jacobian product of the generator at z: dz = (dG/dz)^T dy for a cotangent dy shaped like G(z)
        ([N,H,W,C] or [N,H*W*C]).  The forward is recomputed; with want_y it is returned too, as (y, dz), bit-identical
        to forward(z).  With use_bn the batch statistics of the N rows are differentiated."""
        zc = _require_cuda_f32(z, "z")
        dyc = _require_cuda_f32(dy, "dy")
        n = zc.shape[0]
        if zc.numel() != n * self.latent_dim:
            raise ValueError("z must be [N, %d]" % self.latent_dim)
        if dyc.numel() != n * self.hwc or dyc.shape[0] != n:
            raise ValueError("dy must be [N,%d,%d,%d] with the rows of z" % self.image_dim)
        with torch.cuda.device(self.device):
            y = torch.empty((n,) + self.image_dim, dtype=torch.float32, device=self.device) if want_y else None
            dz = torch.empty(n, self.latent_dim, dtype=torch.float32, device=self.device)
            ws, need = self._workspace(n, 1)
            stream = torch.cuda.current_stream(self.device).cuda_stream
            _check(self.lib, self.lib.dgan_vjp(self._handle, _ptr(zc), n, _ptr(dyc), _ptr(y), _ptr(dz), ws, need,
                                               ctypes.c_void_p(stream)), "dgan_vjp")
        return (y, dz) if want_y else dz

    def jvp(self, z: torch.Tensor, t: torch.Tensor, want_y: bool = False):
        """Jacobian-vector product of the generator at z: ty = (dG/dz) t for a tangent t shaped like z ([N, latent_dim]),
        returned as [N,H,W,C].  The forward is recomputed; with want_y it is returned too, as (y, ty), bit-identical to
        forward(z).  With use_bn the batch statistics of the N rows are differentiated."""
        zc = _require_cuda_f32(z, "z")
        tc = _require_cuda_f32(t, "t")
        n = zc.shape[0]
        if zc.numel() != n * self.latent_dim:
            raise ValueError("z must be [N, %d]" % self.latent_dim)
        if tc.numel() != n * self.latent_dim or tc.shape[0] != n:
            raise ValueError("t must be [N, %d] with the rows of z" % self.latent_dim)
        with torch.cuda.device(self.device):
            y = torch.empty((n,) + self.image_dim, dtype=torch.float32, device=self.device) if want_y else None
            ty = torch.empty((n,) + self.image_dim, dtype=torch.float32, device=self.device)
            ws, need = self._workspace(n, 1)
            stream = torch.cuda.current_stream(self.device).cuda_stream
            _check(self.lib, self.lib.dgan_jvp(self._handle, _ptr(zc), n, _ptr(tc), _ptr(y), _ptr(ty), ws, need,
                                               ctypes.c_void_p(stream)), "dgan_jvp")
        return (y, ty) if want_y else ty

    def jacobian(self, z: torch.Tensor, max_rows: int = 4096) -> torch.Tensor:
        """dG/dz at each row of z ([N, latent_dim]) as [N, H, W, C, latent_dim]: column k of image i is jvp(z_i, e_k).
        Runs jvp on each row repeated latent_dim times with identity tangents, whole images per call and at most
        max_rows (at least one image) rows per call; rows are independent, so the chunking does not change a bit.
        Refused with use_bn: the batch statistics couple the rows, so G has no per-row Jacobian."""
        if self.use_bn:
            raise ValueError("generator_jacobian is undefined with BatchNorm (use_bn): its batch statistics couple the "
                             "rows, so the Jacobian of one row depends on the others")
        zc = _require_cuda_f32(z, "z")
        n, k = zc.shape[0], self.latent_dim
        if zc.numel() != n * k:
            raise ValueError("z must be [N, %d]" % k)
        per_call = max(1, int(max_rows) // k)
        eye = torch.eye(k, dtype=torch.float32, device=zc.device)
        out = torch.empty((n, k) + self.image_dim, dtype=torch.float32, device=zc.device)
        for i in range(0, n, per_call):
            m = min(per_call, n - i)
            rows = zc.view(n, k)[i:i + m].repeat_interleave(k, dim=0)
            out[i:i + m] = self.jvp(rows, eye.repeat(m, 1)).view((m, k) + self.image_dim)
        return out.movedim(1, -1).contiguous()


class GeneratorFunction(torch.autograd.Function):
    """y = G(z) through a NativeGenerator (or anything with its forward / vjp / jvp methods), differentiable in z in
    both modes.  The backward recomputes the forward inside `native.vjp`, and the forward-mode rule (`jvp`, used by
    torch.autograd.forward_ad and torch.func.jvp) recomputes it inside `native.jvp`, so a forward-mode call computes G(z)
    twice; both run on the current stream.  The weights are frozen (no gradient), as in the projection.  Only first
    derivatives are available."""

    @staticmethod
    def forward(z, native):
        return native.forward(z)

    @staticmethod
    def setup_context(ctx, inputs, output):
        z, native = inputs
        ctx.native = native
        ctx.save_for_backward(z)
        ctx.save_for_forward(z)

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        (z,) = ctx.saved_tensors
        return ctx.native.vjp(z, dy).reshape(z.shape), None

    @staticmethod
    def jvp(ctx, t, _native_t):
        (z,) = ctx.saved_tensors
        z, t = _unwrap_functorch(z), _unwrap_functorch(t)
        with torch._C._DisableFuncTorch():      # the result buffers must be plain tensors too
            return ctx.native.jvp(z, t)


def _is_functorch_wrapped(z: torch.Tensor) -> bool:
    return bool(torch._C._functorch.is_functorch_wrapped_tensor(z))


def _unwrap_functorch(t: torch.Tensor) -> torch.Tensor:
    """Under torch.func.jvp the forward-mode rule receives functorch-wrapped tensors, which have no storage of their own
    (and tensors it allocates would be wrapped too, unless functorch is disabled); the library reads the tensor they
    wrap."""
    while _is_functorch_wrapped(t):
        t = torch._C._functorch.get_unwrapped(t)
    return t


def generator(native, z: torch.Tensor) -> torch.Tensor:
    """G(z): a tensor with a grad_fn when z requires grad and grad mode is on, a dual tensor carrying J t when z carries a
    forward tangent t (torch.autograd.forward_ad, torch.func.jvp), else exactly native.forward(z)."""
    if ((z.requires_grad and torch.is_grad_enabled()) or _is_functorch_wrapped(z)
            or fwAD.unpack_dual(z).tangent is not None):
        return GeneratorFunction.apply(z, native)
    return native.forward(z)
