"""GPU tests (H100, -m gpu): every layer-direction of the generator checked on its own, against an fp64 reference computed
from the operands the kernel read - its input buffer as the workspace holds it after the call, and the caller's weights
rounded as the handle rounds them - so the only differences left are the kernel's fp32 accumulation order and its output
rounding (tests/layer_ref.py states the bound and the layouts).  The end-to-end tests compare the whole generator, where
fp16 rounding flips ReLU masks and a few percent of error is real; here a missing tap or k-chunk, a wrong weight tile,
mask word or row tile moves elements by far more than the bound, and the failure names the layer-direction, pixel, row,
channel and column block.

Covered, on both precisions, over the matrix below at 1, 300 and 2560 rows:
  dgan_loss_grad (also under every accumulator-slot count the kernel instantiations offer): each GEMM layer's forward
  (with BatchNorm: the fp32 pre-activations as a GEMM, then the stored activations as the batch-statistics BatchNorm of
  the stored pre-activations) and its ReLU masks; the last layer's forward (y, the loss part of every 4x4 block, the
  scaled d(pre)); every backward layer-direction, including the narrow last-layer backward, the split-K Linear
  backward's partial sums, and the backward GEMMs into BatchNorm outputs, checked together with the BatchNorm backward
  that overwrites them in place (the GEMM output's one rounding carried through the BatchNorm map);
  dgan_vjp: the cotangent entry (d(pre) from dy and the stored y, the power-of-two row scales, zeroed tile-padding rows)
  and every backward layer-direction from there;
  dgan_jvp: the tangent entry (z_h = RN16(t * s_n), or v = t), every tangent direction masked by the primal forward's
  masks or through the BatchNorm tangent, the last layer's fp32 tangent of pre and ty = t(pre) * act'(y) / s_n;
  dgan_reconstruct with L = 2: the momentum update (v, z, z_h, the tail's self-resetting counters).
Padded channels of every buffer must be exactly 0.  Real rows are compared with references computed from the real rows
alone, while the tile-padding rows hold non-zero activations (relu(bias)), so no real output depends on them.

Measured on an H100 80GB HBM3 SXM (700 W power limit) over the whole matrix (-s prints the table per case), largest error
beyond the output rounding over its bound: fp16 GEMM outputs 0.058 (Linear.jvp), the narrow last-layer backward 0.13,
the Linear's fp32 BatchNorm pre-activations 0.18, GEMM + BatchNorm outputs 0.85 (last.bwd into MNIST's BatchNorm'd
Generator.3: the bound there is mostly the GEMM output's fp16 rounding, which the kernel does make), the cotangent entry
0.27, ty 0.31, the updated z 0.25 (v exact); on the fp32 path 0.31 at most.  Between 99.2% and 99.97% of the fp16
outputs of a plain GEMM layer-direction are bit-equal to RN16 of the fp64 reference (98.1% for the BatchNorm'd Linear;
60-87% for GEMM + BatchNorm outputs, rounded twice).  No ratio reaches 1: tensor-core fp32 accumulation stays well inside
one rounding per k16 MMA here."""
import ctypes

import numpy as np
import pytest
import torch

import layer_ref as R
from gpu_support import MATRIX, ROWS, gen, read_call
from oracle import defensegan_oracle as O

pytestmark = pytest.mark.gpu


def run_loss_grad(native, w, arch, latent, n_rows, seed=3):
    R_ = 1 if n_rows == 1 else 2
    B = n_rows // R_
    imgs = torch.tensor(O.synthetic_images(arch, w, B, kind="S2", seed=seed, latent_dim=latent)).cuda()
    z = torch.tensor(O.sample_z0(n_rows, latent, seed=seed + 1)).cuda()
    native.loss_grad(imgs, z, R_)
    torch.cuda.synchronize()
    x_rows = imgs.reshape(B, -1).repeat_interleave(R_, dim=0)
    return z, x_rows


@pytest.mark.parametrize("n_rows", ROWS)
@pytest.mark.parametrize("precision", ["fp16", "fp32"])
@pytest.mark.parametrize("arch,latent,net_dim,use_bn", MATRIX)
def test_loss_grad_each_layer_direction(arch, latent, net_dim, use_bn, precision, n_rows):
    w, native = gen(arch, precision, use_bn, latent, net_dim)
    try:
        z, x_rows = run_loss_grad(native, w, arch, latent, n_rows)
        ws, net = read_call(native, w, arch, latent, net_dim, use_bn, precision, n_rows)
        stats = R.Stats()
        R.check_inputs(net, ws, n_rows, z)
        R.check_forward(net, ws, n_rows, stats, "")
        R.check_last_fwd(net, ws, n_rows, x_rows, stats, "")
        R.check_backward(net, ws, n_rows, stats, "")
        print("\n%s %s latent=%d net_dim=%d bn=%d rows=%d" % (precision, arch, latent, net_dim, use_bn, n_rows))
        print("\n".join(stats.lines()))
    finally:
        native.close()


def test_every_slot_count_matches_fp64_per_layer():
    """Every instantiation of the tensor-core kernel a layer-direction can be planned on (dgan_debug_force_slots), each
    checked against the fp64 reference rather than only against the default plan."""
    arch, latent, net_dim, use_bn, n_rows = "mnist", 128, 64, False, 300
    w, native = gen(arch, "fp16", use_bn, latent, net_dim)
    lib = native.lib
    lib.dgan_debug_slot_choices.restype = ctypes.c_int
    lib.dgan_debug_slot_choices.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.POINTER(ctypes.c_int), ctypes.c_int]
    lib.dgan_debug_force_slots.restype = ctypes.c_int
    lib.dgan_debug_force_slots.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int]
    try:
        stats = R.Stats()
        n_dirs = int(lib.dgan_profile_num_kinds(native._handle)) - 1
        tried = 0
        for d in range(n_dirs):
            buf = (ctypes.c_int * 16)()
            for maxb in list(buf[:lib.dgan_debug_slot_choices(native._handle, d, buf, 16)]):
                assert lib.dgan_debug_force_slots(native._handle, d, maxb) == 0, lib.dgan_last_error()
                z, x_rows = run_loss_grad(native, w, arch, latent, n_rows)
                ws, net = read_call(native, w, arch, latent, net_dim, use_bn, "fp16", n_rows)
                tag = "[dir %d, %d slots] " % (d, maxb)
                R.check_forward(net, ws, n_rows, stats, tag)
                R.check_last_fwd(net, ws, n_rows, x_rows, stats, tag)
                R.check_backward(net, ws, n_rows, stats, tag)
                tried += 1
            assert lib.dgan_debug_force_slots(native._handle, d, 0) == 0
        assert tried > n_dirs
        print("\n" + "\n".join(stats.lines()))
    finally:
        native.close()


@pytest.mark.parametrize("n_rows", ROWS)
@pytest.mark.parametrize("precision", ["fp16", "fp32"])
@pytest.mark.parametrize("arch,latent,net_dim,use_bn", MATRIX)
def test_vjp_each_layer_direction(arch, latent, net_dim, use_bn, precision, n_rows):
    """dgan_vjp: the cotangent entry (d(pre) from dy and the stored y, its power-of-two row scales, zeroed tile-padding
    rows), the forward it recomputes, and every backward layer-direction from there."""
    w, native = gen(arch, precision, use_bn, latent, net_dim)
    try:
        g = torch.Generator().manual_seed(n_rows)
        z = torch.tensor(O.sample_z0(n_rows, latent, seed=7)).cuda()
        dy = (torch.randn((n_rows,) + native.image_dim, generator=g) * 0.3).cuda()
        native.vjp(z, dy)
        torch.cuda.synchronize()
        ws, net = read_call(native, w, arch, latent, net_dim, use_bn, precision, n_rows)
        stats = R.Stats()
        R.check_forward(net, ws, n_rows, stats, "")
        R.check_cotangent(net, ws, n_rows, dy, stats, "")
        R.check_backward(net, ws, n_rows, stats, "")
        print("\nvjp %s %s latent=%d net_dim=%d bn=%d rows=%d" % (precision, arch, latent, net_dim, use_bn, n_rows))
        print("\n".join(stats.lines()))
    finally:
        native.close()


@pytest.mark.parametrize("n_rows", ROWS)
@pytest.mark.parametrize("precision", ["fp16", "fp32"])
@pytest.mark.parametrize("arch,latent,net_dim,use_bn", MATRIX)
def test_jvp_each_layer_direction(arch, latent, net_dim, use_bn, precision, n_rows):
    """dgan_jvp: the tangent entry (z_h = RN16(t * s_n), or v = t), every tangent direction on its stored input (masked by
    the primal masks, or through the BatchNorm tangent), the last layer's fp32 tangent of pre and ty."""
    w, native = gen(arch, precision, use_bn, latent, net_dim)
    try:
        g = torch.Generator().manual_seed(n_rows + 1)
        z = torch.tensor(O.sample_z0(n_rows, latent, seed=8)).cuda()
        t = (torch.randn(n_rows, latent, generator=g) * 3.0).cuda()
        ty = native.jvp(z, t)
        torch.cuda.synchronize()
        ws, net = read_call(native, w, arch, latent, net_dim, use_bn, precision, n_rows)
        stats = R.Stats()
        # the tangent of z replaced z_h once the primal Linear had read it
        R.check_forward(net, ws, n_rows, stats, "", skip=("Linear.fwd",) if precision == "fp16" else ())
        R.check_tangent(net, ws, n_rows, t, ty, stats, "")
        print("\njvp %s %s latent=%d net_dim=%d bn=%d rows=%d" % (precision, arch, latent, net_dim, use_bn, n_rows))
        print("\n".join(stats.lines()))
    finally:
        native.close()


@pytest.mark.parametrize("precision", ["fp16", "fp32"])
@pytest.mark.parametrize("arch,latent,net_dim,use_bn", [MATRIX[0], MATRIX[2], MATRIX[5], MATRIX[6]])
def test_momentum_update_after_one_step(arch, latent, net_dim, use_bn, precision):
    """dgan_reconstruct with L = 2 from a given z0: the first step's partial sums stay in g, and z, v, z_h hold the update
    (the tail of the tensor-core Linear backward, or the fp32 path's momentum kernel); the partial sums themselves are
    checked as the Linear backward of the stored d(pre_0)."""
    w, native = gen(arch, precision, use_bn, latent, net_dim)
    try:
        B, Rr, lr = 150, 2, 10.0
        n = B * Rr
        x = torch.tensor(O.synthetic_images(arch, w, B, kind="S2", seed=9, latent_dim=latent)).cuda()
        z0 = torch.tensor(O.sample_z0(n, latent, seed=10)).cuda()
        native.reconstruct(x, Rr, 2, lr, z_init_val=z0, momentum=0.7)
        torch.cuda.synchronize()
        ws, net = read_call(native, w, arch, latent, net_dim, use_bn, precision, n)
        stats = R.Stats()
        R.check_linear_bwd(net, ws, n, stats, "")
        R.check_momentum(net, ws, z0, lr, 0.7, native.hwc, stats, "")
        print("\nmomentum %s %s latent=%d net_dim=%d bn=%d" % (precision, arch, latent, net_dim, use_bn))
        print("\n".join(stats.lines()))
    finally:
        native.close()
