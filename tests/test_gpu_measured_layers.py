"""GPU tests (H100, -m gpu) of the projection from linear measurements layer by layer, at every width of
test_gpu_layers.py's matrix, with and without BatchNorm, on both precisions:
  - each layer-direction of dgan_loss_grad_measured at 1, 300 and 2560 rows against fp64 on the operands it read
    (tests/layer_ref.py): the inputs at the padded latent width, every forward layer-direction, the last layer's
    output y = G(z), the measurement and adjoint products (test_gpu_measured.py's bound), the measured loss of each row
    from the stored residuals, the cotangent entry from the stored dy = (2/m) A^T r with its power-of-two row scales in
    `mscale`, and every backward layer-direction;
  - the measured loop's momentum update (momentum_rows_kernel) after one step of dgan_reconstruct_measured;
  - loss_grad_measured and a short reconstruct_measured loop at the padded widths against the fp64 oracle;
  - exact homogeneity in the operator's scale: A and y times 2^k give G bit for bit, and loss and gradient exactly 4^k
    times; with rec_lr 4^-k times, the loop returns the same rec and idx bit for bit;
  - degenerate operators: A = 0 gives a zero gradient, a loop that stays at z0, restart 0 and loss sum(y^2) / m; a
    repeated row of A is its row scaled by sqrt(2) at the normaliser m + 1;
  - a reconstruction buffer that is not 16-byte aligned is refused by every reconstruct entry, before anything runs.
-s prints, per case, the largest error over its bound of every layer-direction (test_gpu_layers.py's format).

Measured on an H100 80GB HBM3 (700 W power limit) over the whole matrix, largest error beyond the output rounding over
its bound: fp16 plain GEMM layer-directions 0.05 at most (the narrow last-layer backward 0.14), GEMM + BatchNorm outputs
0.85 (last.bwd into MNIST's BatchNorm'd Generator.3, as in test_gpu_layers.py), the cotangent entry 0.26, the
measurement product 0.066, the adjoint product 0.85 (m = 1: one product of two TF32-rounded operands, which nearly
reaches their 2^-10), y 0.03, the measured loss 0.16, the updated z 0.25 (v exact); on the fp32 path 0.31 at most
(the cotangent entry; y 0.10, the measured loss 0.20).  At least 62%
of the fp16 outputs of every layer-direction are bit-equal to RN16 of the fp64 reference (the GEMM + BatchNorm outputs,
rounded twice; 99.2% or more for the plain GEMM layer-directions, 98% for the BatchNorm'd Linear).  The operator-scale
test holds bit for bit on both precisions."""
import ctypes

import numpy as np
import pytest
import torch

import layer_ref as R
import measured_oracle as MO
from gpu_support import HWC, MATRIX, ROWS, SHAPE, TOL, check_products, gen, layout, read_call, views
from gpu_support import release_cached_memory  # noqa: F401
from oracle import defensegan_oracle as O

pytestmark = pytest.mark.gpu

MEASURED = ("am", "amt", "ym", "r", "dym", "mloss_part", "mscale")


def _m(arch):
    """The sketch size: no multiple of the 64-column tile, several N tiles."""
    return 200 if arch == "mnist" else 1000


def _measure(a, x):
    """y = A x for images x [B, ...] (torch, on the GPU), in fp64, stored as fp32."""
    return (x.reshape(x.shape[0], -1).double() @ a.double().t()).float()


def _read(native, w, arch, latent, net_dim, use_bn, precision, n_rows, m):
    """The workspace of the last measured call: the common buffers (typed) and the measured ones, by name."""
    ws, net = read_call(native, w, arch, latent, net_dim, use_bn, precision, n_rows)
    wsm = views(native, layout(native, "_measured", n_rows, m)[0][0])
    for k in MEASURED:
        ws[k] = wsm[k]
    return ws, net


@pytest.mark.parametrize("precision", ["fp16", "fp32"])
@pytest.mark.parametrize("arch,latent,net_dim,use_bn", MATRIX)
def test_loss_grad_measured_each_layer_direction(arch, latent, net_dim, use_bn, precision):
    w, native = gen(arch, precision, use_bn, latent, net_dim)
    try:
        hwc = HWC[arch]
        for n_rows in ROWS:
            R_ = 1 if n_rows == 1 else 2
            B = n_rows // R_
            m = 1 if n_rows == 1 else _m(arch)
            imgs = torch.tensor(O.synthetic_images(arch, w, B, kind="S2", seed=3, latent_dim=latent)).cuda()
            a = torch.tensor(MO.gaussian_operator(m, hwc, seed=m)).cuda()
            y = _measure(a, imgs)
            z = torch.tensor(O.sample_z0(n_rows, latent, seed=4)).cuda()
            native.loss_grad_measured(y, a, z, R_)
            torch.cuda.synchronize()
            ws, net = _read(native, w, arch, latent, net_dim, use_bn, precision, n_rows, m)
            stats = R.Stats()
            R.check_inputs(net, ws, n_rows, z)
            R.check_forward(net, ws, n_rows, stats, "")
            R.check_last_y(net, ws, n_rows, stats, "")
            r_ratio, dy_ratio = check_products(ws, n_rows, R_, m, hwc, precision)
            stats.add("measurement product (r)", r_ratio, None)
            stats.add("adjoint product (dy)", dy_ratio, None)
            R.check_measured_loss(ws, n_rows, m, stats, "")
            R.check_cotangent(net, ws, n_rows, ws["dym"][:n_rows], stats, "", scale="mscale")
            R.check_backward(net, ws, n_rows, stats, "")
            print("\nmeasured %s %s latent=%d net_dim=%d bn=%d rows=%d m=%d"
                  % (precision, arch, latent, net_dim, use_bn, n_rows, m))
            print("\n".join(stats.lines()))
    finally:
        native.close()


@pytest.mark.parametrize("precision", ["fp16", "fp32"])
@pytest.mark.parametrize("arch,latent,net_dim,use_bn", [MATRIX[0], MATRIX[2], MATRIX[5], MATRIX[6]])
def test_momentum_rows_after_one_step(arch, latent, net_dim, use_bn, precision):
    """dgan_reconstruct_measured with L = 2 from a given z0.  After the loop, the step-0 values that the update read are
    still in the workspace: the L-1 iteration runs only the forward (act, mask, pre, y) and the measurement product
    (r, mloss_part), then the loss finish (loss) and the select.  So g, dact.0, mscale and the updated z, v, z_h are
    step 0's: the partial sums are checked as the Linear backward of the stored d(pre_0), then the update."""
    w, native = gen(arch, precision, use_bn, latent, net_dim)
    try:
        B, Rr, m = 150, 2, _m(arch)
        n = B * Rr
        lr = 10.0 * m / HWC[arch]
        x = torch.tensor(O.synthetic_images(arch, w, B, kind="S2", seed=9, latent_dim=latent)).cuda()
        a = torch.tensor(MO.gaussian_operator(m, HWC[arch], seed=5)).cuda()
        z0 = torch.tensor(O.sample_z0(n, latent, seed=10)).cuda()
        native.reconstruct_measured(_measure(a, x), a, Rr, 2, lr, z_init_val=z0, momentum=0.7)
        torch.cuda.synchronize()
        ws, net = _read(native, w, arch, latent, net_dim, use_bn, precision, n, m)
        stats = R.Stats()
        R.check_linear_bwd(net, ws, n, stats, "")
        R.check_momentum_rows(net, ws, z0, lr, 0.7, n, stats, "")
        print("\nmeasured momentum %s %s latent=%d net_dim=%d bn=%d" % (precision, arch, latent, net_dim, use_bn))
        print("\n".join(stats.lines()))
    finally:
        native.close()


# test_gpu_parity.py's BatchNorm golden cases (R = 2, L = 3, lr 0.5) and their tolerances: the batch statistics couple
# every row's rounding into every row
BN_TOL = {"fp32": dict(y=5e-5, loss=1e-5, grad=1e-3, rec=1e-3, lmin=1e-4),
          "fp16": dict(y=1e-2, loss=1e-3, grad=6e-2, rec=1e-1, lmin=1e-3)}


@pytest.mark.parametrize("precision", ["fp32", "fp16"])
@pytest.mark.parametrize("arch,latent,net_dim,use_bn", MATRIX)
def test_measured_calls_at_padded_widths(arch, latent, net_dim, use_bn, precision):
    """loss_grad_measured against the fp64 oracle and a short loop against the fp64 oracle's, at the matrix's widths:
    without BatchNorm (L = 6 at test_gpu_measured.py's step) within test_gpu_measured.py's tolerances, with BatchNorm
    (L = 3 at the golden cases' step lr 0.5, scaled by m / HWC as test_gpu_measured.py scales its steps) within
    test_gpu_parity.py's BatchNorm tolerances.  The BatchNorm rows run 8 MNIST or 4 CelebA images: with the 6 rows of
    3 MNIST images the problem itself is ill-conditioned (the fp32 and fp64 oracles' gradients differ by 1% of their
    largest element), and so is the CelebA loop of 2 images (0.8% between the oracles' reconstructions)."""
    w, native = gen(arch, precision, use_bn, latent, net_dim)
    try:
        if use_bn:
            B, R_ = (8, 2) if arch == "mnist" else (4, 2)
        else:
            B, R_ = (3, 2) if arch == "mnist" else (2, 2)
        m, hwc = _m(arch), HWC[arch]
        imgs = O.synthetic_images(arch, w, B, kind="S2", seed=5, latent_dim=latent)
        z = O.sample_z0(B * R_, latent, seed=6)
        a = MO.gaussian_operator(m, hwc, seed=3)
        y = (imgs.reshape(B, -1).astype(np.float64) @ a.T.astype(np.float64)).astype(np.float32)
        g64, loss64, grad64 = MO.loss_and_grad(arch, w, a, y, z, R_, use_bn=use_bn, dtype=torch.float64)
        g, loss, grad = native.loss_grad_measured(torch.tensor(y).cuda(), torch.tensor(a).cuda(), torch.tensor(z).cuda(), R_)
        g, loss, gr = g.cpu().numpy(), loss.cpu().numpy(), grad.cpu().numpy()
        gerr, lerr = np.abs(g - g64).max(), np.abs(loss - loss64).max() / max(1.0, float(np.abs(loss64).max()))
        grel = np.abs(gr - grad64).max() / np.abs(grad64).max()
        cos = float((gr * grad64).sum() / np.sqrt((gr * gr).sum() * (grad64 * grad64).sum()))
        if use_bn:
            t = BN_TOL[precision]
            L, lr = 3, 0.5 * m / hwc
            assert gerr <= t["y"] and lerr <= t["loss"] and grel <= t["grad"], (gerr, lerr, grel)
        else:
            t = TOL[precision]
            L, lr = 6, 10.0 * m / hwc
            assert gerr <= t["fwd"] and lerr <= t["loss"] and grel <= t["grad_rel"] and cos >= t["grad_cos"], \
                (gerr, lerr, grel, cos)
        z0 = O.sample_z0(B * R_, latent, seed=7)
        ref = MO.reconstruct(arch, w, a, y, R_, L, rec_lr=lr, z_init_val=z0, use_bn=use_bn, dtype=torch.float64)
        rec, lmin, idx = native.reconstruct_measured(torch.tensor(y).cuda(), torch.tensor(a).cuda(), R_, L, lr,
                                                     z_init_val=torch.tensor(z0).cuda(), return_aux=True)
        agree = idx.cpu().numpy() == ref["idx"]
        drec = np.abs(rec.cpu().numpy() - ref["rec"]).reshape(B, -1).max(axis=1)
        rerr = float(drec[agree].max()) if agree.any() else 0.0
        merr = float(np.abs(lmin.cpu().numpy() - ref["loss_min"]).max())
        print("\n%s %s latent=%d net_dim=%d bn=%d: |dG| %.2e |dloss| %.2e grad rel %.2e cos %.7f | loop L=%d |drec| %.2e "
              "|dloss_min| %.2e restart agreement %.2f" % (precision, arch, latent, net_dim, use_bn, gerr, lerr, grel,
                                                            cos, L, rerr, merr, agree.mean()))
        assert agree.all() if precision == "fp32" else agree.mean() >= 0.5
        if use_bn:
            assert rerr <= t["rec"] and merr <= t["lmin"], (rerr, merr)
        else:
            assert rerr <= t["fwd"] and merr <= t["loss"], (rerr, merr)
    finally:
        native.close()


@pytest.mark.parametrize("precision", ["fp16", "fp32"])
@pytest.mark.parametrize("arch,latent,net_dim,use_bn", [MATRIX[0], MATRIX[1], MATRIX[5]])
def test_operator_scale_is_exact(arch, latent, net_dim, use_bn, precision):
    """A and y times 2^k: every scaling is by a power of two - TF32 rounding commutes with it, the cotangent's row scale
    absorbs the 4^k of d(pre) exactly (on the fp32 path the backward is linear in it), no value leaves the normal fp32
    range at these k - so G is bit-identical and loss and gradient are exactly 4^k times the k = 0 result; with rec_lr
    4^-k times, every step moves z by the same bits, and rec, idx are bit-identical, the loss exactly 4^k times."""
    w, native = gen(arch, precision, use_bn, latent, net_dim)
    try:
        B, R_, L, m = 4, 3, 5, _m(arch)
        lr = 0.5 if use_bn else 10.0 * m / HWC[arch]
        x = torch.tensor(O.synthetic_images(arch, w, B, kind="S2", seed=2, latent_dim=latent)).cuda()
        a = torch.tensor(MO.gaussian_operator(m, HWC[arch], seed=8)).cuda()
        y = _measure(a, x)
        z0 = torch.tensor(O.sample_z0(B * R_, latent, seed=4)).cuda()
        g0, l0, d0 = [t.clone() for t in native.loss_grad_measured(y, a, z0, R_)]
        rec0, lm0, idx0 = [t.clone() for t in native.reconstruct_measured(y, a, R_, L, lr, z_init_val=z0, return_aux=True)]
        assert bool(d0.abs().max() > 0)
        for k in (-20, -6, 6, 20):
            s, s2 = 2.0 ** k, 4.0 ** k
            g, l, d = native.loss_grad_measured(y * s, a * s, z0, R_)
            assert torch.equal(g, g0), k
            assert torch.equal(l, l0 * s2), (k, float((l / l0).min()), float((l / l0).max()))
            assert torch.equal(d, d0 * s2), (k, float((d - d0 * s2).abs().max() / (d0 * s2).abs().max()))
            rec, lm, idx = native.reconstruct_measured(y * s, a * s, R_, L, lr / s2, z_init_val=z0, return_aux=True)
            assert torch.equal(rec, rec0) and torch.equal(idx, idx0), k
            assert torch.equal(lm, lm0 * s2), k
    finally:
        native.close()


@pytest.mark.parametrize("precision", ["fp16", "fp32"])
def test_zero_operator(precision):
    """A = 0 (m = 50), y != 0: r = -y whatever z is, so the gradient is exactly 0, the loop never leaves z0 (L = 7 returns
    L = 1's bits), every restart of an image has the same loss bits (restart 0 is chosen), and the loss is sum(y^2) / m
    as the kernels sum it: one partial per 64-column tile, the tiles in a fixed order - within the fp32 bound of any
    order of m + 1 additions and the two roundings of the 1/m multiply."""
    arch, latent, B, R_, m = "mnist", 128, 4, 3, 50
    w, native = gen(arch, precision, False, latent, 64)
    try:
        a = torch.zeros(m, HWC[arch], device="cuda")
        y = torch.randn(B, m, generator=torch.Generator().manual_seed(12)).cuda()
        z0 = torch.tensor(O.sample_z0(B * R_, latent, seed=4)).cuda()
        _, loss, grad = native.loss_grad_measured(y, a, z0, R_)
        assert torch.equal(grad, torch.zeros_like(grad))
        one = [t.clone() for t in native.reconstruct_measured(y, a, R_, 1, 10.0, z_init_val=z0, return_aux=True)]
        seven = native.reconstruct_measured(y, a, R_, 7, 10.0, z_init_val=z0, return_aux=True)
        assert all(torch.equal(p, q) for p, q in zip(one, seven))
        assert not bool(seven[2].any())
        y2 = (y.double() ** 2).sum(dim=1)
        want = y2 / m
        lim = (m + 3) * 2.0 ** -24 * want
        for got in (seven[1], loss.reshape(B, R_).t()):
            assert bool(((got.double() - want).abs() <= lim).all()), float(((got.double() - want).abs() / lim).max())
    finally:
        native.close()


@pytest.mark.parametrize("precision", ["fp16", "fp32"])
def test_repeated_row_is_the_row_scaled_by_sqrt2(precision):
    """A with row j repeated (and y_j) is, at the normaliser m + 1, the m-row operator with row j and y_j scaled by
    sqrt(2): its loss is m / (m + 1) times that one's, and with rec_lr (m + 1) / m times it takes the same steps."""
    arch, B, R_, L, m, j = "mnist", 4, 3, 8, 64, 5
    w, native = gen(arch, precision, False, 128, 64)
    try:
        x = torch.tensor(O.synthetic_images(arch, w, B, kind="S2", seed=2)).cuda()
        z0 = torch.tensor(O.sample_z0(B * R_, 128, seed=4)).cuda()
        a = torch.tensor(MO.gaussian_operator(m, 784, seed=9)).cuda()
        y = _measure(a, x)
        lr = 10.0 * m / 784
        a2, y2 = a.clone(), y.clone()
        a2[j] *= 2.0 ** 0.5
        y2[:, j] *= 2.0 ** 0.5
        rec, loss, idx = native.reconstruct_measured(y2, a2, R_, L, lr, z_init_val=z0, return_aux=True)
        rec, loss, idx = rec.clone(), loss.clone(), idx.clone()
        ar = torch.cat([a, a[j:j + 1]])
        yr = torch.cat([y, y[:, j:j + 1]], dim=1)
        rec1, loss1, idx1 = native.reconstruct_measured(yr, ar, R_, L, lr * (m + 1) / m, z_init_val=z0, return_aux=True)
        t = TOL[precision]
        print("\n%s: |drec| %.3g |dloss| %.3g" % (precision, float((rec1 - rec).abs().max()),
                                                  float((loss1 * (m + 1) / m - loss).abs().max())))
        assert float((rec1 - rec).abs().max()) <= t["fwd"]
        assert float((loss1 * (m + 1) / m - loss).abs().max()) <= t["loss"]
        assert torch.equal(idx1, idx)
    finally:
        native.close()


@pytest.mark.parametrize("precision", ["fp16", "fp32"])
def test_misaligned_out_is_refused(precision):
    """rec_dev is stored 16 bytes at a time: a reconstruction buffer 4 bytes into an allocation is refused by every
    reconstruct entry with DGAN_ERR_INVALID_ARG before anything is enqueued (the buffer and the launch count stay as
    they were), the binding raises ValueError, and the same call into an aligned buffer returns the bits it returned
    before."""
    from defensegan_b200 import _native
    arch, B, R_, L, m = "mnist", 3, 2, 3, 100
    w, native = gen(arch, precision, False, 128, 64)
    lib = native.lib
    try:
        hwc = HWC[arch]
        x = torch.tensor(O.synthetic_images(arch, w, B, kind="S2", seed=2)).cuda()
        z0 = torch.tensor(O.sample_z0(B * R_, 128, seed=4)).cuda()
        pw = torch.rand(x.shape, generator=torch.Generator().manual_seed(3)).cuda()
        a = torch.tensor(MO.gaussian_operator(m, hwc, seed=1)).cuda()
        y = _measure(a, x)
        entries = {
            "plain": (lambda out=None: native.reconstruct(x, R_, L, 1.0, z_init_val=z0, out=out, return_aux=True),
                      lambda prm, rec, loss, idx, ws, need, st: lib.dgan_reconstruct(
                          native._handle, ctypes.byref(prm), x.data_ptr(), z0.data_ptr(), rec, loss, idx, ws, need, st),
                      dict()),
            "weighted": (lambda out=None: native.reconstruct(x, R_, L, 1.0, z_init_val=z0, out=out, return_aux=True,
                                                             pixel_weights=pw),
                         lambda prm, rec, loss, idx, ws, need, st: lib.dgan_reconstruct_weighted(
                             native._handle, ctypes.byref(prm), x.data_ptr(), pw.data_ptr(), z0.data_ptr(), rec, loss, idx,
                             ws, need, st),
                         dict(weighted=True)),
            "measured": (lambda out=None: native.reconstruct_measured(y, a, R_, L, 1.0, z_init_val=z0, out=out,
                                                                      return_aux=True),
                         lambda prm, rec, loss, idx, ws, need, st: lib.dgan_reconstruct_measured(
                             native._handle, ctypes.byref(prm), a.data_ptr(), m, y.data_ptr(), z0.data_ptr(), rec, loss,
                             idx, ws, need, st),
                         dict(m=m)),
        }
        for name, (call, abi, ws_kw) in entries.items():
            want = [t.clone() for t in call()]
            launches = native.last_launch_count
            buf = torch.full((B * hwc + 8,), float("nan"), device="cuda")
            bad = buf[1:1 + B * hwc]
            assert bad.data_ptr() % 16 != 0
            loss = torch.empty(B, device="cuda")
            idx = torch.empty(B, dtype=torch.int32, device="cuda")
            ws, need = native._workspace(B, R_, **ws_kw)
            stream = torch.cuda.current_stream().cuda_stream
            # Probe first with batch = 0, which no library runs: one that checks the alignment refuses the buffer
            # (the check comes before the hyper-parameters'), one without the check refuses the batch.  Only the
            # former may see the real call below, which a library without the check would run to the misaligned stores.
            rc = abi(_native.dgan_rec_params(0, R_, L, 1.0, 0.7, 0, 0, 0), bad.data_ptr(), loss.data_ptr(),
                     idx.data_ptr(), ws, need, stream)
            if rc != -1 or b"16-byte aligned" not in lib.dgan_last_error():
                pytest.fail("%s: the library does not refuse a misaligned rec_dev (%d: %r): rebuild it "
                            "(__graft_entry__.build())" % (name, rc, lib.dgan_last_error()))
            prm = _native.dgan_rec_params(B, R_, L, 1.0, 0.7, 0, 0, 0)
            rc = abi(prm, bad.data_ptr(), loss.data_ptr(), idx.data_ptr(), ws, need, stream)
            assert rc == -1, (name, rc)                                       # DGAN_ERR_INVALID_ARG
            assert b"16-byte aligned" in lib.dgan_last_error(), (name, lib.dgan_last_error())
            assert native.last_launch_count == launches, name
            torch.cuda.synchronize()
            assert bool(buf.isnan().all()), name                             # nothing was written
            with pytest.raises(ValueError, match="16-byte aligned"):
                call(out=bad.view(B, *SHAPE[arch]))
            good = buf[4:4 + B * hwc].view(B, *SHAPE[arch])                  # 16 bytes in: aligned
            got = call(out=good)
            assert got[0].data_ptr() == good.data_ptr()
            assert all(torch.equal(p, q) for p, q in zip(got, want)), name
            assert all(torch.equal(p, q) for p, q in zip(call(), want)), name
    finally:
        native.close()
