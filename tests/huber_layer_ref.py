"""The fp64 checks of the Huber loss epilogues (dgan_loss_grad_huber, dgan_loss_grad_measured_huber) on the operands the
kernels read, with the bounds of tests/layer_ref.py and tests/weighted_layer_ref.py.

Last-layer forward: y is stored as the squared-error epilogue stores it; with d = y - x, c = psi_delta(d) and e = w c
(w = 1 unweighted), d(pre) = e act'(y) (tensor cores: dblk = RN16(gscale e act'(y))) and the loss part of a 4x4 block
sums e (2 d - c) = w rho_delta(d).  psi_delta is 1-Lipschitz with |psi_delta(d)| <= |d|, and rho_delta' = 2 psi_delta,
rho_delta'' <= 2, so every error term of the squared-error bound holds unchanged; the reference is evaluated at the
reference y, on either side of the clipping threshold.

Measured product: the stored residual is c = psi_delta(r) with r = A G - y; it is compared with psi_delta of the fp64 r
within the product's bound (psi_delta does not enlarge an error), and the row loss (1/m) sum_j rho_delta(r_j) with the
fp64 value within its terms' rounding plus 2 |c| times r's bound per measurement."""
from __future__ import annotations

import numpy as np
import torch

import huber_oracle as H
import layer_ref as R


def check_last_fwd_huber(net, ws, n, x_img_rows, w_img_rows, delta, stats, tag):
    """The last layer's Huber forward: y, the loss part of each 4x4 block (tensor cores) and d(pre); x_img_rows and
    w_img_rows (None: unweighted) are the image and weights of each latent row, [n][H*W*C].  Returns the share of the
    pixels whose reference residual is clipped."""
    delta = float(np.float32(delta))                        # the value the kernel compares with
    tc = net.precision == "fp16"
    y, dact, dy = R.check_last_y(net, ws, n, stats, tag)
    w_out = 2 * net.fh
    C = net.c_img
    x = x_img_rows.double().reshape(n, w_out, w_out, C)
    wt = torch.ones_like(x) if w_img_rows is None else w_img_rows.double().reshape(n, w_out, w_out, C)
    d = y - x
    c = H.clip(d, delta)
    dpre = wt * c * dact
    # d/dy of psi(y - x) act'(y) is at most 1.25 (sigmoid) or 5 (tanh) in magnitude, as for the squared error
    dd = wt * dy * (1.25 if net.act == "sigmoid" else 5.0)
    if tc:
        got = R.blocks_to_nhwc(ws["dblk"], n, w_out, C)
        R.check_close(tag + "last.fwd.huber (dblk)", got, R.GRAD_SCALE * dpre, torch.zeros_like(dpre), 0.0, "f16", stats,
                      extra=R.GRAD_SCALE * dd, where=["row", "i", "j", "c"])
        nb = w_out // 4
        lp = H.terms(d, delta, wt).reshape(n, nb, 4, nb, 4, C).sum(dim=(2, 4, 5)).reshape(n, nb * nb).t()
        tol = (wt * (2 * c.abs() + dy) * dy).reshape(n, nb, 4, nb, 4, C).sum(dim=(2, 4, 5)).reshape(n, nb * nb).t()
        R.check_close(tag + "last.fwd.huber (loss part)", ws["loss_part"][:, :n], lp, torch.zeros_like(lp), 0.0, "f32",
                      stats, extra=tol + 2.0 ** -20 * lp, where=["block", "row"])
    else:
        got = ws["dpre"][:n].reshape(n, w_out, w_out, C)
        R.check_close(tag + "last.fwd.huber (dpre)", got, dpre, torch.zeros_like(dpre), 0.0, "f32", stats, extra=dd,
                      where=["row", "i", "j", "c"])
    return float((d.abs() > delta).double().mean())


def check_measured_huber(ws, n, rec_rr, m, hwc, delta, precision, stats, tag):
    """The Huber measurement product of the last call on n latent rows: the stored residual c = psi_delta(A G - y)
    against fp64 on the operands it read (ws: the measured workspace's buffers, as test_gpu_measured._buffers reads
    them) and the row loss from the parts it left; the padded measurements of r exact zeros.  Returns the share of the
    residuals that are clipped.  The adjoint product dy = (2/m) A^T c is checked on the stored c, as the squared error's
    is on the stored r (test_gpu_measured.check_products)."""
    delta = float(np.float32(delta))
    u = 2.0 ** -24
    rnd = 2.0 ** -10 if precision == "fp16" else 0.0      # two operands rounded to TF32, 2^-11 each
    g = ws["y"][:n]
    y_rows = ws["ym"][:n // rec_rr].repeat_interleave(rec_rr, dim=0)
    r64 = g.double() @ ws["am"].double().t() - y_rows.double()
    lim = (rnd + hwc * u / (1 - hwc * u)) * (g.abs().double() @ ws["am"].abs().double().t()) + u * r64.abs() + 1e-30
    c64 = H.clip(r64, delta)
    got = ws["r"][:n].double()
    R.check_close(tag + "measurement product.huber (r)", got, c64, torch.zeros_like(c64), 0.0, "f32", stats, extra=lim,
                  where=["row", "j"])
    assert not ws["r"][:n, m:].any()                       # padded measurements are exact zeros
    t64 = H.terms(r64[:, :m], delta)
    ref = t64.sum(dim=1) / m
    extra = (m + 4) * u * t64.sum(dim=1) / m + (2 * c64[:, :m].abs() * lim[:, :m] + lim[:, :m] ** 2).sum(dim=1) / m
    R.check_close(tag + "measured loss.huber", ws["loss"][:n], ref, torch.zeros_like(ref), 0.0, "f32", stats, extra=extra,
                  where=["row"])
    m_ld = ws["am"].shape[0]
    r = ws["r"][:n]
    dy64 = (2.0 / m) * (r.double() @ ws["amt"].double().t())
    dlim = (2.0 / m) * (rnd + m_ld * u / (1 - m_ld * u)) * (r.abs().double() @ ws["amt"].abs().double().t()) * (1 + 2 * u)
    dlim = dlim + 2 * u * dy64.abs() + 1e-30
    R.check_close(tag + "adjoint product.huber (dy)", ws["dym"][:n], dy64, torch.zeros_like(dy64), 0.0, "f32", stats,
                  extra=dlim, where=["row", "p"])
    return float((r64[:, :m].abs() > delta).double().mean())
