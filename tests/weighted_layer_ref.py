"""The fp64 check of the weighted last-layer forward (dgan_loss_grad_weighted), on the operands the kernel read, with the
bound of tests/layer_ref.py.  Shared by test_gpu_weighted.py (the workspace a call leaves) and test_host_weighted.py (a
CPU emulation, and the same emulation with seeded weighting defects, which the bound must reject).

The weighted epilogue stores y as the unweighted one does; with e = w (y - x) per pixel, d(pre) = e act'(y) (tensor cores:
dblk = RN16(gscale e act'(y))) and the loss part of a 4x4 block sums e (y - x).  Every error term of the unweighted bound
is scaled by w <= 1."""
from __future__ import annotations

import torch

import layer_ref as R


def check_last_fwd_weighted(net, ws, n, x_img_rows, w_img_rows, stats, tag):
    """The last layer's weighted forward: y, the weighted loss part of each 4x4 block (tensor cores) and the weighted
    d(pre); x_img_rows and w_img_rows are the image and weights of each latent row, [n][H*W*C]."""
    tc = net.precision == "fp16"
    L = net.layers[-1]
    x_store = ws[("act_h.%d" if tc else "act.%d") % (net.nl - 1)]
    pre, ab = R.last_fwd_ref(net, x_store, n)
    gamma = net.gamma(net.pairs(net.nl, "fwd"), L["c_out_p"])
    y, dact = R.act_fwd(net, pre)
    dy = dact * gamma * ab + R.ACT_EPS[net.precision]           # |y - y_ref|
    w_out = 2 * net.fh
    C = net.c_img
    R.check_close(tag + "last.fwd (y)", ws["y"][:n].reshape(n, w_out, w_out, C), y, torch.zeros_like(y), 0.0, "f32", stats,
                  extra=dy, where=["row", "i", "j", "c"])
    x = x_img_rows.double().reshape(n, w_out, w_out, C)
    wt = w_img_rows.double().reshape(n, w_out, w_out, C)
    d = wt * (y - x) * dact
    # d/dy of (y - x) act'(y) is at most 1.25 (sigmoid) or 5 (tanh) in magnitude
    dd = wt * dy * (1.25 if net.act == "sigmoid" else 5.0)
    if tc:
        got = R.blocks_to_nhwc(ws["dblk"], n, w_out, C)
        R.check_close(tag + "last.fwd (dblk)", got, R.GRAD_SCALE * d, torch.zeros_like(d), 0.0, "f16", stats,
                      extra=R.GRAD_SCALE * dd, where=["row", "i", "j", "c"])
        # loss part of block (by, bx): sum over its 16 pixels of w (y - x)^2
        e = wt * (y - x) ** 2
        nb = w_out // 4
        lp = e.reshape(n, nb, 4, nb, 4, C).sum(dim=(2, 4, 5)).reshape(n, nb * nb).t()
        tol = (wt * (2 * (y - x).abs() + dy) * dy).reshape(n, nb, 4, nb, 4, C).sum(dim=(2, 4, 5)).reshape(n, nb * nb).t()
        R.check_close(tag + "last.fwd (loss part)", ws["loss_part"][:, :n], lp, torch.zeros_like(lp), 0.0, "f32", stats,
                      extra=tol + 2.0 ** -20 * lp, where=["block", "row"])
    else:
        got = ws["dpre"][:n].reshape(n, w_out, w_out, C)
        R.check_close(tag + "last.fwd (dpre)", got, d, torch.zeros_like(d), 0.0, "f32", stats, extra=dd,
                      where=["row", "i", "j", "c"])
