"""CPU oracle of the projection with sparse deviations (an extension: the reference has none; Sparse-Gen, Dhar, Grover and
Ermon 2018), built on tests/huber_oracle.py (its data terms: image or measured loss, weighted or not, squared error at
delta = +inf or Huber), tests/prior_oracle.py, tests/adam_oracle.py and oracle/defensegan_oracle.py.

Each restart row carries nu (H*W*C values, starting at 0) and minimises
  J(z, nu) = D(G(z) + nu) + lambda ||z||^2 + l1 ||nu||_1
with D the counterpart's data term and its normaliser (1/n, n = H*W*C, or 1/m).  Iteration t evaluates D, J and
g = dD/du at (z_t, nu_t), u = G(z_t) + nu_t; unless it is the last, z takes the counterpart's update (momentum or Adam on
dD/dz + 2 lambda z) and nu the ISTA step nu <- S_tau(nu - eta g), eta = step n / 2 (step m / 2), tau = eta l1.  The
returned loss and the arg-min (lowest index on ties) are J at iteration L-1; rec is G(z), dev is nu of that restart."""
from __future__ import annotations

from typing import Optional

import numpy as np
import torch

import adam_oracle as AO
import huber_oracle as H
from oracle import defensegan_oracle as O

INF = float("inf")


def shrink(a: torch.Tensor, tau: float) -> torch.Tensor:
    """The soft threshold S_tau(a) = sign(a) max(|a| - tau, 0)."""
    return torch.sign(a) * torch.clamp(a.abs() - tau, min=0.0)


def _problem(arch, weights, rec_rr, delta, images, pixel_weights, operator, measurements, use_bn, dtype, device="cpu"):
    return H._Problem(arch, weights, rec_rr, delta, images, pixel_weights, operator, measurements, use_bn, dtype, device)


def data_term(p: "H._Problem", u: torch.Tensor) -> torch.Tensor:
    """D per row at u [N, H, W, C] (or [N, H*W*C]) for the problem p."""
    if p.a is not None:
        return H.measured_loss(u, p.a, p.target, p.delta)
    return H.image_loss(u.reshape(p.target.shape), p.target, p.delta, p.pw)


def n_values(p: "H._Problem") -> int:
    """n of eta = step n / 2: m for a measured problem, H*W*C for the image loss."""
    return int(p.a.shape[0]) if p.a is not None else int(np.prod(p.target.shape[1:]))


def objective(p: "H._Problem", z: torch.Tensor, nu: torch.Tensor, lam: float, l1: float):
    """(G(z), u, D(u), J) per row for the problem p at (z, nu); nu is [N, H*W*C]."""
    y = O.generator_forward(p.arch, p.w, z, use_bn=p.use_bn)
    u = y.reshape(y.shape[0], -1) + nu
    d = data_term(p, u)
    return y, u, d, d + lam * (z * z).sum(dim=1) + l1 * nu.abs().sum(dim=1)


def reconstruct(arch: str, weights, rec_rr: int, rec_iters: int, rec_lr: float, l1: float, step: float,
                lam: float = 0.0, delta: float = INF, images: Optional[np.ndarray] = None,
                pixel_weights: Optional[np.ndarray] = None, operator: Optional[np.ndarray] = None,
                measurements: Optional[np.ndarray] = None, z_init_val: Optional[np.ndarray] = None,
                momentum: float = 0.7, adam=None, use_bn: bool = False, dtype=torch.float64,
                emulate_dead_decay: bool = True, seed: int = O.Z0_SEED, device="cpu"):
    """The R x L loop on J.  Returns dict(rec, dev, loss_min, idx, loss_all, data_all, rec_all, nu_all, z_final) as numpy
    arrays; loss_* are J, data_all is D, nu_all is every row's nu at iteration L-1."""
    lam, l1, step = (float(np.float32(v)) for v in (lam, l1, step))
    p = _problem(arch, weights, rec_rr, delta, images, pixel_weights, operator, measurements, use_bn, dtype, device)
    b = p.target.shape[0] // rec_rr
    eta = step * n_values(p) / 2.0
    tau = eta * l1
    if z_init_val is None:
        z_init_val = O.sample_z0(b * rec_rr, p.latent, seed)
    z = torch.as_tensor(np.asarray(z_init_val)).to(dtype).to(device).clone().reshape(b * rec_rr, p.latent)
    hwc = int(p.a.shape[1]) if p.a is not None else int(np.prod(p.target.shape[1:]))
    nu = torch.zeros((b * rec_rr, hwc), dtype=dtype, device=device)
    if adam is not None:
        beta1, beta2, eps = (float(np.float32(v)) for v in adam)
    v = torch.zeros_like(z)
    s = torch.zeros_like(z)
    y = d = j = None
    for t in range(rec_iters):
        zt = z.detach().clone().requires_grad_(True)
        nt = nu.detach().clone().requires_grad_(True)
        y, u, d, j = objective(p, zt, nt, lam, l1)
        if t == rec_iters - 1:
            break                                               # the pre-update forward of iteration L-1
        gz, gu = torch.autograd.grad(d.sum() + lam * (zt * zt).sum(), (zt, nt))
        if adam is None:
            lr = O.effective_learning_rate(rec_lr, rec_iters, t, emulate_dead_decay)
            v = momentum * v + gz
            z = z - lr * v
        else:
            c1, c2 = AO.adam_constants(rec_lr, t, beta1, beta2)
            v = beta1 * v + (1 - beta1) * gz
            s = beta2 * s + (1 - beta2) * gz * gz
            z = z - c1 * v / (torch.sqrt(s) * c2 + eps)
        nu = shrink(nu - eta * gu, tau)
    y, d, j = y.detach().cpu(), d.detach().cpu(), j.detach().cpu()
    nu = nu.detach().cpu()
    idx = torch.argmin(j.reshape(b, rec_rr), dim=1)              # lowest index on ties
    rows = torch.arange(b) * rec_rr + idx
    return dict(rec=y[rows].numpy(), dev=nu[rows].reshape(y[rows].shape).numpy(), loss_min=j[rows].numpy(),
                idx=idx.numpy().astype(np.int32), loss_all=j.numpy(), data_all=d.numpy(), rec_all=y.numpy(),
                nu_all=nu.numpy(), z_final=z.detach().cpu().numpy())
