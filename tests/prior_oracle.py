"""CPU oracle of the projection with a latent prior (an extension: the reference has none), built on
tests/huber_oracle.py (its problem: image or measured loss, weighted or not, squared error at delta = +inf or Huber),
tests/adam_oracle.py and oracle/defensegan_oracle.py.

For lambda >= 0 each restart minimises
  J(z) = D(z) + lambda ||z||^2
with D the counterpart's data term and its normaliser (1/HWC or 1/m).  Its gradient is g + 2 lambda z with g the data
term's gradient; the update (momentum or Adam) takes it in place of g.  J is evaluated on the z its D is computed on: the
pre-update forward of iteration L-1 for the returned loss and the arg-min select (lowest index on ties)."""
from __future__ import annotations

from typing import Optional

import numpy as np
import torch

import adam_oracle as AO
import huber_oracle as H
from oracle import defensegan_oracle as O

INF = float("inf")


def prior_term(z: torch.Tensor, lam: float) -> torch.Tensor:
    """lambda ||z||^2 per row of z [N, latent]."""
    return lam * (z * z).sum(dim=1)


def objective(p: "H._Problem", z: torch.Tensor, lam: float):
    """(G(z), D(z), J(z)) per row for the problem p."""
    y, d = p.loss(z)
    return y, d, d + prior_term(z, lam)


def _problem(arch, weights, rec_rr, delta, images, pixel_weights, operator, measurements, use_bn, dtype, device="cpu"):
    return H._Problem(arch, weights, rec_rr, delta, images, pixel_weights, operator, measurements, use_bn, dtype, device)


def loss_and_grad(arch: str, weights, z: np.ndarray, rec_rr: int, lam: float, delta: float = INF,
                  images: Optional[np.ndarray] = None, pixel_weights: Optional[np.ndarray] = None,
                  operator: Optional[np.ndarray] = None, measurements: Optional[np.ndarray] = None,
                  use_bn: bool = False, dtype=torch.float64):
    """(G(z), per-row D, per-row J, d(sum J)/dz) at z [B*rec_rr, latent]; delta = +inf is the squared error."""
    p = _problem(arch, weights, rec_rr, delta, images, pixel_weights, operator, measurements, use_bn, dtype)
    zt = torch.as_tensor(np.asarray(z)).to(dtype).clone().requires_grad_(True)
    y, d, j = objective(p, zt, lam)
    (g,) = torch.autograd.grad(j.sum(), zt)
    return y.detach().numpy(), d.detach().numpy(), j.detach().numpy(), g.numpy()


def reconstruct(arch: str, weights, rec_rr: int, rec_iters: int, rec_lr: float, lam: float, delta: float = INF,
                images: Optional[np.ndarray] = None, pixel_weights: Optional[np.ndarray] = None,
                operator: Optional[np.ndarray] = None, measurements: Optional[np.ndarray] = None,
                z_init_val: Optional[np.ndarray] = None, momentum: float = 0.7, adam=None, use_bn: bool = False,
                dtype=torch.float64, emulate_dead_decay: bool = True, seed: int = O.Z0_SEED, device="cpu"):
    """The R x L loop on J: momentum (the oracle's) or, with adam = (beta1, beta2, eps), Adam (adam_oracle's).  Returns
    dict(rec, loss_min, idx, loss_all, data_all, rec_all, z_final) as numpy arrays; loss_* are J, data_all is D."""
    lam = float(np.float32(lam))
    p = _problem(arch, weights, rec_rr, delta, images, pixel_weights, operator, measurements, use_bn, dtype, device)
    b = p.target.shape[0] // rec_rr
    if z_init_val is None:
        z_init_val = O.sample_z0(b * rec_rr, p.latent, seed)
    z = torch.as_tensor(np.asarray(z_init_val)).to(dtype).to(device).clone().reshape(b * rec_rr, p.latent)
    if adam is not None:
        beta1, beta2, eps = (float(np.float32(v)) for v in adam)
    v = torch.zeros_like(z)
    s = torch.zeros_like(z)
    y = d = j = None
    for t in range(rec_iters):
        zt = z.detach().clone().requires_grad_(True)
        y, d, j = objective(p, zt, lam)
        if t == rec_iters - 1:
            break                                               # the pre-update forward of iteration L-1
        (g,) = torch.autograd.grad(j.sum(), zt)
        if adam is None:
            lr = O.effective_learning_rate(rec_lr, rec_iters, t, emulate_dead_decay)
            v = momentum * v + g
            z = z - lr * v
        else:
            c1, c2 = AO.adam_constants(rec_lr, t, beta1, beta2)
            v = beta1 * v + (1 - beta1) * g
            s = beta2 * s + (1 - beta2) * g * g
            z = z - c1 * v / (torch.sqrt(s) * c2 + eps)
    y, d, j = y.detach().cpu(), d.detach().cpu(), j.detach().cpu()
    idx = torch.argmin(j.reshape(b, rec_rr), dim=1)              # lowest index on ties
    rows = torch.arange(b) * rec_rr + idx
    return dict(rec=y[rows].numpy(), loss_min=j[rows].numpy(), idx=idx.numpy().astype(np.int32), loss_all=j.numpy(),
                data_all=d.numpy(), rec_all=y.numpy(), z_final=z.detach().cpu().numpy())
