"""CPU oracle of the per-pixel weighted projection (an extension: the reference has no weighting), built on
oracle/defensegan_oracle.py.  With pixel_weights=None each function is the oracle's own, unchanged.

The weighted per-row loss is (1/HWC) sum_p w[n // R, p] (G(z_n)_p - x_p)^2, evaluated per pixel in the kernels' order:
d = y - x, e = w * d, loss term e * d (so that w == 1 gives e == d and the unweighted oracle's bits)."""
from __future__ import annotations

from typing import Optional

import numpy as np
import torch

from oracle import defensegan_oracle as O


def weighted_loss(y: torch.Tensor, x_tiled: torch.Tensor, w_tiled: torch.Tensor) -> torch.Tensor:
    """Per-row (1/HWC) sum of w (y - x)^2 with e = w * d, term e * d."""
    d = y - x_tiled
    e = w_tiled * d
    return (e * d).mean(dim=tuple(range(1, y.dim())))


def loss_and_grad(arch: str, weights, images: np.ndarray, z: np.ndarray, rec_rr: int, use_bn: bool = False,
                  dtype=torch.float32, pixel_weights: Optional[np.ndarray] = None):
    """O.loss_and_grad with the weighted loss when pixel_weights [B,H,W,C] is given."""
    if pixel_weights is None:
        return O.loss_and_grad(arch, weights, images, z, rec_rr, use_bn=use_bn, dtype=dtype)
    arch = O.canonical_arch(arch)
    w = O.weights_to_torch(weights, dtype)
    x_tiled = O.tile_images(torch.as_tensor(np.asarray(images)).to(dtype), rec_rr)
    w_tiled = O.tile_images(torch.as_tensor(np.asarray(pixel_weights)).to(dtype), rec_rr)
    zt = torch.as_tensor(np.asarray(z)).to(dtype).clone().requires_grad_(True)
    y = O.generator_forward(arch, w, zt, use_bn=use_bn)
    loss = weighted_loss(y, x_tiled, w_tiled)
    (g,) = torch.autograd.grad(loss.sum(), zt)
    return y.detach().numpy(), loss.detach().numpy(), g.numpy()


def reconstruct(arch: str, weights, images: np.ndarray, rec_rr: int, rec_iters: int, rec_lr: float = 10.0,
                z_init_val: Optional[np.ndarray] = None, momentum: float = 0.7, use_bn: bool = False, dtype=torch.float32,
                emulate_dead_decay: bool = True, seed: int = O.Z0_SEED, pixel_weights: Optional[np.ndarray] = None):
    """O.reconstruct (the same loop, momentum and select) on the weighted loss when pixel_weights [B,H,W,C] is given."""
    if pixel_weights is None:
        return O.reconstruct(arch, weights, images, rec_rr, rec_iters, rec_lr=rec_lr, z_init_val=z_init_val,
                             momentum=momentum, use_bn=use_bn, dtype=dtype, emulate_dead_decay=emulate_dead_decay, seed=seed)
    arch = O.canonical_arch(arch)
    w = O.weights_to_torch(weights, dtype)
    x = torch.as_tensor(np.asarray(images)).to(dtype)
    b = x.shape[0]
    n_rows = b * rec_rr
    latent_dim = w["Generator.Input/Generator.Input.W"].shape[0]
    x_tiled = O.tile_images(x, rec_rr)
    w_tiled = O.tile_images(torch.as_tensor(np.asarray(pixel_weights)).to(dtype), rec_rr)
    if z_init_val is None:
        z_init_val = O.sample_z0(n_rows, latent_dim, seed)
    z = torch.as_tensor(np.asarray(z_init_val)).to(dtype).clone().reshape(n_rows, latent_dim)
    v = torch.zeros_like(z)
    y = loss = None
    for t in range(rec_iters):
        zt = z.detach().clone().requires_grad_(True)
        y = O.generator_forward(arch, w, zt, use_bn=use_bn)
        loss = weighted_loss(y, x_tiled, w_tiled)
        (g,) = torch.autograd.grad(loss.sum(), zt)
        lr = O.effective_learning_rate(rec_lr, rec_iters, t, emulate_dead_decay)
        v = momentum * v + g
        z = z - lr * v
    y, loss = y.detach(), loss.detach()
    idx = torch.argmin(loss.reshape(b, rec_rr), dim=1)           # lowest index on ties
    rows = torch.arange(b) * rec_rr + idx
    return dict(rec=y[rows].reshape(x.shape).numpy(), loss_min=loss[rows].numpy(), idx=idx.numpy().astype(np.int32),
                loss_all=loss.numpy(), rec_all=y.numpy(), z_final=z.detach().numpy())
