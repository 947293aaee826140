"""CPU oracle of the projection from linear measurements (an extension: the reference has none), built on
oracle/defensegan_oracle.py.

Row n minimises loss_n = (1/m) sum_j ((A G(z_n))_j - y[n // R]_j)^2 for an operator A [m, H*W*C] (NHWC pixel order) and
measurements y [B, m]; the loop, momentum, z0 stream and arg-min select are the oracle's."""
from __future__ import annotations

from typing import Optional

import numpy as np
import torch

from oracle import defensegan_oracle as O


def measured_loss(g: torch.Tensor, a: torch.Tensor, y_tiled: torch.Tensor) -> torch.Tensor:
    """Per-row (1/m) ||A g - y||^2 for g [N, H, W, C], a [m, H*W*C], y_tiled [N, m]."""
    r = g.reshape(g.shape[0], -1) @ a.t() - y_tiled
    return (r * r).mean(dim=1)


def _tiled(measurements, rec_rr: int, dtype) -> torch.Tensor:
    return torch.as_tensor(np.asarray(measurements)).to(dtype).repeat_interleave(rec_rr, dim=0)


def loss_and_grad(arch: str, weights, operator: np.ndarray, measurements: np.ndarray, z: np.ndarray, rec_rr: int,
                  use_bn: bool = False, dtype=torch.float32):
    """(G(z), per-row measured loss, d(sum loss)/dz) at z [B*rec_rr, latent]."""
    arch = O.canonical_arch(arch)
    w = O.weights_to_torch(weights, dtype)
    a = torch.as_tensor(np.asarray(operator)).to(dtype)
    zt = torch.as_tensor(np.asarray(z)).to(dtype).clone().requires_grad_(True)
    g = O.generator_forward(arch, w, zt, use_bn=use_bn)
    loss = measured_loss(g, a, _tiled(measurements, rec_rr, dtype))
    (grad,) = torch.autograd.grad(loss.sum(), zt)
    return g.detach().numpy(), loss.detach().numpy(), grad.numpy()


def reconstruct(arch: str, weights, operator: np.ndarray, measurements: np.ndarray, rec_rr: int, rec_iters: int,
                rec_lr: float = 10.0, z_init_val: Optional[np.ndarray] = None, momentum: float = 0.7, use_bn: bool = False,
                dtype=torch.float32, emulate_dead_decay: bool = True, seed: int = O.Z0_SEED):
    """O.reconstruct (the same loop, momentum and select) on the measured loss."""
    arch = O.canonical_arch(arch)
    w = O.weights_to_torch(weights, dtype)
    a = torch.as_tensor(np.asarray(operator)).to(dtype)
    y_tiled = _tiled(measurements, rec_rr, dtype)
    b = y_tiled.shape[0] // rec_rr
    n_rows = b * rec_rr
    latent_dim = w["Generator.Input/Generator.Input.W"].shape[0]
    if z_init_val is None:
        z_init_val = O.sample_z0(n_rows, latent_dim, seed)
    z = torch.as_tensor(np.asarray(z_init_val)).to(dtype).clone().reshape(n_rows, latent_dim)
    v = torch.zeros_like(z)
    g = loss = None
    for t in range(rec_iters):
        zt = z.detach().clone().requires_grad_(True)
        g = O.generator_forward(arch, w, zt, use_bn=use_bn)
        loss = measured_loss(g, a, y_tiled)
        (grad,) = torch.autograd.grad(loss.sum(), zt)
        lr = O.effective_learning_rate(rec_lr, rec_iters, t, emulate_dead_decay)
        v = momentum * v + grad
        z = z - lr * v
    g, loss = g.detach(), loss.detach()
    idx = torch.argmin(loss.reshape(b, rec_rr), dim=1)           # lowest index on ties
    rows = torch.arange(b) * rec_rr + idx
    return dict(rec=g[rows].numpy(), loss_min=loss[rows].numpy(), idx=idx.numpy().astype(np.int32),
                loss_all=loss.numpy(), rec_all=g.numpy(), z_final=z.detach().numpy())


def gaussian_operator(m: int, hwc: int, seed: int = 0) -> np.ndarray:
    """A compressed-sensing sketch: i.i.d. N(0, 1/hwc) entries (rows of about unit norm), [m, hwc] fp32."""
    return (np.random.RandomState(seed).standard_normal((m, hwc)) / np.sqrt(hwc)).astype(np.float32)


def block_average_operator(h: int, w: int, c: int, k: int = 2) -> np.ndarray:
    """A low-resolution copy: the mean of each k x k block of pixels per channel, [(h/k)(w/k)c, h*w*c] in NHWC order."""
    a = np.zeros(((h // k) * (w // k) * c, h * w * c), dtype=np.float32)
    for i in range(h):
        for j in range(w):
            for ch in range(c):
                a[((i // k) * (w // k) + j // k) * c + ch, (i * w + j) * c + ch] = 1.0 / (k * k)
    return a
