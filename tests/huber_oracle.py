"""CPU oracle of the projection with a Huber data term (an extension: the reference's loss is the squared error), built
on oracle/defensegan_oracle.py, tests/measured_oracle.py and tests/adam_oracle.py.

Per residual d (d = y - x per pixel on the image loss, r = (A G(z))_j - y_j per measurement on the measured loss), in the
kernels' order, with delta > 0 (+inf allowed):
  c = |d| > delta ? copysign(delta, d) : d;  e = w c (e = c without weights);  term = e (2 d - c)
The row loss is the mean of the terms (1/HWC, or 1/m), so term = w rho_delta(d) with rho = 2 huber_loss, and its
gradient with respect to d is 2 e.  When no |d| exceeds delta, c == d and 2 d - c == d exactly: every loss is the
squared-error oracles' to the bit, and so are the unweighted and measured gradients (2 (g e) == g (2 d)); the weighted
oracle differentiates e d term by term, so its gradients differ from 2 g e by rounding only.  The loop (momentum or
Adam), z0 stream, pre-update forward of iteration L-1 and arg-min select (lowest index on ties) are those oracles'."""
from __future__ import annotations

from typing import Optional

import numpy as np
import torch

import adam_oracle as AO
from oracle import defensegan_oracle as O


def clip(d: torch.Tensor, delta: float) -> torch.Tensor:
    """psi_delta(d): d clipped to [-delta, delta] with the sign of d; NaN passes through."""
    dl = torch.as_tensor(float(delta), dtype=d.dtype, device=d.device)
    return torch.where(d.abs() > dl, torch.copysign(dl, d), d)


def terms(d: torch.Tensor, delta: float, w: Optional[torch.Tensor] = None) -> torch.Tensor:
    """w rho_delta(d) per element as e (2 d - c), differentiable in d with gradient 2 e (c is held constant: it is d
    itself wherever it is not constant, and 2 e is the derivative of both pieces)."""
    c = clip(d, delta).detach()
    e = c if w is None else w * c
    return e * (2 * d - c)


def image_loss(y: torch.Tensor, x_tiled: torch.Tensor, delta: float, w_tiled: Optional[torch.Tensor] = None):
    """Per-row (1/HWC) sum_p w_p rho_delta(y_p - x_p)."""
    return terms(y - x_tiled, delta, w_tiled).mean(dim=tuple(range(1, y.dim())))


def measured_loss(g: torch.Tensor, a: torch.Tensor, y_tiled: torch.Tensor, delta: float):
    """Per-row (1/m) sum_j rho_delta((A g)_j - y_j) for g [N, H, W, C], a [m, H*W*C], y_tiled [N, m]."""
    r = g.reshape(g.shape[0], -1) @ a.t() - y_tiled
    return terms(r, delta).mean(dim=1)


class _Problem:
    """The generator's weights and the tiled target of one call: images (pixel weights optional) or measurements
    through an operator."""

    def __init__(self, arch, weights, rec_rr, delta, images=None, pixel_weights=None, operator=None, measurements=None,
                 use_bn=False, dtype=torch.float64, device="cpu"):
        self.arch = O.canonical_arch(arch)
        self.w = {k: v.to(device) for k, v in O.weights_to_torch(weights, dtype).items()}
        self.delta, self.use_bn = float(np.float32(delta)), use_bn
        self.a = self.pw = None
        if operator is not None:
            self.a = torch.as_tensor(np.asarray(operator)).to(dtype).to(device)
            self.target = torch.as_tensor(np.asarray(measurements)).to(dtype).to(device).repeat_interleave(rec_rr, dim=0)
        else:
            self.target = O.tile_images(torch.as_tensor(np.asarray(images)).to(dtype).to(device), rec_rr)
            if pixel_weights is not None:
                self.pw = O.tile_images(torch.as_tensor(np.asarray(pixel_weights)).to(dtype).to(device), rec_rr)
        self.latent = self.w["Generator.Input/Generator.Input.W"].shape[0]

    def loss(self, z: torch.Tensor):
        y = O.generator_forward(self.arch, self.w, z, use_bn=self.use_bn)
        if self.a is not None:
            return y, measured_loss(y, self.a, self.target, self.delta)
        return y, image_loss(y, self.target, self.delta, self.pw)


def loss_and_grad(arch: str, weights, z: np.ndarray, rec_rr: int, delta: float, images: Optional[np.ndarray] = None,
                  pixel_weights: Optional[np.ndarray] = None, operator: Optional[np.ndarray] = None,
                  measurements: Optional[np.ndarray] = None, use_bn: bool = False, dtype=torch.float64):
    """(G(z), per-row Huber loss, d(sum loss)/dz) at z [B*rec_rr, latent] on images or measurements."""
    p = _Problem(arch, weights, rec_rr, delta, images, pixel_weights, operator, measurements, use_bn, dtype)
    zt = torch.as_tensor(np.asarray(z)).to(dtype).clone().requires_grad_(True)
    y, loss = p.loss(zt)
    (g,) = torch.autograd.grad(loss.sum(), zt)
    return y.detach().numpy(), loss.detach().numpy(), g.numpy()


def reconstruct(arch: str, weights, rec_rr: int, rec_iters: int, rec_lr: float, delta: float,
                images: Optional[np.ndarray] = None, pixel_weights: Optional[np.ndarray] = None,
                operator: Optional[np.ndarray] = None, measurements: Optional[np.ndarray] = None,
                z_init_val: Optional[np.ndarray] = None, momentum: float = 0.7, adam=None, use_bn: bool = False,
                dtype=torch.float64, emulate_dead_decay: bool = True, seed: int = O.Z0_SEED, device="cpu"):
    """The R x L loop on the Huber loss: momentum (the oracle's) or, with adam = (beta1, beta2, eps), Adam (adam_oracle's).
    Returns dict(rec, loss_min, idx, loss_all, rec_all, z_final) as numpy arrays."""
    p = _Problem(arch, weights, rec_rr, delta, images, pixel_weights, operator, measurements, use_bn, dtype, device)
    b = p.target.shape[0] // rec_rr
    if z_init_val is None:
        z_init_val = O.sample_z0(b * rec_rr, p.latent, seed)
    z = torch.as_tensor(np.asarray(z_init_val)).to(dtype).to(device).clone().reshape(b * rec_rr, p.latent)
    if adam is not None:
        beta1, beta2, eps = (float(np.float32(v)) for v in adam)
    v = torch.zeros_like(z)
    s = torch.zeros_like(z)
    y = loss = None
    for t in range(rec_iters):
        zt = z.detach().clone().requires_grad_(True)
        y, loss = p.loss(zt)
        if adam is not None and t == rec_iters - 1:
            break                                               # the pre-update forward of iteration L-1
        (g,) = torch.autograd.grad(loss.sum(), zt)
        if adam is None:
            lr = O.effective_learning_rate(rec_lr, rec_iters, t, emulate_dead_decay)
            v = momentum * v + g
            z = z - lr * v
        else:
            c1, c2 = AO.adam_constants(rec_lr, t, beta1, beta2)
            v = beta1 * v + (1 - beta1) * g
            s = beta2 * s + (1 - beta2) * g * g
            z = z - c1 * v / (torch.sqrt(s) * c2 + eps)
    y, loss = y.detach().cpu(), loss.detach().cpu()
    idx = torch.argmin(loss.reshape(b, rec_rr), dim=1)           # lowest index on ties
    rows = torch.arange(b) * rec_rr + idx
    return dict(rec=y[rows].numpy(), loss_min=loss[rows].numpy(), idx=idx.numpy().astype(np.int32),
                loss_all=loss.numpy(), rec_all=y.numpy(), z_final=z.detach().cpu().numpy())
