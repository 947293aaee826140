"""The projection with the Adam update, evaluated eagerly (fp64 by default) on top of the momentum oracles: the loop of
oracle/defensegan_oracle.reconstruct on the image loss (optionally weighted per pixel) or of tests/measured_oracle.py on
the measured loss, with z updated by Adam as dgan_reconstruct_adam defines it - for latent row n at iteration t, k = t + 1:
  m = b1 m + (1 - b1) g;  s = b2 s + (1 - b2) g^2;  z = z - c1 m / (sqrt(s) c2 + eps)
  c1 = lr_t / (1 - b1^k), c2 = 1 / sqrt(1 - b2^k)
The z0 stream, the pre-update forward of iteration L-1 and the arg-min select (lowest index on ties) are the oracle's."""
from __future__ import annotations

import math
from typing import Optional

import numpy as np
import torch

import measured_oracle as MO
from oracle import defensegan_oracle as O


def adam_constants(lr: float, t: int, beta1: float, beta2: float):
    """(c1, c2) of iteration t in double, from the fp32 values the library reads."""
    b1, b2, k = float(np.float32(beta1)), float(np.float32(beta2)), t + 1
    return float(np.float32(lr)) / (1.0 - b1 ** k), 1.0 / math.sqrt(1.0 - b2 ** k)


def reconstruct(arch: str, weights, rec_rr: int, rec_iters: int, rec_lr: float, adam, images: Optional[np.ndarray] = None,
                pixel_weights: Optional[np.ndarray] = None, operator: Optional[np.ndarray] = None,
                measurements: Optional[np.ndarray] = None, z_init_val: Optional[np.ndarray] = None,
                dtype=torch.float64, device="cpu"):
    """Adam on the image loss (images [B,H,W,C], pixel_weights optional) or on the measured loss (operator [m, H*W*C],
    measurements [B, m]).  Returns dict(rec, loss_min, idx, loss_all, rec_all, z_final) as numpy arrays."""
    beta1, beta2, eps = (float(np.float32(v)) for v in adam)
    arch = O.canonical_arch(arch)
    w = {k: v.to(device) for k, v in O.weights_to_torch(weights, dtype).items()}
    latent = w["Generator.Input/Generator.Input.W"].shape[0]
    if operator is not None:
        a = torch.as_tensor(np.asarray(operator)).to(dtype).to(device)
        target = torch.as_tensor(np.asarray(measurements)).to(dtype).to(device).repeat_interleave(rec_rr, dim=0)
    else:
        x = torch.as_tensor(np.asarray(images)).to(dtype).to(device)
        target = O.tile_images(x, rec_rr)
        pw = None
        if pixel_weights is not None:
            pw = O.tile_images(torch.as_tensor(np.asarray(pixel_weights)).to(dtype).to(device), rec_rr)
    b = target.shape[0] // rec_rr
    z = torch.as_tensor(np.asarray(z_init_val)).to(dtype).to(device).clone().reshape(b * rec_rr, latent)
    m = torch.zeros_like(z)
    s = torch.zeros_like(z)
    y = loss = None
    for t in range(rec_iters):
        zt = z.detach().clone().requires_grad_(True)
        y = O.generator_forward(arch, w, zt)
        if operator is not None:
            loss = MO.measured_loss(y, a, target)
        else:
            d2 = (y - target) ** 2
            loss = (d2 if pw is None else pw * d2).mean(dim=tuple(range(1, y.dim())))
        if t == rec_iters - 1:
            break                                               # the pre-update forward of iteration L-1
        (g,) = torch.autograd.grad(loss.sum(), zt)
        c1, c2 = adam_constants(rec_lr, t, beta1, beta2)
        m = beta1 * m + (1 - beta1) * g
        s = beta2 * s + (1 - beta2) * g * g
        z = z - c1 * m / (torch.sqrt(s) * c2 + eps)
    y, loss = y.detach().cpu(), loss.detach().cpu()
    idx = torch.argmin(loss.reshape(b, rec_rr), dim=1)
    rows = torch.arange(b) * rec_rr + idx
    return dict(rec=y[rows].numpy(), loss_min=loss[rows].numpy(), idx=idx.numpy().astype(np.int32), loss_all=loss.numpy(),
                rec_all=y.numpy(), z_final=z.detach().cpu().numpy())
