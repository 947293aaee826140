"""Structured measurement operators for the projection from linear measurements (DefenseGANBase.reconstruct_measured).

ConvOperator is a 2-D convolution applied per channel with a stride and zero padding - a blur, a box downsample, a blur
followed by decimation - with one kernel shared by every image or one kernel per image.  The library applies it as a
stencil (dgan_reconstruct_measured_conv in include/defensegan_b200.h), without a matrix or an index list.
"""
from __future__ import annotations

import numbers
from typing import Sequence, Tuple, Union

import numpy as np
import torch

__all__ = ["ConvOperator"]

MAX_KERNEL = 32       # largest kh and kw the library accepts
MAX_STRIDE = 16


def _int(v, name: str) -> int:
    if isinstance(v, bool) or not isinstance(v, numbers.Integral):
        raise ValueError("%s = %r is not an integer" % (name, v))
    return int(v)


class ConvOperator(object):
    """A per-channel 2-D cross-correlation with stride and zero padding, for images [B, H, W, C] in NHWC order:

        Ho = (H + 2 ph - kh) // s + 1,  Wo = (W + 2 pw - kw) // s + 1,  m = Ho * Wo * C
        y[(u * Wo + v) * C + c] = sum over in-bounds (a, b) of k[a][b] * x[s u + a - ph][s v + b - pw][c]

    The kernel is not flipped, and the same kernel applies to every channel: torch's conv2d with groups = C.
    `kernel` is [kh, kw] (one for every image) or [B, kh, kw] (image i's kernel at i), 1 <= kh, kw <= 32; `stride` s in
    1 .. 16; `padding` an int or (ph, pw) with 0 <= 2 ph <= kh - 1 and 0 <= 2 pw <= kw - 1.  Geometry and values
    (finite) are checked here, a ValueError naming the bad value; that the kernel fits the image is checked by
    out_shape."""

    def __init__(self, kernel, stride: int = 1, padding: Union[int, Sequence[int]] = 0):
        k = kernel if isinstance(kernel, torch.Tensor) else torch.as_tensor(np.asarray(kernel))
        if k.dim() not in (2, 3):
            raise ValueError("kernel must be [kh, kw] or [B, kh, kw], got shape %s" % (tuple(k.shape),))
        if k.dim() == 3 and k.shape[0] == 0:
            raise ValueError("kernel [B, kh, kw] needs B >= 1, got shape %s" % (tuple(k.shape),))
        kh, kw = int(k.shape[-2]), int(k.shape[-1])
        for name, v in (("kh", kh), ("kw", kw)):
            if not 1 <= v <= MAX_KERNEL:
                raise ValueError("kernel %s = %d must be in [1, %d]" % (name, v, MAX_KERNEL))
        s = _int(stride, "stride")
        if not 1 <= s <= MAX_STRIDE:
            raise ValueError("stride = %d must be in [1, %d]" % (s, MAX_STRIDE))
        if isinstance(padding, numbers.Integral) and not isinstance(padding, bool):
            ph = pw = int(padding)
        else:
            try:
                pad = tuple(padding)
            except TypeError:
                raise ValueError("padding = %r must be an int or a (ph, pw) pair" % (padding,)) from None
            if len(pad) != 2:
                raise ValueError("padding = %r must be an int or a (ph, pw) pair" % (padding,))
            ph, pw = _int(pad[0], "padding ph"), _int(pad[1], "padding pw")
        if not 0 <= 2 * ph <= kh - 1:
            raise ValueError("padding ph = %d must satisfy 0 <= 2 ph <= kh - 1 = %d" % (ph, kh - 1))
        if not 0 <= 2 * pw <= kw - 1:
            raise ValueError("padding pw = %d must satisfy 0 <= 2 pw <= kw - 1 = %d" % (pw, kw - 1))
        if not (k.dtype.is_floating_point or k.dtype in (torch.int8, torch.int16, torch.int32, torch.int64,
                                                          torch.uint8)):
            raise ValueError("kernel must hold real numbers, got dtype %s" % (k.dtype,))
        k = k.to(torch.float32)
        if not bool(torch.isfinite(k).all()):
            raise ValueError("kernel values must be finite")
        self.kernel = k.contiguous()
        self.stride = s
        self.padding = (ph, pw)

    # -- constructors ---------------------------------------------------------------------------------------------
    @classmethod
    def gaussian(cls, size: int, sigma: float) -> "ConvOperator":
        """A size x size Gaussian blur at full resolution (stride 1, padding (size - 1) // 2): the outer product of the
        normalised 1-D taps exp(-x^2 / (2 sigma^2)), x = -(size - 1)/2 .. (size - 1)/2, formed in float64 and rounded to
        fp32 once."""
        size = _int(size, "size")
        if not 1 <= size <= MAX_KERNEL:
            raise ValueError("size = %d must be in [1, %d]" % (size, MAX_KERNEL))
        if not (isinstance(sigma, numbers.Real) and np.isfinite(sigma) and sigma > 0):
            raise ValueError("sigma = %r must be finite and > 0" % (sigma,))
        t = np.exp(-0.5 * ((np.arange(size) - (size - 1) / 2) / sigma) ** 2)
        t /= t.sum()
        return cls(np.outer(t, t).astype(np.float32), stride=1, padding=(size - 1) // 2)

    @classmethod
    def box(cls, factor: int) -> "ConvOperator":
        """The block average of factor x factor pixels per channel: a low-resolution copy (stride = factor, no padding)."""
        factor = _int(factor, "factor")
        if not 1 <= factor <= MAX_STRIDE:
            raise ValueError("factor = %d must be in [1, %d]" % (factor, MAX_STRIDE))
        return cls(np.full((factor, factor), 1.0 / (factor * factor), dtype=np.float32), stride=factor, padding=0)

    # -- geometry ---------------------------------------------------------------------------------------------------
    @property
    def kernel_size(self) -> Tuple[int, int]:
        return int(self.kernel.shape[-2]), int(self.kernel.shape[-1])

    @property
    def per_image(self) -> bool:
        """True when the kernel is [B, kh, kw] (one per image)."""
        return self.kernel.dim() == 3

    def out_shape(self, image_dim) -> Tuple[int, int, int]:
        """(Ho, Wo, C) for images of shape image_dim = (H, W, C); a ValueError when the kernel does not fit."""
        h, w, c = (int(v) for v in image_dim)
        kh, kw = self.kernel_size
        if kh > h or kw > w:
            raise ValueError("kernel %dx%d does not fit the %dx%d image" % (kh, kw, h, w))
        ph, pw = self.padding
        return (h + 2 * ph - kh) // self.stride + 1, (w + 2 * pw - kw) // self.stride + 1, c

    def num_measurements(self, image_dim) -> int:
        ho, wo, c = self.out_shape(image_dim)
        return ho * wo * c

    def kernels(self, batch: int, device=None) -> torch.Tensor:
        """The kernels as a contiguous fp32 [batch, kh, kw] tensor: a shared kernel repeated, per-image ones as they are
        (their count must be batch)."""
        k = self.kernel if device is None else self.kernel.to(device)
        if self.per_image:
            if k.shape[0] != batch:
                raise ValueError("the operator has %d per-image kernels for %d images" % (k.shape[0], batch))
            return k.contiguous()
        return k.unsqueeze(0).expand(batch, -1, -1).contiguous()

    def _with_kernels(self, k: torch.Tensor) -> "ConvOperator":
        """This geometry with kernels k [B, kh, kw] already checked (no second host read)."""
        op = object.__new__(ConvOperator)
        op.kernel, op.stride, op.padding = k, self.stride, self.padding
        return op

    # -- application --------------------------------------------------------------------------------------------------
    def __call__(self, images: torch.Tensor) -> torch.Tensor:
        """y [B, m] = A_i x_i for images [B, H, W, C], in the order above (torch's conv2d in the images' dtype: a helper
        for making measurements, not the projection's path)."""
        x = images if isinstance(images, torch.Tensor) else torch.as_tensor(np.asarray(images))
        if x.dim() != 4:
            raise ValueError("images must be [B, H, W, C], got shape %s" % (tuple(x.shape),))
        b, h, w, c = x.shape
        self.out_shape((h, w, c))
        k = self.kernels(b, x.device).to(x.dtype)
        kh, kw = self.kernel_size
        xn = x.permute(0, 3, 1, 2).reshape(1, b * c, h, w)
        wt = k.repeat_interleave(c, dim=0).reshape(b * c, 1, kh, kw)
        out = torch.nn.functional.conv2d(xn, wt, stride=self.stride, padding=self.padding, groups=b * c)
        return out.reshape(b, c, out.shape[-2], out.shape[-1]).permute(0, 2, 3, 1).reshape(b, -1)

    def to_sparse_csr(self, image_dim, image: int = 0) -> torch.Tensor:
        """Image `image`'s operator as a torch CSR matrix [m, H*W*C] (fp32, columns ascending within each row, zero taps
        left out), built from the stencil without a dense matrix."""
        ho, wo, c = self.out_shape(image_dim)
        h, w, _ = (int(v) for v in image_dim)
        k = self.kernel[image] if self.per_image else self.kernel
        k = k.detach().cpu().numpy()
        kh, kw = self.kernel_size
        ph, pw = self.padding
        u, v, ch = np.meshgrid(np.arange(ho), np.arange(wo), np.arange(c), indexing="ij")
        row = ((u * wo + v) * c + ch).reshape(-1)
        u, v, ch = u.reshape(-1), v.reshape(-1), ch.reshape(-1)
        rows, cols, vals = [], [], []
        for a in range(kh):
            for b in range(kw):
                if k[a, b] == 0:
                    continue
                i, j = self.stride * u + a - ph, self.stride * v + b - pw
                ok = (i >= 0) & (i < h) & (j >= 0) & (j < w)
                rows.append(row[ok])
                cols.append(((i * w + j) * c + ch)[ok])
                vals.append(np.full(int(ok.sum()), k[a, b], dtype=np.float32))
        m, n = ho * wo * c, h * w * c
        if not rows:
            return torch.sparse_csr_tensor(torch.zeros(m + 1, dtype=torch.int64), torch.zeros(0, dtype=torch.int64),
                                           torch.zeros(0, dtype=torch.float32), size=(m, n))
        rows, cols, vals = np.concatenate(rows), np.concatenate(cols), np.concatenate(vals)
        order = np.lexsort((cols, rows))
        rows, cols, vals = rows[order], cols[order], vals[order]
        crow = np.zeros(m + 1, dtype=np.int64)
        np.cumsum(np.bincount(rows, minlength=m), out=crow[1:])
        return torch.sparse_csr_tensor(torch.from_numpy(crow), torch.from_numpy(cols.astype(np.int64)),
                                       torch.from_numpy(vals), size=(m, n))

    def __repr__(self):
        return "ConvOperator(kernel=%s%s, stride=%d, padding=%s)" % (
            "[%d, " % self.kernel.shape[0] if self.per_image else "[", "%d, %d]" % self.kernel_size, self.stride,
            self.padding)
