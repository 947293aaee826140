"""Sparse linear operators for the tests and the benchmark of the projection from sparse measurements: a full-resolution
5 x 5 blur, pixel subsampling, a grayscale copy and a random sparse matrix with an empty and a fully dense row.  Each is
returned as a dense [m, H*W*C] fp32 array (NHWC pixel order), which callers turn into CSR; the 2x2 block average is
measured_oracle.block_average_operator."""
from __future__ import annotations

import numpy as np


def blur_operator(h: int, w: int, c: int, sigma: float = 1.0) -> np.ndarray:
    """A blurred copy at full resolution: a separable 5 x 5 Gaussian per channel with zero boundary, [h*w*c, h*w*c] in
    NHWC order (at most 25 non-zeros per row)."""
    t = np.exp(-0.5 * (np.arange(-2, 3) / sigma) ** 2)
    t /= t.sum()
    a = np.zeros((h * w * c, h * w * c), dtype=np.float32)
    for i in range(h):
        for j in range(w):
            for di in range(-2, 3):
                for dj in range(-2, 3):
                    if 0 <= i + di < h and 0 <= j + dj < w:
                        for ch in range(c):
                            a[(i * w + j) * c + ch, ((i + di) * w + j + dj) * c + ch] = t[di + 2] * t[dj + 2]
    return a


def subsample_operator(m: int, hwc: int, seed: int = 0) -> np.ndarray:
    """Random pixel subsampling: m distinct entries of the image, in ascending order, [m, hwc] (one 1 per row)."""
    cols = np.sort(np.random.RandomState(seed).choice(hwc, size=m, replace=False))
    a = np.zeros((m, hwc), dtype=np.float32)
    a[np.arange(m), cols] = 1.0
    return a


def grayscale_operator(h: int, w: int) -> np.ndarray:
    """A grayscale copy of an RGB image (ITU-R BT.601 luma weights), [h*w, h*w*3] in NHWC order (3 non-zeros per row)."""
    a = np.zeros((h * w, h * w * 3), dtype=np.float32)
    for p in range(h * w):
        a[p, 3 * p:3 * p + 3] = (0.299, 0.587, 0.114)
    return a


def random_sparse_operator(m: int, hwc: int, density: float = 0.01, seed: int = 0) -> np.ndarray:
    """A random sparse matrix [m, hwc] with N(0, 1/(density hwc)) non-zeros at a fraction `density` of the entries, whose
    row 1 is empty and whose last row is fully dense (N(0, 1/hwc)); m >= 3."""
    rs = np.random.RandomState(seed)
    a = (rs.standard_normal((m, hwc)) * (rs.uniform(size=(m, hwc)) < density) / np.sqrt(density * hwc)).astype(np.float32)
    a[1] = 0.0
    a[-1] = (rs.standard_normal(hwc) / np.sqrt(hwc)).astype(np.float32)
    return a
