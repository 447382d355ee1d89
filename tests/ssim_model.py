"""Float64 NumPy model of the fused SSIM op (csrc/ssim.cu): the separable 11-tap window with zero padding, the SSIM map,
its means, and a hand-written VJP with respect to img1.  Written from the formula, not from the reference's text;
tests/test_ssim_cpu.py pins it to the reference's own outputs (tests/golden/ssim_*.npz) and its VJP to finite differences.
"""
import math

import numpy as np

R = 5
C1, C2 = 0.01 ** 2, 0.03 ** 2


def window():
    """The 11 weights as the reference builds them: float32 of exp(double), divided by their float32 sum (torch's sum of
    these values is their exact sum rounded once)."""
    g = np.array([math.exp(-(i - R) ** 2 / (2 * 1.5 ** 2)) for i in range(2 * R + 1)], np.float32)
    s = np.float32(np.sum(g.astype(np.float64)))
    return (g / s).astype(np.float64)


def filt(a):
    """The window along the last two axes, zero outside the image (conv2d with padding=5)."""
    w = window()
    H, W = a.shape[-2:]
    p = np.pad(np.asarray(a, np.float64), [(0, 0)] * (a.ndim - 2) + [(R, R), (R, R)])
    h = sum(w[k] * p[..., :, k:k + W] for k in range(2 * R + 1))
    return sum(w[k] * h[..., k:k + H, :] for k in range(2 * R + 1))


def _stats(x, y):
    mu1, mu2 = filt(x), filt(y)
    s11, s22, s12 = filt(x * x) - mu1 * mu1, filt(y * y) - mu2 * mu2, filt(x * y) - mu1 * mu2
    n1, n2 = 2 * mu1 * mu2 + C1, 2 * s12 + C2
    d1, d2 = mu1 * mu1 + mu2 * mu2 + C1, s11 + s22 + C2
    den = d1 * d2 + 1e-10
    return mu1, mu2, n1, n2, d1, d2, den


def ssim_map(x, y):
    x, y = np.asarray(x, np.float64), np.asarray(y, np.float64)
    _, _, n1, n2, _, _, den = _stats(x, y)
    return n1 * n2 / den


def ssim(x, y, size_average=True):
    """Mean over everything, or with size_average=False the per-image mean over (C,H,W) of an (N,C,H,W) input."""
    m = ssim_map(x, y)
    return m.mean() if size_average else m.reshape(m.shape[0], -1).mean(1)


def maps(x, y):
    """A = dm/dmu1 - 2 mu1 dm/ds11 - mu2 dm/ds12, B = dm/ds11, Cm = dm/ds12 (include/surfel_ssim.h)."""
    mu1, mu2, n1, n2, d1, d2, den = _stats(np.asarray(x, np.float64), np.asarray(y, np.float64))
    m = n1 * n2 / den
    dmu1 = (2 * mu2 * n2 - m * 2 * mu1 * d2) / den
    ds11 = -m * d1 / den
    ds12 = 2 * n1 / den
    return dmu1 - 2 * mu1 * ds11 - mu2 * ds12, ds11, ds12


def vjp(x, y, g_map):
    """dL/dx for dL/dm = g_map (same shape as x): the window is symmetric, so its adjoint is the same filter."""
    x, y = np.asarray(x, np.float64), np.asarray(y, np.float64)
    A, B, Cm = maps(x, y)
    return filt(g_map * A) + 2 * x * filt(g_map * B) + y * filt(g_map * Cm)


def vjp_mean(x, y, g, size_average=True):
    """dL/dx of L = g * ssim(x, y, size_average) (g a scalar, or (N,) per image)."""
    x = np.asarray(x, np.float64)
    if size_average:
        gm = np.full(x.shape, float(g) / x.size)
    else:
        per = x[0].size
        gm = np.broadcast_to(np.asarray(g, np.float64).reshape((-1,) + (1,) * (x.ndim - 1)) / per, x.shape)
    return vjp(x, y, gm)
