"""TEST INFRASTRUCTURE -- the fused SSIM op (csrc/ssim.cu) restated operation for operation, with its rounding-error bound.

ssim_fwd, ssim_reduce, ssim_bwd and ssim_bkgd_reduce are restated here in NumPy in the kernels' order, on the kernels' own
fp32 inputs, as running-error values (tests/error_bound.py): every value carries its float64 value, a bound B (units of
u = 2^-24) on the error of its fp32 evaluation, and an fp32 shadow evaluation.  The tests hold the GPU (and, on the CPU,
the shadow) to |x - value| <= K u B + FLOOR.

  * Window: the fp32 weights of ssim_model.window(), exact leaves.  The constants C1 = 0.01f * 0.01f, C2 = 0.03f * 0.03f
    and 1e-10f carry their value as ssim_model uses it and their fp32 rounding as bound.
  * Composite: x = img1 + (1 - alpha) bkgd[ch].  nvcc may contract it into an FMA, differently in the forward and the
    backward; the two roundings charged bound either.
  * Filters: the horizontal then the vertical 11-tap fmaf chains, zero outside the image.  fma() charges the product's
    rounding and the sum's: fmaf rounds once, and the same charge covers an a * b + c that nvcc contracts or not.
  * Means: a pixel's value enters a per-thread chain of SS_ROWS adds (the first onto an exact 0.f), a 5-level xor
    butterfly over the warp and a chain of SS_THREADS / 32 warp totals (the first again exact): LEVELS roundings, each
    at most u sum |t| over the CTA.  The tiles' float64 sums and the final float rounding follow.
  * Backward: on the kernel's own fp32 maps as leaves, so its bound is free of the forward's error.  dL/dbkgd's per-CTA
    partials take the same LEVELS, then their float64 sum, its float rounding and the += onto the prefill.

Ill-conditioned pixels: where the first-order bound of d2 or den exceeds 1/64 of its value (HDR flat regions, where the
cancellation in sigma^2 = E[x^2] - mu^2 leaves an error near C2), the quotients' first-order bound means nothing.  Those
pixels' maps are not compared, nor the means of an image holding one; the tests count them.
"""
import zlib

import numpy as np

from . import ssim_model as sm
from .error_bound import _E, _c, _rnd

U = 2.0 ** -24
K = 2.0
FLOOR = float(np.finfo(np.float32).tiny)
KNIFE_REL = 2.0 ** -6

# csrc/ssim.cu's launch constants
SS_T, SS_R, SS_THREADS = 32, 5, 256
WARPS = SS_THREADS // 32
SS_ROWS = SS_T // WARPS
LEVELS = (SS_ROWS - 1) + 5 + (WARPS - 1)
U64 = 2.0 ** -53 / U          # one float64 rounding, in units of u

ZERO = _E(0.0, None, np.float32(0.0))
ONE = _E(1.0, None, np.float32(1.0))


def _k(c64, c32):
    """A constant the kernel rounds to fp32: the value ssim_model uses, its actual fp32 rounding as bound, the fp32 shadow."""
    return _E(c64, abs(float(np.float32(c32)) - c64) / U, np.float32(c32))


C1 = _k(sm.C1, np.float32(0.01) * np.float32(0.01))
C2 = _k(sm.C2, np.float32(0.03) * np.float32(0.03))
EPS = _E.const(1e-10)
WIN = [_E.leaf(w) for w in sm.window().astype(np.float32)]


def fma(a, b, c):
    """a * b + c: the product's rounding and the sum's (none where exact); the shadow is the float64 sum of the exact fp32
    product rounded once to fp32."""
    a, b, c = _c(a), _c(b), _c(c)
    p = a.v * b.v
    v = p + c.v
    ex = (a.b == 0) & (b.b == 0)
    bd = np.abs(a.v) * b.b + np.abs(b.v) * a.b + c.b + _rnd(p, ex) + _rnd(v, ex & (c.b == 0))
    f = None
    if a.f is not None and b.f is not None and c.f is not None:
        f = (a.f.astype(np.float64) * b.f + c.f).astype(np.float32)
    return _E(v, bd, f)


def _pad(t):
    p = [(0, 0)] * (t.v.ndim - 2) + [(SS_R, SS_R), (SS_R, SS_R)]
    return _E(np.pad(t.v, p), np.pad(t.b, p), None if t.f is None else np.pad(t.f, p))


def filt(t):
    """ssim_fwd / ssim_bwd's separable window over the last two axes, zero outside the image: for each staged row the
    horizontal fmaf chain over taps 0..10, then for each output row the vertical one."""
    H, W = t.v.shape[-2:]
    p = _pad(t)
    h = ZERO
    for k in range(2 * SS_R + 1):
        h = fma(WIN[k], p[..., :, k:k + W], h)
    v = ZERO
    for k in range(2 * SS_R + 1):
        v = fma(WIN[k], h[..., k:k + H, :], v)
    return v


def image_x(img1, alpha, bkgd):
    """image_x: img1, or img1 + (1 - alpha) bkgd[ch] with alpha (N,H,W) and bkgd (3,) fp32."""
    x = _E.leaf(img1)
    if alpha is None:
        return x
    return x + (ONE - _E.leaf(alpha[:, None])) * _E.leaf(np.asarray(bkgd, np.float32).reshape(1, -1, 1, 1))


def _ill(e):
    return U * e.b > KNIFE_REL * np.abs(e.v)


# ------------------------------------------------------------------------------------------------ reductions
def _tiles(a):
    """(N,C,H,W) -> (N,C,tiles,SS_T,SS_T), zero outside the image, tiles in the kernel's order (row-major)."""
    N, C, H, W = a.shape
    TY, TX = -(-H // SS_T), -(-W // SS_T)
    p = np.zeros((N, C, TY * SS_T, TX * SS_T), a.dtype)
    p[..., :H, :W] = a
    return p.reshape(N, C, TY, SS_T, TX, SS_T).transpose(0, 1, 2, 4, 3, 5).reshape(N, C, TY * TX, SS_T, SS_T)


def _block_sum_f(f):
    """block_sum of per-pixel fp32 terms (…, SS_T rows, SS_T columns) exactly as the kernel adds them: thread (warp rg,
    lane c) sums rows rg * SS_ROWS + j of column c in order, the xor butterfly, then the warps in order."""
    part = np.zeros(f.shape[:-2] + (WARPS, SS_T), np.float32)
    rows = f.reshape(f.shape[:-2] + (WARPS, SS_ROWS, SS_T))
    for j in range(SS_ROWS):
        part = part + rows[..., :, j, :]
    lane = np.arange(SS_T)
    for o in (16, 8, 4, 2, 1):
        part = part + part[..., lane ^ o]
    t = np.zeros(f.shape[:-2], np.float32)
    for w in range(WARPS):
        t = t + part[..., w, 0]
    return t


def block_sums(t):
    """Each CTA's fp32 block_sum of a per-pixel _E t (N,C,H,W): (N,C,tiles) value, bound, shadow."""
    v, a = _tiles(t.v), _tiles(np.abs(t.v))
    b = _tiles(t.b)
    return _E(v.sum((-2, -1)), b.sum((-2, -1)) + LEVELS * a.sum((-2, -1)),
              None if t.f is None else _block_sum_f(_tiles(t.f)))


def _f64_sum(parts, axes, scale):
    """warp_row_sum / the block's sum: float64 sums of fp32 partials over `axes`, times a float64 scale, rounded once to
    fp32.  The float64 roundings are charged n u64 sum |t| (n terms)."""
    n = int(np.prod([parts.v.shape[a] for a in axes]))
    v = parts.v.sum(axes) * scale
    b = (parts.b.sum(axes) + (n + 2) * U64 * np.abs(parts.v).sum(axes)) * scale
    f = None if parts.f is None else (parts.f.astype(np.float64).sum(axes) * scale).astype(np.float32)
    return _E(v, b + np.abs(v), f)


# ------------------------------------------------------------------------------------------------ forward
def forward(img1, img2, alpha=None, bkgd=None):
    """ssim_fwd + ssim_reduce on fp32 (N,C,H,W) inputs; alpha (N,H,W) (the plane the kernel reads) and bkgd (3,) for the
    background composite.  Returns dict of _E: A, B, Cm, m (N,C,H,W), ssim_img (N,), ssim_mean (); ill (N,C,H,W)."""
    N, C, H, W = img1.shape
    x, y = image_x(img1, alpha, bkgd), _E.leaf(img2)
    mu1, mu2 = filt(x), filt(y)
    e11, e22, e12 = filt(x * x), filt(y * y), filt(x * y)
    mu1_sq, mu2_sq, mu12 = mu1 * mu1, mu2 * mu2, mu1 * mu2
    s11, s22, s12 = e11 - mu1_sq, e22 - mu2_sq, e12 - mu12
    n1, n2 = mu12.scale(2.0) + C1, s12.scale(2.0) + C2
    d1, d2 = (mu1_sq + mu2_sq) + C1, (s11 + s22) + C2
    den = d1 * d2 + EPS
    m = (n1 * n2) / den
    inv = ONE / den
    dmu1 = ((mu2.scale(2.0) * n2) - (m.scale(2.0) * mu1) * d2) * inv
    ds11 = (-m * d1) * inv
    ds12 = n1.scale(2.0) * inv
    A = (dmu1 - mu1.scale(2.0) * ds11) - mu2 * ds12
    ill = _ill(d2) | _ill(den)
    parts = block_sums(m)
    pix = float(H) * W
    return dict(A=A, B=ds11, Cm=ds12, m=m, ill=ill, parts=parts,
                ssim_img=_f64_sum(parts, (1, 2), 1.0 / (C * pix)),
                ssim_mean=_f64_sum(parts, (0, 1, 2), 1.0 / (N * C * pix)))


# ------------------------------------------------------------------------------------------------ backward
def backward(img1, img2, maps, dL_dssim, per_image, alpha=None, bkgd=None, dimg1=None, dalpha=None, dbkgd=None):
    """ssim_bwd + ssim_bkgd_reduce.  maps (3,N,C,H,W): the forward's maps as fp32 leaves, or float64 (exact, no shadow) to
    pin the values to ssim_model, or the forward's (A, B, Cm) _E values when the GPU's maps are not at hand.  dL_dssim: the fp32 upstream array the kernel indexes ([n] with per_image, else [0]).
    dimg1 (N,C,H,W): the prefill under accumulate = 1, or None.  dalpha (N,H,W) and dbkgd (N,3): the prefills the
    composite adds onto.  Returns dict of _E: dimg1, and with alpha dalpha and dbkgd."""
    N, C, H, W = img1.shape
    count = (1.0 if per_image else float(N)) * C * H * W
    inv_count = _E.const(1.0 / count)
    up = _E.leaf(np.asarray(dL_dssim, np.float32).reshape(-1))
    g = (up[np.arange(N)] if per_image else up[np.zeros(N, int)]) * inv_count
    g = g[:, None, None, None]
    if isinstance(maps[0], _E):                  # the forward's running-error maps: their bound carries through
        mp = list(maps)
    elif np.asarray(maps).dtype == np.float32:
        mp = [_E.leaf(a) for a in maps]
    else:
        mp = [_E(np.asarray(a, np.float64)) for a in maps]
    v0, v1, v2 = filt(mp[0]), filt(mp[1]), filt(mp[2])
    x, y = image_x(img1, alpha, bkgd), _E.leaf(img2)
    gxv = g * ((v0 + x.scale(2.0) * v1) + y * v2)
    out = dict(gxv=gxv, dimg1=gxv if dimg1 is None else _E.leaf(dimg1) + gxv)
    if alpha is not None:
        bk = [_E.leaf(np.float32(b)) for b in bkgd]
        da = ZERO
        for ch in range(C):
            da = fma(gxv[:, ch], bk[ch], da)
        out["dalpha"] = _E.leaf(dalpha) - da
        t = gxv * (ONE - _E.leaf(alpha[:, None]))
        parts = block_sums(t)
        s = _f64_sum(parts, (2,), 1.0)
        out["dbkgd"] = _E.leaf(dbkgd) + s
    return out


def fp32_maps(fw):
    """The forward's maps as the fp32 tensor the kernel writes (its shadow)."""
    return np.stack([fw["A"].f, fw["B"].f, fw["Cm"].f])


# ------------------------------------------------------------------------------------------------ inputs
def content(kind, shape, rng):
    """img1, img2 (fp32 (N,C,H,W)) of one kind:
    textured   uniform [0, 1] with img2 a noisy copy;
    patches    piecewise-constant 6x6 patches, half of them with img1 == img2, the rest different constants (sigma = 0:
               the 1/C2 amplification peaks);
    nearconst  0.5 +- 1e-3 (E[x^2] - mu^2 cancels to ~1e-6);
    zeros      textured, with both images exactly 0 over a region;
    hdr        values in [-0.5, 8], with flat patches."""
    N, C, H, W = shape
    if kind == "textured":
        a = rng.uniform(0, 1, shape)
        b = np.clip(a + 0.2 * rng.normal(size=shape), 0, 1)
    elif kind == "patches":
        ny, nx = -(-H // 6), -(-W // 6)
        pa = rng.uniform(0, 1, (N, C, ny, nx))
        pb = np.where(rng.uniform(size=pa.shape) < 0.5, pa, rng.uniform(0, 1, pa.shape))
        up = lambda p: np.repeat(np.repeat(p, 6, -2), 6, -1)[..., :H, :W]  # noqa: E731
        a, b = up(pa), up(pb)
    elif kind == "nearconst":
        a = 0.5 + rng.uniform(-1e-3, 1e-3, shape)
        b = 0.5 + rng.uniform(-1e-3, 1e-3, shape)
    elif kind == "zeros":
        a = rng.uniform(0, 1, shape)
        b = np.clip(a + 0.2 * rng.normal(size=shape), 0, 1)
        a[..., H // 4:H // 4 + max(1, H // 2), :max(1, W // 2)] = 0.0
        b[..., H // 4:H // 4 + max(1, H // 2), :max(1, W // 2)] = 0.0
    elif kind == "hdr":
        a = rng.uniform(-0.5, 8.0, shape)
        b = np.clip(a + rng.normal(size=shape), -0.5, 8.0)
        a[..., :max(1, H // 3), :max(1, W // 3)] = 6.5
        b[..., :max(1, H // 3), :max(1, W // 3)] = 6.0
    else:
        raise ValueError(kind)
    return np.asarray(a, np.float32), np.asarray(b, np.float32)


def upstream(N, per_image, rng):
    """dL/dssim: per image 1 .. 1e-6 with, for N >= 3, the second one negative and, for N >= 2, the last exactly 0; or one
    scalar."""
    if not per_image:
        return np.array([-0.7], np.float32)
    g = 10.0 ** (-6.0 * np.arange(N) / max(N - 1, 1))
    if N >= 3:
        g[1] = -g[1]
    if N >= 2:
        g[-1] = 0.0
    return g.astype(np.float32)


def alpha_plane(N, H, W, rng):
    """alpha in (0, 1) with an exact-0 band of columns and an exact-1 band of rows."""
    a = rng.uniform(0, 1, (N, H, W))
    a[..., :, :max(1, W // 4)] = 0.0
    a[..., -max(1, H // 4):, :] = 1.0
    return a.astype(np.float32)


BKGD = np.array([0.3, 0.0, 0.7], np.float32)


# each case: shape (N,C,H,W), content, per_image, accumulate, background composite (None, "hw" or "allmap") and the edge
# it asserts
CASES = {
    # the whole image inside one window (H or W <= 11), one 32-px tile
    "px_1x1": ((1, 1, 1, 1), "textured", 0, 0, None),
    "row_1x37": ((1, 1, 1, 37), "patches", 1, 1, None),
    "col_37x1": ((1, 1, 37, 1), "nearconst", 0, 1, None),
    "win_5x7": ((2, 3, 5, 7), "textured", 1, 0, "hw"),
    "win_10x11": ((2, 3, 10, 11), "zeros", 1, 1, "allmap"),
    "win_11x12": ((1, 3, 11, 12), "hdr", 0, 0, None),
    # tile seams and one-pixel last tiles
    "seam_31x33": ((2, 3, 31, 33), "textured", 1, 1, "hw"),
    "seam_32x32": ((1, 3, 32, 32), "patches", 0, 0, None),
    "seam_33x65": ((2, 3, 33, 65), "nearconst", 1, 0, "allmap"),
    "seam_64x63": ((2, 1, 64, 63), "zeros", 1, 1, None),
    "seam_65x97": ((1, 3, 65, 97), "hdr", 0, 1, None),
    # channel counts other than 1 and 3
    "c2_40x33": ((3, 2, 40, 33), "patches", 1, 0, None),
    "c5_33x34": ((2, 5, 33, 34), "textured", 0, 1, None),
    # the per-image upstream spread over 1 .. 1e-6, one negative, one 0, with and without accumulate
    "spread_acc": ((5, 3, 20, 30), "textured", 1, 1, "allmap"),
    "spread": ((5, 1, 40, 9), "patches", 1, 0, None),
    "hdr_allmap": ((3, 3, 45, 50), "hdr", 1, 1, "allmap"),
    # render_loss_batch's shape and layout: M = 4, 3 x 120 x 160, alpha plane 1 of 8
    "production": ((4, 3, 120, 160), "textured", 1, 1, "allmap"),
}


def make_case(name):
    """The inputs of CASES[name]: dict img1, img2, per_image, accumulate, dL_dssim, composite, and with the composite
    alpha (N,H,W) and bkgd; prefills dimg1 (None without accumulate), dalpha (N,H,W), dbkgd (N,3)."""
    shape, kind, per_image, acc, comp = CASES[name]
    N, C, H, W = shape
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    a, b = content(kind, shape, rng)
    out = dict(img1=a, img2=b, per_image=per_image, accumulate=acc, composite=comp,
               dL_dssim=upstream(N, per_image, rng), alpha=None, bkgd=None,
               dimg1=rng.normal(size=shape).astype(np.float32) if acc else None)
    if comp is not None:
        out.update(alpha=alpha_plane(N, H, W, rng), bkgd=BKGD, dalpha=rng.normal(size=(N, H, W)).astype(np.float32),
                   dbkgd=rng.normal(size=(N, 3)).astype(np.float32))
    return out


def fixture_case(name):
    """A tests/golden/ssim_*.npz input as a case: a (C,H,W) input counts as N = 1 with a scalar upstream, an (N,C,H,W) one
    takes its per-image upstream."""
    from .conftest import load_golden
    g = load_golden(name)
    x, y, gup = g["in_img1"], g["in_img2"], g["in_gup"]
    per_image = int(x.ndim == 4)
    if x.ndim == 3:
        x, y = x[None], y[None]
    return dict(img1=np.ascontiguousarray(x, np.float32), img2=np.ascontiguousarray(y, np.float32), per_image=per_image,
                accumulate=0, composite=None, alpha=None, bkgd=None, dimg1=None,
                dL_dssim=np.asarray(gup, np.float32).reshape(-1))


def run_model(case, maps=None):
    """The forward, and the backward on `maps` (default: the forward's fp32 shadow maps)."""
    fw = forward(case["img1"], case["img2"], case["alpha"], case["bkgd"])
    bw = backward(case["img1"], case["img2"], fp32_maps(fw) if maps is None else maps, case["dL_dssim"], case["per_image"],
                  case["alpha"], case["bkgd"], case["dimg1"], case.get("dalpha"), case.get("dbkgd"))
    return fw, bw


def within(x, e, skip=None):
    """The largest |x - value| / (K u B + FLOOR) outside `skip` (NaN counts as infinite)."""
    x = np.asarray(x, np.float64)
    r = np.abs(x - e.v) / (K * U * e.b + FLOOR)
    r = np.where(np.isnan(x), np.inf, r)
    if skip is not None:
        r = np.where(skip, 0.0, r)
    return float(r.max()) if r.size else 0.0
