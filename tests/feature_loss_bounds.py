"""TEST INFRASTRUCTURE -- the fused feature-plane losses (csrc/loss.cu: feat_loss_kernel, feat_loss_scale_kernel)
restated operation for operation, with their rounding-error bound (tests/error_bound.py).

On the kernels' own fp32 inputs, per pixel:
  * feature term:  d_c = f_c - t_c;  ss = 0, ss += d_c * d_c over the Cf channels;  nrm = sqrtf(ss);  wpx = mask * det;
    v = nrm * wpx;  on = v > 0;  k = on ? wpx / nrm : 0;  g_c = (f_c - t_c) * k.  nvcc may contract ss += d * d into one
    FMA; the product's rounding and the sum's, both charged, bound the contracted and the uncontracted evaluation.
  * Gaussian-mask term:  d = f_gm - alpha;  v = d * d;  on = v > 0;  g_gm = on ? 2 d : 0 (2 d is exact).
  * scale:  s = w / (float)C with C the batch-wide count of on pixels (0 when C = 0), one rounding;  every touched plane
    element g *= s, one rounding;  the per-frame term: each block sums its on values with a 5-level xor butterfly per
    warp and a chain of the 8 warp partials, then one fp32 atomicAdd per block onto the memset 0, in no fixed order:
    (5 + 8 + blocks) u sum |v| in all;  then term *= s, one rounding.

Knife pixels: where the float64 v lies within its own bound of 0 (|v| <= K u B, B > 0), the kernel's `v > 0` may go
either way -- v = nrm * mask can underflow to 0 for a tiny mask, and d * d for |d| near 1e-23.  Their plane elements are
not compared; the counts may differ from the model's by at most their number; the term's bound takes their |v| in.  The
model scales with the counts it is given (the GPU's own), as the rasterizer oracles composite from the GPU's records.

shadow() is the same computation in float32 NumPy, decision for decision and in the kernels' summation order; `mutate`
plants one of the mistakes the CPU tests must see fall outside the bound.
"""
from __future__ import annotations

import numpy as np

from .error_bound import TINY_U, _E, _where

U = 2.0 ** -24
K = 2.0
FLOOR = float(np.finfo(np.float32).tiny)
BX, BY = 32, 8                         # the kernels' block: 32 x 8 pixels, 8 warps of one row each
MUTATIONS = ("no_is_detected", "per_frame_count", "v_ge_0", "no_factor_2", "no_wpx_in_k")


def _nblocks(H, W):
    return -(-W // BX) * -(-H // BY)


def _arr(x, shape=None):
    return None if x is None else np.ascontiguousarray(np.asarray(x, np.float32) if shape is None
                                                       else np.broadcast_to(np.asarray(x, np.float32), shape))


def pixel_terms(feat, target, mask, is_detected, alpha, gm):
    """The unscaled per-pixel quantities as running-error values.  Returns a dict with, per term k in (0 feature,
    1 Gaussian mask) present: v[k] (M,H,W) _E, knife[k] (M,H,W) bool, grad planes g[c] (M,H,W) _E unscaled (value where
    the float64 v > 0, else exactly 0)."""
    feat = _arr(feat)
    M, F, H, W = feat.shape
    out = {"v": {}, "knife": {}, "g": {}}
    if target is not None:
        tg = _arr(target)
        Cf = tg.shape[1]
        det = np.ones(M, np.float32) if is_detected is None else _arr(is_detected)
        wpx = _E.leaf(mask) * _E.leaf(np.broadcast_to(det[:, None, None], (M, H, W)))
        d = [_E.leaf(feat[:, c]) - _E.leaf(tg[:, c]) for c in range(Cf)]
        ss = _E(np.zeros((M, H, W)), None, np.zeros((M, H, W), np.float32))
        for c in range(Cf):
            ss = ss + d[c] * d[c]
        nrm = ss.sqrt()
        v = nrm * wpx
        on = v.v > 0
        k = _where(on, wpx / _where(on, nrm, 1.0), 0.0)
        out["v"][0] = v
        out["knife"][0] = (v.b > 0) & (np.abs(v.v) <= K * U * v.b)
        for c in range(Cf):
            out["g"][c] = d[c] * k
    if gm is not None and gm >= 0:
        d = _E.leaf(feat[:, gm]) - _E.leaf(alpha)
        v = d * d
        on = v.v > 0
        out["v"][1] = v
        out["knife"][1] = (v.b > 0) & (np.abs(v.v) <= K * U * v.b)
        out["g"][gm] = _where(on, d.scale(2.0), 0.0)
    return out


def scaled(px, counts, weights, gm):
    """The scale kernel on the model's unscaled values with the given (M,2) counts (the GPU's own): per term the scale
    s = w / C as an _E, the planes g[c] * s and the per-frame terms sum(v on) * s with the reduction's bound."""
    counts = np.asarray(counts, np.int64)
    w = np.asarray(weights, np.float32)
    M, H, W = next(iter(px["v"].values())).v.shape
    depth = 5 + 8 + _nblocks(H, W)
    s, terms, g = {}, {}, {}
    for k, v in px["v"].items():
        C = int(counts[:, k].sum())
        s[k] = _E(0.0) if C == 0 else _E.leaf(w[k]) / _E(float(C))      # (float)C: exact below 2^24
        kn = px["knife"][k]
        on = (v.v > 0) & ~kn
        av = np.abs(v.v)
        sv = np.where(on, v.v, 0.0).reshape(M, -1).sum(1)
        sb = (np.where(on, v.b, 0.0) + depth * np.where(on, av, 0.0)).reshape(M, -1).sum(1)
        # a knife pixel's v may be in the GPU's sum or not: it brings in at most |v| + K u B
        sb = sb + np.where(kn, av / (K * U) + v.b + depth * (av + K * U * v.b), 0.0).reshape(M, -1).sum(1)
        terms[k] = _E(sv, sb) * s[k]
    for c, e in px["g"].items():
        g[c] = e * s[1 if c == gm else 0]
    return s, terms, g


def shadow(feat, target, mask, is_detected, alpha, gm, weights, mutate=None, fma=False):
    """The two kernels in float32 NumPy, in their order.  Returns (terms (M,2), counts (M,2), grad (M,F,H,W)).
    fma: evaluate ss += d * d as one fused multiply-add (nvcc's contraction) instead of two roundings."""
    assert mutate in (None,) + MUTATIONS, mutate
    feat = _arr(feat)
    M, F, H, W = feat.shape
    f32 = np.float32
    part = np.zeros((2, M, H, W), f32)
    on = np.zeros((2, M, H, W), bool)
    grad = np.zeros_like(feat)
    with np.errstate(all="ignore"):
        if target is not None:
            tg = _arr(target)
            Cf = tg.shape[1]
            det = np.ones(M, f32) if is_detected is None else _arr(is_detected)
            if mutate == "no_is_detected":
                det = np.ones(M, f32)
            wpx = _arr(mask) * det[:, None, None]
            ss = np.zeros((M, H, W), f32)
            for c in range(Cf):
                d = feat[:, c] - tg[:, c]
                ss = (d.astype(np.float64) * d + ss).astype(f32) if fma else ss + d * d
            nrm = np.sqrt(ss)
            v = nrm * wpx
            on[0] = v >= 0 if mutate == "v_ge_0" else v > 0
            k = np.where(on[0], (f32(1.0) if mutate == "no_wpx_in_k" else wpx) / nrm, f32(0.0))
            for c in range(Cf):
                grad[:, c] = (feat[:, c] - tg[:, c]) * k
            part[0] = np.where(on[0], v, f32(0.0))
        if gm is not None and gm >= 0:
            d = feat[:, gm] - _arr(alpha)
            v = d * d
            on[1] = v > 0
            grad[:, gm] = np.where(on[1], d if mutate == "no_factor_2" else f32(2.0) * d, f32(0.0))
            part[1] = np.where(on[1], v, f32(0.0))
        counts = on.reshape(2, M, -1).sum(-1).T.astype(np.int64)
        sums = np.stack([_block_sums(part[k]) for k in range(2)], 1)
        w = np.asarray(weights, f32)
        terms = np.zeros((M, 2), f32)
        for k in range(2):
            C = counts[:, k] if mutate == "per_frame_count" else np.full(M, counts[:, k].sum())
            s = np.where(C > 0, w[k] / np.maximum(C, 1).astype(f32), f32(0.0)).astype(f32)
            terms[:, k] = sums[:, k] * s
            if k == 0:
                chans = range(tg.shape[1]) if target is not None else []
            else:
                chans = [gm] if gm is not None and gm >= 0 else []
            for c in chans:
                grad[:, c] = grad[:, c] * s[:, None, None]
    return terms, counts, grad


def _block_sums(p):
    """Per frame, the fp32 term as the kernel forms it: per block the xor butterfly of each warp (one 32-pixel row),
    the 8 warp partials in order, then the blocks' totals added in block order onto 0."""
    M, H, W = p.shape
    TY, TX = -(-H // BY), -(-W // BX)
    q = np.zeros((M, TY * BY, TX * BX), np.float32)
    q[:, :H, :W] = p
    q = q.reshape(M, TY, BY, TX, BX).transpose(0, 1, 3, 2, 4).reshape(M, TY * TX, BY, BX)
    lane = np.arange(BX)
    for o in (16, 8, 4, 2, 1):
        q = q + q[..., lane ^ o]
    t = np.zeros((M, TY * TX), np.float32)
    for wp in range(BY):
        t = t + q[..., wp, 0]
    out = np.zeros(M, np.float32)
    for b in range(TY * TX):
        out = out + t[:, b]
    return out


def check(name, terms, counts, grad, px, weights, gm, F, report=None):
    """Every element of a GPU (or shadow) result against the model: counts exact outside the knife, within the knife
    count in all; plane elements outside the knife under the bound, untouched channels exactly 0; the per-frame terms
    under theirs.  Returns the headroom per tensor (largest err / (K u B + FLOOR)); asserts it is <= 1."""
    terms = np.asarray(terms, np.float64)
    counts = np.asarray(counts, np.int64)
    grad = np.asarray(grad, np.float64)
    report = {} if report is None else report
    assert not np.isnan(grad).any() and not np.isnan(terms).any(), name
    for k, v in px["v"].items():
        kn = px["knife"][k]
        want = ((v.v > 0) & ~kn).reshape(len(counts), -1).sum(1)
        nk = kn.reshape(len(counts), -1).sum(1)
        assert np.all((counts[:, k] >= want) & (counts[:, k] <= want + nk)), (name, k, counts[:, k], want, nk)
    _, tm, g = scaled(px, counts, weights, gm)
    for k in range(2):
        if k in tm:
            _within(name, f"terms[{k}]", terms[:, k], tm[k], report)
        else:
            assert (terms[:, k] == 0).all() and (counts[:, k] == 0).all(), (name, k)
    for c in range(F):
        if c not in g:
            assert (grad[:, c] == 0).all(), (name, "untouched channel", c)
            continue
        kn = px["knife"][1 if c == gm else 0]
        _within(name, "grad_gm" if c == gm else "grad_feat", grad[:, c], g[c], report, skip=kn)
    return report


def ratio(x, e, skip=None):
    """err / (K u B + FLOOR) element by element (NaN is infinite), 0 under `skip`."""
    x = np.asarray(x, np.float64)
    r = np.abs(x - e.v) / (K * U * e.b + FLOOR)
    r = np.where(np.isnan(x), np.inf, r)
    return r if skip is None else np.where(skip, 0.0, r)


def _within(name, what, x, e, report, skip=None):
    r = ratio(x, e, skip)
    i = int(np.argmax(r)) if r.size else 0
    m = float(r.flat[i]) if r.size else 0.0
    report[what] = max(report.get(what, 0.0), m)
    assert m <= 1.0, (name, what, "element", np.unravel_index(i, r.shape), "got", np.asarray(x).flat[i], "model",
                      e.v.flat[i], "bound", K * U * e.b.flat[i] + FLOOR)


# ------------------------------------------------------------------------------------------------ inputs
WEIGHTS = np.array([1e-2, 7e-3], np.float32)

# the seeded configurations the CPU and GPU tests share: Cf = F, Cf = 1, the Gaussian-mask term alone, F = 32, one frame
# undetected and one at 0.5, a batch where nothing is positive; ragged sizes on the 32 x 8 grid
CONFIGS = {
    "f22_det_0_half": dict(M=3, W=65, H=33, F=22, Cf=16, gm=21, det=(1.0, 0.0, 0.5)),
    "cf_eq_f": dict(M=2, W=33, H=9, F=16, Cf=16, gm=-1, det=(0.5, 1.0)),
    "cf_1": dict(M=2, W=40, H=17, F=4, Cf=1, gm=3, det=None),
    "gm_only": dict(M=2, W=97, H=9, F=5, Cf=0, gm=2, det=None),
    "f32": dict(M=1, W=64, H=16, F=32, Cf=16, gm=31, det=None),
    "nothing_positive": dict(M=2, W=33, H=9, F=22, Cf=16, gm=21, det=None, empty=True),
}


def config_inputs(name):
    """CONFIGS[name]'s planted inputs: (feat, target, mask, det, alpha, gm, planted)."""
    c = CONFIGS[name]
    feat, target, mask, det, alpha, planted = planted_inputs(c["M"], c["W"], c["H"], c["F"], c["Cf"], c["gm"],
                                                             seed=sum(map(ord, name)), det=c["det"])
    if c.get("empty"):
        mask[:] = 0.0
        feat[:, c["gm"]] = alpha
    return feat, target, mask, det, alpha, c["gm"], planted


PLANTS =("feat_eq_target", "gm_eq_alpha", "mask_zero", "mask_frac", "mask_1e-30", "d_1e-20")


def _sites(H, W):
    """(seam site, border site) for a plant: the first column of the second 32-wide block (or a row seam), and the last
    column of the image."""
    seam = (min(8, H - 1), min(32, W - 1)) if W > 32 else (min(8, H - 1), W // 2)
    return seam, (H // 2, W - 1)


def planted_inputs(M, W, H, F, Cf, gm, seed, det=None):
    """Seeded planes (M,F,H,W), target (M,Cf,H,W) (None for Cf = 0), mask (M,H,W), is_detected (M,), alpha (M,H,W),
    with each PLANTS kind put on a block seam and on the image border of some frame.  Returns the inputs and the
    planted list [(kind, frame, y, x)]."""
    rng = np.random.default_rng(seed)
    f32 = np.float32
    feat = rng.normal(size=(M, F, H, W)).astype(f32)
    target = rng.normal(size=(M, Cf, H, W)).astype(f32) if Cf > 0 else None
    mask = np.where(rng.uniform(size=(M, H, W)) < 0.6, rng.uniform(0.1, 1.0, (M, H, W)), 0.0).astype(f32)
    alpha = rng.uniform(0, 1, (M, H, W)).astype(f32)
    alpha[rng.uniform(size=(M, H, W)) < 0.1] = 0.0
    if det is None:
        det = np.ones(M, f32)
    det = np.asarray(det, f32)
    planted = []
    for i, kind in enumerate(PLANTS):
        for j, (y, x) in enumerate(_sites(H, W)):
            f = (i + j) % M
            if kind == "feat_eq_target" and target is not None:
                feat[f, :Cf, y, x] = target[f, :, y, x]
            elif kind == "gm_eq_alpha" and gm >= 0:
                feat[f, gm, y, x] = alpha[f, y, x]
            elif kind == "mask_zero":
                mask[f, y, x] = 0.0
            elif kind == "mask_frac":
                mask[f, y, x] = f32(0.375)
            elif kind == "mask_1e-30":           # on the seam v = 1e-30 * (a 1e-20-sized nrm) underflows to 0
                mask[f, y, x] = f32(1e-30)
                if target is not None and j == 0:
                    target[f, :, y, x] = 0.0
                    feat[f, :Cf, y, x] = f32(1e-20) * np.sign(rng.normal(size=Cf)).astype(f32)
            elif kind == "d_1e-20":             # d * d underflows to a subnormal (feature) / to 0 (|d| ~ 1e-23)
                if target is not None:
                    target[f, :, y, x] = 0.0
                    feat[f, :Cf, y, x] = (1e-20 * rng.uniform(0.5, 2.0, Cf)).astype(f32)
                    mask[f, y, x] = 1.0
                if gm >= 0:
                    alpha[f, y, x] = 0.0
                    feat[f, gm, y, x] = f32(1e-20 if j == 0 else 3e-24)
            else:
                continue
            planted.append((kind, f, y, x))
    return feat, target, mask, det, alpha, planted
