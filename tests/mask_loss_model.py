"""Float64 NumPy restatement of Stage 3's fused silhouette loss (csrc/mask_loss.cu, sr_mask_loss_batch) and of its
gradient, with a first-order bound on the kernels' fp32 rounding (tests/error_bound.py).  Pinned to the reference's own
code by the tests/golden/maskloss_*.npz fixtures (tests/golden/make_mask_loss_golden.py):

    lab4d/engine/model.py:587-611    get_mask_balance_wt: vd = vis2d * is_detected;  pos_wt = sum(vd) / sum(mask[vd > 0]),
                                     neg_wt = sum(vd) / sum(1 - mask[vd > 0]);  bw = 0.5 pos_wt mask + 0.5 neg_wt (1 - mask)
                                     if sum(mask) > 0 and sum(1 - mask) > 0, else 1
    lab4d/engine/model.py:648-650    v = (acc - mask)^2 * bw
    lab4d/engine/model.py:950-967    v *= vis2d, then v *= is_detected[frame]
    lab4d/engine/model.py:1000-1012  loss = w * mean(v[v > 0]) over the whole batch, or w * mean(v) if nothing is > 0

Planes are (M,H,W); is_detected (M,) or None; vis2d (M,H,W) or None.  The three passes are modelled as the kernels run
them: the five sums in float64, rounded to fp32, then fp32 divisions (mask_stats); v and dv/dacc per pixel in the kernels'
fp32 operation order (mask_loss); the scale w / C in fp32 and the per-frame shares in float64 (mask_loss_scale).
"""
from __future__ import annotations

import numpy as np

from .error_bound import _E

U = 2.0 ** -24


def balance(mask, vis2d, is_detected):
    """(pos_wt, neg_wt, branch) as mask_stats forms them: float64 sums rounded to fp32, fp32 divisions."""
    m = np.asarray(mask, np.float32)
    M = m.shape[0]
    vis = np.ones_like(m) if vis2d is None else np.asarray(vis2d, np.float32)
    det = np.ones(M, np.float32) if is_detected is None else np.asarray(is_detected, np.float32)
    vd = vis * det[:, None, None]                              # one fp32 product: exact in float32 arithmetic
    n = np.float32(1.0) - m
    on = vd > 0
    s = [np.float32(x.astype(np.float64).sum()) for x in (vd, np.where(on, m, 0), np.where(on, n, 0), m, n)]
    with np.errstate(divide="ignore", invalid="ignore"):
        pos, neg = np.float32(s[0] / s[1]), np.float32(s[0] / s[2])
    return pos, neg, bool(s[3] > 0 and s[4] > 0)


def mask_loss(alpha, mask, vis2d, is_detected, weight):
    """Returns a dict: "terms" (M,) each frame's share of the loss, "counts" (M,) of v > 0, "grad" (M,H,W) d loss / d alpha,
    "pos_wt" / "neg_wt" / "branch" (the balance weights, fp32), and the bounds (absolute, float64) of the kernels' fp32
    evaluation: "terms_bound" (M,), "grad_bound" (M,H,W).  "v" is the fp32 value of v the kernels form (its shadow)."""
    a = _E.leaf(alpha)
    m = _E.leaf(mask)
    M, H, W = a.v.shape
    vis = _E.leaf(np.ones((M, H, W), np.float32) if vis2d is None else vis2d)
    det = _E.leaf(np.broadcast_to((np.ones(M, np.float32) if is_detected is None else np.asarray(is_detected, np.float32))
                                  [:, None, None], (M, H, W)))
    pos, neg, on = balance(mask, vis2d, is_detected)
    w = float(np.float32(weight))
    one = _E.leaf(np.ones((M, H, W), np.float32))
    with np.errstate(all="ignore"):
        if on:
            bw = _E.leaf(np.full((M, H, W), pos)).scale(0.5) * m + _E.leaf(np.full((M, H, W), neg)).scale(0.5) * (one - m)
        else:
            bw = one
        d = a - m
        v = d * d * bw * vis * det
        dv = det * vis * bw * d.scale(2.0)
        positive = v.f > 0                                     # the kernels' decision, on their own fp32 v
        cnt = positive.reshape(M, -1).sum(1)
        C = int(cnt.sum())
        if C > 0:
            scale, inv = np.float32(np.float32(w) / np.float32(C)), w / C
            sums = np.where(positive, v.v, 0.0).reshape(M, -1).sum(1)
            sums_b = np.where(positive, v.b, 0.0).reshape(M, -1).sum(1)
            sel = positive
        else:
            n = float(M * H * W)
            scale, inv = np.float32(np.float32(w) / np.float32(n)), w / n
            sums, sums_b, sel = v.v.reshape(M, -1).sum(1), v.b.reshape(M, -1).sum(1), np.ones_like(positive)
        terms = sums * inv
        terms_bound = (sums_b * U + 1e-12 * np.abs(sums)) * inv + np.abs(terms) * U      # + the fp32 rounding of the share
        g_exact = np.where(sel, float(scale) * dv.v, 0.0)
        g_bound = np.where(sel, float(scale) * dv.b * U + np.abs(g_exact) * U, 0.0)
        # the scale itself: w / C rounded once against the exact quotient
        g_bound = g_bound + np.where(sel, np.abs(dv.v) * abs(float(scale) - inv), 0.0)
        grad = np.where(sel, inv * dv.v, 0.0)
    return {"terms": terms, "counts": cnt.astype(np.int64), "grad": grad, "pos_wt": pos, "neg_wt": neg, "branch": on,
            "terms_bound": terms_bound, "grad_bound": g_bound, "v": v.f, "scale": scale}
