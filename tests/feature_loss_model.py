"""Float64 NumPy restatement of the Stage-3 losses on the feature planes and of their gradient (csrc/loss.cu,
sr_feature_loss_batch), pinned to the reference's own code by the tests/golden/featloss_*.npz fixtures
(tests/golden/make_feature_loss_golden.py):

    lab4d/engine/model.py:663-667    feature = ||feat_r - feat_gt||_2 over the target's channels
    lab4d/engine/model.py:742-745    reg_gauss_mask = (gauss_mask_r - acc.detach())^2
    lab4d/engine/model.py:952-967    feature *= mask (keys_fg), then *= is_detected[frame]; reg_gauss_mask unmasked
    lab4d/engine/model.py:1000-1012  term = w * mean(v[v > 0]) over the whole batch, or v.mean() if nothing is > 0

Planes are (M,C,H,W); mask (M,H,W); is_detected (M,) or None; alpha (M,H,W) is allmap plane 1.
"""
from __future__ import annotations

import numpy as np


def _positive_mean(v):
    """(per-frame share of mean(v[v > 0]), per-frame count of v > 0, d term / d v); v (M,H,W) float64."""
    on = v > 0
    cnt = on.reshape(len(v), -1).sum(1)
    C = int(cnt.sum())
    if C == 0:        # v.mean(): v >= 0 here (norms and squares times non-negative masks), so the mean is 0
        return np.zeros(len(v)), cnt, np.zeros_like(v)
    return np.where(on, v, 0.0).reshape(len(v), -1).sum(1) / C, cnt, on / C


def feature_losses(features, target, mask, is_detected, alpha, gauss_mask_channel, weights):
    """Returns (terms (M,2) per-frame shares of the weighted {feature, reg_gauss_mask} terms, counts (M,2) of v > 0,
    grad (M,F,H,W) of the sum of the two terms w.r.t. the feature planes).  target None: no feature term;
    gauss_mask_channel -1 / None: no Gaussian-mask term."""
    feat = np.asarray(features, np.float64)
    M, F = feat.shape[:2]
    terms, counts, grad = np.zeros((M, 2)), np.zeros((M, 2), np.int64), np.zeros_like(feat)
    if target is not None:
        tg = np.asarray(target, np.float64)
        Cf = tg.shape[1]
        d = feat[:, :Cf] - tg
        nrm = np.sqrt((d * d).sum(1))
        det = np.ones(M) if is_detected is None else np.asarray(is_detected, np.float64)
        wpx = np.asarray(mask, np.float64) * det[:, None, None]
        share, counts[:, 0], dv = _positive_mean(nrm * wpx)
        terms[:, 0] = weights[0] * share
        with np.errstate(invalid="ignore", divide="ignore"):
            unit = np.where(nrm[:, None] > 0, d / nrm[:, None], 0.0)        # torch's norm gradient is 0 at ||d|| = 0
        grad[:, :Cf] = weights[0] * (dv * wpx)[:, None] * unit
    if gauss_mask_channel is not None and gauss_mask_channel >= 0:
        d = feat[:, gauss_mask_channel] - np.asarray(alpha, np.float64)
        share, counts[:, 1], dv = _positive_mean(d * d)
        terms[:, 1] = weights[1] * share
        grad[:, gauss_mask_channel] += weights[1] * dv * 2.0 * d
    return terms, counts, grad
