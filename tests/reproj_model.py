"""TEST INFRASTRUCTURE -- float64 torch restatement of Stage 3's feat_reproj loss (csrc/match.cu, vidu4d_b200.registration).

    lab4d/nnutils/deformable_gaussian.py:1436-1486   global_match (num_grad = K): scores against the drawn candidates, top-K,
                                                     softmax at temperature exp(logsigma), prob-weighted xyz
    lab4d/nnutils/deformable_gaussian.py:1488-1513   forward_project: the bob warp of oracle/warp_oracle.py on each frame's
                                                     matched points, then pinhole_projection K x / (z + 1e-6)
    lab4d/engine/model.py:669-672,915,961-967,994-1012   ||xy - hxy[..., :2]|| * mask * is_detected; weight * mean over
                                                     the batch's positive values / train_res
Autograd of these expressions is the gradient oracle.  The top-K order is the kernel's: larger score first, the lower
candidate position first among equal scores.  Pinned to tests/golden/reproj_*.npz by tests/test_reproj_cpu.py.
"""
from __future__ import annotations

import torch

from oracle import warp_oracle as wo


def q2dq(q, t):
    """quaternion_translation_to_dual_quaternion (quat_transform.py): (q, 0.5 (0,t) q)."""
    return q, 0.5 * wo.qmul(torch.cat((torch.zeros_like(t[..., :1]), t), -1), q)


def all_scores(feat_px, regist_feat, cand):
    """(M*H*W, C) scores feat_px . regist_feat[cand mod P]."""
    return feat_px.reshape(-1, feat_px.shape[-1]) @ regist_feat[cand.long() % regist_feat.shape[0]].T


def global_match(feat_px, regist_feat, xyz, cand, logsigma, K, order=None):
    """Returns xyz_matched (M,H,W,3), the top-K candidate positions (N,K), their probs (N,K) and all scores (N,C).
    `order` (N,K), optional: use these candidate sets instead of the top-K (e.g. a kernel's, once checked to be valid)."""
    score = all_scores(feat_px, regist_feat, cand)
    if order is None:
        order = torch.sort(-score.detach(), dim=1, stable=True).indices[:, :K]
    prob = torch.softmax(score.gather(1, order) * logsigma.exp(), 1)
    xyz_c = xyz[cand.long() % xyz.shape[0]]
    xyz_m = (prob[..., None] * xyz_c[order]).sum(1)
    return xyz_m.reshape(feat_px.shape[:-1] + (3,)), order, prob, score


def weighted_xyz(xyz, cand, order, prob):
    """The prob-weighted canonical xyz of given top-K sets (N,K)."""
    return (prob[..., None] * xyz[cand.long() % xyz.shape[0]][order]).sum(1)


def reproj(xyz_m, Kmat, rest_dq, inv_gauss, se3, field2cam, delta=None):
    """xy_reproj (M,H,W,2): each frame's matched points warped by that frame's bones and field2cam, then projected."""
    M, H, W = xyz_m.shape[:3]
    B = inv_gauss.shape[0]
    out = []
    for m in range(M):
        pts = xyz_m[m].reshape(-1, 3)
        rot = torch.zeros((pts.shape[0], 4), dtype=pts.dtype, device=pts.device)
        rot[:, 0] = 1.0
        d = None if delta is None else delta[m].reshape(-1, B)
        xc, _, _ = wo.bob_warp(pts, rot, rest_dq, inv_gauss, (se3[0][m:m + 1], se3[1][m:m + 1]),
                               (field2cam[0][m:m + 1], field2cam[1][m:m + 1]), d)
        h = xc[0] @ Kmat[m].T
        out.append(h[:, :2] / (h[:, 2:] + 1e-6))
    return torch.stack(out).reshape(M, H, W, 2)


def reproj_loss(xy, hxy, mask, det, weight, train_res):
    """Returns loss, per-frame terms (M,), per-frame counts (M,)."""
    v = (xy - hxy[..., :2]).norm(dim=-1) * mask * det[:, None, None]
    on = v > 0
    c = int(on.sum())
    per_frame = torch.where(on, v, torch.zeros_like(v)).sum((1, 2))
    terms = per_frame * (weight / (c * train_res)) if c > 0 else per_frame * 0.0
    return terms.sum(), terms, on.sum((1, 2))


def run_fixture(g, dtype=torch.float64, device="cpu", order=None):
    """The model on the inputs of a reproj_*.npz fixture (numpy arrays under in_*), with leaf tensors requiring grad.
    `order`: optional candidate sets to use instead of the top-K (global_match).  Returns (leaves, outputs)."""
    skip = ("in_cand", "in_meta", "in_feat_px", "in_Kmat", "in_hxy", "in_mask", "in_is_detected", "in_weight")
    t = {k[3:]: torch.tensor(v, dtype=dtype, device=device).requires_grad_(True) for k, v in g.items()
         if k.startswith("in_") and k not in skip}
    K, train_res = (int(v) for v in g["in_meta"])
    cand = torch.from_numpy(g["in_cand"]).to(device)
    f = lambda k: torch.tensor(g[k], dtype=dtype, device=device)  # noqa: E731
    M = g["in_feat_px"].shape[0]
    xyz_m, order, prob, score = global_match(f("in_feat_px"), t["regist_feat"], t["xyz"], cand, t["logsigma"], K, order)
    rest = q2dq(t["rest_q"], t["rest_t"])
    art = q2dq(t["art_q"], t["art_t"])
    rest_m = (rest[0][None].expand(M, -1, -1), rest[1][None].expand(M, -1, -1))
    se3 = wo.dq_mul(art, wo.dq_inverse(rest_m))
    xy = reproj(xyz_m, f("in_Kmat"), rest, torch.exp(-t["log_gauss"]), se3, (t["cam_q"], t["cam_t"]), t.get("delta"))
    loss, terms, counts = reproj_loss(xy, f("in_hxy"), f("in_mask"), f("in_is_detected"), float(g["in_weight"][0]), train_res)
    return t, dict(xyz_matched=xyz_m, order=order, prob=prob, score=score, xy_reproj=xy, loss=loss, terms=terms, counts=counts)
