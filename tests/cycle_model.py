"""TEST INFRASTRUCTURE -- float64 torch restatement of Stage 3's deformation-cycle regulariser (csrc/cycle.cu,
vidu4d_b200.warp.cycle_loss), built on the warp algebra of oracle/warp_oracle.py:

    lab4d/nnutils/deformable_gaussian.py:1517-1574   cycle_loss: cam_to_field, backward warp, apply_qt_to_gaussian, |.|
    lab4d/nnutils/deformable_gaussian.py:738-764     cam_to_field (quat_transform.py:286-291 quaternion_translation_inverse)
    lab4d/nnutils/warping.py:378-444                 SkinningWarp.forward(backward=True): skinning on t_articulation,
                                                     per-bone se3 = rest_articulation o t_articulation^-1
    lab4d/engine/model.py:850-853,994-1012           reg_deform_cyc / reg_delta_skin / reg_skin_entropy, v[v > 0].mean() * wt

Autograd of these expressions is the gradient oracle.  Pinned to tests/golden/cycle_*.npz by tests/test_cycle_cpu.py.
"""
from __future__ import annotations

import torch

from oracle import warp_oracle as wo


def cycle_values(xyz, xyz_cam, rest_dq, t_dq, inv_gauss, field2cam, delta=None):
    """Per frame and surfel: cyc (M,P), dsk (M,P), ent (M,P).

    xyz (P,3) canonical surfels; xyz_cam (M,P,3) the same surfels warped into each frame's camera space; rest_dq
    ((B,4),(B,4)) and t_dq ((M,B,4),(M,B,4)) bone-to-object dual quaternions; inv_gauss (B,3); field2cam ((M,4),(M,3));
    delta (M,P,B) or None."""
    qc, tc = field2cam
    qi = wo.qconj(qc)                                            # cam2field = quaternion_translation_inverse(field2cam)
    ti = wo.qapply(qi, -tc)
    x_t = wo.qapply(qi[:, None], xyz_cam) + ti[:, None]          # (M,P,3) object space at time t
    B = t_dq[0].shape[-2]
    q_ob, t_ob = wo.dq_to_qt(*wo.dq_inverse(t_dq))               # (M,B,4), (M,B,3) object -> bone of t_articulation
    xb = wo.qapply(q_ob[:, None], x_t[:, :, None, :].expand(-1, -1, B, -1)) + t_ob[:, None]      # (M,P,B,3)
    d2 = ((xb * inv_gauss) ** 2).sum(-1)
    logits = -(d2 + delta) if delta is not None else -d2
    w = torch.softmax(logits, -1)                                # (M,P,B)
    M = t_dq[0].shape[0]
    rest_m = (rest_dq[0][None].expand(M, -1, -1), rest_dq[1][None].expand(M, -1, -1))
    qr, qd = wo.dq_mul(rest_m, wo.dq_inverse(t_dq))              # (M,B,4) rest o t^-1
    anchor = w.argmax(-1)                                        # (M,P)
    qa = torch.gather(qr, 1, anchor[..., None].expand(-1, -1, 4))                           # (M,P,4)
    sign = ((qa[:, :, None, :] * qr[:, None, :, :]).sum(-1) > 0).to(xyz.dtype) * 2 - 1     # (M,P,B)
    ws = w * sign
    qr_w = torch.einsum("mpb,mbl->mpl", ws, qr)
    qd_w = torch.einsum("mpb,mbl->mpl", ws, qd)
    inv = 1.0 / qr_w.norm(dim=-1, keepdim=True)
    q, t = wo.dq_to_qt(qr_w * inv, qd_w * inv)
    x_c = wo.qapply(q, x_t) + t
    cyc = (x_c - xyz[None]).norm(dim=-1)
    dsk = (delta ** 2).mean(-1) if delta is not None else torch.zeros_like(cyc)
    return cyc, dsk, wo.skin_entropy(logits)


def positive_mean_terms(values, weights):
    """apply_loss_weights (model.py:994-1012) of each (M,P) value tensor: weight * mean over the values > 0, 0 when there
    are none; a value = 0 gets no gradient.  Returns loss, terms (M,K) each frame's share, counts (M,K)."""
    terms, counts = [], []
    for v, wt in zip(values, weights):
        pos = v > 0
        c = pos.sum(-1)                                          # (M,)
        total = int(c.sum())
        s = wt / total if total else 0.0
        terms.append(torch.where(pos, v, torch.zeros_like(v)).sum(-1) * s)
        counts.append(c)
    terms = torch.stack(terms, -1)
    return terms.sum(), terms, torch.stack(counts, -1)


def cycle_loss(xyz, xyz_cam, rest_dq, t_dq, inv_gauss, field2cam, delta=None, weights=(0.01, 5e-3, 5e-4)):
    """loss, terms (M,3), counts (M,3), values (cyc, dsk, ent) of {reg_deform_cyc, reg_delta_skin, reg_skin_entropy}."""
    vals = cycle_values(xyz, xyz_cam, rest_dq, t_dq, inv_gauss, field2cam, delta)
    loss, terms, counts = positive_mean_terms(vals, weights)
    return loss, terms, counts, vals
