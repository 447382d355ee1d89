"""Fused bob-skinning warp: canonical surfels -> every frame's camera space (SURVEY.md section 8(f) rows N2/N3).

Python host side of csrc/warp.cu.  Mirrors what the reference computes in
    lab4d/nnutils/deformable_gaussian.py:1395-1434   DeformableGaussian.forward_warp
    lab4d/nnutils/warping.py:378-444                 SkinningWarp.forward (forward direction, return_qt=True)
with the same argument meaning: per-frame bone articulations and the rest articulation as dual quaternions
((…,B,4),(…,B,4)), per-bone log Gaussian scales, optional delta skinning logits, field2cam as (quaternion, translation).
The small per-bone / per-frame tables are prepared here with ordinary differentiable torch ops (they are tens of floats);
the per-surfel work -- where the reference allocates (M,P,B,4) temporaries -- is one CUDA kernel each way.
"""
from __future__ import annotations

import torch

from . import _capi


# Hamilton product as ONE gather + two multiplies + one sum (out_i = sum_j SGN[i][j] * a[IDX[i][j]] * b[j]) instead of the
# 28 elementwise kernels (and ~60 in the backward) of the unbind / stack formulation: the bone tables are tens of floats, so
# their cost is pure launch count -- ~600 of the ~800 kernels of a captured Stage-3 step before this (r2h launch list).
_Q_IDX = ((0, 1, 2, 3), (1, 0, 3, 2), (2, 3, 0, 1), (3, 2, 1, 0))
_Q_SGN = ((1.0, -1.0, -1.0, -1.0), (1.0, 1.0, -1.0, 1.0), (1.0, 1.0, 1.0, -1.0), (1.0, -1.0, 1.0, 1.0))
_q_tables: dict = {}


def _qt(device, dtype):
    key = (str(device), dtype)
    t = _q_tables.get(key)
    if t is None:
        t = (torch.tensor(_Q_IDX, device=device), torch.tensor(_Q_SGN, device=device, dtype=dtype),
             torch.tensor((1.0, -1.0, -1.0, -1.0), device=device, dtype=dtype))
        _q_tables[key] = t
    return t


def _qmul(a, b):
    idx, sgn, _ = _qt(a.device, a.dtype)
    return ((a[..., idx] * sgn) * b[..., None, :]).sum(-1)


def _qconj(q):
    return q * _qt(q.device, q.dtype)[2]


class _BobWarp(torch.autograd.Function):
    @staticmethod
    def forward(ctx, xyz, rot, o2b_q, o2b_t, inv_gauss, se3_r, se3_d, cam_q, cam_t, delta):
        lib = _capi.load()
        f = lambda t: None if t is None else t.detach().to(torch.float32).contiguous()  # noqa: E731
        xyz, rot, o2b_q, o2b_t, inv_gauss, se3_r, se3_d, cam_q, cam_t, delta = map(f, (xyz, rot, o2b_q, o2b_t, inv_gauss, se3_r,
                                                                                      se3_d, cam_q, cam_t, delta))
        if not xyz.is_cuda:
            raise RuntimeError("bob_warp needs CUDA tensors (there is no CPU fallback)")
        P, B, M = int(xyz.shape[0]), int(o2b_q.shape[0]), int(se3_r.shape[0])
        dev = xyz.device
        xyz_cam = torch.empty((M, P, 3), dtype=torch.float32, device=dev)
        rot_cam = torch.empty((M, P, 4), dtype=torch.float32, device=dev)
        ent = torch.empty((P,), dtype=torch.float32, device=dev)
        ptr = lambda t: None if t is None else t.data_ptr()  # noqa: E731
        with torch.cuda.device(dev):
            rc = lib.sr_bob_warp_forward(P, B, M, ptr(xyz), ptr(rot), ptr(o2b_q), ptr(o2b_t), ptr(inv_gauss), ptr(delta), ptr(se3_r),
                                         ptr(se3_d), ptr(cam_q), ptr(cam_t), ptr(xyz_cam), ptr(rot_cam), ptr(ent),
                                         torch.cuda.current_stream(dev).cuda_stream)
        _capi.check(rc, "sr_bob_warp_forward")
        ctx.dims = (P, B, M)
        ctx.has_delta = delta is not None
        ctx.save_for_backward(xyz, rot, o2b_q, o2b_t, inv_gauss, se3_r, se3_d, cam_q, cam_t,
                              delta if delta is not None else torch.empty((0,), device=dev))
        return xyz_cam, rot_cam, ent

    @staticmethod
    def backward(ctx, g_xyz_cam, g_rot_cam, g_ent):
        lib = _capi.load()
        P, B, M = ctx.dims
        xyz, rot, o2b_q, o2b_t, inv_gauss, se3_r, se3_d, cam_q, cam_t, delta = ctx.saved_tensors
        dev = xyz.device
        z = lambda g, shape: torch.zeros(shape, dtype=torch.float32, device=dev) if g is None else g.to(torch.float32).contiguous()  # noqa: E731
        g_xyz_cam, g_rot_cam = z(g_xyz_cam, (M, P, 3)), z(g_rot_cam, (M, P, 4))
        g_ent = None if g_ent is None else g_ent.to(torch.float32).contiguous()
        g_xyz = torch.empty((P, 3), dtype=torch.float32, device=dev)
        g_rot = torch.empty((P, 4), dtype=torch.float32, device=dev)
        g_delta = torch.empty((P, B), dtype=torch.float32, device=dev) if ctx.has_delta else None
        nt = int(lib.sr_bob_warp_table_floats(B, M))
        g_tab = torch.empty((nt,), dtype=torch.float32, device=dev)
        ptr = lambda t: None if t is None else t.data_ptr()  # noqa: E731
        with torch.cuda.device(dev):
            rc = lib.sr_bob_warp_backward(P, B, M, ptr(xyz), ptr(rot), ptr(o2b_q), ptr(o2b_t), ptr(inv_gauss),
                                          ptr(delta) if ctx.has_delta else None, ptr(se3_r), ptr(se3_d), ptr(cam_q), ptr(cam_t),
                                          ptr(g_xyz_cam), ptr(g_rot_cam), ptr(g_ent), ptr(g_xyz), ptr(g_rot), ptr(g_delta),
                                          ptr(g_tab), torch.cuda.current_stream(dev).cuda_stream)
        _capi.check(rc, "sr_bob_warp_backward")
        g_oq, g_ot, g_ig, g_sr, g_sd, g_cq, g_ct = split_table_grads(g_tab, B, M)
        return g_xyz, g_rot, g_oq, g_ot, g_ig, g_sr, g_sd, g_cq, g_ct, g_delta


def split_table_grads(g_tab, B, M):
    """Views of a flat g_tables buffer (sr_bob_warp_table_floats order): g_o2b_q, g_o2b_t, g_inv_gauss, g_se3_r, g_se3_d,
    g_cam_q, g_cam_t."""
    o = 0
    outs = []
    for shape in ((B, 4), (B, 3), (B, 3), (M, B, 4), (M, B, 4), (M, 4), (M, 3)):
        n = 1
        for s_ in shape:
            n *= s_
        outs.append(g_tab[o:o + n].view(shape)); o += n
    return outs


def bob_warp_tables(xyz, rot, o2b_q, o2b_t, inv_gauss, se3, field2cam, delta=None):
    """Low-level entry: the tables already prepared.  se3 = ((M,B,4),(M,B,4)), field2cam = ((M,4),(M,3)).
    Returns xyz_cam (M,P,3), rot_cam (M,P,4), skin_entropy (P,)."""
    return _BobWarp.apply(xyz, rot, o2b_q, o2b_t, inv_gauss, se3[0], se3[1], field2cam[0], field2cam[1], delta)


def bob_warp(xyz, rot, rest_articulation, t_articulation, log_gauss, field2cam, delta=None):
    """forward_warp for M frames (deformable_gaussian.py:1395-1434 with warping.py:404-413).

    xyz (P,3), rot (P,4): canonical surfels.  rest_articulation ((B,4),(B,4)) and t_articulation ((M,B,4),(M,B,4)): bone-to-
    object dual quaternions.  log_gauss (B,3).  field2cam ((M,4),(M,3)).  delta (P,B): optional delta skinning term
    (relu(mlp) * 0.1 of skinning.py:104-119; the MLP itself stays in PyTorch).
    Returns xyz_cam (M,P,3), rot_cam (M,P,4), skin_entropy (P,)."""
    o2b_q, o2b_t, inv_gauss, se3_r, se3_d = warp_tables(rest_articulation, t_articulation, log_gauss)
    return _BobWarp.apply(xyz, rot, o2b_q, o2b_t, inv_gauss, se3_r, se3_d, field2cam[0], field2cam[1], delta)


def warp_tables(rest_articulation, t_articulation, log_gauss):
    """The per-bone / per-frame tables of the warp kernels from the reference's arguments, with differentiable torch ops:
    o2b_q (B,4), o2b_t (B,3), inv_gauss (B,3), se3_r (M,B,4), se3_d (M,B,4)."""
    rr, rd = rest_articulation
    # object -> bone of the rest pose: (q, t) of the inverse dual quaternion (transforms.py:20, quat_transform.py:341-349)
    ir, idq = _qconj(rr), _qconj(rd)
    o2b_q = ir
    o2b_t = 2.0 * _qmul(idq, _qconj(ir))[..., 1:]
    # per frame and bone: t_articulation o rest_articulation^-1 (warping.py:410-413, quat_transform.py:435-443)
    tr, td = t_articulation
    se3_r = _qmul(tr, ir[None])
    se3_d = _qmul(tr, idq[None]) + _qmul(td, ir[None])
    return o2b_q, o2b_t, torch.exp(-log_gauss), se3_r, se3_d
