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

B_MAX = 64                    # bones per call (the warp, reprojection, cycle and feature-row kernels)
TABLE_SMEM_MAX = 200 * 1024   # bytes of shared memory the bone / frame tables may take (SR_TABLE_SMEM_MAX)

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
        _capi.call("sr_bob_warp_forward", dev, P, B, M, xyz, rot, o2b_q, o2b_t, inv_gauss, delta, se3_r, se3_d, cam_q, cam_t,
                   xyz_cam, rot_cam, ent)
        ctx.dims = (P, B, M)
        ctx.has_delta = delta is not None
        ctx.save_for_backward(xyz, rot, o2b_q, o2b_t, inv_gauss, se3_r, se3_d, cam_q, cam_t,
                              delta if delta is not None else torch.empty((0,), device=dev))
        return xyz_cam, rot_cam, ent

    @staticmethod
    def backward(ctx, g_xyz_cam, g_rot_cam, g_ent):
        P, B, M = ctx.dims
        xyz, rot, o2b_q, o2b_t, inv_gauss, se3_r, se3_d, cam_q, cam_t, delta = ctx.saved_tensors
        dev = xyz.device
        z = lambda g, shape: torch.zeros(shape, dtype=torch.float32, device=dev) if g is None else g.to(torch.float32).contiguous()  # noqa: E731
        g_xyz_cam, g_rot_cam = z(g_xyz_cam, (M, P, 3)), z(g_rot_cam, (M, P, 4))
        g_ent = None if g_ent is None else g_ent.to(torch.float32).contiguous()
        g_xyz = torch.empty((P, 3), dtype=torch.float32, device=dev)
        g_rot = torch.empty((P, 4), dtype=torch.float32, device=dev)
        g_delta = torch.empty((P, B), dtype=torch.float32, device=dev) if ctx.has_delta else None
        g_tab = torch.empty((int(_capi.load().sr_bob_warp_table_floats(B, M)),), dtype=torch.float32, device=dev)
        _capi.call("sr_bob_warp_backward", dev, P, B, M, xyz, rot, o2b_q, o2b_t, inv_gauss, delta if ctx.has_delta else None,
                   se3_r, se3_d, cam_q, cam_t, g_xyz_cam, g_rot_cam, g_ent, g_xyz, g_rot, g_delta, g_tab)
        g_oq, g_ot, g_ig, g_sr, g_sd, g_cq, g_ct = split_table_grads(g_tab, B, M)
        return g_xyz, g_rot, g_oq, g_ot, g_ig, g_sr, g_sd, g_cq, g_ct, g_delta


def table_views(flat, shapes):
    """Consecutive views of the flat buffer `flat`, one per shape, from its start."""
    views, o = [], 0
    for shape in shapes:
        n = 1
        for s_ in shape:
            n *= s_
        views.append(flat[o:o + n].view(shape)); o += n
    return views


def split_table_grads(g_tab, B, M):
    """Views of a flat g_tables buffer (sr_bob_warp_table_floats order): g_o2b_q, g_o2b_t, g_inv_gauss, g_se3_r, g_se3_d,
    g_cam_q, g_cam_t."""
    return table_views(g_tab, ((B, 4), (B, 3), (B, 3), (M, B, 4), (M, B, 4), (M, 4), (M, 3)))


def check_pairs(named):
    """Raise RuntimeError unless every (name, pair, shapes) has two tensors of the two given shapes."""
    for name, pair, shapes in named:
        if len(pair) != 2 or tuple(pair[0].shape) != shapes[0] or tuple(pair[1].shape) != shapes[1]:
            raise RuntimeError(f"{name} must be tensors of shapes {shapes}, got {[tuple(t.shape) for t in pair]}")


def check_articulations(B, M, rest_articulation, t_articulation, field2cam):
    """The shapes of the warp's articulation and camera arguments: ((B,4),(B,4)), ((M,B,4),(M,B,4)), ((M,4),(M,3))."""
    check_pairs((("rest_articulation", rest_articulation, ((B, 4), (B, 4))),
                 ("t_articulation", t_articulation, ((M, B, 4), (M, B, 4))),
                 ("field2cam", field2cam, ((M, 4), (M, 3)))))


def bob_warp_tables(xyz, rot, o2b_q, o2b_t, inv_gauss, se3, field2cam, delta=None):
    """Low-level entry: the tables already prepared.  se3 = ((M,B,4),(M,B,4)), field2cam = ((M,4),(M,3)).
    Returns xyz_cam (M,P,3), rot_cam (M,P,4), skin_entropy (P,)."""
    return _BobWarp.apply(xyz, rot, o2b_q, o2b_t, inv_gauss, se3[0], se3[1], field2cam[0], field2cam[1], delta)


def bob_warp(xyz, rot, rest_articulation, t_articulation, log_gauss, field2cam, delta=None):
    """forward_warp for M frames (deformable_gaussian.py:1395-1434 with warping.py:404-413).

    xyz (P,3), rot (P,4): canonical surfels.  rest_articulation ((B,4),(B,4)) and t_articulation ((M,B,4),(M,B,4)): bone-to-
    object dual quaternions.  log_gauss (B,3).  field2cam ((M,4),(M,3)).  delta (P,B): optional delta skinning term
    (relu(mlp) * 0.1 of skinning.py:104-119: delta_skin(xyz, rest_articulation, log_gauss, mlp, cond)).
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


# ---------------------------------------------------------------------------------------------------------------------
# Deformation-cycle regulariser (csrc/cycle.cu): the backward warp of every frame's warped surfels back to the canonical
# space, with the backward warp's skin-entropy and delta-skin terms.

CYCLE_TERMS = ("reg_deform_cyc", "reg_delta_skin", "reg_skin_entropy")


def cycle_tables(rest_articulation, t_articulation, log_gauss):
    """The per-frame tables of the cycle kernels from the reference's arguments, with differentiable torch ops:
    o2b_q (M,B,4), o2b_t (M,B,3) (object -> bone of t_articulation, the bones the backward warp skins on), inv_gauss (B,3),
    se3_r, se3_d (M,B,4) = rest_articulation o t_articulation^-1 (warping.py:407-411)."""
    rr, rd = rest_articulation
    tr, td = t_articulation
    itr, itd = _qconj(tr), _qconj(td)
    o2b_q = itr
    o2b_t = 2.0 * _qmul(itd, tr)[..., 1:]                     # 2 (conj(td) (x) conj(conj(tr)))[1:]
    se3_r = _qmul(rr[None], itr)
    se3_d = _qmul(rr[None], itd) + _qmul(rd[None], itr)
    return o2b_q, o2b_t, torch.exp(-log_gauss), se3_r, se3_d


def _check_cycle(xyz, xyz_cam, rest_articulation, t_articulation, log_gauss, field2cam, delta, weights):
    if xyz.dim() != 2 or xyz.shape[1] != 3:
        raise RuntimeError(f"xyz must be (P,3), got {tuple(xyz.shape)}")
    P = int(xyz.shape[0])
    if xyz_cam.dim() != 3 or tuple(xyz_cam.shape[1:]) != (P, 3) or xyz_cam.shape[0] < 1:
        raise RuntimeError(f"xyz_cam must be (M,P,3) with P = {P}, got {tuple(xyz_cam.shape)}")
    M = int(xyz_cam.shape[0])
    B = int(log_gauss.shape[0]) if log_gauss.dim() == 2 else -1
    if not 1 <= B <= B_MAX or tuple(log_gauss.shape) != (B, 3):
        raise RuntimeError(f"log_gauss must be (B,3) with 1 <= B <= {B_MAX}, got {tuple(log_gauss.shape)}")
    check_articulations(B, M, rest_articulation, t_articulation, field2cam)
    if delta is not None and tuple(delta.shape) != (M, P, B):
        raise RuntimeError(f"delta must be (M,P,B) = ({M},{P},{B}), got {tuple(delta.shape)}")
    if torch.is_tensor(weights):
        if tuple(weights.shape) != (3,) or weights.dtype != torch.float32:
            raise RuntimeError(f"weights must be 3 floats or a (3,) float32 tensor, got {tuple(weights.shape)} {weights.dtype}")
    elif len(weights) != 3:
        raise RuntimeError(f"weights must be 3 floats (reg_deform_cyc, reg_delta_skin, reg_skin_entropy), got {weights!r}")
    if 2 * 4 * (M * B * 15 + B * 3 + M * 7) > TABLE_SMEM_MAX:    # sr_cycle_loss_table_floats, twice, in shared memory
        raise RuntimeError(f"the bone / frame tables of B = {B}, M = {M} frames do not fit in shared memory: split the frames")
    named = [("xyz", xyz), ("xyz_cam", xyz_cam), ("log_gauss", log_gauss), ("rest_articulation", rest_articulation[0]),
             ("rest_articulation", rest_articulation[1]), ("t_articulation", t_articulation[0]),
             ("t_articulation", t_articulation[1]), ("field2cam", field2cam[0]), ("field2cam", field2cam[1])]
    named += [(n, t) for n, t in (("delta", delta), ("weights", weights)) if torch.is_tensor(t)]
    _capi.check_tensors(named, "xyz", xyz)
    return P, B, M


class _CycleLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, xyz, xyz_cam, o2b_q, o2b_t, inv_gauss, se3_r, se3_d, cam_q, cam_t, delta, weights, dims):
        P, B, M = dims
        f = lambda t: None if t is None else t.detach().contiguous()  # noqa: E731
        ins = tuple(map(f, (xyz, xyz_cam, o2b_q, o2b_t, inv_gauss, delta, se3_r, se3_d, cam_q, cam_t)))
        dev = xyz.device
        terms = torch.empty((M, 3), dtype=torch.float32, device=dev)
        counts = torch.empty((M, 3), dtype=torch.int32, device=dev)
        scale = torch.empty((3,), dtype=torch.float32, device=dev)
        loss = torch.empty((), dtype=torch.float32, device=dev)
        _capi.call("sr_cycle_loss_forward", dev, P, B, M, *ins, weights, terms, counts, scale, loss)
        ctx.dims = dims
        ctx.ins = ins
        ctx.scale = scale
        ctx.mark_non_differentiable(terms, counts)
        return loss, terms, counts

    @staticmethod
    def backward(ctx, g_loss, _g_terms, _g_counts):
        P, B, M = ctx.dims
        ins = ctx.ins
        delta = ins[5]
        if g_loss is None:
            return (None,) * 12
        dev = ins[0].device
        g_loss = g_loss.to(torch.float32).contiguous()
        g_xyz = torch.empty((P, 3), dtype=torch.float32, device=dev)
        g_xyz_cam = torch.empty((M, P, 3), dtype=torch.float32, device=dev)
        g_delta = torch.empty((M, P, B), dtype=torch.float32, device=dev) if delta is not None else None
        g_tab = torch.empty((int(_capi.load().sr_cycle_loss_table_floats(B, M)),), dtype=torch.float32, device=dev)
        _capi.call("sr_cycle_loss_backward", dev, P, B, M, *ins, ctx.scale, g_loss, g_xyz_cam, g_xyz, g_delta, g_tab)
        g_oq, g_ot, g_ig, g_sr, g_sd, g_cq, g_ct = table_views(g_tab, ((M, B, 4), (M, B, 3), (B, 3), (M, B, 4), (M, B, 4), (M, 4),
                                                                      (M, 3)))
        return g_xyz, g_xyz_cam, g_oq, g_ot, g_ig, g_sr, g_sd, g_cq, g_ct, g_delta, None, None


def cycle_loss(xyz, xyz_cam, rest_articulation, t_articulation, log_gauss, field2cam, delta=None, weights=(0.01, 5e-3, 5e-4)):
    """Stage 3's deformation-cycle regulariser (deformable_gaussian.py:1272-1275,1517-1574) with the backward warp's
    skin-entropy and delta-skin terms, reduced as model.py:850-853 and apply_loss_weights (:994-1012) do.

    xyz (P,3): canonical surfels.  xyz_cam (M,P,3): bob_warp's output for the same surfels, so autograd chains through
    both kernels.  rest_articulation ((B,4),(B,4)), t_articulation ((M,B,4),(M,B,4)), log_gauss (B,3), field2cam
    ((M,4),(M,3)): as for bob_warp.  delta (M,P,B) or None: the frame-conditioned delta skinning term (relu(mlp) * 0.1 of
    skinning.py:104-119) evaluated on the surfels in object space at time t: delta_skin(xyz_t, t_articulation, log_gauss, mlp,
    cond) with xyz_t (M,P,3) and the frames' cond (M,C).  weights: the weights of
    {reg_deform_cyc, reg_delta_skin, reg_skin_entropy}, 3 floats or a (3,) float32 CUDA tensor read at run time (refill it
    in place between CUDA-graph replays).

    Per frame m and surfel p: cyc = |x_cycled - xyz[p]|, dsk = mean_b delta^2 (0 without delta), ent = logsumexp - max of
    the backward warp's skinning logits.  Returns {"loss": sum_k weight_k * mean(v_k[v_k > 0]) (0 for a term with no
    v_k > 0), differentiable in xyz, xyz_cam, the articulations, log_gauss, field2cam and delta; "terms": (M,3) each frame's
    share of the three weighted terms; "counts": (M,3) int32 values > 0}.  No host synchronisation, nothing allocated
    beyond the outputs and gradients."""
    P, B, M = _check_cycle(xyz, xyz_cam, rest_articulation, t_articulation, log_gauss, field2cam, delta, weights)
    o2b_q, o2b_t, inv_gauss, se3_r, se3_d = cycle_tables(rest_articulation, t_articulation, log_gauss)
    if not torch.is_tensor(weights):
        w = torch.empty((3,), dtype=torch.float32, device=xyz.device)
        for i, v in enumerate(weights):
            w[i].fill_(float(v))
        weights = w
    loss, terms, counts = _CycleLoss.apply(xyz, xyz_cam, o2b_q, o2b_t, inv_gauss, se3_r, se3_d, field2cam[0], field2cam[1],
                                           delta, weights, (P, B, M))
    return {"loss": loss, "terms": terms, "counts": counts}


# ---------------------------------------------------------------------------------------------------------------------
# Per-surfel feature rows (csrc/feature_rows.cu): [regist | flow / s | normal | Gaussian-bone density] per frame, the
# (M,P,Cf+6) channels render_loss_batch(features=) composites next to the colour.

def _check_feature_rows(regist_feat, xyz, scaling, xyz_cam, rot_cam, Kmat, field2cam, rest_articulation, logibeta):
    if xyz.dim() != 2 or xyz.shape[1] != 3:
        raise RuntimeError(f"xyz must be (P,3), got {tuple(xyz.shape)}")
    P = int(xyz.shape[0])
    if regist_feat.dim() != 2 or regist_feat.shape[0] != P or regist_feat.shape[1] + 6 > _capi.FEATURES_MAX:
        raise RuntimeError(f"regist_feat must be (P,Cf) with P = {P} and Cf + 6 <= {_capi.FEATURES_MAX}, got {tuple(regist_feat.shape)}")
    Cf = int(regist_feat.shape[1])
    if tuple(scaling.shape) != (P, 2):
        raise RuntimeError(f"scaling must be (P,2) (the two tangent scales) with P = {P}, got {tuple(scaling.shape)}")
    if xyz_cam.dim() != 3 or tuple(xyz_cam.shape[1:]) != (P, 3) or xyz_cam.shape[0] < 1:
        raise RuntimeError(f"xyz_cam must be (M,P,3) with P = {P}, got {tuple(xyz_cam.shape)}")
    M = int(xyz_cam.shape[0])
    if M > 1 and M % 2:
        raise RuntimeError(f"M must be 1 or even: the flow pairs frames 2k and 2k+1 (flip_pair), got M = {M}")
    if M > 1024:
        raise RuntimeError(f"M must be at most 1024, got {M}")
    if tuple(rot_cam.shape) != (M, P, 4):
        raise RuntimeError(f"rot_cam must be (M,P,4) = ({M},{P},4), got {tuple(rot_cam.shape)}")
    if tuple(Kmat.shape) != (M, 3, 3):
        raise RuntimeError(f"Kmat must be (M,3,3) with M = {M}, got {tuple(Kmat.shape)}")
    if len(field2cam) != 2 or tuple(field2cam[0].shape) != (M, 4):
        raise RuntimeError(f"field2cam must be ((M,4),(M,3)) with M = {M}, got {[tuple(t.shape) for t in field2cam]}")
    B = int(rest_articulation[0].shape[0]) if rest_articulation[0].dim() == 2 else -1
    if (len(rest_articulation) != 2 or not 1 <= B <= B_MAX or tuple(rest_articulation[0].shape) != (B, 4)
            or tuple(rest_articulation[1].shape) != (B, 4)):
        raise RuntimeError(f"rest_articulation must be ((B,4),(B,4)) with 1 <= B <= {B_MAX}, "
                           f"got {[tuple(t.shape) for t in rest_articulation]}")
    if logibeta.numel() != 1:
        raise RuntimeError(f"logibeta must hold one value, got shape {tuple(logibeta.shape)}")
    named = [("regist_feat", regist_feat), ("xyz", xyz), ("scaling", scaling), ("xyz_cam", xyz_cam), ("rot_cam", rot_cam),
             ("Kmat", Kmat), ("field2cam", field2cam[0]), ("rest_articulation", rest_articulation[0]),
             ("rest_articulation", rest_articulation[1]), ("logibeta", logibeta)]
    _capi.check_tensors(named, "xyz", xyz)
    return P, M, B, Cf


class _FeatureRows(torch.autograd.Function):
    @staticmethod
    def forward(ctx, regist, xyz, xyz_cam, rot_cam, cam_q, centres, beta, scaling, Kmat, dims):
        P, M, B, Cf = dims
        f = lambda t: t.detach().contiguous()  # noqa: E731
        regist, xyz, xyz_cam, rot_cam, cam_q, centres, beta, scaling, Kmat = map(f, (regist, xyz, xyz_cam, rot_cam, cam_q, centres,
                                                                                    beta, scaling, Kmat))
        dev = xyz.device
        rows = torch.empty((M, P, Cf + 6), dtype=torch.float32, device=dev)
        density = torch.empty((P, 1), dtype=torch.float32, device=dev)
        s = torch.empty((), dtype=torch.float32, device=dev)
        aux = torch.empty((3,), dtype=torch.int32, device=dev)
        _capi.call("sr_feature_rows_forward", dev, P, M, B, Cf, regist if Cf else None, xyz, scaling, xyz_cam, rot_cam, Kmat, cam_q,
                   centres, beta, rows, density, s, aux)
        ctx.dims = dims
        ctx.save_for_backward(xyz, scaling, xyz_cam, rot_cam, Kmat, cam_q, centres, beta, s, aux)
        return rows, s, density

    @staticmethod
    def backward(ctx, g_rows, g_s, g_density):
        P, M, B, Cf = ctx.dims
        xyz, scaling, xyz_cam, rot_cam, Kmat, cam_q, centres, beta, s, aux = ctx.saved_tensors
        dev = xyz.device
        g_rows = torch.zeros((M, P, Cf + 6), dtype=torch.float32, device=dev) if g_rows is None else g_rows.to(torch.float32).contiguous()
        g_s = None if g_s is None else g_s.to(torch.float32).contiguous()
        g_density = None if g_density is None else g_density.to(torch.float32).contiguous()
        g_regist = torch.empty((P, Cf), dtype=torch.float32, device=dev)
        g_xyz = torch.empty((P, 3), dtype=torch.float32, device=dev)
        g_xyz_cam = torch.empty((M, P, 3), dtype=torch.float32, device=dev)
        g_rot_cam = torch.empty((M, P, 4), dtype=torch.float32, device=dev)
        g_tab = torch.empty((M * 4 + B * 3 + 2,), dtype=torch.float32, device=dev)
        _capi.call("sr_feature_rows_backward", dev, P, M, B, Cf, xyz, scaling, xyz_cam, rot_cam, Kmat, cam_q, centres, beta, s, aux,
                   g_rows, g_density, g_s, g_regist if Cf else None, g_xyz, g_xyz_cam, g_rot_cam, g_tab)
        g_cq, g_cen, g_beta = table_views(g_tab, ((M, 4), (B, 3), (1,)))
        return g_regist, g_xyz, g_xyz_cam, g_rot_cam, g_cq, g_cen, g_beta, None, None, None


def feature_rows(regist_feat, xyz, scaling, xyz_cam, rot_cam, Kmat, field2cam, rest_articulation, logibeta):
    """Stage 3's per-surfel feature rows (deformable_gaussian.py:1106-1182): for frame m and surfel p the row
    [regist_feat[p] (Cf) | flow[m,p] / s (2) | normal[m,p] (3) | gauss_density[p] (1)], the channels the reference renders
    next to the colour (render_view(override_color=concated_feat)); the Gaussian-mask channel is Cf + 5.

    regist_feat (P,Cf): `_regist_feat` (a FlatSurfelModel view is fine).  xyz (P,3): the canonical `_xyz`.  scaling (P,2):
    `get_scaling`.  xyz_cam (M,P,3), rot_cam (M,P,4): bob_warp's first two outputs.  Kmat (M,3,3): Kmatinv(Kinv).
    field2cam ((M,4),(M,3)).  rest_articulation ((B,4),(B,4)): the rest bones as dual quaternions
    (samples_dict["rest_articulation"][..][0]).  logibeta (1,): the SkinningWarp's.  M is 1 or even: frames 2k and 2k+1
    are each other's flow partner (compute_flow's flip_pair); a single frame is its own partner and its flow is 0.

      flow[m,p] = pi(K[m'], xyz_cam[m',p]) - pi(K[m], xyz_cam[m,p]), pi(K,x) = (Kx)[0:2] / (Kx)[2], m' = m xor 1;
      s = max(max(flow), |min(flow)|) + 1e-6, NOT detached (as in the reference);
      normal = field2cam[0][m] applied to rot_cam[m,p] applied to e_a, where e_a is e_x or e_y, whichever of the two
          tangent scales is smaller (e_x on ties) -- the reference's axis, which is never the surfel normal e_z; rot_cam
          already holds the camera rotation, which is applied a second time as in the reference; no quaternion is
          normalised;
      gauss_density = exp(logibeta) * max_b exp(-0.5 |xyz - c_b|^2 / 0.01^2), c_b the rest bones' translations.

    Returns {"rows": (M,P,Cf+6), "flow_scale": 0-d tensor s, "gauss_density": (P,1)}, all differentiable: gradients reach
    regist_feat, xyz, xyz_cam, rot_cam (through bob_warp: the canonical surfels and the articulations), field2cam[0],
    rest_articulation and logibeta.  scaling, Kmat and field2cam[1] are data.  The caller multiplies the flow planes it
    renders back by flow_scale (:1193), which adds its own gradient to s.  No host synchronisation; nothing is allocated
    beyond the outputs and the gradients."""
    P, M, B, Cf = _check_feature_rows(regist_feat, xyz, scaling, xyz_cam, rot_cam, Kmat, field2cam, rest_articulation, logibeta)
    rr, rd = rest_articulation
    centres = 2.0 * _qmul(rd, _qconj(rr))[..., 1:]              # dual_quaternion_to_quaternion_translation
    beta = torch.exp(logibeta.reshape(1))
    rows, s, density = _FeatureRows.apply(regist_feat, xyz, xyz_cam, rot_cam, field2cam[0], centres, beta, scaling, Kmat,
                                          (P, M, B, Cf))
    return {"rows": rows, "flow_scale": s, "gauss_density": density}


# ---------------------------------------------------------------------------------------------------------------------
# Delta-skinning MLP (csrc/skin_mlp.cu): delta = relu(delta_field([xyz_bone | t_embed | inst_code])) * 0.1 of
# skinning.py:104-119, the `delta=` argument of bob_warp, cycle_loss and reproj_loss.

SKIN_MLP_WIDTH = 64           # hidden units of the reference's delta_field (CondMLP(D=2, W=64), skinning.py:74-85)
SKIN_MLP_DEPTH = 2


class DeltaSkinMLP(torch.nn.Module):
    """The reference's `SkinningField.delta_field` (CondMLP(D=2, W=64), base.py:17-150) with the fused op as its forward.

    Parameters carry the reference's names and shapes -- linear_1.0.weight (64, 3B+C), linear_1.0.bias, linear_2.0.weight
    (64,64), linear_2.0.bias, linear_final.weight (B,64), linear_final.bias -- so load_state_dict of the reference's
    delta_field state (without its inst_embedding entries) works.  cond_channels C = 128 time + 32 instance channels."""

    def __init__(self, num_bones, cond_channels=160):
        super().__init__()
        if not 1 <= num_bones <= B_MAX:
            raise RuntimeError(f"num_bones must be in [1, {B_MAX}], got {num_bones}")
        if cond_channels < 0:
            raise RuntimeError(f"cond_channels must be >= 0, got {cond_channels}")
        self.num_bones, self.cond_channels = int(num_bones), int(cond_channels)
        relu = torch.nn.ReLU(True)
        self.linear_1 = torch.nn.Sequential(torch.nn.Linear(3 * num_bones + cond_channels, SKIN_MLP_WIDTH), relu)
        self.linear_2 = torch.nn.Sequential(torch.nn.Linear(SKIN_MLP_WIDTH, SKIN_MLP_WIDTH), relu)
        self.linear_final = torch.nn.Linear(SKIN_MLP_WIDTH, num_bones)

    def forward(self, points, articulation, log_gauss, cond):
        return delta_skin(points, articulation, log_gauss, self, cond)


def delta_skin_tables(articulation, log_gauss, W1, b1, cond):
    """The first layer folded per frame: F (Mt,64,4) float32 with W1 [xyz_bone | cond] + b1 = F [x; 1], Mt = 1 when the
    bones and cond are shared and M when either is per frame.  xyz_bone[b] = (R_b x + t_b) exp(-log_gauss[b]) with
    (R_b, t_b) the inverse of bone b's articulation (transforms.py:9-25, skinning.py:126-142), so the product with W1's
    first 3B columns is a (64,3) matrix and a 64-vector; W1's other columns times cond, and b1, join that vector.  Built
    in float64 with differentiable torch ops and rounded once."""
    r, d = articulation[0].double(), articulation[1].double()
    if r.dim() == 2:
        r, d = r[None], d[None]
    q = _qconj(r)                                               # object -> bone, as warp_tables / cycle_tables
    t = 2.0 * _qmul(_qconj(d), r)[..., 1:]                      # (Mb,B,3)
    w, x, y, z = q.unbind(-1)
    R = torch.stack((w * w + x * x - y * y - z * z, 2 * (x * y - w * z), 2 * (x * z + w * y),
                     2 * (x * y + w * z), w * w - x * x + y * y - z * z, 2 * (y * z - w * x),
                     2 * (x * z - w * y), 2 * (y * z + w * x), w * w - x * x - y * y + z * z), -1)
    B = int(log_gauss.shape[0])
    R = R.view(R.shape[0], B, 3, 3)                             # q v q* as a matrix, q not normalised (nor is it there)
    ig = torch.exp(-log_gauss.double())                         # (B,3)
    W1 = W1.double()
    Wx = W1[:, :3 * B].view(1, -1, B, 3) * ig                   # (1,64,B,3)
    # tens of thousands of products: plain broadcast sums, no GEMM call
    A = (Wx[..., None] * R[:, None]).sum((2, 3))                # (Mb,64,3)
    c = (Wx * t[:, None]).sum((2, 3))                           # (Mb,64)
    cond = cond.double()
    if cond.dim() == 1:
        cond = cond[None]
    c = c + (cond[:, None, :] * W1[None, :, 3 * B:]).sum(-1) + b1.double()      # (Mt,64): (1 | M) broadcast with (1 | M)
    A = A.expand(c.shape[0], -1, -1)
    return torch.cat((A, c[..., None]), -1).to(torch.float32)


def _check_delta_skin(points, articulation, log_gauss, mlp, cond):
    if points.dim() not in (2, 3, 4) or points.shape[-1] != 3 or any(s_ < 1 for s_ in points.shape):
        raise RuntimeError(f"points must be (N,3), (M,N,3) or (M,H,W,3) with every dimension >= 1, got {tuple(points.shape)}")
    M = int(points.shape[0]) if points.dim() > 2 else 1
    B = int(log_gauss.shape[0]) if log_gauss.dim() == 2 else -1
    if not 1 <= B <= B_MAX or tuple(log_gauss.shape) != (B, 3):
        raise RuntimeError(f"log_gauss must be (B,3) with 1 <= B <= {B_MAX}, got {tuple(log_gauss.shape)}")
    if not isinstance(mlp, DeltaSkinMLP):
        raise RuntimeError(f"mlp must be a DeltaSkinMLP, got {type(mlp).__name__}")
    if mlp.num_bones != B:
        raise RuntimeError(f"mlp has {mlp.num_bones} bones, log_gauss {B}")
    shapes = [tuple(t.shape) for t in articulation] if len(articulation) == 2 else None
    if shapes not in ([(B, 4)] * 2, [(M, B, 4)] * 2):
        raise RuntimeError(f"articulation must be ((B,4),(B,4)) or ((M,B,4),(M,B,4)) with B = {B}, M = {M}, got {shapes}")
    C = mlp.cond_channels
    if tuple(cond.shape) not in ((C,), (M, C)):
        raise RuntimeError(f"cond must be (C,) or (M,C) with C = {C}, M = {M}, got {tuple(cond.shape)}")
    named = [("points", points), ("articulation", articulation[0]), ("articulation", articulation[1]), ("log_gauss", log_gauss),
             ("cond", cond)] + [("mlp." + n, p) for n, p in mlp.named_parameters()]
    _capi.check_tensors(named, "points", points)
    return M, B


class _DeltaSkin(torch.autograd.Function):
    @staticmethod
    def forward(ctx, points, F, W2, b2, W3, b3, dims):
        M, N, B = dims
        ins = tuple(t.detach().contiguous() for t in (points, F, W2, b2, W3, b3))
        dev = points.device
        delta = torch.empty((M, N, B), dtype=torch.float32, device=dev)
        _capi.call("sr_delta_skin_forward", dev, M, N, B, int(F.shape[0]), SKIN_MLP_WIDTH, SKIN_MLP_DEPTH, *ins, delta)
        ctx.dims = dims
        ctx.save_for_backward(*ins)
        return delta

    @staticmethod
    def backward(ctx, g_delta):
        M, N, B = ctx.dims
        ins = ctx.saved_tensors
        F, W2, b2, W3, b3 = ins[1:]
        dev = F.device
        g_delta = g_delta.to(torch.float32).contiguous()
        g_points = torch.empty((M, N, 3), dtype=torch.float32, device=dev)
        grads = tuple(torch.empty_like(t) for t in (F, W2, b2, W3, b3))
        nbytes = int(_capi.load().sr_delta_skin_scratch_bytes(M, N, B))
        scratch = torch.empty((nbytes,), dtype=torch.uint8, device=dev)
        _capi.call("sr_delta_skin_backward", dev, M, N, B, int(F.shape[0]), SKIN_MLP_WIDTH, SKIN_MLP_DEPTH, *ins, g_delta, g_points,
                   *grads, scratch, nbytes)
        return (g_points,) + grads + (None,)


def delta_skin(points, articulation, log_gauss, mlp, cond):
    """The delta skinning term of skinning.py:104-119, delta = relu(delta_field([xyz_bone | cond])) * 0.1, as one fused
    CUDA op each way (csrc/skin_mlp.cu) -- the `delta=` of bob_warp, cycle_loss and reproj_loss.

    points (N,3), (M,N,3) or (M,H,W,3): object-space points.  articulation ((B,4),(B,4)) shared by every frame or
    ((M,B,4),(M,B,4)) per frame: the bones the skinning is evaluated on as dual quaternions (rest_articulation for the
    forward warps, t_articulation for the cycle's backward warp).  log_gauss (B,3).  mlp: a DeltaSkinMLP.  cond (C,)
    shared or (M,C) per frame: cat(t_embed, inst_code), the time code (the mean embedding, or the frame's) and the instance
    code, which stay the caller's few torch ops.

    Returns delta of shape points.shape[:-1] + (B,), differentiable in points, both halves of articulation, log_gauss,
    cond and the MLP's six parameters.  The first layer is folded per frame into a (64,4) table in float64 (see
    delta_skin_tables); the kernels never form xyz_bone, the (…,3B+C) input or a stored activation.  The backward holds
    sr_delta_skin_scratch_bytes of scratch (a few MB) for the fixed-order sum of the weight gradients: results are
    bit-identical from run to run.  No host synchronisation."""
    M, B = _check_delta_skin(points, articulation, log_gauss, mlp, cond)
    F = delta_skin_tables(articulation, log_gauss, mlp.linear_1[0].weight, mlp.linear_1[0].bias, cond)
    N = points.numel() // (3 * M)
    delta = _DeltaSkin.apply(points.reshape(M, N, 3), F, mlp.linear_2[0].weight, mlp.linear_2[0].bias, mlp.linear_final.weight,
                             mlp.linear_final.bias, (M, N, B))
    return delta.view(tuple(points.shape[:-1]) + (B,))
