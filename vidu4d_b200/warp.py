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


# ---------------------------------------------------------------------------------------------------------------------
# Deformation-cycle regulariser (csrc/cycle.cu): the backward warp of every frame's warped surfels back to the canonical
# space, with the backward warp's skin-entropy and delta-skin terms.

B_MAX = 64
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
    for name, pair, shapes in (("rest_articulation", rest_articulation, ((B, 4), (B, 4))),
                               ("t_articulation", t_articulation, ((M, B, 4), (M, B, 4))),
                               ("field2cam", field2cam, ((M, 4), (M, 3)))):
        if len(pair) != 2 or tuple(pair[0].shape) != shapes[0] or tuple(pair[1].shape) != shapes[1]:
            raise RuntimeError(f"{name} must be tensors of shapes {shapes}, got {[tuple(t.shape) for t in pair]}")
    if delta is not None and tuple(delta.shape) != (M, P, B):
        raise RuntimeError(f"delta must be (M,P,B) = ({M},{P},{B}), got {tuple(delta.shape)}")
    if torch.is_tensor(weights):
        if tuple(weights.shape) != (3,) or weights.dtype != torch.float32:
            raise RuntimeError(f"weights must be 3 floats or a (3,) float32 tensor, got {tuple(weights.shape)} {weights.dtype}")
    elif len(weights) != 3:
        raise RuntimeError(f"weights must be 3 floats (reg_deform_cyc, reg_delta_skin, reg_skin_entropy), got {weights!r}")
    if 2 * 4 * (M * B * 15 + B * 3 + M * 7) > 200 * 1024:        # sr_cycle_loss_table_floats, twice, in shared memory
        raise RuntimeError(f"the bone / frame tables of B = {B}, M = {M} frames do not fit in shared memory: split the frames")
    named = [("xyz", xyz), ("xyz_cam", xyz_cam), ("log_gauss", log_gauss), ("rest_articulation", rest_articulation[0]),
             ("rest_articulation", rest_articulation[1]), ("t_articulation", t_articulation[0]),
             ("t_articulation", t_articulation[1]), ("field2cam", field2cam[0]), ("field2cam", field2cam[1])]
    named += [(n, t) for n, t in (("delta", delta), ("weights", weights)) if torch.is_tensor(t)]
    for name, t in named:
        if t.dtype != torch.float32:
            raise RuntimeError(f"{name} must be float32, got {t.dtype}")
        if not t.is_cuda:
            raise RuntimeError(f"{name} must be a CUDA tensor (there is no CPU fallback)")
        if t.device != xyz.device:
            raise RuntimeError(f"{name} is on {t.device}, xyz on {xyz.device}")
    return P, B, M


class _CycleLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, xyz, xyz_cam, o2b_q, o2b_t, inv_gauss, se3_r, se3_d, cam_q, cam_t, delta, weights, dims):
        P, B, M = dims
        lib = _capi.load()
        f = lambda t: None if t is None else t.detach().contiguous()  # noqa: E731
        ins = tuple(map(f, (xyz, xyz_cam, o2b_q, o2b_t, inv_gauss, delta, se3_r, se3_d, cam_q, cam_t)))
        dev = xyz.device
        terms = torch.empty((M, 3), dtype=torch.float32, device=dev)
        counts = torch.empty((M, 3), dtype=torch.int32, device=dev)
        scale = torch.empty((3,), dtype=torch.float32, device=dev)
        loss = torch.empty((), dtype=torch.float32, device=dev)
        ptr = lambda t: None if t is None else t.data_ptr()  # noqa: E731
        with torch.cuda.device(dev):
            rc = lib.sr_cycle_loss_forward(P, B, M, *map(ptr, ins), ptr(weights.detach()), ptr(terms), ptr(counts), ptr(scale),
                                           ptr(loss), torch.cuda.current_stream(dev).cuda_stream)
        _capi.check(rc, "sr_cycle_loss_forward")
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
        lib = _capi.load()
        g_tab = torch.empty((int(lib.sr_cycle_loss_table_floats(B, M)),), dtype=torch.float32, device=dev)
        ptr = lambda t: None if t is None else t.data_ptr()  # noqa: E731
        with torch.cuda.device(dev):
            rc = lib.sr_cycle_loss_backward(P, B, M, *map(ptr, ins), ptr(ctx.scale), ptr(g_loss), ptr(g_xyz_cam), ptr(g_xyz),
                                            ptr(g_delta), ptr(g_tab), torch.cuda.current_stream(dev).cuda_stream)
        _capi.check(rc, "sr_cycle_loss_backward")
        o = 0
        g = []
        for shape in ((M, B, 4), (M, B, 3), (B, 3), (M, B, 4), (M, B, 4), (M, 4), (M, 3)):
            n = 1
            for s_ in shape:
                n *= s_
            g.append(g_tab[o:o + n].view(shape)); o += n
        g_oq, g_ot, g_ig, g_sr, g_sd, g_cq, g_ct = g
        return g_xyz, g_xyz_cam, g_oq, g_ot, g_ig, g_sr, g_sd, g_cq, g_ct, g_delta, None, None


def cycle_loss(xyz, xyz_cam, rest_articulation, t_articulation, log_gauss, field2cam, delta=None, weights=(0.01, 5e-3, 5e-4)):
    """Stage 3's deformation-cycle regulariser (deformable_gaussian.py:1272-1275,1517-1574) with the backward warp's
    skin-entropy and delta-skin terms, reduced as model.py:850-853 and apply_loss_weights (:994-1012) do.

    xyz (P,3): canonical surfels.  xyz_cam (M,P,3): bob_warp's output for the same surfels, so autograd chains through
    both kernels.  rest_articulation ((B,4),(B,4)), t_articulation ((M,B,4),(M,B,4)), log_gauss (B,3), field2cam
    ((M,4),(M,3)): as for bob_warp.  delta (M,P,B) or None: the frame-conditioned delta skinning term (relu(mlp) * 0.1 of
    skinning.py:104-119) that the caller evaluates on the surfels in object space at time t.  weights: the weights of
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
