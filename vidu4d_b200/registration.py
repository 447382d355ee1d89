"""Stage 3's feature-matching reprojection loss ("feat_reproj"), fused: Python host side of csrc/match.cu.

Mirrors what the reference computes with rgb_loss_only off:
    lab4d/nnutils/deformable_gaussian.py:1305-1324   global_match + forward_project on every pixel's feature
    lab4d/nnutils/deformable_gaussian.py:1436-1486   global_match (num_grad = 8)
    lab4d/nnutils/deformable_gaussian.py:1488-1513   forward_project: forward_warp without rotation + pinhole_projection
    lab4d/engine/model.py:669-672,915,961-967,994-1012   the feat_reproj term, its masking and its reduction
in two autograd functions, because the caller's delta-skinning MLP runs on the matched points between them:

    cand = draw_candidates(M, P, 2048, device=dev)
    xyz_m = global_match(feat_px, model._regist_feat, model._xyz, cand, logsigma, num_grad=8)      # (M,H,W,3)
    delta = delta_skin(xyz_m, rest_articulation, log_gauss, mlp, cond_mean)         # warp.delta_skin: (M,H,W,B); or None
    out = reproj_loss(xyz_m, hxy, Kmat, rest_articulation, t_articulation, log_gauss, field2cam, mask_fg, is_detected,
                      weight=wt, train_res=256, delta=delta)

Neither call allocates anything the size of the (M*H*W, C) score matrix, synchronises with the host, or needs a count on
the host, so a step that uses them can be captured in a CUDA graph (vidu4d_b200.graph.GraphedStep).  The candidate
indices, logsigma and the weight are read from device memory: refill them in place between replays.
"""
from __future__ import annotations

import torch

from . import _capi
from .warp import B_MAX, check_articulations, split_table_grads, warp_tables

FEAT = 16          # width of the registration feature (_regist_feat)
NUM_GRAD_MAX = 8


def draw_candidates(M: int, P: int, num_candidates: int = 2048, generator=None, device=None):
    """The candidate draw of global_match (deformable_gaussian.py:1461-1462): the first min(num_candidates, M*P) entries of
    torch.randperm(M*P) -- indices into the M-fold expanded surfels, candidate c being surfel idx[c] mod P -- as int32 on
    `device`.  With generator=None the draw uses torch's default CPU generator, as the reference does."""
    C = min(int(num_candidates), M * P)
    gdev = generator.device if generator is not None else "cpu"
    return torch.randperm(M * P, generator=generator, device=gdev)[:C].to(device=device, dtype=torch.int32)


def _check_match(feat_px, regist_feat, xyz, cand, logsigma, num_grad):
    if feat_px.dim() != 4 or feat_px.shape[-1] != FEAT:
        raise RuntimeError(f"feat_px must be (M,H,W,{FEAT}) (the registration feature's width), got {tuple(feat_px.shape)}")
    M = int(feat_px.shape[0])
    if regist_feat.dim() != 2 or regist_feat.shape[1] != FEAT:
        raise RuntimeError(f"regist_feat must be (P,{FEAT}), got {tuple(regist_feat.shape)}")
    P = int(regist_feat.shape[0])
    if xyz.shape != (P, 3):
        raise RuntimeError(f"xyz must be (P,3) = ({P},3), got {tuple(xyz.shape)}")
    if cand.dim() != 1 or cand.dtype != torch.int32 or not 1 <= cand.shape[0] <= M * P:
        raise RuntimeError(f"cand must be a 1-D int32 tensor of 1..M*P = {M * P} indices (draw_candidates), got "
                           f"{tuple(cand.shape)} {cand.dtype}")
    if logsigma.numel() != 1:
        raise RuntimeError(f"logsigma must hold one value, got {tuple(logsigma.shape)}")
    C = int(cand.shape[0])
    if not isinstance(num_grad, int) or isinstance(num_grad, bool) or not 1 <= num_grad <= min(NUM_GRAD_MAX, C):
        raise RuntimeError(f"num_grad must be an int in [1, min({NUM_GRAD_MAX}, C = {C})], got {num_grad!r}")
    floats = (("feat_px", feat_px), ("regist_feat", regist_feat), ("xyz", xyz), ("logsigma", logsigma))
    _capi.check_tensors(floats[:3] + (("cand", cand),) + floats[3:], "feat_px", feat_px, floats=floats)
    return M, int(feat_px.shape[1]), int(feat_px.shape[2]), P, C


class _GlobalMatch(torch.autograd.Function):
    @staticmethod
    def forward(ctx, feat_px, regist_feat, xyz, cand, logsigma, dims):
        M, H, W, P, C, K = dims
        feat_px, regist_feat, xyz, cand, logsigma = (t.detach().contiguous() for t in (feat_px, regist_feat, xyz, cand, logsigma))
        dev = feat_px.device
        xyz_m = torch.empty((M, H, W, 3), dtype=torch.float32, device=dev)
        idx = torch.empty((M, H, W, K), dtype=torch.int32, device=dev)
        prob = torch.empty((M, H, W, K), dtype=torch.float32, device=dev)
        score = torch.empty((M, H, W, K), dtype=torch.float32, device=dev)
        _capi.call("sr_global_match_forward", dev, M, H, W, P, C, K, feat_px, regist_feat, xyz, cand, logsigma, xyz_m, idx, prob,
                   score)
        ctx.dims = dims
        ctx.save_for_backward(feat_px, xyz, cand, logsigma, idx, prob, score)
        ctx.mark_non_differentiable(idx, prob)
        return xyz_m, idx, prob

    @staticmethod
    def backward(ctx, g_xyz_m, _g_idx, _g_prob):
        M, H, W, P, C, K = ctx.dims
        feat_px, xyz, cand, logsigma, idx, prob, score = ctx.saved_tensors
        dev = feat_px.device
        if g_xyz_m is None:
            return None, None, None, None, None, None
        g = g_xyz_m.to(torch.float32).contiguous()
        g_cand = torch.empty((C, FEAT + 3), dtype=torch.float32, device=dev)
        g_rf = torch.empty((P, FEAT), dtype=torch.float32, device=dev)
        g_xyz = torch.empty((P, 3), dtype=torch.float32, device=dev)
        g_log = torch.empty((1,), dtype=torch.float32, device=dev)
        _capi.call("sr_global_match_backward", dev, M, H, W, P, C, K, feat_px, xyz, cand, logsigma, idx, prob, score, g, g_cand,
                   g_rf, g_xyz, g_log)
        return None, g_rf, g_xyz, None, g_log.view(logsigma.shape), None


def global_match(feat_px, regist_feat, xyz, cand, logsigma, num_grad: int = NUM_GRAD_MAX, return_topk: bool = False):
    """global_match (deformable_gaussian.py:1436-1486) with num_grad = K, without the (M*H*W, C) score matrix.

    feat_px (M,H,W,16): pixel features (data: no gradient).  regist_feat (P,16), xyz (P,3): the canonical surfels'
    registration feature and position.  cand (C,) int32: draw_candidates(M, P, ...).  logsigma (1,) or (): log
    temperature.  Returns xyz_matched (M,H,W,3), differentiable in regist_feat, xyz and logsigma; with return_topk also
    the chosen candidate positions (M,H,W,K) int32 (best first; among equal scores the lower position first; -1 if
    none) and their softmax probabilities (M,H,W,K)."""
    M, H, W, P, C = _check_match(feat_px, regist_feat, xyz, cand, logsigma, num_grad)
    xyz_m, idx, prob = _GlobalMatch.apply(feat_px, regist_feat, xyz, cand, logsigma, (M, H, W, P, C, num_grad))
    return (xyz_m, idx, prob) if return_topk else xyz_m


def _check_reproj(xyz_m, hxy, Kmat, rest_articulation, t_articulation, log_gauss, field2cam, mask, is_detected, weight,
                  train_res, delta):
    if xyz_m.dim() != 4 or xyz_m.shape[-1] != 3:
        raise RuntimeError(f"xyz_matched must be (M,H,W,3), got {tuple(xyz_m.shape)}")
    M, H, W = (int(v) for v in xyz_m.shape[:3])
    if hxy.dim() != 4 or tuple(hxy.shape[:3]) != (M, H, W) or hxy.shape[3] not in (2, 3):
        raise RuntimeError(f"hxy must be (M,H,W,2) or (M,H,W,3) = ({M},{H},{W},2|3), got {tuple(hxy.shape)}")
    if tuple(Kmat.shape) != (M, 3, 3):
        raise RuntimeError(f"Kmat must be (M,3,3) = ({M},3,3), got {tuple(Kmat.shape)}")
    if tuple(mask.shape) not in ((M, H, W), (M, H, W, 1)):
        raise RuntimeError(f"mask_fg must be (M,H,W) or (M,H,W,1) = ({M},{H},{W}), got {tuple(mask.shape)}")
    if is_detected is not None and tuple(is_detected.shape) != (M,):
        raise RuntimeError(f"is_detected must be (M,) = ({M},), got {tuple(is_detected.shape)}")
    B = int(log_gauss.shape[0])
    if not 1 <= B <= B_MAX or tuple(log_gauss.shape) != (B, 3):
        raise RuntimeError(f"log_gauss must be (B,3) with 1 <= B <= {B_MAX}, got {tuple(log_gauss.shape)}")
    check_articulations(B, M, rest_articulation, t_articulation, field2cam)
    if delta is not None and tuple(delta.shape) != (M, H, W, B):
        raise RuntimeError(f"delta must be (M,H,W,B) = ({M},{H},{W},{B}), got {tuple(delta.shape)}")
    if torch.is_tensor(weight) and (weight.numel() != 1 or weight.dtype != torch.float32):
        raise RuntimeError(f"weight must be a float or a one-element float32 tensor, got {tuple(weight.shape)} {weight.dtype}")
    if not float(train_res) > 0:
        raise RuntimeError(f"train_res must be > 0, got {train_res}")
    named = [("xyz_matched", xyz_m), ("hxy", hxy), ("Kmat", Kmat), ("mask_fg", mask), ("log_gauss", log_gauss),
             ("rest_articulation", rest_articulation[0]), ("rest_articulation", rest_articulation[1]),
             ("t_articulation", t_articulation[0]), ("t_articulation", t_articulation[1]), ("field2cam", field2cam[0]),
             ("field2cam", field2cam[1])]
    named += [(n, t) for n, t in (("is_detected", is_detected), ("delta", delta), ("weight", weight)) if torch.is_tensor(t)]
    _capi.check_tensors(named, "xyz_matched", xyz_m, floats=())     # the forward converts to float32
    return M, H, W, B


class _ReprojLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, xyz_m, o2b_q, o2b_t, inv_gauss, se3_r, se3_d, cam_q, cam_t, delta, Kmat, hxy, mask, det, weight, cfg):
        M, H, W, B, train_res = cfg
        f = lambda t: None if t is None else t.detach().to(torch.float32).contiguous()  # noqa: E731
        ins = tuple(map(f, (xyz_m, o2b_q, o2b_t, inv_gauss, se3_r, se3_d, cam_q, cam_t, delta, Kmat, hxy, mask, det, weight)))
        xyz_m, o2b_q, o2b_t, inv_gauss, se3_r, se3_d, cam_q, cam_t, delta, Kmat, hxy, mask, det, weight = ins
        dev = xyz_m.device
        xy = torch.empty((M, H, W, 2), dtype=torch.float32, device=dev)
        terms = torch.empty((M,), dtype=torch.float32, device=dev)
        counts = torch.empty((M,), dtype=torch.int32, device=dev)
        scale = torch.empty((1,), dtype=torch.float32, device=dev)
        loss = torch.empty((), dtype=torch.float32, device=dev)
        _capi.call("sr_reproj_loss_forward", dev, M, H, W, B, int(hxy.shape[-1]), float(train_res), xyz_m, o2b_q, o2b_t, inv_gauss,
                   delta, se3_r, se3_d, cam_q, cam_t, Kmat, hxy, mask, det, weight, xy, terms, counts, scale, loss)
        ctx.cfg = cfg
        ctx.ins = ins
        ctx.scale = scale
        ctx.mark_non_differentiable(xy, terms, counts)
        return loss, xy, terms, counts

    @staticmethod
    def backward(ctx, g_loss, _g_xy, _g_terms, _g_counts):
        M, H, W, B, _ = ctx.cfg
        xyz_m, o2b_q, o2b_t, inv_gauss, se3_r, se3_d, cam_q, cam_t, delta, Kmat, hxy, mask, det, _w = ctx.ins
        none = (None,) * 6
        if g_loss is None:
            return (None,) * 9 + none
        dev = xyz_m.device
        g_loss = g_loss.to(torch.float32).contiguous()
        g_xyz_m = torch.empty((M, H, W, 3), dtype=torch.float32, device=dev)
        g_delta = torch.empty((M, H, W, B), dtype=torch.float32, device=dev) if delta is not None else None
        g_tab = torch.empty((int(_capi.load().sr_bob_warp_table_floats(B, M)),), dtype=torch.float32, device=dev)
        _capi.call("sr_reproj_loss_backward", dev, M, H, W, B, int(hxy.shape[-1]), xyz_m, o2b_q, o2b_t, inv_gauss, delta, se3_r,
                   se3_d, cam_q, cam_t, Kmat, hxy, mask, det, ctx.scale, g_loss, g_xyz_m, g_delta, g_tab)
        g_oq, g_ot, g_ig, g_sr, g_sd, g_cq, g_ct = split_table_grads(g_tab, B, M)
        return (g_xyz_m, g_oq, g_ot, g_ig, g_sr, g_sd, g_cq, g_ct, g_delta) + none


def reproj_loss(xyz_matched, hxy, Kmat, rest_articulation, t_articulation, log_gauss, field2cam, mask_fg, is_detected=None,
                weight=5e-2, train_res=256, delta=None):
    """forward_project of the matched points and the feat_reproj loss (deformable_gaussian.py:1488-1513,
    model.py:669-672,915,961-967,994-1012).

    xyz_matched (M,H,W,3): global_match's output.  hxy (M,H,W,2|3): pixel coordinates (the first two are read).  Kmat
    (M,3,3): each frame's intrinsics (Kmatinv of the reference's Kinv).  rest_articulation ((B,4),(B,4)), t_articulation
    ((M,B,4),(M,B,4)), log_gauss (B,3), field2cam ((M,4),(M,3)): as for vidu4d_b200.warp.bob_warp.  mask_fg (M,H,W[,1]);
    is_detected (M,) or None (= 1).  weight: feat_reproj_wt, a float or a one-element float32 CUDA tensor read at run
    time.  delta (M,H,W,B) or None: the delta-skinning term of the matched points.

    Returns {"loss": weight * mean(v[v > 0]) / train_res (0 when no v > 0), differentiable in xyz_matched, the warp
    tables' inputs and delta; "terms": (M,) each frame's share of it; "counts": (M,) int32 pixels with v > 0;
    "xy_reproj": (M,H,W,2)}, where v = ||xy_reproj - hxy[..., :2]|| * mask_fg * is_detected."""
    M, H, W, B = _check_reproj(xyz_matched, hxy, Kmat, rest_articulation, t_articulation, log_gauss, field2cam, mask_fg,
                               is_detected, weight, train_res, delta)
    o2b_q, o2b_t, inv_gauss, se3_r, se3_d = warp_tables(rest_articulation, t_articulation, log_gauss)
    if not torch.is_tensor(weight):
        weight = torch.full((1,), float(weight), dtype=torch.float32, device=xyz_matched.device)
    loss, xy, terms, counts = _ReprojLoss.apply(xyz_matched, o2b_q, o2b_t, inv_gauss, se3_r, se3_d, field2cam[0], field2cam[1],
                                                delta, Kmat, hxy, mask_fg, is_detected, weight, (M, H, W, B, float(train_res)))
    return {"loss": loss, "terms": terms, "counts": counts, "xy_reproj": xy}
