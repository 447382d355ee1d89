"""Dense point tracking through a reconstructed sequence, on the anchors render_frames(..., anchors=K) keeps.

A pixel of frame s is the blend of the few surfels it was rendered from, each hit at a known point of its disc.  With
each surfel's position and orientation in every frame (Stage 3: the bob-warped copies), the pixel's surface point is
known in every frame, and so are its projection and whether that frame sees it: correspondences over the whole
sequence, for evaluating a 4D reconstruction or propagating an edit or a label from one frame to all others.

track_pixels is one CUDA launch (csrc/track.cu, include/surfel_track.h) over (query, target frame) that writes the
outputs and nothing else.  Nothing here differentiates.
"""
from __future__ import annotations

import torch

from . import _capi

DEPTH_TOLERANCE = 0.05


def _check_anchors(anchors, device):
    """render_frames' three anchor tensors, checked: ids (S,K,H,W) int32, weights (S,K,H,W) and uv (S,K,2,H,W) float32,
    contiguous, on `device`.  Returns (ids, weights, uv, S, K, H, W)."""
    if not isinstance(anchors, (tuple, list)) or len(anchors) != 3:
        raise RuntimeError("anchors must be render_frames' (anchor_ids, anchor_weights, anchor_uv)")
    ids, w, uv = anchors
    for name, t in (("anchor_ids", ids), ("anchor_weights", w), ("anchor_uv", uv)):
        if not torch.is_tensor(t):
            raise RuntimeError(f"{name} must be a tensor, got {type(t).__name__}")
        if t.device != torch.device(device):
            raise RuntimeError(f"{name} must be on the surfels' device {device}, got {t.device}")
        if not t.is_contiguous():
            raise RuntimeError(f"{name} must be contiguous")
    if ids.dtype != torch.int32 or ids.ndim != 4:
        raise RuntimeError(f"anchor_ids must be an int32 (S,K,H,W) tensor, got {ids.dtype} {tuple(ids.shape)}")
    S, K, H, W = (int(x) for x in ids.shape)
    if K not in _capi.ANCHOR_SLOTS:
        raise RuntimeError(f"anchor_ids must have K in {_capi.ANCHOR_SLOTS} slots, got {K}")
    if w.dtype != torch.float32 or tuple(w.shape) != (S, K, H, W):
        raise RuntimeError(f"anchor_weights must be a float32 {(S, K, H, W)} tensor, got {w.dtype} {tuple(w.shape)}")
    if uv.dtype != torch.float32 or tuple(uv.shape) != (S, K, 2, H, W):
        raise RuntimeError(f"anchor_uv must be a float32 {(S, K, 2, H, W)} tensor, got {uv.dtype} {tuple(uv.shape)}")
    return ids, w, uv, S, K, H, W


def track_pixels(anchors, queries, cameras, pc, means3D=None, rotations=None, depth=None,
                 depth_tolerance=DEPTH_TOLERANCE):
    """Follow pixels through T target frames on their anchors.

    anchors: (anchor_ids, anchor_weights, anchor_uv), render_frames(..., anchors=K)'s three outputs for any S frames.
    queries: (N,3) int32 CUDA tensor of (anchor frame s in [0, S), x, y): pixel (x, y) of anchors' frame s.
    cameras: a BatchCameras of the T target frames, scalar or with the `intrinsics` table, at the anchors' resolution.
    pc, means3D (T,P,3), rotations (T,P,4): the surfels, as render_frames takes them -- default pc.get_xyz and
    pc.get_rotation in every frame; Stage 3 passes the bob-warped copies and identity views.  pc.get_scaling is shared.
    depth: optional (T,H,W) float32 per-frame depth, e.g. render_frames' surf_depth[:, 0], for the occlusion test.

    For every query n and target frame t, over the query's non-empty slots k (csrc/track.cu):

        X = sum_k w_k (mean_t + u_k s_u t_u,t + v_k s_v t_v,t) / sum_k w_k

    with the surfel's frame-t mean, the first two columns of its frame-t rotation matrix and its scale, as the
    rasterizer's preprocess builds them.  X is projected through frame t's view and intrinsics into the rasterizer's
    continuous pixel coordinates, where pixel (x, y) is centred at (x + 0.5, y + 0.5): a query tracked into its own frame
    with its own surfels lands on its pixel's centre.

    Returns {"xy": (N,T,2), "z": (N,T) view depth, "visible": (N,T) bool -- z >= 0.2, inside the image and, with depth,
    |z - depth[t, floor(y), floor(x)]| <= depth_tolerance * z --, "coverage": (N,) sum_k w_k, which the caller compares
    with the pixel's acc to see how much of it the K slots hold}.  A query on a pixel no surfel covers, with an anchor
    frame or pixel out of range, or with an id >= P gets coverage 0, NaN xy and z and visible False in every frame; the
    kernel checks this without a host synchronisation."""
    from .rasterizer import _check_intrinsics, _f32c
    from .renderer import BatchCameras, _cam_tans, stack_cameras
    if not isinstance(cameras, BatchCameras):
        cameras = stack_cameras(cameras)
    xyz = pc.get_xyz if means3D is None else means3D
    P, dev = int(xyz.shape[-2]), xyz.device
    ids, w, uv, S, K, H, W = _check_anchors(anchors, dev)
    T = len(cameras)
    if (int(cameras.image_height), int(cameras.image_width)) != (H, W):
        raise RuntimeError(f"cameras are {int(cameras.image_width)}x{int(cameras.image_height)}, the anchors {W}x{H}")
    if not 1 <= T <= 65535:
        raise RuntimeError(f"cameras must hold 1..65535 target frames, got {T}")
    if not torch.is_tensor(queries) or queries.dtype != torch.int32 or queries.ndim != 2 or int(queries.shape[1]) != 3:
        raise RuntimeError("queries must be an (N,3) int32 tensor of (anchor frame, x, y)")
    if queries.device != torch.device(dev):
        raise RuntimeError(f"queries must be on the surfels' device {dev}, got {queries.device}")
    for name, t, tail in (("means3D", means3D, 3), ("rotations", rotations, 4)):
        if t is not None and (t.ndim != 3 or tuple(t.shape) != (T, P, tail)):
            raise RuntimeError(f"{name} must be (T,P,{tail}) = ({T},{P},{tail}) or None, got {tuple(t.shape)}")
    if depth is not None:
        if not torch.is_tensor(depth) or depth.dtype != torch.float32 or tuple(depth.shape) != (T, H, W):
            raise RuntimeError(f"depth must be a float32 (T,H,W) = ({T},{H},{W}) tensor")
        if depth.device != torch.device(dev):
            raise RuntimeError(f"depth must be on the surfels' device {dev}, got {depth.device}")
    tol = float(depth_tolerance)
    if not tol >= 0.0:
        raise RuntimeError(f"depth_tolerance must be >= 0, got {depth_tolerance!r}")
    intr = _check_intrinsics(cameras.intrinsics, T, xyz)
    tanx, tany = (0.0, 0.0) if intr is not None else _cam_tans(cameras)
    N = int(queries.shape[0])
    with torch.no_grad(), torch.cuda.device(dev):
        mu = _f32c(xyz.detach(), "means3D")
        rot = _f32c((pc.get_rotation if rotations is None else rotations).detach(), "rotations")
        sc = _f32c(pc.get_scaling.detach(), "scales")
        vm = _f32c(cameras.world_view_transform.detach(), "world_view_transform")
        dp = None if depth is None else depth.detach().contiguous()
        xy = torch.empty((N, T, 2), dtype=torch.float32, device=dev)
        z = torch.empty((N, T), dtype=torch.float32, device=dev)
        vis = torch.empty((N, T), dtype=torch.bool, device=dev)
        cov = torch.empty((N,), dtype=torch.float32, device=dev)
        if N:
            _capi.call("sr_track_pixels", dev, N, T, S, P, K, W, H, queries.contiguous(), ids, w, uv, K * H * W, mu,
                       3 * P if means3D is not None else 0, sc, rot, 4 * P if rotations is not None else 0, vm,
                       float(tanx), float(tany), intr, dp, tol, xy, z, vis, cov)
    return {"xy": xy, "z": z, "visible": vis, "coverage": cov}
