"""render() twin and the caller-side contract of the hot path.

Mirrors (same names, argument meaning, dict keys and error behaviour):

    render(viewpoint_camera, pc, pipe, bg_color, scaling_modifier=1.0, override_color=None)
                                           gs/gaussian_renderer/__init__.py:21-164
    depths_to_points / depth_to_normal     gs/utils/point_utils.py:9-37
    MiniCam / KCamera input contract       gs/scene/cameras.py:59-162

`pc` is duck-typed exactly as the reference uses it: get_xyz (P,3), get_opacity (P,1), get_scaling (P,2),
get_rotation (P,4), get_features (P,K,3), active_sh_degree, get_covariance().  `pipe` needs
compute_cov3D_python and depth_ratio.  lab4d's DeformableGaussian.render_view
(lab4d/nnutils/deformable_gaussian.py:178-190) can call this render() unchanged.

The ~25 small torch ops of the post-processing stay in PyTorch this round (SURVEY.md section 8(f) row N1 is the
fused version); what is removed here are the reference's per-call host synchronisations other than
`num_rendered` (tan(FoV) on a CUDA tensor, torch.tensor(...).cuda() + .inverse() per frame,
point_utils.py:9-18): the per-camera ray table is built once and cached.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import torch

from .rasterizer import GaussianRasterizationSettings, GaussianRasterizer


def _tan_half(fov) -> float:
    if torch.is_tensor(fov):
        return float(torch.tan(fov * 0.5).item())
    return math.tan(float(fov) * 0.5)


def _cam_tans(cam):
    """(tan(FoVx/2), tan(FoVy/2)) of a camera, computed ONCE per camera object: the reference's KCamera keeps FoVx/FoVy as
    tensors (gs/scene/cameras.py:86-87), possibly on the GPU, and reading them costs a host sync per call -- which
    also makes the call uncapturable in a CUDA graph.  The pair is cached on the object (cameras are immutable in Vidu4D)."""
    t = getattr(cam, "_sr_tans", None)
    if t is None:
        t = (_tan_half(cam.FoVx), _tan_half(cam.FoVy))
        try:
            object.__setattr__(cam, "_sr_tans", t)
        except Exception:
            pass
    return t


# ---------------------------------------------------------------------------------------------
# cameras (gs/scene/cameras.py, gs/utils/graphics_utils.py) -- input contract only
# ---------------------------------------------------------------------------------------------
def getWorld2View2(R, t, translate=(0.0, 0.0, 0.0), scale=1.0):
    """gs/utils/graphics_utils.py:38-51 (R is camera-to-world rotation, t world-to-camera translation)."""
    R = torch.as_tensor(R, dtype=torch.float32)
    t = torch.as_tensor(t, dtype=torch.float32)
    Rt = torch.zeros((4, 4), dtype=torch.float32)
    Rt[:3, :3] = R.T
    Rt[:3, 3] = t
    Rt[3, 3] = 1.0
    C2W = torch.inverse(Rt)
    C2W[:3, 3] = (C2W[:3, 3] + torch.as_tensor(translate, dtype=torch.float32)) * scale
    return torch.inverse(C2W).float()


def getProjectionMatrix(znear, zfar, fovX, fovY):
    """gs/utils/graphics_utils.py:53-76"""
    tanHalfFovY, tanHalfFovX = math.tan(fovY / 2), math.tan(fovX / 2)
    top, right = tanHalfFovY * znear, tanHalfFovX * znear
    bottom, left = -top, -right
    P = torch.zeros(4, 4)
    P[0, 0] = 2.0 * znear / (right - left)
    P[1, 1] = 2.0 * znear / (top - bottom)
    P[0, 2] = (right + left) / (right - left)
    P[1, 2] = (top + bottom) / (top - bottom)
    P[3, 2] = 1.0
    P[2, 2] = zfar / (zfar - znear)
    P[2, 3] = -(zfar * znear) / (zfar - znear)
    return P


@dataclass
class MiniCam:
    """gs/scene/cameras.py:59-71 -- everything render() reads from a camera."""
    image_width: int
    image_height: int
    FoVy: float
    FoVx: float
    znear: float
    zfar: float
    world_view_transform: torch.Tensor   # (4,4) = W2C transposed (row-vector convention)
    full_proj_transform: torch.Tensor    # (4,4)
    camera_center: torch.Tensor = None

    def __post_init__(self):
        if self.camera_center is None:
            self.camera_center = torch.inverse(self.world_view_transform)[3][:3]


def make_camera(width, height, fovx, fovy, R=None, T=None, device="cuda", znear=0.01, zfar=100.0) -> MiniCam:
    """Camera from a camera-to-world rotation R (3,3) and world-to-camera translation T (3,), as
    gs/scene/cameras.py:17-57 builds it.  R=None,T=None gives the Stage-3 identity camera (cameras.py:84-85)."""
    R = torch.eye(3) if R is None else torch.as_tensor(R, dtype=torch.float32)
    T = torch.zeros(3) if T is None else torch.as_tensor(T, dtype=torch.float32)
    wvt = getWorld2View2(R, T).transpose(0, 1)
    proj = getProjectionMatrix(znear, zfar, fovx, fovy).transpose(0, 1)
    full = wvt.unsqueeze(0).bmm(proj.unsqueeze(0)).squeeze(0)
    center = torch.inverse(wvt)[3, :3]
    return MiniCam(int(width), int(height), float(fovy), float(fovx), znear, zfar, wvt.to(device).contiguous(),
                   full.to(device).contiguous(), center.to(device).contiguous())


# ---------------------------------------------------------------------------------------------
# gs/utils/point_utils.py
# ---------------------------------------------------------------------------------------------
_dir_cache: dict = {}


def _rays(view, device):
    """rays_d (H*W,3) and rays_o (3,) of depths_to_points (point_utils.py:9-21).  The camera-space pixel
    directions (pixel grid times K^-1) are cached per (W,H,fov); the per-frame camera-to-world factor uses
    the adjugate formula, so the reference's per-call torch.tensor(...).cuda(), .inverse() and math.tan(cuda
    tensor) syncs are gone."""
    W, H = int(view.image_width), int(view.image_height)
    tx, ty = _cam_tans(view)
    key = (W, H, tx, ty, str(device))
    dirs = _dir_cache.get(key)
    if dirs is None:
        fx, fy = W / (2 * tx), H / (2 * ty)
        intrins = torch.tensor([[fx, 0., W / 2.], [0., fy, H / 2.], [0., 0., 1.0]], dtype=torch.float32)
        grid_x, grid_y = torch.meshgrid(torch.arange(W).float(), torch.arange(H).float(), indexing='xy')
        points = torch.stack([grid_x, grid_y, torch.ones_like(grid_x)], dim=-1).reshape(-1, 3)
        dirs = (points @ intrins.inverse().T).to(device)
        if len(_dir_cache) > 16:
            _dir_cache.clear()
        _dir_cache[key] = dirs
    # camera-to-world of the affine view matrix by the adjugate formula: plain elementwise torch ops -- no host
    # synchronisation, no solver workspace, capturable in a CUDA graph (the reference calls .inverse() per frame)
    w2c = view.world_view_transform.T
    A, t = w2c[:3, :3], w2c[:3, 3]
    c0 = torch.linalg.cross(A[1], A[2]); c1 = torch.linalg.cross(A[2], A[0]); c2 = torch.linalg.cross(A[0], A[1])
    Ainv = torch.stack([c0, c1, c2], dim=1) / (A[0] * c0).sum()
    rays_d = dirs @ Ainv.T
    rays_o = -(Ainv @ t)
    return rays_d, rays_o


def depths_to_points(view, depthmap):
    rays_d, rays_o = _rays(view, depthmap.device)
    return depthmap.reshape(-1, 1) * rays_d + rays_o


def depth_to_normal(view, depth):
    """view: camera; depth: (1,H,W).  Returns (H,W,3) pseudo surface normals (point_utils.py:23-37)."""
    points = depths_to_points(view, depth).reshape(*depth.shape[1:], 3)
    output = torch.zeros_like(points)
    dx = points[2:, 1:-1] - points[:-2, 1:-1]
    dy = points[1:-1, 2:] - points[1:-1, :-2]
    normal_map = torch.nn.functional.normalize(torch.cross(dx, dy, dim=-1), dim=-1)
    output[1:-1, 1:-1, :] = normal_map
    return output


# ---------------------------------------------------------------------------------------------
# gs/gaussian_renderer/__init__.py:21-164
# ---------------------------------------------------------------------------------------------
def render(viewpoint_camera, pc, pipe, bg_color: torch.Tensor, scaling_modifier=1.0, override_color=None, features=None):
    """Render the scene.  Background tensor (bg_color) must be on GPU!

    features (P,F), 1 <= F <= 32 (not in the reference): per-surfel channels composited with the colour's weights next to
    the SH colour; "render" is then (3+F,H,W) -- RGB, then the F feature planes over bg_color[3:] (bg_color of 3+F values)
    or a zero background (bg_color of 3).  Vidu4D's 22-channel vector (deformable_gaussian.py:1182-1207) goes here."""
    xyz = pc.get_xyz
    screenspace_points = torch.zeros_like(xyz, dtype=xyz.dtype, requires_grad=True, device=xyz.device) + 0
    try:
        screenspace_points.retain_grad()
    except Exception:
        pass

    tanfovx, tanfovy = _cam_tans(viewpoint_camera)
    raster_settings = GaussianRasterizationSettings(
        image_height=int(viewpoint_camera.image_height),
        image_width=int(viewpoint_camera.image_width),
        tanfovx=tanfovx,
        tanfovy=tanfovy,
        bg=bg_color,
        scale_modifier=scaling_modifier,
        viewmatrix=viewpoint_camera.world_view_transform,
        projmatrix=viewpoint_camera.full_proj_transform,
        sh_degree=pc.active_sh_degree,
        campos=viewpoint_camera.camera_center,
        prefiltered=False,
        debug=False,
    )
    rasterizer = GaussianRasterizer(raster_settings=raster_settings)
    means3D = xyz
    means2D = screenspace_points
    opacity = pc.get_opacity

    scales = None
    rotations = None
    cov3D_precomp = None
    if pipe.compute_cov3D_python:
        cov3D_precomp = pc.get_covariance(scaling_modifier)
    else:
        scales = pc.get_scaling
        rotations = pc.get_rotation

    # the reference always passes SHs *and* override_color; with a non-None override_color the rasterizer
    # raises (gaussian_renderer/__init__.py:91-92 vs RAST/.../__init__.py:192-193) -- preserved.
    shs = pc.get_features
    colors_precomp = override_color

    try:
        means3D.retain_grad()
    except Exception:
        pass
    if features is None:
        rendered_image, radii, allmap = rasterizer(
            means3D=means3D, means2D=means2D, shs=shs, colors_precomp=colors_precomp, opacities=opacity,
            scales=scales, rotations=rotations, cov3D_precomp=cov3D_precomp)
    else:
        rendered_image, radii, allmap = rasterizer.forward_features(
            means3D=means3D, means2D=means2D, opacities=opacity, features=features, shs=shs,
            colors_precomp=colors_precomp, scales=scales, rotations=rotations, cov3D_precomp=cov3D_precomp)

    rets = {"render": rendered_image,
            "viewspace_points": means2D,
            "visibility_filter": radii > 0,
            "radii": radii}

    render_alpha = allmap[1:2]
    render_normal = allmap[2:5]
    render_normal = (render_normal.permute(1, 2, 0) @ (viewpoint_camera.world_view_transform[:3, :3].T)).permute(2, 0, 1)
    render_depth_median = allmap[5:6]
    render_depth_median = torch.nan_to_num(render_depth_median, 0, 0)
    render_depth_expected = allmap[0:1]
    render_depth_expected = (render_depth_expected / render_alpha)
    render_depth_expected = torch.nan_to_num(render_depth_expected, 0, 0)
    render_dist = allmap[6:7]
    surf_depth = render_depth_expected * (1 - pipe.depth_ratio) + (pipe.depth_ratio) * render_depth_median
    surf_normal = depth_to_normal(viewpoint_camera, surf_depth)
    surf_normal = surf_normal.permute(2, 0, 1)
    surf_normal = surf_normal * (render_alpha).detach()

    rets.update({
        'acc': render_alpha,
        'rend_normal': render_normal,
        'rend_dist': render_dist,
        'surf_depth': torch.cat([surf_depth] * 3, 0),
        'render_depth_median': torch.cat([render_depth_median] * 3, 0),
        'render_depth_expected': torch.cat([render_depth_expected] * 3, 0),
        'surf_normal': surf_normal,
    })
    return rets


class _RenderPost(torch.autograd.Function):
    """allmap (8,H,W) -> (acc, rend_normal, rend_dist, depth_median, depth_expected, surf_depth, surf_normal) in one
    CUDA kernel each way (csrc/postprocess.cu); same maths as the torch expressions in render()."""

    @staticmethod
    def forward(ctx, allmap, wvt, tanx, tany, depth_ratio):
        from . import _capi
        allmap = allmap.contiguous()
        wvt = wvt.contiguous()
        _, H, W = allmap.shape
        dev = allmap.device
        mk = lambda c: torch.empty((c, H, W), dtype=torch.float32, device=dev)  # noqa: E731
        acc, rn, dist, med, ex, sd, sn = mk(1), mk(3), mk(1), mk(1), mk(1), mk(1), mk(3)
        _capi.call("sr_post_forward", dev, W, H, tanx, tany, depth_ratio, allmap, wvt, acc, rn, dist, med, ex, sd, sn)
        ctx.save_for_backward(allmap, wvt, sd)
        ctx.cfg = (W, H, tanx, tany, depth_ratio)
        return acc, rn, dist, med, ex, sd, sn

    @staticmethod
    def backward(ctx, g_acc, g_rn, g_dist, g_med, g_ex, g_sd, g_sn):
        from . import _capi
        allmap, wvt, sd = ctx.saved_tensors
        W, H, tanx, tany, depth_ratio = ctx.cfg
        dev = allmap.device
        z = lambda g, c: torch.zeros((c, H, W), dtype=torch.float32, device=dev) if g is None else g.contiguous()  # noqa: E731
        g_acc, g_rn, g_dist, g_med, g_ex, g_sd, g_sn = z(g_acc, 1), z(g_rn, 3), z(g_dist, 1), z(g_med, 1), z(g_ex, 1), z(g_sd, 1), z(g_sn, 3)
        g_allmap = torch.empty_like(allmap)
        _capi.call("sr_post_backward", dev, W, H, tanx, tany, depth_ratio, allmap, wvt, sd, g_acc, g_rn, g_dist, g_med, g_ex, g_sd,
                   g_sn, g_allmap)
        return g_allmap, None, None, None, None


def render_fused(viewpoint_camera, pc, pipe, bg_color: torch.Tensor, scaling_modifier=1.0, override_color=None,
                 features=None):
    """Same contract, `features` and dict keys as render(); the post-processing of `allmap` runs in one fused CUDA kernel each
    way instead of ~35 forward / ~60 backward PyTorch kernels (SURVEY.md section 8(f) row N1).  The three depth
    entries are (3,H,W) broadcast VIEWS of one plane (render() materialises three copies with torch.cat)."""
    xyz = pc.get_xyz
    screenspace_points = torch.zeros_like(xyz, dtype=xyz.dtype, requires_grad=True, device=xyz.device) + 0
    try:
        screenspace_points.retain_grad()
    except Exception:
        pass
    tanfovx, tanfovy = _cam_tans(viewpoint_camera)
    raster_settings = GaussianRasterizationSettings(
        image_height=int(viewpoint_camera.image_height), image_width=int(viewpoint_camera.image_width),
        tanfovx=tanfovx, tanfovy=tanfovy, bg=bg_color, scale_modifier=scaling_modifier,
        viewmatrix=viewpoint_camera.world_view_transform, projmatrix=viewpoint_camera.full_proj_transform,
        sh_degree=pc.active_sh_degree, campos=viewpoint_camera.camera_center, prefiltered=False, debug=False)
    rasterizer = GaussianRasterizer(raster_settings=raster_settings)
    scales = rotations = cov3D_precomp = None
    if pipe.compute_cov3D_python:
        cov3D_precomp = pc.get_covariance(scaling_modifier)
    else:
        scales, rotations = pc.get_scaling, pc.get_rotation
    try:
        xyz.retain_grad()
    except Exception:
        pass
    kw = dict(means3D=xyz, means2D=screenspace_points, shs=pc.get_features, colors_precomp=override_color,
              opacities=pc.get_opacity, scales=scales, rotations=rotations, cov3D_precomp=cov3D_precomp)
    rendered_image, radii, allmap = rasterizer(**kw) if features is None else rasterizer.forward_features(features=features, **kw)
    acc, rn, dist, med, ex, sd, sn = _RenderPost.apply(allmap, viewpoint_camera.world_view_transform, tanfovx, tanfovy,
                                                       float(pipe.depth_ratio))
    return {"render": rendered_image, "viewspace_points": screenspace_points, "visibility_filter": radii > 0,
            "radii": radii, "acc": acc, "rend_normal": rn, "rend_dist": dist, "surf_depth": sd.expand(3, -1, -1),
            "render_depth_median": med.expand(3, -1, -1), "render_depth_expected": ex.expand(3, -1, -1),
            "surf_normal": sn}


@dataclass
class PipelineParams:
    """gs/arguments/__init__.py PipelineParams, as instantiated at deformable_gaussian.py:158-160."""
    convert_SHs_python: bool = False
    compute_cov3D_python: bool = False
    depth_ratio: float = 0.0
    debug: bool = False


# ---------------------------------------------------------------------------------------------
# Batched Stage-3 inner loop: M frames -> rasterize -> post-process -> image losses, one launch set each way
# (SURVEY.md section 8(f) row N1).  Replaces the Python frame loop of lab4d/nnutils/deformable_gaussian.py:1175-1188 and
# the ~40 torch kernels per frame of lab4d/engine/model.py:674-692,817-842.
# ---------------------------------------------------------------------------------------------
@dataclass
class BatchCameras:
    """M cameras sharing resolution and field of view (Stage 3: gs/scene/cameras.py:72-162 builds them per frame)."""
    image_width: int
    image_height: int
    FoVx: float
    FoVy: float
    world_view_transform: torch.Tensor   # (M,4,4), each W2C transposed
    full_proj_transform: torch.Tensor    # (M,4,4)
    camera_center: torch.Tensor          # (M,3)

    def __len__(self):
        return int(self.world_view_transform.shape[0])


def stack_cameras(cams) -> BatchCameras:
    c0 = cams[0]
    return BatchCameras(int(c0.image_width), int(c0.image_height), c0.FoVx, c0.FoVy,
                        torch.stack([c.world_view_transform for c in cams]).contiguous(),
                        torch.stack([c.full_proj_transform for c in cams]).contiguous(),
                        torch.stack([c.camera_center for c in cams]).contiguous())


class _RasterLossBatch(torch.autograd.Function):
    """rasterize M frames -> fused post-processing + losses.  The loss kernel already produced dL/dcolor and dL/dallmap,
    so backward() is just the rasterizer backward with the upstream scalar as `grad_scale`.  Optional feature planes are a
    further differentiable output; their incoming gradient (already scaled) goes to the same rasterizer backward."""

    @staticmethod
    def forward(ctx, means3D, means2D, sh, opacities, scales, rotations, bkgd, cfg, features=None, feature_loss=None,
                mask_loss=None):
        from . import _capi
        from .rasterizer import _C
        (cams, bg, sh_degree, target, vis, mask, mask_wt, depth_ratio, w_rgb, w_mask, lam_n, lam_d, tanx, tany, target_stream,
         w_ssim) = cfg
        M, H, W = len(cams), cams.image_height, cams.image_width
        dev = means3D.device
        e = torch.empty((0,), dtype=torch.float32, device=dev)
        kw = {} if features is None else {"features": features, "concat": False}
        out = _C.rasterize_gaussians_batch(
            bg, means3D, e, opacities, scales, rotations, 1.0, cams.world_view_transform, cams.full_proj_transform, tanx, tany,
            H, W, sh, sh_degree, cams.camera_center, **kw)
        nr, color, allmap, radii, gb, bb, ib = out[:7]
        feat = out[7] if features is not None else None
        terms = torch.empty((M, 4), dtype=torch.float32, device=dev)
        dLc = torch.empty_like(color)
        dLa = torch.empty_like(allmap)
        dLb = torch.empty((M, 3), dtype=torch.float32, device=dev) if bkgd is not None else None
        scratch = torch.empty((M, H, W), dtype=torch.float32, device=dev)
        f32 = lambda t: None if t is None else t.to(dtype=torch.float32).contiguous()  # noqa: E731
        target, vis, mask, mask_wt = f32(target), f32(vis), f32(mask), f32(mask_wt)
        bk = f32(bkgd.detach()) if bkgd is not None else None
        wvt = f32(cams.world_view_transform)         # (M,4,4) packed: callers may hand in a strided view
        if target_stream is not None:       # the targets are still being uploaded on another stream: join it only now,
            torch.cuda.current_stream(dev).wait_stream(target_stream)   # after the rasterizer forward has been queued
        _capi.call("sr_render_loss_batch", dev, M, W, H, tanx, tany, float(depth_ratio), color, allmap, wvt, target, vis, mask,
                   mask_wt, bk, float(w_rgb), float(w_mask), float(lam_n), float(lam_d), terms, dLc, dLa, dLb, scratch)
        total = terms.sum()
        sterms = None
        if w_ssim > 0.0:                    # D-SSIM on the final colour: csrc/ssim.cu, its gradient added into dLc / dLa / dLb
            sterms = _ssim_term(M, H, W, color, allmap, target, bk, w_ssim, dLc, dLa, dLb)
            total = total + sterms.sum()
        mterms = None
        if mask_loss is not None:           # after SSIM: the silhouette term's gradient is the last addend of dL/dalpha
            is_det, weight = mask_loss
            mterms, mcounts = _mask_term(M, H, W, allmap, mask, vis, f32(is_det), weight, dLa)
            total = total + mterms.sum()
        dLf = None
        if feature_loss is not None:        # the losses on the feature planes: csrc/loss.cu, sr_feature_loss_batch
            ftarget, is_det, gm, weights = feature_loss
            F = feat.shape[1]
            fterms = torch.empty((M, 2), dtype=torch.float32, device=dev)
            counts = torch.empty((M, 2), dtype=torch.int32, device=dev)
            dLf = torch.empty_like(feat)
            ftarget, is_det = f32(ftarget), f32(is_det)
            _capi.call("sr_feature_loss_batch", dev, M, W, H, F, 0 if ftarget is None else int(ftarget.shape[1]), gm, feat, ftarget,
                       mask, is_det, allmap, weights, fterms, counts, dLf)
            total = total + fterms.sum()
        ctx.cfg = (cams, bg, sh_degree, tanx, tany)
        ctx.has_bkgd = bkgd is not None
        ctx.save_for_backward(means3D, scales, rotations, radii, sh, opacities, gb, bb, ib, dLc, dLa,
                              dLb if dLb is not None else e, features, dLf)
        ctx.has_features = features is not None
        outs = (total, terms, color, allmap, radii) + (() if feat is None else (feat,)) + (() if dLf is None else (fterms, counts))
        outs = outs + (() if sterms is None else (sterms,)) + (() if mterms is None else (mterms, mcounts))
        ctx.mark_non_differentiable(terms, color, allmap, radii, *(o for o in outs[5:] if o is not feat))
        return outs

    @staticmethod
    def backward(ctx, g_total, g_terms, g_color, g_allmap, g_radii, g_feat=None, *_):
        from .rasterizer import _C, _reduce_like
        cams, bg, sh_degree, tanx, tany = ctx.cfg
        means3D, scales, rotations, radii, sh, opacities, gb, bb, ib, dLc, dLa, dLb, features, dLf = ctx.saved_tensors
        e = torch.empty((0,), dtype=torch.float32, device=means3D.device)
        kw = {}
        if ctx.has_features:
            if dLf is not None:
                # the fused feature losses' plane gradient scales with the upstream scalar like dLc / dLa; the caller's own
                # use of out["features"] (g_feat) does not -- so the two are summed here and handed over unscaled
                g_feat = dLf * g_total if g_feat is None else torch.addcmul(g_feat, dLf, g_total)
            elif g_feat is None:
                g_feat = torch.zeros((dLc.shape[0], features.shape[-1]) + tuple(dLc.shape[2:]), dtype=torch.float32,
                                     device=means3D.device)
            kw = {"features": features, "dL_dout_features": g_feat}
        grads = _C.rasterize_gaussians_backward_batch(
            bg, means3D, radii, e, scales, rotations, 1.0, cams.world_view_transform, cams.full_proj_transform, tanx, tany,
            dLc, dLa, sh, sh_degree, cams.camera_center, gb, bb, ib, grad_scale=g_total, sum_shared=True,
            opacity_shared=opacities.ndim == 2, want_transmat=False, **kw)
        g2d, gcol, gop, g3d, gtm, gsh, gsc, grot = grads[:8]
        g_bk = (dLb.sum(0) * g_total) if ctx.has_bkgd else None
        return (_reduce_like(g3d, means3D), g2d, _reduce_like(gsh, sh), _reduce_like(gop, opacities),
                _reduce_like(gsc, scales), _reduce_like(grot, rotations), g_bk, None,
                _reduce_like(grads[8], features) if ctx.has_features else None, None, None)


def _ssim_term(M, H, W, color, allmap, target, bkgd, w_ssim, dLc, dLa, dLb):
    """Each frame's w_ssim * (1 - SSIM(color + (1 - alpha) * bkgd, target)), (M,), with its gradient ADDED into dL/dcolor,
    dL/dalpha (allmap plane 1) and dL/dbkgd -- unscaled, like the other terms' (the backward applies the upstream scalar)."""
    from . import _capi
    dev = color.device
    nbytes = int(_capi.load().sr_ssim_scratch_bytes(M, 3, H, W))
    scratch = torch.empty((nbytes,), dtype=torch.uint8, device=dev)
    per_frame = torch.empty((M,), dtype=torch.float32, device=dev)
    mean = torch.empty((1,), dtype=torch.float32, device=dev)
    maps = torch.empty((3, M, 3, H, W), dtype=torch.float32, device=dev)
    alpha, d_alpha = (allmap[:, 1], dLa[:, 1]) if bkgd is not None else (None, None)
    stride = 8 * H * W
    _capi.call("sr_ssim_forward", dev, M, 3, H, W, color, target, alpha, stride, bkgd, per_frame, mean, maps, scratch, nbytes)
    g = torch.full((M,), -float(w_ssim), dtype=torch.float32, device=dev)      # d(w (1 - ssim_f)) / d ssim_f
    _capi.call("sr_ssim_backward", dev, M, 3, H, W, color, target, alpha, stride, bkgd, maps, g, 1, dLc, 1, d_alpha, dLb,
               scratch, nbytes)
    return (1.0 - per_frame) * float(w_ssim)


def _mask_term(M, H, W, allmap, mask, vis, is_detected, weight, dLa):
    """Stage 3's silhouette term as the reference weighs it (csrc/mask_loss.cu): returns each frame's share (M,) and count of
    positive values (M,) int32, and ADDS its gradient into dL/dalpha (allmap plane 1) -- unscaled, like the other terms'."""
    from . import _capi
    dev = allmap.device
    nbytes = int(_capi.load().sr_mask_loss_scratch_bytes(M, W, H))
    scratch = torch.empty((nbytes,), dtype=torch.uint8, device=dev)
    terms = torch.empty((M,), dtype=torch.float32, device=dev)
    counts = torch.empty((M,), dtype=torch.int32, device=dev)
    balance = torch.empty((3,), dtype=torch.float32, device=dev)
    _capi.call("sr_mask_loss_batch", dev, M, W, H, allmap[:, 1], 8 * H * W, mask, vis, is_detected, weight, terms, counts,
               balance, dLa[:, 1], scratch, nbytes)
    return terms, counts


def _check_mask_loss(M, device, mask_gt, mask_wt, w_mask, is_detected, mask_loss_weight):
    """Validate the fused silhouette term's arguments of render_loss_batch before anything runs on the device; returns
    (is_detected, weight)."""
    if mask_gt is None:
        raise RuntimeError("mask_loss_weight needs mask_gt")
    if mask_wt is not None or w_mask != 0.0:
        raise RuntimeError("mask_loss_weight replaces the plain mask term: pass neither mask_wt nor w_mask != 0 with it")
    if tuple(mask_loss_weight.shape) != (1,) or mask_loss_weight.dtype != torch.float32:
        raise RuntimeError(f"mask_loss_weight must be a float32 (1,) tensor, got {mask_loss_weight.dtype} "
                           f"{tuple(mask_loss_weight.shape)}")
    if is_detected is not None and tuple(is_detected.shape) != (M,):
        raise RuntimeError(f"is_detected must be (M,) = ({M},), got {tuple(is_detected.shape)}")
    for name, t in (("mask_loss_weight", mask_loss_weight), ("is_detected", is_detected)):
        if t is not None and (not t.is_cuda or t.device != device):
            raise RuntimeError(f"{name} must be a CUDA tensor on the rasterizer's device {device}, got {t.device}")
    return is_detected, mask_loss_weight.contiguous()


def _check_feature_losses(M, H, W, features, feature_target, mask_gt, is_detected, gauss_mask_channel, feature_loss_weights):
    """Validate the fused feature-loss arguments of render_loss_batch before anything runs on the device (shapes and
    channels first, then devices); returns (feature_target, is_detected, gauss_mask_channel (-1 = off), weights)."""
    if features is None:
        raise RuntimeError("fused feature losses (feature_target / gauss_mask_channel) need features=")
    F = int(features.shape[-1])
    Cf = 0
    if feature_target is not None:
        Cf = int(feature_target.shape[1]) if feature_target.ndim == 4 else -1
        if Cf < 1 or Cf > F or tuple(feature_target.shape[::2]) != (M, H) or feature_target.shape[3] != W:
            raise RuntimeError(f"feature_target must be (M,Cf,H,W) = ({M},Cf,{H},{W}) with 1 <= Cf <= F = {F}, "
                               f"got {tuple(feature_target.shape)}")
        if mask_gt is None:
            raise RuntimeError("the feature term needs mask_gt (the reference masks it with batch['mask'])")
    gm = -1 if gauss_mask_channel is None else int(gauss_mask_channel)
    if gauss_mask_channel is not None and not Cf <= gm < F:
        raise RuntimeError(f"gauss_mask_channel must be in [Cf, F) = [{Cf}, {F}), got {gauss_mask_channel}")
    if is_detected is not None and tuple(is_detected.shape) != (M,):
        raise RuntimeError(f"is_detected must be (M,) = ({M},), got {tuple(is_detected.shape)}")
    if feature_loss_weights is not None and (tuple(feature_loss_weights.shape) != (2,)
                                             or feature_loss_weights.dtype != torch.float32):
        raise RuntimeError("feature_loss_weights must be a float32 (2,) tensor [feature_wt, reg_gauss_mask_wt]")
    for name, t in (("features", features), ("feature_target", feature_target), ("mask_gt", mask_gt),
                    ("is_detected", is_detected), ("feature_loss_weights", feature_loss_weights)):
        if t is not None and not t.is_cuda:
            raise RuntimeError(f"{name} must be a CUDA tensor")
    if feature_loss_weights is None:        # config.py:82,102 defaults; pass a device tensor to change them without re-capture
        feature_loss_weights = torch.tensor([1e-2, 1e-2], dtype=torch.float32, device=features.device)
    return feature_target, is_detected, gm, feature_loss_weights.contiguous()


def _check_loss_inputs(M, H, W, device, target_rgb, vis2d, mask_gt, mask_wt, learnable_bkgd):
    """Validate the image-loss arguments of render_loss_batch before anything runs on the device (shapes first, then
    devices).  The loss kernel reads them as raw (M,3,H,W) / (M,H,W) / (3,) buffers on the rasterizer's device: a (H,W)
    mask for M > 1 frames or a host tensor would make it read past the end of the buffer."""
    if target_rgb is None or tuple(target_rgb.shape) != (M, 3, H, W):
        raise RuntimeError(f"target_rgb must be (M,3,H,W) = ({M},3,{H},{W}), got "
                           f"{None if target_rgb is None else tuple(target_rgb.shape)}")
    for name, t in (("vis2d", vis2d), ("mask_gt", mask_gt), ("mask_wt", mask_wt)):
        if t is not None and tuple(t.shape) != (M, H, W):
            raise RuntimeError(f"{name} must be (M,H,W) = ({M},{H},{W}) or None, got {tuple(t.shape)}")
    if mask_wt is not None and mask_gt is None:
        raise RuntimeError("mask_wt weights the mask term: it needs mask_gt")
    if learnable_bkgd is not None and learnable_bkgd.numel() != 3:
        raise RuntimeError(f"learnable_bkgd must have 3 elements, got shape {tuple(learnable_bkgd.shape)}")
    for name, t in (("target_rgb", target_rgb), ("vis2d", vis2d), ("mask_gt", mask_gt), ("mask_wt", mask_wt),
                    ("learnable_bkgd", learnable_bkgd)):
        if t is not None and (not t.is_cuda or t.device != device):
            raise RuntimeError(f"{name} must be a CUDA tensor on the rasterizer's device {device}, got {t.device}")


def render_loss_batch(cameras, pc, pipe, bg_color, target_rgb, vis2d=None, mask_gt=None, mask_wt=None, learnable_bkgd=None,
                      w_rgb=1.0, w_mask=0.0, lambda_normal=0.0, lambda_dist=0.0, means3D=None, rotations=None, target_stream=None,
                      features=None, feature_target=None, is_detected=None, gauss_mask_channel=None, feature_loss_weights=None,
                      w_ssim=0.0, mask_loss_weight=None):
    """The Stage-3 inner loop for M frames in one call: rasterize every frame (batched launch set), post-process and
    evaluate the image losses in one fused kernel, and hand autograd a single scalar.

    cameras: BatchCameras (or a list of cameras, stacked here).  pc: as in render().  means3D (M,P,3) / rotations (M,P,4):
    optional per-frame overrides -- the bob-warped surfels of each frame (DeformableGaussian._override_xyz/_rotation,
    lab4d/nnutils/deformable_gaussian.py:163-176); default = pc.get_xyz / pc.get_rotation shared by all frames.
    target_rgb (M,3,H,W); vis2d / mask_gt / mask_wt (M,H,W) or None; learnable_bkgd (3,) or None.
    target_stream: CUDA stream on which target_rgb (and the masks) are still being produced, e.g. an H2D copy running
    beside the rasterizer forward; it is joined right before the loss kernel (None: the tensors are ready).
    features: optional per-surfel channels, (P,F) shared or (M,P,F) per frame, 1 <= F <= 32, composited with the colour's
    weights (bg_color may then have 3+F values).

    Fused losses on the feature planes (csrc/loss.cu, lab4d/engine/model.py:663-667,742-745,952-967,1000-1012), on when
    feature_target or gauss_mask_channel is given (both need features=):
      feature_target (M,Cf,H,W), Cf <= F: feature_wt * mean over the batch's positive values of
          ||planes[:Cf] - feature_target|| * mask_gt * is_detected[frame]; needs mask_gt.
      gauss_mask_channel c in [Cf, F): reg_gauss_mask_wt * the same positive mean of (planes[c] - alpha.detach())^2.
      is_detected (M,) or None (= all detected); feature_loss_weights: (2,) float32 DEVICE tensor
          [feature_wt, reg_gauss_mask_wt], read by the kernel at run time -- update it in place (e.g. the reference's
          linear ramp of reg_gauss_mask_wt) between replays of a captured step; None = [1e-2, 1e-2].

    Returns {"loss": scalar (sum over frames and terms, differentiable), "terms": (M,4) weighted rgb/mask/normal/dist
    (detached), "render": (M,3,H,W), "allmap": (M,8,H,W), "radii": (M,P), "visibility_filter": (M,P),
    "viewspace_points": (M,P,3) whose .grad receives the densification proxy}; with features also "features": (M,F,H,W),
    differentiable, so that a caller's own losses on the planes backpropagate through the same rasterizer backward; with
    the fused feature losses also "feature_terms": (M,2) each frame's share of the weighted feature / reg_gauss_mask
    terms (detached, included in "loss") and "feature_counts": (M,2) int32, each frame's number of positive values.

    w_ssim > 0 adds, per frame, w_ssim * (1 - SSIM(final colour, target_rgb)) to "loss" (csrc/ssim.cu; gs/train.py's D-SSIM
    term): the final colour includes learnable_bkgd, and SSIM is unmasked.  "ssim_terms": (M,) each frame's share
    (detached).  Stage 3's setting is w_rgb = 1 - lambda_dssim, w_ssim = lambda_dssim.  w_ssim = 0 launches nothing more.

    mask_loss_weight: (1,) float32 DEVICE tensor mask_wt (read at run time, like feature_loss_weights) turns on Stage 3's
    silhouette term as the reference weighs it (csrc/mask_loss.cu, lab4d/engine/model.py:587-611,648-650,950-967,
    1000-1012): mask_wt * mean over the batch's positive values of (alpha - mask_gt)^2 * bw * vis2d * is_detected[frame],
    with the batch's class-balance weights bw of get_mask_balance_wt (or v.mean() if no value is positive).  Needs
    mask_gt; excludes mask_wt and w_mask != 0 (the plain per-frame mask term).  "mask_terms": (M,) each frame's share
    (detached, included in "loss"); "mask_counts": (M,) int32, each frame's number of positive values.  Its gradient is
    added into dL/dalpha after the SSIM term's.  None launches nothing more."""
    if not isinstance(cameras, BatchCameras):
        cameras = stack_cameras(cameras)
    M = len(cameras)
    xyz = pc.get_xyz if means3D is None else means3D
    _check_loss_inputs(M, cameras.image_height, cameras.image_width, xyz.device, target_rgb, vis2d, mask_gt, mask_wt,
                       learnable_bkgd)
    feature_loss = None
    if feature_target is not None or gauss_mask_channel is not None:
        feature_loss = _check_feature_losses(M, cameras.image_height, cameras.image_width, features, feature_target, mask_gt,
                                             is_detected, gauss_mask_channel, feature_loss_weights)
    mask_loss = None
    if mask_loss_weight is not None:
        mask_loss = _check_mask_loss(M, xyz.device, mask_gt, mask_wt, w_mask, is_detected, mask_loss_weight)
    rot = pc.get_rotation if rotations is None else rotations
    P = int(xyz.shape[-2])
    screenspace_points = torch.zeros((M, P, 3), dtype=xyz.dtype, requires_grad=True, device=xyz.device)
    tanx, tany = _cam_tans(cameras)
    cfg = (cameras, bg_color, pc.active_sh_degree, target_rgb, vis2d, mask_gt, mask_wt, float(pipe.depth_ratio),
           w_rgb, w_mask, lambda_normal, lambda_dist, tanx, tany, target_stream, float(w_ssim))
    outs = _RasterLossBatch.apply(xyz, screenspace_points, pc.get_features, pc.get_opacity, pc.get_scaling, rot,
                                  learnable_bkgd, cfg, features, feature_loss, mask_loss)
    total, terms, color, allmap, radii = outs[:5]
    out = {"loss": total, "terms": terms, "render": color, "allmap": allmap, "radii": radii,
           "visibility_filter": radii > 0, "viewspace_points": screenspace_points}
    if features is not None:
        out["features"] = outs[5]
    if feature_loss is not None:
        out["feature_terms"], out["feature_counts"] = outs[6], outs[7]
    k = 5 + (features is not None) + 2 * (feature_loss is not None)
    if w_ssim > 0.0:
        out["ssim_terms"] = outs[k]
        k += 1
    if mask_loss is not None:
        out["mask_terms"], out["mask_counts"] = outs[k], outs[k + 1]
    return out
