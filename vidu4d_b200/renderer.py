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
from dataclasses import dataclass, replace
from typing import Optional

import torch

from .rasterizer import GaussianRasterizationSettings, GaussianRasterizer, _check_intrinsics


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
    """M cameras sharing resolution (Stage 3: gs/scene/cameras.py:72-162 builds them per frame).  Without `intrinsics` they
    also share the field of view FoVx / FoVy, with the principal point at the image centre.  intrinsics: optional (M,4)
    float32 CUDA table of each frame's (tan_fovx, tan_fovy, cx_off, cy_off) -- see camera_table() -- that the rasterizer
    and the loss pass read on the device instead: FoVx / FoVy are then not read at all (no host synchronisation), and a
    captured step renders with whatever the table holds at replay."""
    image_width: int
    image_height: int
    FoVx: float
    FoVy: float
    world_view_transform: torch.Tensor   # (M,4,4), each W2C transposed
    full_proj_transform: torch.Tensor    # (M,4,4)
    camera_center: torch.Tensor          # (M,3)
    intrinsics: Optional[torch.Tensor] = None   # (M,4) per-frame camera table, or None

    def __len__(self):
        return int(self.world_view_transform.shape[0])


def camera_table(width, height, K) -> torch.Tensor:
    """The (M,4) per-frame camera table (tan_fovx, tan_fovy, cx_off, cy_off) of BatchCameras.intrinsics from pinhole
    intrinsics K (M,3,3), the same K feature_rows and reproj_loss project with:
        tan_fovx = W / (2 K[:,0,0]),  tan_fovy = H / (2 K[:,1,1]),  cx_off = K[:,0,2] - W/2,  cy_off = K[:,1,2] - H/2.
    float32 torch ops on K's device, with no host synchronisation, so it can sit inside a captured step; K gets no
    gradient through it (nothing differentiates the rasterizer with respect to its camera).  The reference's KCamera
    derives its FoV from the focal length with arctan and the rasterizer takes tan of half of it again, so its tangent may
    differ from this one in the last bit."""
    if K.ndim != 3 or tuple(K.shape[1:]) != (3, 3):
        raise RuntimeError(f"K must be (M,3,3), got {tuple(K.shape)}")
    K = K.detach().to(torch.float32)
    W, H = float(width), float(height)
    fx, fy = K[:, 0, 0], K[:, 1, 1]
    # tensor / tensor: a Python number over a tensor would multiply by the reciprocal, which is not the IEEE quotient
    tan_x = torch.full_like(fx, W) / (2.0 * fx)
    tan_y = torch.full_like(fy, H) / (2.0 * fy)
    return torch.stack((tan_x, tan_y, K[:, 0, 2] - 0.5 * W, K[:, 1, 2] - 0.5 * H), dim=1).contiguous()


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
        if cams.intrinsics is not None:
            kw["intrinsics"] = cams.intrinsics
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
        if cams.intrinsics is None:
            _capi.call("sr_render_loss_batch", dev, M, W, H, tanx, tany, float(depth_ratio), color, allmap, wvt, target, vis,
                       mask, mask_wt, bk, float(w_rgb), float(w_mask), float(lam_n), float(lam_d), terms, dLc, dLa, dLb, scratch)
        else:
            _capi.call("sr_render_loss_batch_cameras", dev, M, W, H, cams.intrinsics, float(depth_ratio), color, allmap, wvt,
                       target, vis, mask, mask_wt, bk, float(w_rgb), float(w_mask), float(lam_n), float(lam_d), terms, dLc, dLa,
                       dLb, scratch)
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
        if cams.intrinsics is not None:
            kw["intrinsics"] = cams.intrinsics
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

    cameras: BatchCameras (or a list of cameras, stacked here); with cameras.intrinsics every frame is rendered, and its
    normals are derived, with its own focal length and principal point.  pc: as in render().  means3D (M,P,3) / rotations (M,P,4):
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
    if cameras.intrinsics is not None:
        cameras = replace(cameras, intrinsics=_check_intrinsics(cameras.intrinsics, M, xyz))
        tanx = tany = None                  # not read: the table replaces them
    else:
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


# ---------------------------------------------------------------------------------------------
# Forward-only rendering of a trained sequence: what lab4d/engine/model.py:186-284 (evaluate) renders frame pair by
# frame pair under torch.no_grad(), in chunks of frames with no backward state (include/surfel_render.h).
# ---------------------------------------------------------------------------------------------
@dataclass
class SurfelContributions:
    """What every surfel contributes to a set of rendered frames, added into by render_frames(contributions=...).

    A pair (frame, pixel, surfel) contributes when the composite blends it; its weight is w = T * alpha, rounded once to
    float32 (the feature plane of a feature equal to 1), and its quantised weight q(w) = round-half-even(w * 2^32).  Per
    surfel, over every contributing pair (include/surfel_render.h, sr_contrib):
      weight_q   (P,) int64: the sum of q(w), an unsigned 64-bit word (it stays below 2^63)
      max_weight (P,) int32: the largest w, as its float32 bits (max_weight.view(torch.float32) is the value)
      pixels     (P,) int64: the number of contributing (frame, pixel) pairs
      frames     (P,) int64: the number of rendered frames with radii > 0 (those whose preprocess kept the surfel)
    With silhouettes (zeros(..., silhouettes=True); render_frames(..., masks=) fills them, include/surfel_render.h,
    sr_contrib_mask), over the contributing pairs on the frames' background pixels:
      weight_bg_q (P,) int64: the sum of q(w)
      pixels_bg   (P,) int64: the number of those pairs
    Without them both are None.  Every entry is an integer sum or maximum, so the totals have the same bits for any order
    of the frames, any chunking and, after distributed.allreduce_contributions, any split over ranks.  torch's
    collectives take no unsigned 64-bit type: the words live in int64 and int32 tensors."""
    weight_q: torch.Tensor
    max_weight: torch.Tensor
    pixels: torch.Tensor
    frames: torch.Tensor
    weight_bg_q: Optional[torch.Tensor] = None
    pixels_bg: Optional[torch.Tensor] = None

    @classmethod
    def zeros(cls, P: int, device, silhouettes: bool = False) -> "SurfelContributions":
        z = lambda dt: torch.zeros((int(P),), dtype=dt, device=device)  # noqa: E731
        bg = (z(torch.int64), z(torch.int64)) if silhouettes else (None, None)
        return cls(z(torch.int64), z(torch.int32), z(torch.int64), z(torch.int64), *bg)

    @property
    def silhouettes(self) -> bool:
        """True when the background words are present."""
        return self.weight_bg_q is not None or self.pixels_bg is not None

    @property
    def P(self) -> int:
        return int(self.weight_q.shape[0])

    @property
    def weight(self) -> torch.Tensor:
        """(P,) float64: each surfel's summed weight, weight_q / 2^32."""
        return self.weight_q.to(torch.float64) / 4294967296.0

    @property
    def background_fraction(self) -> torch.Tensor:
        """(P,) float64: the share of each surfel's summed weight that fell on background pixels, weight_bg_q / weight_q
        (each word converted to float64, then divided); 0 where weight_q == 0.  Needs the background words."""
        if self.weight_bg_q is None:
            raise RuntimeError("background_fraction needs the background words: SurfelContributions.zeros(P, device, "
                               "silhouettes=True), filled by render_frames(..., masks=)")
        wq = self.weight_q.to(torch.float64)
        return torch.where(wq > 0, self.weight_bg_q.to(torch.float64) / wq.clamp_min(1.0), torch.zeros_like(wq))

    def prune_mask(self, min_weight: float = 0.0, min_pixels: int = 1,
                   max_background_fraction: Optional[float] = None) -> torch.Tensor:
        """(P,) bool: the surfels with weight < min_weight or pixels < min_pixels and, when max_background_fraction f is
        given (it needs the background words), those whose background_fraction is above f."""
        mask = (self.weight < float(min_weight)) | (self.pixels < int(min_pixels))
        if max_background_fraction is not None:
            f = max_background_fraction
            if isinstance(f, bool) or not isinstance(f, (int, float)) or not 0.0 <= float(f) <= 1.0:
                raise RuntimeError(f"max_background_fraction must be a number in [0, 1] or None, got {f!r}")
            mask |= self.background_fraction > float(f)
        return mask

    def check(self, P: int, device) -> None:
        """Raise RuntimeError unless the four tensors, and the two background words when present (both or neither), are
        contiguous (P,) tensors of their dtypes on `device`."""
        if (self.weight_bg_q is None) != (self.pixels_bg is None):
            raise RuntimeError("contributions.weight_bg_q and contributions.pixels_bg must both be tensors or both None")
        names = [("weight_q", torch.int64), ("max_weight", torch.int32), ("pixels", torch.int64), ("frames", torch.int64)]
        if self.silhouettes:
            names += [("weight_bg_q", torch.int64), ("pixels_bg", torch.int64)]
        for name, dt in names:
            t = getattr(self, name)
            if not torch.is_tensor(t) or t.dtype != dt or tuple(t.shape) != (P,) or not t.is_contiguous():
                raise RuntimeError(f"contributions.{name} must be a contiguous {dt} (P,) = ({P},) tensor, got "
                                   f"{tuple(t.shape) if torch.is_tensor(t) else type(t).__name__}"
                                   f"{' ' + str(t.dtype) if torch.is_tensor(t) else ''}")
            if t.device != torch.device(device):
                raise RuntimeError(f"contributions.{name} must be on the rasterizer's device {device}, got {t.device}")


@dataclass
class SurfelLift:
    """Per-pixel maps lifted onto the surfels, added into by render_frames(..., contributions=, lift=, values=): for each
    surfel i and channel c, over the contributing pairs (frame, pixel, surfel i) of the rendered frames,

      sums[i, c] += q,   q = round-half-even(fl(w * v) * 2^scale_log2),

    w the pair's weight (SurfelContributions' w = T * alpha) and v the pixel's value of channel c (include/surfel_render.h,
    sr_lift).  sums is (P,C) int64, an exact two's-complement sum: the same bits for any order of the frames, any chunking
    and, after distributed.allreduce_lift, any split over ranks.  saturated (1,) int64 counts the (pair, channel) terms
    that were not exact: a non-finite value contributes 0, and |fl(w * v) * 2^s| > 2^32 contributes +-2^32.

    scale_log2 s is fixed when the accumulator is made, from a bound B on |v|: s = 32 - ceil(log2 B), so that |q| <= 2^32
    for every |v| <= B and a sum cannot overflow below 2^31 pairs.  It is never chosen from the data: sums made with
    different scales do not add.  With v = 1 and B = 1, q is SurfelContributions' q(w), so sums[:, c] == weight_q."""
    sums: torch.Tensor
    saturated: torch.Tensor
    scale_log2: int

    @staticmethod
    def scale_for(value_bound: float) -> int:
        """s = 32 - ceil(log2 B), exactly (no floating-point logarithm); B must be in (2^-33, 2^96]."""
        from . import _capi
        B = value_bound
        if isinstance(B, bool) or not isinstance(B, (int, float)) or not math.isfinite(float(B)) or float(B) <= 0.0:
            raise RuntimeError(f"value_bound must be a finite positive number, got {B!r}")
        m, e = math.frexp(float(B))                  # B = m 2^e, 0.5 <= m < 1
        s = 32 - (e - 1 if m == 0.5 else e)
        if not _capi.LIFT_SCALE_MIN <= s <= _capi.LIFT_SCALE_MAX:
            raise RuntimeError(f"value_bound {B!r} gives scale_log2 {s}, outside [{_capi.LIFT_SCALE_MIN}, "
                               f"{_capi.LIFT_SCALE_MAX}]: value_bound must be in (2^-33, 2^96]")
        return s

    @classmethod
    def zeros(cls, P: int, C: int, device, value_bound: float = 1.0) -> "SurfelLift":
        """An empty accumulator of C channels (1 <= C <= 32) for P surfels, for values with |v| <= value_bound."""
        if isinstance(C, bool) or not isinstance(C, int) or not 1 <= C <= 32:
            raise RuntimeError(f"C must be an int in [1, 32], got {C!r}")
        return cls(torch.zeros((int(P), C), dtype=torch.int64, device=device),
                   torch.zeros((1,), dtype=torch.int64, device=device), cls.scale_for(value_bound))

    @property
    def P(self) -> int:
        return int(self.sums.shape[0])

    @property
    def C(self) -> int:
        return int(self.sums.shape[1])

    def mean(self, contrib: "SurfelContributions") -> torch.Tensor:
        """(P,C) float64: each surfel's weighted mean of the lifted values, (sums 2^-s) / (weight_q 2^-32), each word
        converted to float64 first; 0 where weight_q == 0.  contrib: the SurfelContributions the same render_frames calls
        filled (on several ranks, both all-reduced)."""
        if contrib.P != self.P:
            raise RuntimeError(f"contributions are for {contrib.P} surfels, the lift for {self.P}")
        wq = contrib.weight_q.to(self.sums.device, torch.float64)[:, None] * 2.0 ** -32
        v = self.sums.to(torch.float64) * 2.0 ** -self.scale_log2
        return torch.where(wq > 0, v / torch.where(wq > 0, wq, torch.ones_like(wq)), torch.zeros_like(v))

    def check(self, P: int, device) -> None:
        """Raise RuntimeError unless sums is a contiguous (P,C) int64 tensor with 1 <= C <= 32, saturated a (1,) int64
        tensor, both on `device`, and scale_log2 an int in the library's range."""
        from . import _capi
        t = self.sums
        if not torch.is_tensor(t) or t.dtype != torch.int64 or t.ndim != 2 or int(t.shape[0]) != P \
                or not 1 <= int(t.shape[1]) <= 32 or not t.is_contiguous():
            raise RuntimeError(f"lift.sums must be a contiguous torch.int64 (P,C) tensor with P = {P} and 1 <= C <= 32, "
                               f"got {tuple(t.shape) if torch.is_tensor(t) else type(t).__name__}"
                               f"{' ' + str(t.dtype) if torch.is_tensor(t) else ''}")
        u = self.saturated
        if not torch.is_tensor(u) or u.dtype != torch.int64 or tuple(u.shape) != (1,):
            raise RuntimeError("lift.saturated must be a (1,) torch.int64 tensor")
        for name, x in (("sums", t), ("saturated", u)):
            if x.device != torch.device(device):
                raise RuntimeError(f"lift.{name} must be on the rasterizer's device {device}, got {x.device}")
        s = self.scale_log2
        if isinstance(s, bool) or not isinstance(s, int) or not _capi.LIFT_SCALE_MIN <= s <= _capi.LIFT_SCALE_MAX:
            raise RuntimeError(f"lift.scale_log2 must be an int in [{_capi.LIFT_SCALE_MIN}, {_capi.LIFT_SCALE_MAX}], "
                               f"got {s!r}")


def _lift_values(values, T, C, H, W, device):
    """render_frames' values, checked: a contiguous (T,C,H,W) float32 tensor on `device`.  Nothing is converted or
    copied here; a channels-last (T,H,W,C) map passes as maps.permute(0, 3, 1, 2).contiguous(), one explicit copy."""
    if not torch.is_tensor(values):
        raise RuntimeError(f"values must be a tensor, got {type(values).__name__}")
    if tuple(values.shape) != (T, C, H, W):
        raise RuntimeError(f"values must be (T,C,H,W) = ({T},{C},{H},{W}), got {tuple(values.shape)}")
    if values.dtype != torch.float32:
        raise RuntimeError(f"values must be float32, got {values.dtype}")
    if values.device != torch.device(device):
        raise RuntimeError(f"values must be on the rasterizer's device {device}, got {values.device}")
    if not values.is_contiguous():
        raise RuntimeError("values must be contiguous; a channels-last (T,H,W,C) map passes as "
                           "maps.permute(0, 3, 1, 2).contiguous()")
    return values.detach()


def _check_render_frames(T, P, device, bg_color, means3D, rotations, features, learnable_bkgd, frames_per_call):
    """Validate render_frames' arguments before anything runs on the device; returns F."""
    if isinstance(frames_per_call, bool) or not isinstance(frames_per_call, int) or frames_per_call < 1:
        raise RuntimeError(f"frames_per_call must be an int >= 1, got {frames_per_call!r}")
    for name, t, tail in (("means3D", means3D, 3), ("rotations", rotations, 4)):
        if t is not None and (t.ndim != 3 or tuple(t.shape) != (T, P, tail)):
            raise RuntimeError(f"{name} must be (T,P,{tail}) = ({T},{P},{tail}) or None, got {tuple(t.shape)}")
    F = 0
    if features is not None:
        from .rasterizer import _check_features
        if torch.is_tensor(features) and features.ndim == 3 and int(features.shape[0]) != T:
            raise RuntimeError(f"features must be (P,F) or (T,P,F) with T = {T}, got {tuple(features.shape)}")
        F = _check_features(features, P, bg_color, batched=True)
    elif int(bg_color.numel()) != 3:
        raise RuntimeError(f"bg_color must have 3 values without features, got {int(bg_color.numel())}")
    if learnable_bkgd is not None:
        if learnable_bkgd.numel() != 3:
            raise RuntimeError(f"learnable_bkgd must have 3 elements, got shape {tuple(learnable_bkgd.shape)}")
        if not learnable_bkgd.is_cuda or learnable_bkgd.device != device:
            raise RuntimeError(f"learnable_bkgd must be a CUDA tensor on the rasterizer's device {device}, got {learnable_bkgd.device}")
    return F


def _silhouette_masks(masks, T, H, W, device):
    """render_frames' masks as one contiguous (T,H,W) uint8 tensor on `device`, nonzero = foreground: bool and uint8
    pass as they are (bool is viewed as bytes), a floating mask is foreground where > 0.5, converted once here."""
    if not torch.is_tensor(masks):
        raise RuntimeError(f"masks must be a tensor, got {type(masks).__name__}")
    if tuple(masks.shape) not in ((T, H, W), (T, 1, H, W)):
        raise RuntimeError(f"masks must be (T,H,W) or (T,1,H,W) = ({T},{H},{W}), got {tuple(masks.shape)}")
    if masks.device != torch.device(device):
        raise RuntimeError(f"masks must be on the rasterizer's device {device}, got {masks.device}")
    m = masks.detach().reshape(T, H, W)
    if m.dtype == torch.bool:
        return m.contiguous().view(torch.uint8)
    if m.dtype == torch.uint8:
        return m.contiguous()
    if m.is_floating_point():
        return (m > 0.5).view(torch.uint8)
    raise RuntimeError(f"masks must be bool, uint8 or floating point, got {m.dtype}")


def render_frames(cameras, pc, pipe, bg_color, means3D=None, rotations=None, features=None, learnable_bkgd=None,
                  frames_per_call=8, contributions=None, masks=None, lift=None, values=None, anchors=None):
    """Render T frames forward-only: render_fused()'s outputs for every frame, with a leading frame dimension, and nothing
    differentiable -- no autograd graph is built, even when the inputs require grad.

    cameras: BatchCameras of T frames (or a list of cameras, stacked here), with or without `intrinsics`.  pc, pipe: as in
    render().  means3D (T,P,3) / rotations (T,P,4): optional per-frame surfels (the bob-warped copies, as in
    render_loss_batch); default pc.get_xyz / pc.get_rotation for every frame.  features: optional (P,F) or (T,P,F),
    1 <= F <= 32, composited with the colour's weights (bg_color may then have 3+F values).  learnable_bkgd: optional (3,):
    "render" becomes render + (1 - acc) * learnable_bkgd, as DeformableGaussian.render_view adds it
    (deformable_gaussian.py:188-190).

    The frames are rendered frames_per_call at a time (csrc/composite_fwd.cu's forward-only walk, which keeps no backward
    state and composites the feature channels in the colour's walk; then csrc/postprocess.cu over the chunk) straight into
    the (T,...) outputs.  One arena, sized for the largest chunk, serves every chunk; each chunk reads its instance counts
    back once and re-runs with a larger capacity if it overflowed.  Colour, features, allmap-derived maps and radii are
    bit-identical to the training forward's (_C.rasterize_gaussians_batch) followed by sr_post_forward per frame.

    contributions: optional SurfelContributions of P surfels on the surfels' device (SurfelContributions.zeros(P, device)),
    added into in place with every rendered frame's per-surfel statistics, gathered in the same walk
    (sr_render_forward_contrib).  A sequence rendered in several calls, in any order and with any frames_per_call, adds
    the same bits as one call; a chunk that overflows re-runs only its overflowed frames, so no frame adds twice.  The
    rendered outputs are the same with and without it.

    masks: optional foreground masks, (T,H,W) or (T,1,H,W), on the surfels' device: bool or uint8 (nonzero =
    foreground) or floating point (foreground where > 0.5).  With them `contributions` must have the background words
    (SurfelContributions.zeros(P, device, silhouettes=True)), and each surfel's contributing pairs on background pixels
    are added into weight_bg_q and pixels_bg in the same walk (sr_render_forward_contrib_masked).  The rendered outputs
    and the other statistics have the same bits as without masks.  A pixel the frame cannot judge -- outside vis2d --
    should not count as background: pass masks = mask | ~vis2d.

    lift, values: optional SurfelLift of P surfels and C channels (SurfelLift.zeros(P, C, device, value_bound)) and the
    per-pixel maps to lift, a contiguous (T,C,H,W) float32 tensor on the surfels' device (a channels-last (T,H,W,C) map
    passes as maps.permute(0, 3, 1, 2).contiguous(), one explicit copy).  Each surfel's weighted sums of the values at
    its contributing pairs are added into lift.sums in the same walk (sr_render_forward_lift), with the same frame
    bookkeeping as `contributions`, which a lift needs.  A lift renders colour only (no features) and takes no masks: a
    background indicator channel, 1 on background pixels, lifted with value_bound 1, gives weight_bg_q.  The rendered
    outputs and the statistics have the same bits as without a lift.

    anchors: optional slot count K in {1, 2, 4, 8}.  Each pixel's K heaviest contributing pairs are kept in the same walk
    (sr_render_forward_anchors) and returned as "anchor_ids" (T,K,H,W) int32 (the surfel, -1 for an empty slot),
    "anchor_weights" (T,K,H,W) (the pair's w, SurfelContributions' weight; 0 for an empty slot), sorted descending with
    the front-most pair first among equal weights, and "anchor_uv" (T,K,2,H,W) (where the pixel's ray hits the disc, in
    its scaled tangent frame: the point mean + u*s_u*t_u + v*s_v*t_v; (0, 0), the centre, on the screen-space filter
    branch and in an empty slot).  tracking.track_pixels follows these pixels through the sequence.  Anchors render
    colour only and combine with none of features, contributions, masks or lift.  Every other output has the same bits
    as without anchors.  They take 16 B per slot and pixel: K = 4 at 512 x 512 is 16.8 MB per frame.

    Returns {"render": (T,3,H,W), "features": (T,F,H,W) (with features), "acc": (T,1,H,W), "rend_normal": (T,3,H,W),
    "rend_dist": (T,1,H,W), "surf_depth", "render_depth_median", "render_depth_expected": (T,3,H,W) broadcast views of one
    plane each, "surf_normal": (T,3,H,W), "radii": (T,P) int32, "visibility_filter": (T,P) bool}."""
    from . import _capi
    from .rasterizer import _RenderOut, _batch_inputs, _check_intrinsics, _f32c, _forward
    if not isinstance(cameras, BatchCameras):
        cameras = stack_cameras(cameras)
    T, H, W = len(cameras), int(cameras.image_height), int(cameras.image_width)
    xyz = pc.get_xyz if means3D is None else means3D
    P, dev = int(xyz.shape[-2]), xyz.device
    if lift is not None and features is not None:
        raise RuntimeError("lift renders colour only: features must be None")
    if anchors is not None:
        if isinstance(anchors, bool) or not isinstance(anchors, int) or anchors not in _capi.ANCHOR_SLOTS:
            raise RuntimeError(f"anchors must be a slot count in {_capi.ANCHOR_SLOTS}, got {anchors!r}")
        for name, arg in (("features", features), ("contributions", contributions), ("masks", masks), ("lift", lift)):
            if arg is not None:
                raise RuntimeError(f"anchors render colour only and gather no statistics: {name} must be None")
    F = _check_render_frames(T, P, dev, bg_color, means3D, rotations, features, learnable_bkgd, frames_per_call)
    if contributions is not None:
        if not isinstance(contributions, SurfelContributions):
            raise RuntimeError(f"contributions must be a SurfelContributions, got {type(contributions).__name__}")
        contributions.check(P, dev)
        if contributions.silhouettes and masks is None:
            raise RuntimeError("contributions has the background words (weight_bg_q, pixels_bg) but no masks were given")
    if masks is not None:
        if contributions is None or not contributions.silhouettes:
            raise RuntimeError("masks need contributions with the background words: "
                               "SurfelContributions.zeros(P, device, silhouettes=True)")
        masks = _silhouette_masks(masks, T, H, W, dev)
    if lift is not None:
        if not isinstance(lift, SurfelLift):
            raise RuntimeError(f"lift must be a SurfelLift, got {type(lift).__name__}")
        if contributions is None:
            raise RuntimeError("lift needs contributions: SurfelContributions.zeros(P, device)")
        if masks is not None:
            raise RuntimeError("lift and masks cannot be combined in one call: lift a background indicator channel instead")
        lift.check(P, dev)
        if values is None:
            raise RuntimeError("lift needs values: the (T,C,H,W) maps to lift")
        values = _lift_values(values, T, lift.C, H, W, dev)
    elif values is not None:
        raise RuntimeError("values are lifted into a SurfelLift: pass lift=SurfelLift.zeros(P, C, device)")
    intr = _check_intrinsics(cameras.intrinsics, T, xyz)
    tanx, tany = (0.0, 0.0) if intr is not None else _cam_tans(cameras)     # the table replaces them
    N = H * W
    with torch.no_grad(), torch.cuda.device(dev):
        rot = pc.get_rotation if rotations is None else rotations
        ins, strides = _batch_inputs(T, means3D=(xyz.detach(), (3,)), sh=(pc.get_features.detach(), None),
                                     opacity=(pc.get_opacity.detach(), (1,)), scales=(pc.get_scaling.detach(), (2,)),
                                     rotations=(rot.detach(), (4,)),
                                     features=(None if features is None else features.detach(), None))
        bg = _f32c(bg_color.detach(), "bg_color")
        vm = _f32c(cameras.world_view_transform.detach(), "world_view_transform")
        pm = _f32c(cameras.full_proj_transform.detach(), "full_proj_transform")
        cp = _f32c(cameras.camera_center.detach(), "camera_center")
        bk = None if learnable_bkgd is None else _f32c(learnable_bkgd.detach().reshape(3), "learnable_bkgd")
        mk = lambda *shape, dtype=torch.float32: torch.empty((T,) + shape, dtype=dtype, device=dev)  # noqa: E731
        color, feat = mk(3, H, W), (mk(F, H, W) if F else None)
        acc, rn, dist, med, ex, sd, sn = mk(1, H, W), mk(3, H, W), mk(1, H, W), mk(1, H, W), mk(1, H, W), mk(1, H, W), mk(3, H, W)
        radii = mk(P, dtype=torch.int32)
        n = min(frames_per_call, T)
        allmap = torch.empty((n, 8, H, W), dtype=torch.float32, device=dev)     # one chunk's, reused
        out = _RenderOut(None, None, None, None)
        if contributions is not None:
            out.contrib = _capi.SrContrib(contributions.weight_q.data_ptr(), contributions.max_weight.data_ptr(),
                                          contributions.pixels.data_ptr())
        if masks is not None:
            out.mask = _capi.SrContribMask(None, N, contributions.weight_bg_q.data_ptr(), contributions.pixels_bg.data_ptr())
        if anchors is not None:
            K = anchors
            a_ids = torch.empty((T, K, H, W), dtype=torch.int32, device=dev)
            a_w, a_uv = mk(K, H, W), mk(K, 2, H, W)
            out.anchors = _capi.SrAnchors(K, K * N, None, None, None)
        if lift is not None:
            out.lift = _capi.SrLift(None, lift.C, lift.C * N, lift.scale_log2, lift.sums.data_ptr(),
                                    lift.saturated.data_ptr())

        def forward(a, b, t0):
            """frames [a, b) of the chunk that starts at t0"""
            c = slice(a, b)
            # per-frame inputs are sliced (their strides stay); shared ones pass whole
            sl = {k: (v[c] if v is not None and strides.get(k, 0) else v) for k, v in ins.items()}
            out.color, out.features, out.others, out.radii = color[c], (feat[c] if F else None), allmap[a - t0:b - t0], radii[c]
            if out.mask is not None:
                out.mask.mask = masks[a].data_ptr()                 # this call's frames: a, a + 1, ... (stride H*W)
            if out.lift is not None:
                out.lift.values = values[a].data_ptr()              # (stride C*H*W)
            if out.anchors is not None:                             # (stride K*H*W; uv 2*K*H*W)
                out.anchors.ids, out.anchors.weights, out.anchors.uv = (a_ids[a].data_ptr(), a_w[a].data_ptr(),
                                                                        a_uv[a].data_ptr())
            # P = 0: the empty tensors give the device and F (their pointers pass as NULL)
            xyz_c = sl["means3D"] if sl["means3D"] is not None else xyz
            feat_c = sl["features"] if sl["features"] is not None else features
            _forward(b - a, True, strides, bg, xyz_c, sl["sh"], None, sl["opacity"], sl["scales"], sl["rotations"],
                     feat_c, vm[c], pm[c], cp[c], H, W, pc.active_sh_degree, tanx, tany, 1.0, False, False,
                     intrinsics=None if intr is None else intr[c], render=out)

        for t0 in range(0, T, n):
            t1 = min(T, t0 + n)
            c = slice(t0, t1)
            out.overflowed = []
            forward(t0, t1, t0)
            # with contributions an overflowed chunk is not re-run whole: its frames that fit have added already
            for m in list(out.overflowed):
                forward(t0 + m, t0 + m + 1, t0)
            if contributions is not None:
                contributions.frames += (radii[c] > 0).sum(0)
            # the whole chunk's allmap: after a one-frame re-run out.others is that frame's slice alone
            _capi.call("sr_post_forward_frames", dev, t1 - t0, W, H, tanx, tany, None if intr is None else intr[c],
                       float(pipe.depth_ratio), allmap[:t1 - t0], vm[c], bk, color[c], 3 * N, acc[c], rn[c], dist[c], med[c], ex[c],
                       sd[c], sn[c])
        del out, allmap, masks, values
        rets = {"render": color, "acc": acc, "rend_normal": rn, "rend_dist": dist, "surf_depth": sd.expand(T, 3, H, W),
                "render_depth_median": med.expand(T, 3, H, W), "render_depth_expected": ex.expand(T, 3, H, W),
                "surf_normal": sn, "radii": radii, "visibility_filter": radii > 0}
        if F:
            rets["features"] = feat
        if anchors is not None:
            rets["anchor_ids"], rets["anchor_weights"], rets["anchor_uv"] = a_ids, a_w, a_uv
    return rets
