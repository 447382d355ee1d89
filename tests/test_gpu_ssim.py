"""GPU: the fused SSIM op (csrc/ssim.cu, vidu4d_b200.ssim.ssim) and render_loss_batch's D-SSIM term.

Bounds.  sigma^2 = E[x^2] - mu^2 cancels: each of the five windowed sums carries ~11 float32 roundings per pass, so
sigma^2 is off by a few eps32 * (E[x^2] + mu^2) and m by |dm/dsigma^2| times that, up to 1/C2 ~ 1e3 times it where the
image is flat.  The reference's own float32 run already strays from its float64 run by exactly this kind of error (the
fixtures store both), so ours must stay within 8x that stray, plus 2e-7 for the float32 rounding of a mean near 1.  The
gradient likewise: within 8x the reference's float32 gradient stray plus 1e-6 of its largest element.
At the large sizes, against the float64 model: the mean within 1e-5 (per-pixel |dm/dsigma^2| ~ 1/(sigma^2 + C2) <= ~20 on
these textured images times ~5e-7 of sigma^2 error), the gradient within 1e-4 of its largest element."""
import glob
import os

import numpy as np
import pytest
import torch

from . import ssim_model as sm
from .conftest import GOLDEN_DIR, load_golden

pytestmark = pytest.mark.gpu
CASES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLDEN_DIR, "ssim_*.npz")))


@pytest.fixture(scope="module")
def dev(built):
    from vidu4d_b200 import _capi
    _capi.load()
    return torch.device("cuda:0")


def _run(x, y, size_average, g, dev):
    from vidu4d_b200.ssim import ssim
    a = torch.from_numpy(np.ascontiguousarray(x)).to(dev).requires_grad_(True)
    b = torch.from_numpy(np.ascontiguousarray(y)).to(dev)
    out = ssim(a, b, size_average=size_average)
    out.backward(torch.as_tensor(g, dtype=torch.float32, device=dev).reshape(out.shape))
    return out.detach().cpu().numpy().astype(np.float64), a.grad.cpu().numpy().astype(np.float64)


@pytest.mark.parametrize("case", CASES)
def test_matches_reference_fixtures(case, dev):
    gd = load_golden(case)
    x, y, gup = gd["in_img1"], gd["in_img2"], gd["in_gup"]
    from vidu4d_b200.ssim import ssim
    with torch.no_grad():
        mean = float(ssim(torch.from_numpy(x).to(dev), torch.from_numpy(y).to(dev)))
    stray = abs(float(gd["ref32_mean"]) - float(gd["ref64_mean"]))
    assert abs(mean - float(gd["ref64_mean"])) <= 8 * stray + 2e-7, (case, mean, float(gd["ref64_mean"]), stray)
    if x.ndim == 4:
        per, grad = _run(x, y, False, gup, dev)
        pstray = np.abs(gd["ref32_per_image"] - gd["ref64_per_image"])
        assert (np.abs(per - gd["ref64_per_image"]) <= 8 * pstray + 2e-7).all(), case
    else:
        _, grad = _run(x, y, True, gup, dev)
    ref = gd["ref64_grad"]
    gstray = np.abs(gd["ref32_grad"] - ref).max()
    err = np.abs(grad - ref).max()
    assert err <= 8 * gstray + 1e-6 * np.abs(ref).max() + 1e-30, (case, err, gstray, np.abs(ref).max())


def test_no_grad_writes_no_maps_and_3d_counts_as_one_image(dev):
    from vidu4d_b200.ssim import ssim
    g = torch.Generator(device=dev).manual_seed(3)
    a, b = torch.rand((3, 20, 30), device=dev, generator=g), torch.rand((3, 20, 30), device=dev, generator=g)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    with torch.no_grad():
        v = ssim(a.requires_grad_(True), b, size_average=False)
    assert v.shape == (1,) and v.grad_fn is None
    assert torch.cuda.max_memory_allocated() - base < 3 * 3 * 20 * 30 * 4       # less than the (3,1,3,20,30) maps
    assert torch.equal(v[0], ssim(a.detach(), b))


@pytest.mark.parametrize("shape", [(8, 3, 512, 512), (1, 3, 1080, 1920)])
def test_large_against_model(shape, dev):
    g = torch.Generator(device=dev).manual_seed(11)
    x = torch.rand(shape, device=dev, generator=g)
    y = (x + 0.2 * torch.randn(shape, device=dev, generator=g)).clamp(0, 1)
    up = torch.randn((shape[0],), device=dev, generator=g)
    per, grad = _run(x.cpu().numpy(), y.cpu().numpy(), False, up.cpu().numpy(), dev)
    xn, yn = x.cpu().numpy(), y.cpu().numpy()
    ref_per = sm.ssim(xn, yn, size_average=False)
    assert np.abs(per - ref_per).max() <= 1e-5
    ref_grad = sm.vjp_mean(xn, yn, up.cpu().numpy().astype(np.float64), size_average=False)
    assert np.abs(grad - ref_grad).max() <= 1e-4 * np.abs(ref_grad).max()


def test_batched_equals_single_and_deterministic(dev):
    g = torch.Generator(device=dev).manual_seed(5)
    x = torch.rand((5, 3, 70, 45), device=dev, generator=g) * 1.3 - 0.1
    y = torch.rand((5, 3, 70, 45), device=dev, generator=g)
    up = torch.randn((5,), device=dev, generator=g)
    per, grad = _run(x.cpu().numpy(), y.cpu().numpy(), False, up.cpu().numpy(), dev)
    per2, grad2 = _run(x.cpu().numpy(), y.cpu().numpy(), False, up.cpu().numpy(), dev)
    assert np.array_equal(per, per2) and np.array_equal(grad, grad2)
    for n in range(5):
        p1, g1 = _run(x[n:n + 1].cpu().numpy(), y[n:n + 1].cpu().numpy(), False, up[n:n + 1].cpu().numpy(), dev)
        assert p1[0] == per[n] and np.array_equal(g1[0], grad[n]), n


def test_more_planes_than_grid_y(dev):
    """N*C > 65 535 tiny planes (the planes are not put on gridDim.y / z)."""
    g = torch.Generator(device=dev).manual_seed(9)
    shape = (70000, 1, 3, 2)
    x, y = torch.rand(shape, device=dev, generator=g), torch.rand(shape, device=dev, generator=g)
    up = torch.randn((shape[0],), device=dev, generator=g)
    per, grad = _run(x.cpu().numpy(), y.cpu().numpy(), False, up.cpu().numpy(), dev)
    xn, yn = x.cpu().numpy(), y.cpu().numpy()
    assert np.abs(per - sm.ssim(xn, yn, size_average=False)).max() <= 1e-5
    ref = sm.vjp_mean(xn, yn, up.cpu().numpy().astype(np.float64), size_average=False)
    assert np.abs(grad - ref).max() <= 1e-4 * np.abs(ref).max()


def test_graph_capture_and_no_sync(dev):
    from vidu4d_b200.ssim import ssim
    g = torch.Generator(device=dev).manual_seed(21)
    shape = (2, 3, 64, 48)
    x = torch.rand(shape, device=dev, generator=g).requires_grad_(True)
    y = torch.rand(shape, device=dev, generator=g)

    def step():
        x.grad = None
        v = ssim(x, y)
        v.backward()
        return v.detach(), x.grad
    torch.cuda.set_sync_debug_mode("error")
    try:
        step()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    s = torch.cuda.Stream(device=dev)
    s.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream(dev).wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    x.grad = None
    with torch.cuda.graph(graph):
        v = ssim(x, y)
        v.backward()
    v_g, grad_g = v, x.grad
    for seed in (1, 2):
        gg = torch.Generator(device=dev).manual_seed(seed)
        with torch.no_grad():
            x.copy_(torch.rand(shape, device=dev, generator=gg))
            y.copy_(torch.rand(shape, device=dev, generator=gg))
        graph.replay()
        torch.cuda.synchronize()
        got_v, got_g = v_g.clone(), grad_g.clone()
        x.grad = None
        ev, eg = step()
        assert torch.equal(got_v, ev) and torch.equal(got_g, eg)
        x.grad = grad_g


def _scene(dev, M=3, P=6000, W=160, H=112):
    from vidu4d_b200.renderer import make_camera, stack_cameras
    from vidu4d_b200.synthetic import object_scene, orbit_view
    tanx, tany = 0.5, 0.35
    cams = []
    for f in range(M):
        R, t = orbit_view(5 * f + 2, 64)
        cams.append(make_camera(W, H, 2 * np.arctan(tanx), 2 * np.arctan(tany), R=R.T, T=t, device=dev))
    scene = object_scene(P, seed=21, center=(0.0, 0.0, 0.0))
    gen = torch.Generator(device=dev).manual_seed(7)
    target = torch.rand((M, 3, H, W), device=dev, generator=gen)
    shift = 0.01 * torch.randn((M, P, 3), device=dev, generator=gen)
    return stack_cameras(cams), scene, target, shift, tanx, tany


def test_render_loss_batch_w_ssim_zero_changes_nothing(dev):
    from vidu4d_b200 import _capi
    from vidu4d_b200.renderer import PipelineParams, render_loss_batch
    from vidu4d_b200.synthetic import SurfelCloud
    bc, scene, target, shift, _, _ = _scene(dev)
    res = []
    for kw in ({}, {"w_ssim": 0.0}):
        cloud = SurfelCloud(scene, dev)
        bkgd = torch.tensor([0.3, 0.5, 0.2], device=dev, requires_grad=True)
        torch.cuda.synchronize()
        n0 = _capi.launch_count()
        out = render_loss_batch(bc, cloud, PipelineParams(), torch.zeros(3, device=dev), target, learnable_bkgd=bkgd,
                                means3D=cloud.get_xyz[None] + shift, w_rgb=0.8, lambda_dist=10.0, **kw)
        (out["loss"] * 1.3).backward()
        torch.cuda.synchronize()
        res.append((_capi.launch_count() - n0, sorted(out), out, [p.grad for p in cloud.flat_params()], bkgd.grad,
                    out["viewspace_points"].grad))
    (l0, k0, o0, g0, b0, v0), (l1, k1, o1, g1, b1, v1) = res
    assert l0 == l1 and k0 == k1 and "ssim_terms" not in k1
    for k in ("render", "allmap", "radii"):
        assert torch.equal(o0[k], o1[k]), k
    # the loss terms and gradients come from float atomics in csrc/loss.cu and the rasterizer backward, so even two calls
    # without the keyword may differ in their last bits; with w_ssim = 0 the same launches run (checked above)
    close = lambda a, b: torch.allclose(a, b, rtol=1e-5, atol=1e-7 * float(b.abs().max()))  # noqa: E731
    for k in ("loss", "terms"):
        assert close(o0[k], o1[k]), k
    assert all(close(a, b) for a, b in zip(g0, g1)) and close(b0, b1) and close(v0, v1)


@pytest.mark.parametrize("with_bkgd", [True, False])
def test_render_loss_batch_ssim_matches_oracle(with_bkgd, dev):
    """render_loss_batch's L1 + D-SSIM step against the float64 oracle (oracle/post_oracle.py) plus the model's SSIM VJP on
    the final colour, pushed through the single-frame rasterizer with a non-unit upstream scalar."""
    from oracle import post_oracle as po
    from vidu4d_b200 import rasterizer as RZ
    from vidu4d_b200.renderer import PipelineParams, render_loss_batch
    from vidu4d_b200.synthetic import SurfelCloud
    TOL, UP, W_SSIM, W_RGB = 1e-4, 1.7, 0.2, 0.8
    bc, scene, target, shift, tanx, tany = _scene(dev)
    M, H, W, P = len(bc), bc.image_height, bc.image_width, scene.means3D.shape[0]
    bg = torch.zeros(3, device=dev)
    cloud = SurfelCloud(scene, dev)
    bkgd = torch.tensor([0.3, 0.5, 0.2], device=dev, requires_grad=True) if with_bkgd else None
    out = render_loss_batch(bc, cloud, PipelineParams(), bg, target, learnable_bkgd=bkgd, means3D=cloud.get_xyz[None] + shift,
                            w_rgb=W_RGB, w_ssim=W_SSIM)
    (out["loss"] * UP).backward()
    got = [p.grad.detach().cpu().numpy() for p in cloud.flat_params()]
    assert out["ssim_terms"].shape == (M,) and not out["ssim_terms"].requires_grad
    total = float(out["terms"].sum() + out["ssim_terms"].sum())
    assert abs(total - float(out["loss"].detach())) <= 1e-5 * abs(total)

    cloud2 = SurfelCloud(scene, dev)
    g_bk = np.zeros(3)
    ones, zeros = np.ones((H, W), np.float32), np.zeros((H, W), np.float32)
    for f in range(M):
        rs = RZ.GaussianRasterizationSettings(H, W, tanx, tany, bg, 1.0, bc.world_view_transform[f], bc.full_proj_transform[f],
                                              cloud2.active_sh_degree, bc.camera_center[f], False, False)
        m2d = torch.zeros((P, 3), device=dev, requires_grad=True)
        color, radii, allmap = RZ.GaussianRasterizer(rs)(means3D=cloud2.get_xyz + shift[f], means2D=m2d, shs=cloud2.get_features,
                                                         opacities=cloud2.get_opacity, scales=cloud2.get_scaling,
                                                         rotations=cloud2.get_rotation)
        c64, a64 = color.detach().cpu().numpy().astype(np.float64), allmap.detach().cpu().numpy().astype(np.float64)
        bk = bkgd.detach().cpu().numpy().astype(np.float64) if with_bkgd else np.zeros(3)
        alpha = a64[1]
        final = c64 + (1.0 - alpha)[None] * bk[:, None, None]
        tg = target[f].cpu().numpy().astype(np.float64)
        s_ref = W_SSIM * (1.0 - sm.ssim(final, tg))
        assert abs(float(out["ssim_terms"][f]) - s_ref) <= TOL * max(abs(s_ref), 1e-6), (f, float(out["ssim_terms"][f]), s_ref)
        args = (color.detach().cpu().numpy(), allmap.detach().cpu().numpy(), bc.world_view_transform[f].cpu().numpy(), tanx, tany,
                0.0, target[f].cpu().numpy(), ones, zeros, zeros)
        okw = dict(w_rgb=W_RGB, w_mask=0.0, lambda_normal=0.0, lambda_dist=0.0, bkgd=bk.astype(np.float32) if with_bkgd else None)
        gr = po.stage3_losses_backward(*args, **okw)
        g_color, g_allmap = np.array(gr[0], np.float64), np.array(gr[1], np.float64)
        g_fc = sm.vjp(final, tg, np.full(final.shape, -W_SSIM / final.size))
        g_color += g_fc
        if with_bkgd:
            g_allmap[1] -= (g_fc * bk[:, None, None]).sum(0)
            g_bk += UP * (np.asarray(gr[2], np.float64) + (g_fc * (1.0 - alpha)[None]).sum((1, 2)))
        torch.autograd.backward([color, allmap], [torch.from_numpy((UP * g_color).astype(np.float32)).to(dev),
                                                  torch.from_numpy((UP * g_allmap).astype(np.float32)).to(dev)])
        ref = m2d.grad.cpu().numpy()
        assert np.abs(out["viewspace_points"].grad[f].cpu().numpy() - ref).max() <= TOL * np.abs(ref).max()
    for a, p in zip(got, cloud2.flat_params()):
        ref = p.grad.cpu().numpy()
        assert np.abs(a - ref).max() <= TOL * np.abs(ref).max(), tuple(p.shape)
    if with_bkgd:
        assert np.abs(bkgd.grad.cpu().numpy() - g_bk).max() <= TOL * np.abs(g_bk).max()
