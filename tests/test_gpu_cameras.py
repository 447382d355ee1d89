"""GPU tests of per-frame intrinsics (include/surfel_camera.h): the batched rasterizer and the fused loss pass reading each
frame's (tan_fovx, tan_fovy, cx_off, cy_off) from a device table.

Outputs written without atomics (forward planes, radii, num_rendered, the sorted lists and per-surfel records, the loss
pass's dL/dcolour and dL/dallmap) are compared bit for bit; gradients and loss terms, which reduce with float atomics, up
to the order of those reductions (a relative 2e-5 of the tensor's largest element, as tests/test_gpu_batch.py)."""
import numpy as np
import pytest
import torch

from .test_gpu_batch import _cams
from .test_gpu_loss import TOL, _rel

pytestmark = pytest.mark.gpu

NAMES = ("dL_dmeans2D", "dL_dcolors", "dL_dopacity", "dL_dmeans3D", "dL_dtransMat", "dL_dsh", "dL_dscales", "dL_drotations",
         "dL_dfeatures")
RTOL = 2e-5


@pytest.fixture(scope="module")
def dev(built):
    from vidu4d_b200 import _capi
    _capi.load()
    return torch.device("cuda:0")


def _close(a, b, what):
    if a is None or b is None:
        assert a is None and b is None, what
        return
    assert a.shape == b.shape, what
    assert float((a - b).abs().max()) <= RTOL * float(b.abs().max() + 1e-30), what


def _decoded(gb, bb, ib, M, P, W, H, nr):
    from vidu4d_b200 import debug as dbg
    return [dbg.decode(gb.view(M, -1)[f], bb.view(M, -1)[f], ib.view(M, -1)[f], P, W, H, nr[f]) for f in range(M)]


def _same_lists(da, db, radii):
    """The sorted instance lists, contributor counts and the visible surfels' records (an invisible surfel's record is
    not written) of two forwards, frame by frame, bit for bit."""
    for f, (a, b) in enumerate(zip(da, db)):
        for k in ("point_list", "ranges", "n_contrib", "final_T"):
            assert torch.equal(a[k], b[k]), (f, k)
        vis = radii[f] > 0
        P = vis.numel()
        assert torch.equal(a["surfel_rec"].view(P, -1)[vis], b["surfel_rec"].view(P, -1)[vis]), f


def _setup(M, P, W, H, dev, seed, F=0):
    from vidu4d_b200.synthetic import object_scene
    sc = object_scene(P, seed=seed, center=(0.0, 0.0, 0.0))
    t = sc.to_torch(dev)
    g = torch.Generator(device=dev).manual_seed(seed)
    means = torch.stack([t["means3D"] + 0.005 * f * torch.randn((P, 3), device=dev, generator=g) for f in range(M)])
    feats = torch.rand((P, F), device=dev, generator=g) if F else None
    dLc = torch.randn((M, 3 + F, H, W), device=dev, generator=g)
    dLo = 0.1 * torch.randn((M, 8, H, W), device=dev, generator=g)
    return t, means, feats, dLc, dLo


def _run(t, means, feats, cams, W, H, dLc, dLo, tan, intrinsics=None, sum_shared=False):
    from vidu4d_b200 import rasterizer as RZ
    dev = means.device
    vms, pms, cps = cams
    e = torch.empty((0,), device=dev)
    bg = torch.tensor([0.2, 0.1, 0.4], device=dev)
    kw = {} if intrinsics is None else {"intrinsics": intrinsics}
    fk = {} if feats is None else {"features": feats}
    out = RZ._C.rasterize_gaussians_batch(bg, means, e, t["opacities"], t["scales"], t["rotations"], 1.0, vms, pms, tan[0], tan[1],
                                          H, W, t["shs"], 3, cps, **fk, **kw)
    nr, color, allmap, radii, gb, bb, ib = out[:7]
    grads = RZ._C.rasterize_gaussians_backward_batch(bg, means, radii, e, t["scales"], t["rotations"], 1.0, vms, pms, tan[0],
                                                     tan[1], dLc, dLo, t["shs"], 3, cps, gb, bb, ib, sum_shared=sum_shared,
                                                     **fk, **kw)
    return out, dict(zip(NAMES, grads))


# ------------------------------------------------------------------------------------------------ 1. table == scalars
@pytest.mark.parametrize("F", [0, 22])
@pytest.mark.parametrize("M", [1, 2, 8])
def test_table_with_scalar_tangents_equals_scalar_path(M, F, dev):
    P, W, H = 20000, 136, 88
    t, means, feats, dLc, dLo = _setup(M, P, W, H, dev, seed=10 + M, F=F)
    cams = _cams(M, dev)
    tan = (0.5, 0.41)
    table = torch.tensor([[tan[0], tan[1], 0.0, 0.0]] * M, device=dev)
    for sum_shared in (False, True):
        a, ga = _run(t, means, feats, cams, W, H, dLc, dLo, tan, sum_shared=sum_shared)
        b, gb_ = _run(t, means, feats, cams, W, H, dLc, dLo, (float("nan"), float("nan")), table, sum_shared=sum_shared)
        assert a[0] == b[0] and min(a[0]) > 0
        for i in (1, 2, 3):                                            # colour (+ features), allmap, radii
            assert torch.equal(a[i], b[i]), i
        _same_lists(_decoded(*a[4:7], M, P, W, H, a[0]), _decoded(*b[4:7], M, P, W, H, b[0]), a[3])
        for k in NAMES:
            _close(gb_.get(k), ga.get(k), (M, F, sum_shared, k))


def test_render_loss_batch_with_table_equals_scalar_path(dev):
    """render_loss_batch with intrinsics = the cameras' own tangents and zero offsets: the same planes and loss-pass
    gradients bit for bit, the same terms and parameter gradients up to the order of the atomic reductions."""
    from vidu4d_b200.renderer import PipelineParams, _cam_tans, make_camera, render_loss_batch, stack_cameras
    from vidu4d_b200.synthetic import SurfelCloud, object_scene, orbit_view
    M, P, W, H = 2, 8000, 120, 88
    tanx, tany = 0.5, 0.37
    cams = []
    for f in range(M):
        R, tr = orbit_view(5 * f + 2, 64)
        cams.append(make_camera(W, H, 2 * np.arctan(tanx), 2 * np.arctan(tany), R=R.T, T=tr, device=dev))
    tx, ty = _cam_tans(stack_cameras(cams))                        # what the scalar path passes
    table = torch.tensor([[tx, ty, 0.0, 0.0]] * M, device=dev)
    scene = object_scene(P, seed=4, center=(0.0, 0.0, 0.0))
    gen = torch.Generator(device=dev).manual_seed(4)
    target = torch.rand((M, 3, H, W), device=dev, generator=gen)
    mask = (torch.rand((M, H, W), device=dev, generator=gen) > 0.5).float()
    kw = dict(w_rgb=0.8, w_mask=0.1, lambda_normal=0.05, lambda_dist=100.0, mask_gt=mask, mask_wt=torch.ones_like(mask))
    outs, grads = [], []
    for intr in (None, table):
        cloud = SurfelCloud(scene, dev)
        cam = stack_cameras(cams)
        cam.intrinsics = intr
        if intr is not None:
            cam.FoVx = cam.FoVy = None                               # not read with a table
        o = render_loss_batch(cam, cloud, PipelineParams(), torch.zeros(3, device=dev), target, **kw)
        o["loss"].backward()
        outs.append(o)
        grads.append([p.grad.detach().clone() for p in cloud.flat_params()] + [o["viewspace_points"].grad.detach().clone()])
    a, b = outs
    for k in ("render", "allmap", "radii"):
        assert torch.equal(a[k], b[k]), k
    assert _rel(b["terms"].cpu().numpy(), a["terms"].cpu().numpy()) <= RTOL
    for x, y in zip(grads[1], grads[0]):
        _close(x, y, tuple(y.shape))


# ------------------------------------------------------------------------------------------------ 2. per-frame FoV
def test_per_frame_fov_equals_single_frame_calls(dev):
    from vidu4d_b200 import rasterizer as RZ
    M, P, W, H = 3, 20000, 136, 88
    t, means, _, dLc, dLo = _setup(M, P, W, H, dev, seed=31)
    cams = _cams(M, dev)
    vms, pms, cps = cams
    tans = [(0.5, 0.5), (0.42, 0.37), (0.61, 0.55)]
    table = torch.tensor([[a, b, 0.0, 0.0] for a, b in tans], device=dev)
    out, g = _run(t, means, None, cams, W, H, dLc, dLo, (float("nan"), float("nan")), table)
    _, gsum = _run(t, means, None, cams, W, H, dLc, dLo, (float("nan"), float("nan")), table, sum_shared=True)
    e = torch.empty((0,), device=dev)
    bg = torch.tensor([0.2, 0.1, 0.4], device=dev)
    acc = {}
    for f, (tx, ty) in enumerate(tans):
        o = RZ._C.rasterize_gaussians(bg, means[f], e, t["opacities"], t["scales"], t["rotations"], 1.0, e, vms[f], pms[f], tx, ty,
                                      H, W, t["shs"], 3, cps[f], False, False)
        assert o[0] == out[0][f] and o[0] > 0
        assert torch.equal(o[1], out[1][f]) and torch.equal(o[2], out[2][f]) and torch.equal(o[3], out[3][f])
        gs = RZ._C.rasterize_gaussians_backward(bg, means[f], o[3], e, t["scales"], t["rotations"], 1.0, e, vms[f], pms[f], tx,
                                                ty, dLc[f], dLo[f], t["shs"], 3, cps[f], o[4], o[0], o[5], o[6], False)
        for k, a in zip(NAMES, gs):
            _close(g[k][f], a, (f, k))
            acc[k] = acc.get(k, 0) + a
    for k in ("dL_dcolors", "dL_dopacity", "dL_dsh", "dL_dscales", "dL_drotations"):   # inputs the frames share
        assert gsum[k].shape == acc[k].shape, k
        _close(gsum[k], acc[k], k)
    for k in ("dL_dmeans2D", "dL_dmeans3D"):                                           # per frame either way
        _close(gsum[k], g[k], k)


# ------------------------------------------------------------------------------------------------ 3. off-centre vs oracle
def test_off_centre_principal_point_against_oracle(dev):
    """Per-frame tangents and non-integer offsets of either sign, one frame with the object pushed half out of the image:
    the forward planes and every gradient element hold against the CPU oracle under the rounding-error bound of
    tests/test_gpu_grad_bounds.py, with its knife-edge pixels masked.  The oracle takes the offsets as
    tests/camera_model.py derives them from its centred arithmetic."""
    from oracle import surfel_oracle as so
    from vidu4d_b200.synthetic import object_scene
    from . import camera_model as cm
    from .test_gpu_grad_bounds import (CHAIN, GRADS, K, U, _check_all, _check_forward, _check_knife, _fallback_pairs, _np,
                                       _print)
    M, P, W, H = 3, 20000, 136, 88
    sc = object_scene(P, seed=8, center=(0.0, 0.0, 0.0))
    t = sc.to_torch(dev)
    g = torch.Generator(device=dev).manual_seed(77)
    means = torch.stack([t["means3D"] + 0.002 * f * torch.randn((P, 3), device=dev, generator=g) for f in range(M)]).contiguous()
    cams = _cams(M, dev)
    vms, pms, cps = cams
    rows = [(0.5, 0.45, 7.25, -3.5), (0.44, 0.39, -11.75, 5.125), (0.55, 0.5, 60.5, -30.0)]
    table = torch.tensor(rows, device=dev)
    dLc = torch.randn((M, 3, H, W), device=dev, generator=g)
    dLo = 0.1 * torch.randn((M, 8, H, W), device=dev, generator=g)
    out, _ = _run(t, means, None, cams, W, H, dLc, dLo, (float("nan"), float("nan")), table)
    nr, color, allmap, radii, gb, bb, ib = out
    bg = np.array([0.2, 0.1, 0.4], np.float32)
    frames = []
    decs = _decoded(gb, bb, ib, M, P, W, H, nr)
    for f, (tx, ty, ox, oy) in enumerate(rows):
        dec = decs[f]
        dec["radii"] = _np(radii[f])
        dec["num_rendered"] = nr[f]
        rec = _np(dec["surfel_rec"]).reshape(P, 20)
        cl = _np(dec["clamped"]).astype(np.uint8).reshape(P)
        st, ext = so.from_records(_np(means[f]), sc.opacities, sc.scales, sc.rotations, shs=sc.shs, sh_degree=3, W=W, H=H,
                                  tanfovx=tx, tanfovy=ty, bg=bg, viewmatrix=_np(vms[f]), projmatrix=_np(pms[f]),
                                  campos=_np(cps[f]), transMat=rec[:, 0:9], means2D=rec[:, 9:11],
                                  normal_opacity=rec[:, [12, 13, 14, 11]], rgb=rec[:, 15:18], radii=dec["radii"],
                                  clamped=(cl[:, None] >> np.arange(3)) & 1, point_list=_np(dec["point_list"]).view(np.uint32),
                                  ranges=_np(dec["ranges"]).view(np.uint32))
        # the GPU's own records are the oracle's input above: pin them to the oracle's preprocess, moved by the offsets
        full = so.forward(_np(means[f]), sc.opacities, sc.scales, sc.rotations, shs=sc.shs, sh_degree=3, W=W, H=H, tanfovx=tx,
                          tanfovy=ty, bg=bg, viewmatrix=_np(vms[f]), projmatrix=_np(pms[f]), campos=_np(cps[f]))
        T_ref, c_ref = cm.offset_records(full, ox, oy)
        vis = (dec["radii"] > 0) & (full.radii > 0)
        assert vis.sum() > 0.3 * P, f
        tm = rec[vis, 0:9]
        assert np.abs(T_ref[vis] - tm).max() <= 1e-5 * np.abs(tm).max(), f
        assert np.abs(c_ref[vis] - rec[vis, 9:11]).max() <= 1e-3, f
        fwd = _check_forward(f"off-centre frame {f}", st, ext, _np(color[f]), _np(allmap[f]), dec, W, H)
        keep = torch.from_numpy((~ext["knife"]).astype(np.float32)).to(dev)
        dLc[f] *= keep
        dLo[f] *= keep
        og = so.backward(st, _np(dLc[f]), _np(dLo[f]), bounds=True)
        # _bounds of tests/test_gpu_grad_bounds.py, with the offsets' terms in the dT_w slots
        adds = _np(dec["tiles_touched"]).astype(np.float64) + _fallback_pairs(dec, P)
        B = og["bound"] + (adds[:, None] + CHAIN) * og["asum"]
        B = cm.offset_bound_sums(st, B, og["acc"], og["dL_dtransMat"], ox, oy)
        tol = {k: K * U * v for k, v in so.chain_bound(st, B).items()}
        og = dict(og, **cm.offset_chain(st, og["acc"], og["dL_dtransMat"], ox, oy))
        frames.append((st, ext, og, tol, fwd))
    assert float(allmap[2, 1, :, -1].max()) > 0.5                  # frame 2's object is cut by the image's right edge
    _check_knife("off-centre", sum(int(fr[1]["knife"].sum()) for fr in frames))
    _, gr = _run(t, means, None, cams, W, H, dLc, dLo, (float("nan"), float("nan")), table)
    report = {}
    for f, (st, _, og, tol, _) in enumerate(frames):
        _check_all(f"off-centre frame {f}", st, og, tol, {k: gr[k][f] for k in GRADS}, report)
    _print("off-centre", sum(int(fr[1]["knife"].sum()) for fr in frames), max(fr[4] for fr in frames), report)


@pytest.mark.parametrize("W,H", [(75, 53), (130, 97)])
def test_loss_pass_off_centre_against_post_oracle(W, H, dev):
    """sr_render_loss_batch_cameras with per-frame tangents and offsets against the float64 post_oracle with the same
    offsets (tests/camera_model.py), at ragged image sizes; the offsets matter (the centred oracle disagrees)."""
    from oracle import post_oracle as po
    from vidu4d_b200 import _capi
    from . import camera_model as cm
    M, P = 2, 8000
    t, means, _, dLc, dLo = _setup(M, P, W, H, dev, seed=5)
    cams = _cams(M, dev)
    rows = [(0.5, 0.42, 5.5, -2.25), (0.46, 0.4, -9.75, 6.5)]
    table = torch.tensor(rows, device=dev)
    out, _ = _run(t, means, None, cams, W, H, dLc, dLo, (float("nan"), float("nan")), table)
    color, allmap = out[1], out[2]
    wvt = cams[0].contiguous()
    gen = torch.Generator(device=dev).manual_seed(6)
    target = torch.rand((M, 3, H, W), device=dev, generator=gen)
    vis = (torch.rand((M, H, W), device=dev, generator=gen) > 0.1).float()
    mask = (allmap[:, 1] > 0.5).float()
    wt = torch.ones_like(mask)
    w = dict(w_rgb=0.8, w_mask=0.1, lambda_normal=0.05, lambda_dist=100.0)
    terms = torch.empty((M, 4), device=dev)
    dLcol, dLa = torch.empty_like(color), torch.empty_like(allmap)
    scratch = torch.empty((M, H, W), device=dev)
    _capi.call("sr_render_loss_batch_cameras", dev, M, W, H, table, 0.0, color, allmap, wvt, target, vis, mask, wt, None,
               w["w_rgb"], w["w_mask"], w["lambda_normal"], w["lambda_dist"], terms, dLcol, dLa, None, scratch)
    torch.cuda.synchronize()
    for f, (tx, ty, ox, oy) in enumerate(rows):
        args = (color[f].cpu().numpy(), allmap[f].cpu().numpy(), wvt[f].cpu().numpy(), tx, ty, 0.0, target[f].cpu().numpy(),
                vis[f].cpu().numpy(), mask[f].cpu().numpy(), wt[f].cpu().numpy())
        _, ref = cm.stage3_losses(ox, oy, *args, **w)
        for i, k in enumerate(("rgb", "mask", "normal", "dist")):
            assert abs(float(terms[f, i]) - ref[k]) <= TOL * max(abs(ref[k]), 1e-6), (f, k)
        gc, ga = cm.stage3_losses_backward(ox, oy, *args, **w)
        assert _rel(dLcol[f].cpu().numpy(), gc) <= TOL
        assert _rel(dLa[f].cpu().numpy(), ga) <= TOL
        _, gcentred = po.stage3_losses_backward(*args, **w)
        assert _rel(dLa[f].cpu().numpy(), gcentred) > 10 * TOL, f      # the offsets are not ignored


# ------------------------------------------------------------------------------------------------ 4. feature_rows' pi
def test_footprint_centroid_matches_projection(dev):
    """One opaque surfel facing the camera, about 10 px across, under an off-centre per-frame K: the alpha-weighted
    centroid of its footprint (pixel centres at i + 0.5) is pi(K, x) = (Kx)[0:2] / (Kx)[2], the projection
    feature_rows and reproj_loss use, to within 0.05 px in both frames."""
    from vidu4d_b200 import rasterizer as RZ
    from vidu4d_b200.renderer import camera_table
    M, W, H = 2, 96, 80
    K = torch.tensor([[[110.0, 0.0, 41.3], [0.0, 104.0, 43.8], [0.0, 0.0, 1.0]],
                      [[131.0, 0.0, 55.6], [0.0, 127.5, 35.1], [0.0, 0.0, 1.0]]], device=dev)
    x = torch.tensor([[0.04, -0.03, 2.0], [-0.05, 0.02, 2.2]], device=dev)           # camera space, per frame
    vm = torch.eye(4, device=dev).expand(M, 4, 4).contiguous()
    e = torch.empty((0,), device=dev)
    s = 10.0 / 3.0 * x[:, 2] / K[:, 0, 0]                # 10 px across = about 3 sigma on each side at depth z
    out = RZ._C.rasterize_gaussians_batch(torch.zeros(3, device=dev), x[:, None, :].contiguous(),
                                          torch.ones((1, 3), device=dev), torch.ones((1, 1), device=dev),
                                          torch.stack([s, s], 1)[:, None, :].contiguous(),
                                          torch.tensor([[1.0, 0.0, 0.0, 0.0]], device=dev), 1.0, vm, vm, float("nan"),
                                          float("nan"), H, W, e, 0, torch.zeros((M, 3), device=dev),
                                          intrinsics=camera_table(W, H, K))
    alpha = out[2][:, 1].double()
    ys, xs = torch.meshgrid(torch.arange(H, device=dev, dtype=torch.float64) + 0.5,
                            torch.arange(W, device=dev, dtype=torch.float64) + 0.5, indexing="ij")
    kx = torch.einsum("mij,mj->mi", K.double(), x.double())
    for f in range(M):
        a = alpha[f]
        assert float(a.max()) > 0.5 and 40 < int((a > 0.01).sum()) < 600, f
        c = torch.stack([(a * xs).sum() / a.sum(), (a * ys).sum() / a.sum()])
        pi = kx[f, :2] / kx[f, 2]
        assert float((c - pi).abs().max()) <= 0.05, (f, c.tolist(), pi.tolist())


# ------------------------------------------------------------------------------------------------ 5. capture
def test_captured_step_follows_table_refilled_in_place(dev):
    """A captured render_loss_batch forward + backward that reads the table, replayed after the table was refilled in place
    with another pair's intrinsics, equals an eager call with those intrinsics."""
    from vidu4d_b200.graph import GraphedStep
    from vidu4d_b200.renderer import PipelineParams, camera_table, render_loss_batch, stack_cameras, make_camera
    from vidu4d_b200.synthetic import SurfelCloud, object_scene, orbit_view
    M, P, W, H = 2, 8000, 112, 80
    cams = []
    for f in range(M):
        R, tr = orbit_view(4 * f + 3, 64)
        cams.append(make_camera(W, H, 1.0, 0.8, R=R.T, T=tr, device=dev))
    K1 = torch.tensor([[[100.0, 0, 57.5], [0, 98.0, 38.25], [0, 0, 1]], [[120.0, 0, 52.0], [0, 118.0, 41.5], [0, 0, 1]]], device=dev)
    K2 = torch.tensor([[[90.0, 0, 49.75], [0, 93.0, 44.0], [0, 0, 1]], [[140.0, 0, 60.25], [0, 136.0, 36.0], [0, 0, 1]]], device=dev)
    scene = object_scene(P, seed=12, center=(0.0, 0.0, 0.0))
    gen = torch.Generator(device=dev).manual_seed(12)
    target = torch.rand((M, 3, H, W), device=dev, generator=gen)
    kw = dict(w_rgb=0.8, lambda_normal=0.05, lambda_dist=100.0)
    cloud = SurfelCloud(scene, dev)
    bc = stack_cameras(cams)
    bc.intrinsics = camera_table(W, H, K1)
    res = {}

    def body():
        for p in cloud.flat_params():
            p.grad = None
        o = render_loss_batch(bc, cloud, PipelineParams(), torch.zeros(3, device=dev), target, **kw)
        o["loss"].backward()
        res.update(terms=o["terms"], render=o["render"], allmap=o["allmap"], radii=o["radii"],
                   grads=[p.grad for p in cloud.flat_params()])

    from vidu4d_b200 import rasterizer as RZ
    step = GraphedStep(body, device=dev)
    try:
        step()
        bc.intrinsics.copy_(camera_table(W, H, K2))                # in place: the graph reads the same memory
        step()
        got = {k: ([g.clone() for g in v] if k == "grads" else v.clone()) for k, v in res.items()}
    finally:
        # GraphedStep leaves the host in nosync mode (num_rendered = -1); later tests read num_rendered back
        RZ.set_sync_mode(True)
        RZ._pending.clear()
    cloud2 = SurfelCloud(scene, dev)
    bc2 = stack_cameras(cams)
    bc2.intrinsics = camera_table(W, H, K2)
    o = render_loss_batch(bc2, cloud2, PipelineParams(), torch.zeros(3, device=dev), target, **kw)
    o["loss"].backward()
    for k in ("render", "allmap", "radii"):
        assert torch.equal(got[k], o[k]), k
    assert _rel(got["terms"].cpu().numpy(), o["terms"].detach().cpu().numpy()) <= RTOL
    for a, p in zip(got["grads"], cloud2.flat_params()):
        _close(a, p.grad, tuple(p.shape))
    # and the replay did not keep the captured intrinsics
    bc2.intrinsics = camera_table(W, H, K1)
    o1 = render_loss_batch(bc2, SurfelCloud(scene, dev), PipelineParams(), torch.zeros(3, device=dev), target, **kw)
    assert not torch.equal(o1["render"], got["render"])
