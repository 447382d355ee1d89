"""GPU tests of per-surfel feature channels (sr_forward / sr_backward with F >= 1): F channels composited
with the colour's weights next to the colour.  The colour path must not change at all; a feature plane must be bit for bit
what the colour path renders for the same values; the backward is pinned by linearity against colour-only renders."""
import numpy as np
import pytest
import torch

from .conftest import load_golden

pytestmark = pytest.mark.gpu

NAMES = ("dL_dmeans2D", "dL_dcolors", "dL_dopacity", "dL_dmeans3D", "dL_dtransMat", "dL_dsh", "dL_dscales", "dL_drotations")
GEOM = ("dL_dmeans2D", "dL_dopacity", "dL_dmeans3D", "dL_dscales", "dL_drotations")


@pytest.fixture(scope="module")
def dev(built):
    from vidu4d_b200 import _capi
    _capi.load()
    return torch.device("cuda:0")


def _golden_scene(name, dev):
    g = load_golden(name)
    P, W, H, deg, pre = [int(v) for v in g["in_meta"]]
    t = lambda k: torch.from_numpy(np.ascontiguousarray(g[k], dtype=np.float32)).to(dev)  # noqa: E731
    e = torch.empty((0,), device=dev)
    return dict(P=P, W=W, H=H, deg=deg, means3D=t("in_means3D"), opacities=t("in_opacities").reshape(P, 1),
                scales=t("in_scales"), rotations=t("in_rotations"), shs=e if pre else t("in_shs").reshape(P, -1, 3),
                colors=t("in_colors_precomp").reshape(P, 3) if pre else e, bg=t("in_bg").reshape(3),
                vm=t("in_viewmatrix").reshape(4, 4), pm=t("in_projmatrix").reshape(4, 4), campos=t("in_campos").reshape(3),
                tanx=float(g["in_tanfov"][0]), tany=float(g["in_tanfov"][1]))


def _c2_scene(dev):
    """C2: 100 K surfels, 512^2, one camera in front of an object-centric cloud."""
    from vidu4d_b200.synthetic import object_scene, projection_matrix
    sc = object_scene(100_000, seed=7)
    t = sc.to_torch(dev)
    vm = np.eye(4, dtype=np.float32)
    pm = (vm.astype(np.float64) @ projection_matrix(0.5, 0.5)).astype(np.float32)
    e = torch.empty((0,), device=dev)
    return dict(P=100_000, W=512, H=512, deg=3, means3D=t["means3D"], opacities=t["opacities"], scales=t["scales"],
                rotations=t["rotations"], shs=t["shs"], colors=e, bg=torch.tensor([0.1, 0.2, 0.3], device=dev),
                vm=torch.from_numpy(vm).to(dev), pm=torch.from_numpy(pm).to(dev), campos=torch.zeros(3, device=dev),
                tanx=0.5, tany=0.5)


def _fwd(s, features=None, bg=None, colors=None, shs=None):
    from vidu4d_b200.rasterizer import _C
    args = (s["bg"] if bg is None else bg, s["means3D"], s["colors"] if colors is None else colors, s["opacities"],
            s["scales"], s["rotations"], 1.0, torch.empty((0,), device=s["means3D"].device), s["vm"], s["pm"], s["tanx"],
            s["tany"], s["H"], s["W"], s["shs"] if shs is None else shs, s["deg"], s["campos"], False, False)
    return _C.rasterize_gaussians(*args) if features is None else _C.rasterize_gaussians_features(*args, features)


def _bwd(s, o, dLc, dLo, features=None, bg=None, colors=None, shs=None):
    from vidu4d_b200.rasterizer import _C
    e = torch.empty((0,), device=s["means3D"].device)
    args = (s["bg"] if bg is None else bg, s["means3D"], o[3], s["colors"] if colors is None else colors, s["scales"],
            s["rotations"], 1.0, e, s["vm"], s["pm"], s["tanx"], s["tany"], dLc, dLo, s["shs"] if shs is None else shs,
            s["deg"], s["campos"], o[4], o[0], o[5], o[6], False)
    g = _C.rasterize_gaussians_backward(*args) if features is None else _C.rasterize_gaussians_features_backward(*args, features)
    return dict(zip(NAMES + ("dL_dfeatures",), g))


def _groups(feat, bgf):
    """Columns of the features in groups of 3 (the last one zero-padded), each with its 3 background values."""
    P, F = feat.shape
    n = (F + 2) // 3
    fp = torch.zeros((P, 3 * n), device=feat.device); fp[:, :F] = feat
    bp = torch.zeros((3 * n,), device=feat.device); bp[:F] = bgf
    return [(fp[:, 3 * k:3 * k + 3].contiguous(), bp[3 * k:3 * k + 3].contiguous()) for k in range(n)]


def _close(a, b, tol):
    a, b = a.float(), b.float()
    return float((a - b).abs().max()) <= tol * float(b.abs().max() + 1e-30)


SCENES = ["id_deg3_64", "precomp_init_70x50", "c2"]


def _scene(name, dev):
    return _c2_scene(dev) if name == "c2" else _golden_scene(name, dev)


@pytest.mark.parametrize("name", SCENES)
def test_colour_allmap_radii_unchanged_by_features(name, dev):
    s = _scene(name, dev)
    g = torch.Generator(device=dev).manual_seed(1)
    feat = torch.rand((s["P"], 22), device=dev, generator=g)
    o = _fwd(s)
    for bg in (s["bg"], torch.cat([s["bg"], torch.rand(22, device=dev, generator=g)])):
        of = _fwd(s, feat, bg=bg)
        assert of[0] == o[0] and of[1].shape == (25, s["H"], s["W"])
        assert torch.equal(of[1][:3], o[1]) and torch.equal(of[2], o[2]) and torch.equal(of[3], o[3])


@pytest.mark.parametrize("name", SCENES)
def test_feature_planes_bit_identical_to_colour_renders(name, dev):
    s = _scene(name, dev)
    F = 22
    g = torch.Generator(device=dev).manual_seed(2)
    feat = torch.randn((s["P"], F), device=dev, generator=g)
    bgf = torch.rand(F, device=dev, generator=g)
    of = _fwd(s, feat, bg=torch.cat([s["bg"], bgf]))
    for k, (cols, b3) in enumerate(_groups(feat, bgf)):
        oc = _fwd(s, bg=b3, colors=cols, shs=torch.empty((0,), device=dev))
        n = min(3, F - 3 * k)
        assert torch.equal(of[1][3 + 3 * k:3 + 3 * k + n], oc[1][:n]), k
    # a 3-channel background gives the feature planes a zero background
    oz = _fwd(s, feat)
    oc = _fwd(s, bg=torch.zeros(3, device=dev), colors=feat[:, :3].contiguous(), shs=torch.empty((0,), device=dev))
    assert torch.equal(oz[1][3:6], oc[1])


@pytest.mark.parametrize("name", ["id_deg3_64", "precomp_init_70x50"])
def test_features_match_float64_model(name, dev):
    """Feature planes, dL/dfeatures and the feature planes' alpha term in dL/dopacity against the float64 model of
    tests/feature_model.py, evaluated over the C oracle's forward state of the same scene."""
    from .conftest import oracle_forward_from_golden
    from .feature_model import backward, planes
    g = load_golden(name)
    s = _golden_scene(name, dev)
    F, H, W = 22, s["H"], s["W"]
    rng = np.random.default_rng(3)
    feat = rng.standard_normal((s["P"], F)).astype(np.float32)
    bgf = rng.random(F).astype(np.float32)
    bg = np.concatenate([g["in_bg"].reshape(3), bgf]).astype(np.float32)
    G = rng.standard_normal((F, H, W)).astype(np.float32)
    st = oracle_forward_from_golden(g)
    m = planes(st, feat, bg)
    tf, tb = torch.from_numpy(feat).to(dev), torch.from_numpy(bg).to(dev)
    o = _fwd(s, tf, bg=tb)
    of = o[1][3:].cpu().numpy()
    for f in range(F):
        assert np.abs(of[f] - m[f]).max() <= 1e-4 * (np.abs(m[f]).max() + 1e-30), f
    # backward with the feature planes' gradient only: dL/dopacity is their alpha term alone
    up = torch.cat([torch.zeros((3, H, W), device=dev), torch.from_numpy(G).to(dev)])
    gr = _bwd(s, o, up, torch.zeros((8, H, W), device=dev), features=tf, bg=tb)
    dfeat, dop = backward(st, feat, bg, G)
    assert _close(gr["dL_dfeatures"].cpu().double(), torch.from_numpy(dfeat), 1e-4)
    assert _close(gr["dL_dopacity"].reshape(-1).cpu().double(), torch.from_numpy(dop), 1e-4)


@pytest.mark.parametrize("name", SCENES)
def test_backward_by_linearity(name, dev):
    s = _scene(name, dev)
    F, P, H, W = 22, s["P"], s["H"], s["W"]
    g = torch.Generator(device=dev).manual_seed(4)
    feat = torch.randn((P, F), device=dev, generator=g)
    bgf = torch.rand(F, device=dev, generator=g)
    dLc = torch.randn((3, H, W), device=dev, generator=g)
    dLo = torch.randn((8, H, W), device=dev, generator=g)
    dLf = torch.randn((F, H, W), device=dev, generator=g)
    of = _fwd(s, feat, bg=torch.cat([s["bg"], bgf]))
    gf = _bwd(s, of, torch.cat([dLc, dLf]), dLo, features=feat, bg=torch.cat([s["bg"], bgf]))
    assert gf["dL_dfeatures"].shape == (P, F)
    base = _bwd(s, _fwd(s), dLc, dLo)
    for k in ("dL_dcolors", "dL_dsh"):
        assert torch.equal(gf[k], base[k]) or _close(gf[k], base[k], 1e-5), k
    total = {k: base[k].clone() for k in GEOM}
    e = torch.empty((0,), device=dev)
    zo = torch.zeros((8, H, W), device=dev)
    dfeat = torch.zeros((P, 3 * ((F + 2) // 3)), device=dev)
    dLfp = torch.zeros((3 * ((F + 2) // 3), H, W), device=dev); dLfp[:F] = dLf
    for k, (cols, b3) in enumerate(_groups(feat, bgf)):
        oc = _fwd(s, bg=b3, colors=cols, shs=e)
        gc = _bwd(s, oc, dLfp[3 * k:3 * k + 3].contiguous(), zo, bg=b3, colors=cols, shs=e)
        dfeat[:, 3 * k:3 * k + 3] = gc["dL_dcolors"]
        for n in GEOM:
            total[n] += gc[n]
    assert _close(gf["dL_dfeatures"], dfeat[:, :F], 1e-5)
    for n in GEOM:
        assert _close(gf[n], total[n], 1e-4), n
    vis = of[3] > 0
    assert float(gf["dL_dfeatures"][~vis].abs().max() if (~vis).any() else 0.0) == 0.0


def _cams(M, dev):
    from vidu4d_b200.synthetic import orbit_view, projection_matrix
    Pm = projection_matrix(0.5, 0.5).astype(np.float64)
    vms, pms, cps = [], [], []
    for f in range(M):
        R, t = orbit_view(3 * f + 1, 64)
        W2C = np.eye(4); W2C[:3, :3] = R; W2C[:3, 3] = t
        vms.append(W2C.T.astype(np.float32)); pms.append((W2C.T @ Pm).astype(np.float32)); cps.append((-R.T @ t).astype(np.float32))
    return tuple(torch.from_numpy(np.stack(a)).to(dev) for a in (vms, pms, cps))


@pytest.mark.parametrize("per_frame", [False, True], ids=["shared_features", "per_frame_features"])
@pytest.mark.parametrize("sum_shared", [False, True], ids=["per_frame_grads", "summed_grads"])
def test_batch_equals_single_frame_calls(per_frame, sum_shared, dev):
    from vidu4d_b200 import rasterizer as RZ
    from vidu4d_b200.synthetic import object_scene
    M, P, W, H, F = 4, 20000, 208, 144, 22
    sc = object_scene(P, seed=5, center=(0.0, 0.0, 0.0))
    t = sc.to_torch(dev)
    vms, pms, cps = _cams(M, dev)
    e = torch.empty((0,), device=dev)
    g = torch.Generator(device=dev).manual_seed(6)
    bg = torch.rand(3 + F, device=dev, generator=g)
    feat = torch.randn((M, P, F) if per_frame else (P, F), device=dev, generator=g)
    dLc = torch.randn((M, 3 + F, H, W), device=dev, generator=g)
    dLo = torch.randn((M, 8, H, W), device=dev, generator=g)
    C = RZ._C
    nr, color, allmap, radii, gb, bb, ib, fp = C.rasterize_gaussians_batch(
        bg, t["means3D"], e, t["opacities"], t["scales"], t["rotations"], 1.0, vms, pms, 0.5, 0.5, H, W, t["shs"], 3, cps,
        features=feat)
    assert color.shape == (M, 3 + F, H, W) and torch.equal(fp, color[:, 3:])
    grads = C.rasterize_gaussians_backward_batch(bg, t["means3D"], radii, e, t["scales"], t["rotations"], 1.0, vms, pms, 0.5,
                                                 0.5, dLc, dLo, t["shs"], 3, cps, gb, bb, ib, sum_shared=sum_shared,
                                                 features=feat)
    dfeat = grads[8]
    assert dfeat.shape == ((P, F) if (sum_shared and not per_frame) else (M, P, F))
    acc = torch.zeros((P, F), device=dev)
    for f in range(M):
        ff = feat[f] if per_frame else feat
        o = C.rasterize_gaussians_features(bg, t["means3D"], e, t["opacities"], t["scales"], t["rotations"], 1.0, e, vms[f],
                                           pms[f], 0.5, 0.5, H, W, t["shs"], 3, cps[f], False, False, ff)
        assert o[0] == nr[f] and torch.equal(o[1], color[f]) and torch.equal(o[2], allmap[f]) and torch.equal(o[3], radii[f])
        gs = C.rasterize_gaussians_features_backward(bg, t["means3D"], o[3], e, t["scales"], t["rotations"], 1.0, e, vms[f],
                                                     pms[f], 0.5, 0.5, dLc[f], dLo[f], t["shs"], 3, cps[f], o[4], o[0], o[5],
                                                     o[6], False, ff)
        assert _close(grads[0][f], gs[0], 2e-5)          # the means2D proxy is always per frame
        if dfeat.ndim == 3:
            assert _close(dfeat[f], gs[8], 2e-5)
        acc += gs[8]
        if not sum_shared:
            for n in (3, 6, 7):
                assert _close(grads[n][f], gs[n], 2e-5), NAMES[n]
    if dfeat.ndim == 2:
        assert _close(dfeat, acc, 2e-5)


def test_autograd_paths(dev):
    from vidu4d_b200 import rasterizer as RZ, renderer as RD
    from vidu4d_b200.synthetic import object_scene
    P, W, H, F = 3000, 96, 64, 22
    sc = object_scene(P, seed=9)
    t = sc.to_torch(dev)
    cam = RD.make_camera(W, H, 2 * np.arctan(0.5), 2 * np.arctan(0.5), device=dev)
    g = torch.Generator(device=dev).manual_seed(8)
    featv = torch.randn((P, F), device=dev, generator=g)
    bg = torch.rand(3 + F, device=dev, generator=g)
    up = torch.randn((3 + F, H, W), device=dev, generator=g)

    class PC:
        get_xyz = t["means3D"]; get_opacity = t["opacities"]; get_scaling = t["scales"]; get_rotation = t["rotations"]
        get_features = t["shs"]; active_sh_degree = 3
    pipe = RD.PipelineParams()
    # GaussianRasterizer.forward_features, against the C-level backward
    feat = featv.clone().requires_grad_(True)
    rs = RZ.GaussianRasterizationSettings(H, W, 0.5, 0.5, bg, 1.0, cam.world_view_transform, cam.full_proj_transform, 3,
                                          cam.camera_center, False, False)
    means = t["means3D"].clone().requires_grad_(True)
    color, radii, allmap = RZ.GaussianRasterizer(rs).forward_features(
        means3D=means, means2D=torch.zeros_like(means, requires_grad=True), opacities=t["opacities"], features=feat,
        shs=t["shs"], scales=t["scales"], rotations=t["rotations"])
    assert color.shape == (3 + F, H, W)
    (color * up).sum().backward()
    o = RZ._C.rasterize_gaussians_features(bg, t["means3D"], torch.empty(0, device=dev), t["opacities"], t["scales"],
                                           t["rotations"], 1.0, torch.empty(0, device=dev), cam.world_view_transform,
                                           cam.full_proj_transform, 0.5, 0.5, H, W, t["shs"], 3, cam.camera_center, False,
                                           False, featv)
    ref = RZ._C.rasterize_gaussians_features_backward(bg, t["means3D"], o[3], torch.empty(0, device=dev), t["scales"],
                                                      t["rotations"], 1.0, torch.empty(0, device=dev), cam.world_view_transform,
                                                      cam.full_proj_transform, 0.5, 0.5, up, torch.zeros((8, H, W), device=dev),
                                                      t["shs"], 3, cam.camera_center, o[4], o[0], o[5], o[6], False, featv)
    assert _close(feat.grad, ref[8], 1e-6) and _close(means.grad, ref[3], 1e-6)
    # render(features=) with Vidu4D's in-place edit of render[:3] (deformable_gaussian.py:188-190)
    feat2 = featv.clone().requires_grad_(True)
    out = RD.render(cam, PC, pipe, bg, features=feat2)
    img = out["render"]
    assert img.shape == (3 + F, H, W)
    img[:3] = img[:3] * 0.5 + 0.25
    (img * up).sum().backward()
    assert _close(feat2.grad, ref[8], 1e-6)
    # render_loss_batch(features=): the feature planes are a differentiable output next to the fused losses
    cams = RD.stack_cameras([cam, cam])
    feat3 = featv.clone().requires_grad_(True)
    target = torch.rand((2, 3, H, W), device=dev, generator=g)
    r = RD.render_loss_batch(cams, PC, pipe, bg, target, features=feat3)
    assert r["features"].shape == (2, F, H, W) and r["render"].shape == (2, 3, H, W)
    assert torch.equal(r["features"][0], o[1][3:])
    (r["loss"] * 0 + (r["features"] * up[3:]).sum()).backward()
    assert _close(feat3.grad, 2 * ref[8], 1e-5)


def test_graphed_step_with_features_equals_eager(dev):
    from vidu4d_b200 import rasterizer as RZ
    from vidu4d_b200.graph import GraphedStep
    from vidu4d_b200.synthetic import object_scene
    M, P, W, H, F = 2, 20000, 128, 96, 22
    sc = object_scene(P, seed=11, center=(0.0, 0.0, 0.0))
    t = sc.to_torch(dev)
    vms, pms, cps = _cams(M, dev)
    e = torch.empty((0,), device=dev)
    g = torch.Generator(device=dev).manual_seed(12)
    bg = torch.rand(3 + F, device=dev, generator=g)
    feat = torch.randn((P, F), device=dev, generator=g)
    dLc = torch.randn((M, 3 + F, H, W), device=dev, generator=g)
    dLo = torch.randn((M, 8, H, W), device=dev, generator=g)
    res = {}

    def body():
        out = RZ._C.rasterize_gaussians_batch(bg, t["means3D"], e, t["opacities"], t["scales"], t["rotations"], 1.0, vms, pms,
                                              0.5, 0.5, H, W, t["shs"], 3, cps, features=feat)
        gr = RZ._C.rasterize_gaussians_backward_batch(bg, t["means3D"], out[3], e, t["scales"], t["rotations"], 1.0, vms, pms,
                                                      0.5, 0.5, dLc, dLo, t["shs"], 3, cps, out[4], out[5], out[6],
                                                      sum_shared=True, want_transmat=False, features=feat)
        res["color"], res["dfeat"], res["dmeans"] = out[1], gr[8], gr[3]
    try:
        body()
        eager = {k: v.clone() for k, v in res.items()}
        step = GraphedStep(body, device=dev)
        step()
        torch.cuda.synchronize()
        assert torch.equal(res["color"], eager["color"])
        for k in ("dfeat", "dmeans"):
            assert _close(res[k], eager[k], 1e-5), k
    finally:
        RZ.set_sync_mode(True)
        RZ._pending.clear()


def test_launches_and_empty_scene(dev):
    from vidu4d_b200 import _capi, rasterizer as RZ
    s = _golden_scene("id_deg3_64", dev)
    H, W, F = s["H"], s["W"], 5
    feat = torch.rand((s["P"], F), device=dev)
    dLo = torch.randn((8, H, W), device=dev)

    def run(features):
        _capi.set_profiling(True)
        _capi.get_profile()
        lc = _capi.launch_count()
        o = _fwd(s, features)
        dLc = torch.ones((3 + (F if features is not None else 0), H, W), device=dev)
        _bwd(s, o, dLc, dLo, features=features)
        torch.cuda.synchronize()
        n = _capi.launch_count() - lc
        prof = _capi.get_profile()
        _capi.set_profiling(False)
        return n, prof
    n0, p0 = run(None)
    n1, p1 = run(feat)
    assert n1 == n0 + 2
    assert "feature_fwd" not in p0 and "feature_bwd" not in p0
    assert p1["feature_fwd"]["count"] == 1 and p1["feature_bwd"]["count"] == 1
    assert {k: v["count"] for k, v in p0.items()} == {k: v["count"] for k, v in p1.items() if not k.startswith("feature_")}
    # P = 0: the feature planes are zero, like the colour
    z = torch.zeros((0, 3), device=dev)
    o = RZ._C.rasterize_gaussians_features(s["bg"], z, torch.empty(0, device=dev), torch.zeros((0, 1), device=dev),
                                           torch.zeros((0, 2), device=dev), torch.zeros((0, 4), device=dev), 1.0,
                                           torch.empty(0, device=dev), s["vm"], s["pm"], s["tanx"], s["tany"], H, W,
                                           torch.zeros((0, 16, 3), device=dev), 3, s["campos"], False, False,
                                           torch.zeros((0, F), device=dev))
    assert o[1].shape == (3 + F, H, W) and float(o[1].abs().max()) == 0.0
