"""GPU tests of the fused losses on the feature planes (csrc/loss.cu, sr_feature_loss_batch; render_loss_batch's
feature_target / gauss_mask_channel) and of the registration-feature group of the flat surfel store."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev(built):
    from vidu4d_b200 import _capi
    _capi.load()
    return torch.device("cuda:0")


def _close(a, b, tol):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).abs().max()) <= tol * float(b.abs().max()) + 1e-30


def _inputs(M, W, H, F, Cf, gm, dev, seed):
    """Seeded planes with no v within a few ulp of 0: masks are 0 or >= 0.25, and the pixels with v = 0 have it exactly
    (feature == target, gauss mask == alpha)."""
    g = torch.Generator(device=dev).manual_seed(seed)
    feat = torch.randn((M, F, H, W), device=dev, generator=g)
    target = torch.randn((M, Cf, H, W), device=dev, generator=g)
    same = torch.rand((M, 1, H, W), device=dev, generator=g) < 0.05
    feat[:, :Cf] = torch.where(same, target, feat[:, :Cf])
    on = torch.rand((M, H, W), device=dev, generator=g) < 0.6
    mask = torch.where(on, 0.25 + 0.75 * torch.rand((M, H, W), device=dev, generator=g), torch.zeros((), device=dev))
    allmap = torch.rand((M, 8, H, W), device=dev, generator=g)
    alpha = allmap[:, 1]
    alpha[torch.rand((M, H, W), device=dev, generator=g) < 0.2] = 0.0
    if gm >= 0:
        off = (0.05 + 0.95 * torch.rand((M, H, W), device=dev, generator=g)) * torch.where(
            torch.rand((M, H, W), device=dev, generator=g) < 0.5, -1.0, 1.0)
        eq = torch.rand((M, H, W), device=dev, generator=g) < 0.05
        feat[:, gm] = torch.where(eq, alpha, alpha + off)
    det = torch.ones(M, device=dev)
    if M > 1:
        det[1] = 0.0
    return feat, target, mask, det, allmap


def _call(feat, target, mask, det, allmap, gm, weights):
    from vidu4d_b200 import _capi
    lib = _capi.load()
    M, F, H, W = feat.shape
    dev = feat.device
    terms = torch.full((M, 2), float("nan"), device=dev)
    counts = torch.full((M, 2), -1, dtype=torch.int32, device=dev)
    grad = torch.full_like(feat, float("nan"))
    ptr = lambda t: None if t is None else t.data_ptr()  # noqa: E731
    rc = lib.sr_feature_loss_batch(M, W, H, F, 0 if target is None else target.shape[1], gm, feat.data_ptr(), ptr(target),
                                   ptr(mask), ptr(det), allmap.data_ptr(), weights.data_ptr(), terms.data_ptr(),
                                   counts.data_ptr(), grad.data_ptr(), torch.cuda.current_stream(dev).cuda_stream)
    _capi.check(rc, "sr_feature_loss_batch")
    return terms, counts, grad


@pytest.mark.parametrize("W,H,M,gm,with_target", [(48, 40, 1, 21, True), (48, 40, 2, -1, True), (48, 40, 2, 3, False),
                                                   (256, 256, 2, 21, True), (512, 512, 8, 21, True)])
def test_kernel_matches_float64_model(W, H, M, gm, with_target, dev):
    from . import feature_loss_bounds as fb
    from .feature_loss_model import feature_losses
    F, Cf = 22, 16
    feat, target, mask, det, allmap = _inputs(M, W, H, F, Cf, gm, dev, seed=W + M)
    target = target if with_target else None
    w = torch.tensor([1e-2, 7e-3], device=dev)
    terms, counts, grad = _call(feat, target, mask, det, allmap, gm, w)
    n = lambda t: None if t is None else t.cpu().numpy()  # noqa: E731
    _, rc, _ = feature_losses(n(feat), n(target), n(mask), n(det), n(allmap[:, 1]), gm, [1e-2, 7e-3])
    assert np.array_equal(counts.cpu().numpy(), rc)
    # every element under the restatement's rounding-error bound (tests/feature_loss_bounds.py); untouched channels
    # exactly 0
    px = fb.pixel_terms(n(feat), n(target), n(mask), n(det), n(allmap[:, 1]), gm)
    rep = fb.check(f"{W}x{H} M={M}", n(terms), n(counts), n(grad), px, n(w), gm, F)
    print(f"\n[feature {W}x{H} M={M} gm={gm}] " + ", ".join(f"{k} {v:.3g}" for k, v in rep.items()))
    # no atomics on image data: the planes are bit for bit the same on a second call
    assert torch.equal(_call(feat, target, mask, det, allmap, gm, w)[2], grad)


def test_zero_weights_give_zero_terms_and_planes(dev):
    feat, target, mask, det, allmap = _inputs(2, 48, 40, 22, 16, 21, dev, seed=5)
    terms, counts, grad = _call(feat, target, mask, det, allmap, 21, torch.zeros(2, device=dev))
    assert int(counts.min()) >= 0 and int(counts[0].sum()) > 0
    assert float(terms.abs().max()) == 0.0 and float(grad.abs().max()) == 0.0


# ---------------------------------------------------------------------------------------------- render_loss_batch end to end
def _scene(P, W, H, M, dev, seed=31):
    from vidu4d_b200.renderer import make_camera, stack_cameras
    from vidu4d_b200.synthetic import SurfelCloud, object_scene, orbit_view
    cams = []
    for f in range(M):
        R, t = orbit_view(7 * f + 3, 64)
        cams.append(make_camera(W, H, 2 * np.arctan(0.5), 2 * np.arctan(0.5 * H / W), R=R.T, T=t, device=dev))
    scene = object_scene(P, seed=seed, center=(0.0, 0.0, 0.0))
    return stack_cameras(cams), scene, lambda: SurfelCloud(scene, dev)


def _reference_feature_terms(planes, alpha, target, mask, det, gm, w):
    """lab4d/engine/model.py:663-667,742-745,952-967,1000-1012 written in torch on out["features"] (M,F,H,W)."""
    def positive_mean(v):
        return v.mean() if int((v > 0).sum()) == 0 else v[v > 0].mean()
    Cf = target.shape[1]
    v = (planes[:, :Cf] - target).norm(2, 1) * mask * det[:, None, None]
    g = (planes[:, gm] - alpha.detach()).pow(2)
    return w[0] * positive_mean(v) + w[1] * positive_mean(g)


def test_render_loss_batch_fused_feature_losses_match_torch(dev):
    from vidu4d_b200.renderer import PipelineParams, render_loss_batch
    M, P, W, H, F, Cf, gm = 2, 50000, 128, 128, 22, 16, 21
    bc, scene, mk = _scene(P, W, H, M, dev)
    gen = torch.Generator(device=dev).manual_seed(3)
    rgb = torch.rand((M, 3, H, W), device=dev, generator=gen)
    ftgt = torch.randn((M, Cf, H, W), device=dev, generator=gen) * 0.3
    feat0 = torch.randn((P, F), device=dev, generator=gen) * 0.3
    feat0[:, gm] = torch.rand((P,), device=dev, generator=gen)
    det = torch.tensor([1.0, 1.0], device=dev)
    w = torch.tensor([1e-2, 4e-3], device=dev)
    kw = dict(w_rgb=0.8, w_mask=0.1, lambda_normal=0.05, lambda_dist=10.0)
    pipe, bg = PipelineParams(), torch.zeros(3, device=dev)
    with torch.no_grad():
        pre = render_loss_batch(bc, mk(), pipe, bg, rgb, **dict(kw, w_mask=0.0))
    mask = (pre["allmap"][:, 1] > 0.5).float()
    assert 0 < float(mask.mean()) < 1

    def run(fused):
        cloud = mk()
        feat = feat0.clone().requires_grad_(True)
        extra = dict(feature_target=ftgt, is_detected=det, gauss_mask_channel=gm, feature_loss_weights=w) if fused else {}
        out = render_loss_batch(bc, cloud, pipe, bg, rgb, mask_gt=mask, features=feat, **kw, **extra)
        loss = out["loss"] if fused else out["loss"] + _reference_feature_terms(out["features"], out["allmap"][:, 1], ftgt,
                                                                               mask, det, gm, w)
        # a non-unit upstream scalar, plus a loss of the caller's own on the planes (flow / normal channels)
        (1.7 * loss + 0.3 * out["features"][:, 16:21].square().mean()).backward()
        return out, loss.detach(), [p.grad for p in cloud.flat_params()] + [feat.grad]
    out_f, loss_f, g_f = run(True)
    out_t, loss_t, g_t = run(False)
    assert out_f["feature_terms"].shape == (M, 2) and not out_f["feature_terms"].requires_grad
    assert out_f["terms"].shape == (M, 4) and out_f["feature_counts"].dtype == torch.int32
    assert float(out_f["feature_terms"].abs().min()) > 0
    assert abs(float(loss_f) - float(loss_t)) <= 1e-6 * abs(float(loss_t)), (float(loss_f), float(loss_t))
    for name, a, b in zip(("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation", "features"), g_f, g_t):
        assert float(b.abs().max()) > 0, name
        assert _close(a, b, 1e-5), name


def test_without_new_arguments_nothing_changes(dev, monkeypatch):
    """The launches of render_loss_batch (forward and backward) without the new arguments are the parent commit's:
    without features 15 + 2, with features= 16 + 3; the fused feature losses add their two kernels to the forward.
    With both weights at zero the fused terms contribute exactly nothing: the loss is the image terms' sum bit for bit and
    the rasterizer backward receives bit-identical plane gradients.  (The loss reduction and the rasterizer backward
    accumulate with float atomics, so two calls are compared at those inputs, not at their atomically summed outputs.)"""
    from vidu4d_b200 import _capi
    from vidu4d_b200 import rasterizer as RZ
    from vidu4d_b200.renderer import PipelineParams, render_loss_batch
    M, P, W, H, F = 2, 20000, 96, 64, 22
    bc, scene, mk = _scene(P, W, H, M, dev, seed=41)
    gen = torch.Generator(device=dev).manual_seed(4)
    rgb = torch.rand((M, 3, H, W), device=dev, generator=gen)
    mask = (torch.rand((M, H, W), device=dev, generator=gen) > 0.5).float()
    ftgt = torch.randn((M, 16, H, W), device=dev, generator=gen)
    feat = torch.rand((P, F), device=dev, generator=gen)
    pipe, bg = PipelineParams(), torch.zeros(3, device=dev)
    seen = []
    real = RZ._C.rasterize_gaussians_backward_batch

    def spy(*a, **k):
        seen.append([t.clone() if torch.is_tensor(t) else t for t in (a[11], a[12], k.get("dL_dout_features"),
                                                                        k.get("grad_scale"), k.get("features_grad_scale"))])
        return real(*a, **k)

    def run(features=None, **extra):
        cloud = mk()
        f = None if features is None else features.clone().requires_grad_(True)
        lc = _capi.launch_count()
        out = render_loss_batch(bc, cloud, pipe, bg, rgb, mask_gt=mask, w_mask=0.1, lambda_normal=0.05, features=f, **extra)
        torch.cuda.synchronize()
        n_fwd = _capi.launch_count() - lc
        lc = _capi.launch_count()
        out["loss"].backward()
        torch.cuda.synchronize()
        return out, n_fwd, _capi.launch_count() - lc, [p.grad for p in cloud.flat_params()] + ([f.grad] if f is not None else [])
    run()                                                              # warm-up: learns the instance capacity
    _, f0, b0, _ = run()
    _, f1, b1, _ = run(feat)
    assert (f0, b0) == (15, 2) and (f1, b1) == (16, 3)
    monkeypatch.setattr(RZ._C, "rasterize_gaussians_backward_batch", staticmethod(spy))
    ob, _, _, gb = run(feat)
    oa, fa, ba, ga = run(feat, feature_target=ftgt, gauss_mask_channel=21, feature_loss_weights=torch.zeros(2, device=dev))
    monkeypatch.undo()
    assert (fa, ba) == (f1 + 2, b1)
    assert float(oa["feature_terms"].abs().max()) == 0.0 and int(oa["feature_counts"].sum()) > 0
    assert torch.equal(oa["loss"], oa["terms"].sum()) and torch.equal(ob["loss"], ob["terms"].sum())
    assert torch.equal(oa["features"], ob["features"]) and torch.equal(oa["render"], ob["render"])
    sa, sb = seen
    for i, (x, y) in enumerate(zip(sa, sb)):
        assert (x is None and y is None) or torch.equal(x, y), i
    for a, b in zip(ga, gb):
        assert _close(a, b, 1e-5)


# ---------------------------------------------------------------------------------------------- flat store: regist_feat
def _model(P, dev, seed=0, regist=True):
    from vidu4d_b200.surfel_store import FlatSurfelModel
    from vidu4d_b200.synthetic import object_scene
    sc = object_scene(P, seed=seed, center=(0.0, 0.0, 0.0))
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    op = np.clip(sc.opacities, 1e-6, 1 - 1e-6)
    rf = torch.randn((P, 16), device=dev, generator=torch.Generator(device=dev).manual_seed(seed)) * 0.1 if regist else None
    return FlatSurfelModel(t(sc.means3D), t(sc.shs[:, :1]), t(sc.shs[:, 1:]), t(np.log(op / (1 - op))), t(np.log(sc.scales)),
                           t(sc.rotations), regist_feat=rf)


NAMES = ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation", "regist_feat")


def test_flat_adam_with_regist_feat_matches_torch_adam(dev):
    m = _model(5003, dev)
    assert m.lrs["regist_feat"] == 2.5e-3 and len(m.flat_params()) == 7 and m._regist_feat.shape == (5003, 16)
    ref = [p.detach().clone().requires_grad_(True) for p in m.flat_params()]
    opt = torch.optim.Adam([{"params": [p], "lr": m.lrs[n]} for p, n in zip(ref, NAMES)], lr=0.0, eps=1e-15)
    g = torch.Generator(device=dev).manual_seed(1)
    for step in range(4):
        m.zero_grad_flat()
        for p, r in zip(m.flat_params(), ref):
            gr = torch.randn(p.shape, device=dev, generator=g) * (10.0 ** (step - 2))
            p.grad.copy_(gr)
            r.grad = gr.clone() * 0.25
        m.adam_step(grad_scale=0.25)
        opt.step()
        for p, r, n in zip(m.flat_params(), ref, NAMES):
            assert float((p - r).detach().abs().max()) <= 1e-6 * float(r.abs().max()) + 1e-9, (step, n)
    # the six other groups keep the layout they have without the seventh
    m6 = _model(5003, dev, regist=False)
    assert m6._offsets(5003)[0] == m._offsets(5003)[0][:6] and m.flat.numel() == m6.flat.numel() + 5003 * 16


@pytest.mark.parametrize("max_screen_size", [None, 20])
def test_densify_and_prune_with_regist_feat_matches_reference_procedure(max_screen_size, dev):
    from .test_gpu_store import _reference_densify
    m = _model(20000, dev, seed=3)
    g = torch.Generator(device=dev).manual_seed(5)
    for _ in range(2):
        for p in m.flat_params():
            p.grad.copy_(torch.randn(p.shape, device=dev, generator=g) * 1e-3)
        m.adam_step()
    with torch.no_grad():
        m._opacity[:500] = -8.0
        m._scaling[500:800] += 2.5
    vis = torch.rand((m.P,), device=dev, generator=g) > 0.3
    m.add_densification_stats(torch.randn((m.P, 3), device=dev, generator=g) * 3e-4, vis)
    off, _ = m._offsets(m.P)
    params = {n: p.detach().clone() for n, p in zip(NAMES, m.flat_params())}
    state = {n: (m.exp_avg[o:o + p.numel()].view(p.shape).clone(), m.exp_avg_sq[o:o + p.numel()].view(p.shape).clone())
             for n, p, o in zip(NAMES, m.flat_params(), off)}
    stats = {"accum": m.xyz_gradient_accum.clone(), "denom": m.denom.clone()}
    want_p, want_s = _reference_densify(params, state, stats, m.percent_dense, 2e-4, 0.005, 1.0, max_screen_size,
                                        torch.Generator(device=dev).manual_seed(77))
    info = m.densify_and_prune(2e-4, 0.005, 1.0, max_screen_size, generator=torch.Generator(device=dev).manual_seed(77))
    assert info["cloned"] > 0 and info["split"] > 0 and info["pruned"] > 0
    assert m.P == want_p["regist_feat"].shape[0] == info["P"]
    off, _ = m._offsets(m.P)
    for n, p, o in zip(NAMES, m.flat_params(), off):
        assert torch.equal(p.detach(), want_p[n].view(p.shape)), n
        assert torch.equal(m.exp_avg[o:o + p.numel()].view(p.shape), want_s[n][0].view(p.shape)), n
        assert torch.equal(m.exp_avg_sq[o:o + p.numel()].view(p.shape), want_s[n][1].view(p.shape)), n


def test_grown_model_keeps_rendering_its_features(dev):
    from vidu4d_b200.renderer import PipelineParams, make_camera, render_fused
    m = _model(20000, dev, seed=4)
    cam = make_camera(160, 128, 2 * np.arctan(0.5), 2 * np.arctan(0.4), device=dev)
    bg = torch.zeros(3, device=dev)
    m.xyz_gradient_accum += 1.0
    m.denom += 1.0
    info = m.densify_and_prune(2e-4, 0.005, 1.0, None)
    assert info["P"] > 20000 and m._regist_feat.shape == (m.P, 16)
    m.zero_grad_flat()
    out = render_fused(cam, m, PipelineParams(), bg, features=m._regist_feat)
    assert out["render"].shape == (19, 128, 160) and float(out["render"][3:].abs().max()) > 0
    out["render"][3:].square().mean().backward()
    off, _ = m._offsets(m.P)
    assert float(m.grad_flat[off[6]:].abs().max()) > 0 and m._regist_feat.grad.data_ptr() == m.grad_flat[off[6]:].data_ptr()
    # the planes equal a render with the same features held outside the store
    again = render_fused(cam, m, PipelineParams(), bg, features=m._regist_feat.detach().clone())
    assert torch.equal(again["render"], out["render"].detach())


def test_graphed_step_with_fused_feature_losses_and_regist_feat_matches_eager(dev):
    """render + fused feature losses + backward + FlatSurfelModel.adam_step with regist_feat as one CUDA graph, replayed
    with two different device weights; every replay is compared with an eager step from the same state."""
    from vidu4d_b200 import rasterizer as RZ
    from vidu4d_b200.graph import GraphedStep
    from vidu4d_b200.renderer import PipelineParams, render_loss_batch
    M, P, W, H = 2, 20000, 96, 96
    bc, _, _ = _scene(P, W, H, M, dev, seed=51)
    gen = torch.Generator(device=dev).manual_seed(6)
    rgb = torch.rand((M, 3, H, W), device=dev, generator=gen)
    mask = (torch.rand((M, H, W), device=dev, generator=gen) > 0.4).float()
    ftgt = torch.randn((M, 16, H, W), device=dev, generator=gen) * 0.1
    rest = torch.rand((P, 6), device=dev, generator=gen)                       # flow, normal, Gaussian mask channels
    det = torch.tensor([1.0, 1.0], device=dev)
    pipe, bg = PipelineParams(), torch.zeros(3, device=dev)
    mg, me = _model(P, dev, seed=7), _model(P, dev, seed=7)
    wg, we = torch.tensor([1e-2, 1e-2], device=dev), torch.tensor([1e-2, 1e-2], device=dev)
    loss_g = torch.zeros((), device=dev)

    def step_body(m, w, loss_out):
        m.zero_grad_flat()
        out = render_loss_batch(bc, m, pipe, bg, rgb, mask_gt=mask, w_mask=0.1, features=torch.cat([m._regist_feat, rest], 1),
                                feature_target=ftgt, is_detected=det, gauss_mask_channel=21, feature_loss_weights=w)
        out["loss"].backward()
        m.adam_step()
        loss_out.copy_(out["loss"].detach())
    step = GraphedStep(lambda: step_body(mg, wg, loss_g), device=dev)
    try:
        step()
        baked = mg.step_count                  # adam_step's step count is a launch argument: the graph keeps the captured one
        for wv in ([1e-2, 1e-2], [5e-2, 2e-3]):
            for a, b in ((me.flat, mg.flat), (me.exp_avg, mg.exp_avg), (me.exp_avg_sq, mg.exp_avg_sq)):
                a.copy_(b)
            wg.copy_(torch.tensor(wv, device=dev))
            we.copy_(wg)
            step()
            me.step_count = baked - 1
            loss_e = torch.zeros((), device=dev)
            RZ.set_sync_mode(True)
            step_body(me, we, loss_e)
            RZ.set_sync_mode(False)
            assert abs(float(loss_g) - float(loss_e)) <= 1e-5 * abs(float(loss_e)), wv
            assert _close(mg.grad_flat, me.grad_flat, 1e-5), wv
            off, total = mg._offsets(mg.P)
            for n, a, b in zip(NAMES, off, off[1:] + [total]):
                assert _close(mg.flat[a:b], me.flat[a:b], 1e-5), (wv, n)
        assert step.captures == 1
    finally:
        RZ.set_sync_mode(True)
        RZ._pending.clear()
