"""GPU tests of Stage 3's fused silhouette loss (csrc/mask_loss.cu, sr_mask_loss_batch; render_loss_batch's
mask_loss_weight=): the kernels against the reference's fixtures and the float64 model's rounding bound, run-to-run bit
identity, graph capture with inputs refilled in place, and the term end to end through the rasterizer."""
import numpy as np
import pytest
import torch

from .test_mask_loss_cpu import CASES

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev(built):
    from vidu4d_b200 import _capi
    _capi.load()
    return torch.device("cuda:0")


class _Call:
    """sr_mask_loss_batch on an (M,8,H,W) allmap's alpha plane, with its outputs and scratch allocated once (so that the
    call can be captured and replayed)."""

    def __init__(self, M, H, W, dev):
        from vidu4d_b200 import _capi
        self.lib = _capi.load()
        self.M, self.H, self.W = M, H, W
        self.nb = int(self.lib.sr_mask_loss_scratch_bytes(M, W, H))
        self.scratch = torch.empty((self.nb,), dtype=torch.uint8, device=dev)
        self.terms = torch.empty((M,), device=dev)
        self.counts = torch.empty((M,), dtype=torch.int32, device=dev)
        self.balance = torch.empty((3,), device=dev)
        self.g = torch.zeros((M, 8, H, W), device=dev)

    def __call__(self, allmap, mask, vis, det, weight):
        from vidu4d_b200 import _capi
        ptr = lambda t: None if t is None else t.data_ptr()  # noqa: E731
        M, H, W = self.M, self.H, self.W
        self.g.zero_()
        rc = self.lib.sr_mask_loss_batch(M, W, H, allmap[:, 1].data_ptr(), 8 * H * W, mask.data_ptr(), ptr(vis), ptr(det),
                                         weight.data_ptr(), self.terms.data_ptr(), self.counts.data_ptr(),
                                         self.balance.data_ptr(), self.g[:, 1].data_ptr(), self.scratch.data_ptr(), self.nb,
                                         torch.cuda.current_stream(allmap.device).cuda_stream)
        _capi.check(rc, "sr_mask_loss_batch")
        return self.terms, self.counts, self.balance, self.g


def _allmap(alpha, dev, seed=0):
    M, H, W = alpha.shape
    am = torch.rand((M, 8, H, W), device=dev, generator=torch.Generator(device=dev).manual_seed(seed))
    am[:, 1] = torch.as_tensor(alpha, device=dev)
    return am


def _check_against_model(r, terms, counts, balance, g):
    """terms, counts, weights and every dL/dalpha element against the model, within its rounding bound."""
    assert np.array_equal(counts.cpu().numpy(), r["counts"])
    assert np.array_equal(balance.cpu().numpy()[:2], [r["pos_wt"], r["neg_wt"]], equal_nan=True)
    assert float(balance[2]) == float(r["branch"])
    t = terms.cpu().numpy().astype(np.float64)
    fin = np.isfinite(r["terms"])
    assert np.array_equal(np.isnan(t), np.isnan(r["terms"]))
    assert np.all(np.abs(t[fin] - r["terms"][fin]) <= r["terms_bound"][fin] + 1e-30), (t, r["terms"], r["terms_bound"])
    ga = g[:, 1].cpu().numpy().astype(np.float64)
    assert np.array_equal(np.isnan(ga), np.isnan(r["grad"])) and np.array_equal(np.isinf(ga), np.isinf(r["grad"]))
    fin = np.isfinite(r["grad"])
    assert np.all(np.abs(ga[fin] - r["grad"][fin]) <= r["grad_bound"][fin])
    others = g[:, [0, 2, 3, 4, 5, 6, 7]]
    assert float(others.abs().max()) == 0.0                  # only the alpha plane is touched


@pytest.mark.parametrize("name", CASES)
def test_kernels_match_reference_fixture_and_model(name, dev):
    from .conftest import load_golden
    from .mask_loss_model import mask_loss
    gd = load_golden(name)
    M, H, W = gd["in_alpha"].shape
    am = _allmap(gd["in_alpha"], dev)
    t = lambda k: torch.from_numpy(gd[k]).to(dev)  # noqa: E731
    call = _Call(M, H, W, dev)
    terms, counts, balance, g = call(am, t("in_mask"), t("in_vis2d"), t("in_is_detected"), t("in_weight"))
    torch.cuda.synchronize()
    # the reference's weights bit for bit where its sums are exact (binary masks)
    binary = np.isin(gd["in_mask"], (0.0, 1.0)).all()
    if gd["ref_branch"][0] and binary:
        assert np.array_equal(balance.cpu().numpy()[:2], [gd["ref_pos_wt"][0], gd["ref_neg_wt"][0]], equal_nan=True)
    assert float(balance[2]) == float(gd["ref_branch"][0])
    assert np.array_equal(counts.cpu().numpy(), gd["ref_counts"])
    # inf / NaN exactly where the reference has them
    loss, ref = float(terms.double().sum()), float(gd["ref_loss"][0])
    assert np.isnan(loss) == np.isnan(ref)
    rg = gd["ref_grad_alpha"]
    ga = g[:, 1].cpu().numpy()
    assert np.array_equal(np.isnan(ga), np.isnan(rg)) and np.array_equal(np.isinf(ga), np.isinf(rg))
    if not np.isnan(ref):
        assert abs(loss - ref) <= 2e-6 * abs(ref) + 1e-30, (loss, ref)
    r = mask_loss(gd["in_alpha"], gd["in_mask"], gd["in_vis2d"], gd["in_is_detected"], gd["in_weight"][0])
    _check_against_model(r, terms, counts, balance, g)
    # bit-identical from run to run
    first = [x.clone() for x in (terms, counts, balance, g)]
    again = call(am, t("in_mask"), t("in_vis2d"), t("in_is_detected"), t("in_weight"))
    for a, b in zip(first, again):
        assert torch.equal(a.nan_to_num(), b.nan_to_num()) and torch.equal(a.isnan(), b.isnan())


def _inputs(M, H, W, dev, seed, frac=False):
    g = torch.Generator(device=dev).manual_seed(seed)
    r = lambda: torch.rand((M, H, W), device=dev, generator=g)  # noqa: E731
    mask = (r() < 0.4).float() * (r() if frac else 1.0)
    vis = (r() < 0.9).float()
    alpha = r()
    alpha = torch.where(r() < 0.05, mask, alpha)
    det = (torch.rand((M,), device=dev, generator=g) < 0.8).float()
    det[0] = 1.0
    return alpha, mask, vis, det


@pytest.mark.parametrize("M,W,H,frac", [(2, 256, 256, False), (8, 512, 512, False), (3, 97, 33, True), (1, 1, 1, False)])
def test_kernels_match_model_at_full_size(M, W, H, frac, dev):
    from .mask_loss_model import mask_loss
    alpha, mask, vis, det = _inputs(M, H, W, dev, seed=M + W, frac=frac)
    am = _allmap(alpha, dev, seed=1)
    w = torch.tensor([0.1], device=dev)
    out = _Call(M, H, W, dev)(am, mask, vis, det, w)
    n = lambda x: x.cpu().numpy()  # noqa: E731
    r = mask_loss(n(alpha), n(mask), n(vis), n(det), 0.1)
    _check_against_model(r, *out)


def test_null_vis2d_and_is_detected_mean_all_ones(dev):
    alpha, mask, _, _ = _inputs(2, 40, 48, dev, seed=3)
    am = _allmap(alpha, dev)
    w = torch.tensor([0.1], device=dev)
    a = [x.clone() for x in _Call(2, 40, 48, dev)(am, mask, None, None, w)]
    b = _Call(2, 40, 48, dev)(am, mask, torch.ones_like(mask), torch.ones(2, device=dev), w)
    for x, y in zip(a, b):
        assert torch.equal(x, y)


def test_graph_replay_with_inputs_refilled_in_place_matches_eager(dev):
    M, H, W = 2, 40, 48
    alpha, mask, vis, det = _inputs(M, H, W, dev, seed=5)
    am = _allmap(alpha, dev)
    w = torch.tensor([0.1], device=dev)
    call = _Call(M, H, W, dev)
    call(am, mask, vis, det, w)                              # warm-up outside the capture
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        call(am, mask, vis, det, w)
    eager = _Call(M, H, W, dev)
    cases = [_inputs(M, H, W, dev, seed=s) + (wv,) for s, wv in ((6, 0.1), (7, 0.37), (8, 2.0))]
    a9, m9, v9, _ = _inputs(M, H, W, dev, seed=9)
    cases.append((a9, m9, v9, torch.zeros(M, device=dev), 0.5))      # no detected frame: NaN weights and loss
    for a2, m2, v2, d2, wv in cases:
        am[:, 1].copy_(a2); mask.copy_(m2); vis.copy_(v2); det.copy_(d2); w.fill_(wv)
        graph.replay()
        want = eager(am, mask, vis, det, w)
        torch.cuda.synchronize()
        for x, y in zip((call.terms, call.counts, call.balance, call.g), want):
            assert torch.equal(x.nan_to_num(), y.nan_to_num()) and torch.equal(x.isnan(), y.isnan()), wv
    assert bool(call.terms.isnan().all())


# ---------------------------------------------------------------------------------------------- render_loss_batch end to end
def _scene(P, W, H, M, dev, seed=31):
    from vidu4d_b200.renderer import make_camera, stack_cameras
    from vidu4d_b200.synthetic import SurfelCloud, object_scene, orbit_view
    cams = []
    for f in range(M):
        R, t = orbit_view(7 * f + 3, 64)
        cams.append(make_camera(W, H, 2 * np.arctan(0.5), 2 * np.arctan(0.5 * H / W), R=R.T, T=t, device=dev))
    scene = object_scene(P, seed=seed, center=(0.0, 0.0, 0.0))
    return stack_cameras(cams), lambda: SurfelCloud(scene, dev)


def _reference_mask_term(acc, mask, vis, det, w):
    """lab4d/engine/model.py:587-611,648-650,950-967,1000-1012 written in torch on out["allmap"][:, 1]."""
    vd = vis * det[:, None, None]
    if mask.sum() > 0 and (1 - mask).sum() > 0:
        pos_wt = vd.sum() / mask[vd > 0].sum()
        neg_wt = vd.sum() / (1 - mask[vd > 0]).sum()
        bw = 0.5 * pos_wt * mask + 0.5 * neg_wt * (1 - mask)
    else:
        bw = 1
    v = (acc - mask).pow(2) * bw * vis * det[:, None, None]
    return w * (v.mean() if int((v > 0).sum()) == 0 else v[v > 0].mean())


@pytest.mark.parametrize("w_ssim", [0.0, 0.2])
def test_render_loss_batch_mask_term_matches_torch(w_ssim, dev):
    """out["loss"] and the gradients reaching the surfels against the reference's statements on the alpha plane of the
    same rasterizer's differentiable batch forward (out["allmap"] itself is detached), backpropagated through the same
    rasterizer backward, to 1e-5 of each gradient's largest element (the rasterizer backward sums with float atomics).
    With w_ssim > 0 and a learnable background the SSIM term's dL/dalpha comes first."""
    from vidu4d_b200.rasterizer import GaussianRasterizationSettings, rasterize_gaussians_batch
    from vidu4d_b200.renderer import PipelineParams, _cam_tans, render_loss_batch
    M, P, W, H = 2, 50000, 128, 96
    bc, mk = _scene(P, W, H, M, dev)
    gen = torch.Generator(device=dev).manual_seed(3)
    rgb = torch.rand((M, 3, H, W), device=dev, generator=gen)
    vis = (torch.rand((M, H, W), device=dev, generator=gen) > 0.1).float()
    det = torch.tensor([1.0, 1.0], device=dev)
    w = torch.tensor([0.1], device=dev)
    kw = dict(vis2d=vis, w_rgb=0.8, lambda_normal=0.05, lambda_dist=10.0, w_ssim=w_ssim)
    pipe, bg = PipelineParams(), torch.zeros(3, device=dev)
    with torch.no_grad():
        pre = render_loss_batch(bc, mk(), pipe, bg, rgb, **kw)
    mask = (pre["allmap"][:, 1] > 0.5).float()
    assert 0 < float(mask.mean()) < 1

    def run(fused):
        cloud = mk()
        bk = torch.tensor([0.2, 0.3, 0.4], device=dev, requires_grad=True) if w_ssim else None
        extra = dict(is_detected=det, mask_loss_weight=w) if fused else {}
        out = render_loss_batch(bc, cloud, pipe, bg, rgb, mask_gt=mask, learnable_bkgd=bk, **kw, **extra)
        loss = out["loss"]
        if not fused:
            tx, ty = _cam_tans(bc)
            rs = GaussianRasterizationSettings(H, W, tx, ty, bg, 1.0, bc.world_view_transform, bc.full_proj_transform,
                                               cloud.active_sh_degree, bc.camera_center, False, False)
            _, _, allmap = rasterize_gaussians_batch(cloud.get_xyz, torch.zeros((M, P, 3), device=dev), cloud.get_features,
                                                     None, cloud.get_opacity, cloud.get_scaling, cloud.get_rotation, rs)
            assert torch.equal(allmap.detach(), out["allmap"])
            loss = loss + _reference_mask_term(allmap[:, 1], mask, vis, det, w[0])
        (1.7 * loss).backward()
        return out, loss.detach(), [p.grad for p in cloud.flat_params()] + ([bk.grad] if bk is not None else [])
    out_f, loss_f, g_f = run(True)
    out_t, loss_t, g_t = run(False)
    assert out_f["mask_terms"].shape == (M,) and not out_f["mask_terms"].requires_grad
    assert out_f["mask_counts"].dtype == torch.int32 and int(out_f["mask_counts"].min()) > 0
    assert ("ssim_terms" in out_f) == (w_ssim > 0)
    assert abs(float(loss_f) - float(loss_t)) <= 1e-6 * abs(float(loss_t)), (float(loss_f), float(loss_t))
    names = ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation", "bkgd")
    for name, a, b in zip(names, g_f, g_t):
        assert float(b.abs().max()) > 0, name
        assert float((a - b).abs().max()) <= 1e-5 * float(b.abs().max()), name


def test_without_mask_loss_weight_nothing_changes(dev):
    """Without mask_loss_weight the forward and backward launch what the parent commit launches (15 + 2) and out has the
    parent's keys; with it the forward adds the term's three kernels and two outputs, and the weight tensor is read at
    run time."""
    from vidu4d_b200 import _capi
    from vidu4d_b200.renderer import PipelineParams, render_loss_batch
    M, P, W, H = 2, 20000, 96, 64
    bc, mk = _scene(P, W, H, M, dev, seed=41)
    gen = torch.Generator(device=dev).manual_seed(4)
    rgb = torch.rand((M, 3, H, W), device=dev, generator=gen)
    mask = (torch.rand((M, H, W), device=dev, generator=gen) > 0.5).float()
    pipe, bg = PipelineParams(), torch.zeros(3, device=dev)

    def run(**extra):
        cloud = mk()
        lc = _capi.launch_count()
        out = render_loss_batch(bc, cloud, pipe, bg, rgb, mask_gt=mask, lambda_normal=0.05, **extra)
        torch.cuda.synchronize()
        n_fwd = _capi.launch_count() - lc
        lc = _capi.launch_count()
        out["loss"].backward()
        torch.cuda.synchronize()
        return out, n_fwd, _capi.launch_count() - lc
    run()
    o0, f0, b0 = run(w_mask=0.1)
    assert (f0, b0) == (15, 2)
    assert set(o0) == {"loss", "terms", "render", "allmap", "radii", "visibility_filter", "viewspace_points"}
    w = torch.tensor([0.0], device=dev)
    o1, f1, b1 = run(mask_loss_weight=w)
    assert (f1, b1) == (f0 + 3, b0) and set(o1) == set(o0) | {"mask_terms", "mask_counts"}
    assert float(o1["mask_terms"].abs().max()) == 0.0 and int(o1["mask_counts"].sum()) > 0
    assert torch.equal(o1["render"], o0["render"]) and torch.equal(o1["allmap"], o0["allmap"])
    w.fill_(0.25)
    o2, _, _ = run(mask_loss_weight=w)
    assert float(o2["mask_terms"].sum()) > 0
