"""GPU tests of the deterministic rasterizer backward (include/surfel_deterministic.h, DESIGN.md 3.4b).

  * run to run: at the headline size (300 K surfels, 512 x 512, M = 8, per-frame intrinsics), with F = 0 and F = 22 and
    with sum_shared off and on, two backward calls with another workload between them give the same bits in all nine
    gradient tensors;
  * batch independence: each frame's (M,P,.) gradients of the batch equal, bit for bit, a one-frame call on that frame
    -- the grid and the interleaving of the CTAs differ, so any order that depends on scheduling fails here;
  * correctness: the golden and constructed cases of test_gpu_grad_bounds.py and test_gpu_feature_bounds.py (dense and
    overflowing chunks included) stay within their K u B' bound against the oracle, with the accumulator term counting
    one add per tile touched and no pair past the buffer (the deterministic path has no direct path);
  * the trigger: torch.use_deterministic_algorithms(True) or set_deterministic(True) selects the deterministic kernels,
    neither runs the default ones;
  * capture: a GraphedStep of render_loss_batch with F = 22 feature losses (scratch allocated inside the capture)
    replays the eager step's gradient bit for bit;
  * training: two 30-step Stage-3 runs -- render_loss_batch with F = 22 feature losses and no learnable background,
    FlatSurfelModel clip_grad_norm_ + step(), densify_and_prune every 10 steps -- have the same P and the same flat
    buffers after every step.
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

NAMES = ("dL_dmeans2D", "dL_dcolors", "dL_dopacity", "dL_dmeans3D", "dL_dtransMat", "dL_dsh", "dL_dscales", "dL_drotations",
         "dL_dfeatures")


@pytest.fixture(scope="module")
def dev(built):
    from vidu4d_b200 import _capi
    _capi.load()
    return torch.device("cuda:0")


@pytest.fixture
def det():
    from vidu4d_b200 import rasterizer as RZ
    RZ.set_deterministic(True)
    yield
    RZ.set_deterministic(False)


def _headline(dev, M=8, P=300_000, res=512, F=0, seed=0):
    """Stage-3-like batch: per-frame positions and orientations, shared SH / opacities / scales / features, one orbit
    camera and one (tan, tan, cx_off, cy_off) row per frame."""
    from vidu4d_b200.synthetic import object_scene, orbit_view, projection_matrix
    sc = object_scene(P, seed=seed, opacity="trained", center=(0.0, 0.0, 0.0))
    t = sc.to_torch(dev)
    g = torch.Generator(device=dev).manual_seed(seed + 7)
    Pm = projection_matrix(0.5, 0.5).astype(np.float64)
    vms, pms, cps = [], [], []
    for f in range(M):
        R, tr = orbit_view(5 * f, 64)
        W2C = np.eye(4); W2C[:3, :3] = R; W2C[:3, 3] = tr
        vms.append(W2C.T.astype(np.float32)); pms.append((W2C.T @ Pm).astype(np.float32)); cps.append((-R.T @ tr).astype(np.float32))
    vms, pms, cps = (torch.from_numpy(np.stack(a)).to(dev) for a in (vms, pms, cps))
    intr = torch.tensor([[0.5 + 0.01 * f, 0.5 - 0.005 * f, 1.5 * f - 4.0, 3.0 - f] for f in range(M)], dtype=torch.float32, device=dev)
    means = torch.stack([t["means3D"] + 0.003 * f * torch.randn((P, 3), device=dev, generator=g) for f in range(M)])
    rots = torch.stack([torch.nn.functional.normalize(t["rotations"] + 0.02 * f * torch.randn((P, 4), device=dev, generator=g), dim=-1)
                        for f in range(M)])
    feats = torch.randn((P, F), device=dev, generator=g) if F else None
    bg = torch.tensor([0.2, 0.1, 0.4] + [0.05 * i for i in range(F)], device=dev)
    dLc = torch.randn((M, 3 + F, res, res), device=dev, generator=g)
    dLo = 0.1 * torch.randn((M, 8, res, res), device=dev, generator=g)
    return dict(t=t, means=means, rots=rots, feats=feats, bg=bg, vms=vms, pms=pms, cps=cps, intr=intr, dLc=dLc, dLo=dLo, M=M, res=res)


def _fwd(h, f=None):
    from vidu4d_b200.rasterizer import _C
    e = torch.empty((0,), device=h["bg"].device)
    sl = (lambda x: x[f:f + 1]) if f is not None else (lambda x: x)
    kw = {"features": h["feats"]} if h["feats"] is not None else {}
    out = _C.rasterize_gaussians_batch(h["bg"], sl(h["means"]), e, h["t"]["opacities"], h["t"]["scales"], sl(h["rots"]), 1.0,
                                       sl(h["vms"]), sl(h["pms"]), 0.5, 0.5, h["res"], h["res"], h["t"]["shs"], 3, sl(h["cps"]),
                                       intrinsics=sl(h["intr"]), **kw)
    return out[3:7]


def _bwd(h, fw, sum_shared, f=None):
    from vidu4d_b200.rasterizer import _C
    e = torch.empty((0,), device=h["bg"].device)
    sl = (lambda x: x[f:f + 1]) if f is not None else (lambda x: x)
    radii, gb, bb, ib = fw
    kw = {"features": h["feats"]} if h["feats"] is not None else {}
    g = _C.rasterize_gaussians_backward_batch(h["bg"], sl(h["means"]), radii, e, h["t"]["scales"], sl(h["rots"]), 1.0,
                                              sl(h["vms"]), sl(h["pms"]), 0.5, 0.5, sl(h["dLc"]), sl(h["dLo"]), h["t"]["shs"], 3,
                                              sl(h["cps"]), gb, bb, ib, sum_shared=sum_shared, want_transmat=True,
                                              intrinsics=sl(h["intr"]), **kw)
    return dict(zip(NAMES, g))


def _same(a, b, what):
    for k in a:
        if a[k] is None:
            assert b[k] is None, (what, k)
            continue
        assert a[k].shape == b[k].shape, (what, k)
        n = int((a[k].view(torch.int32) != b[k].view(torch.int32)).sum())
        assert n == 0, f"{what}: {k} differs in {n} of {a[k].numel()} elements"


@pytest.mark.parametrize("F", [0, 22])
@pytest.mark.parametrize("sum_shared", [False, True], ids=["per_frame_grads", "sum_shared"])
def test_run_to_run_headline(F, sum_shared, dev, det):
    h = _headline(dev, F=F)
    fw = _fwd(h)
    first = _bwd(h, fw, sum_shared)
    # another workload between the two calls: a different upstream gradient through the default and the deterministic path
    from vidu4d_b200 import rasterizer as RZ
    h2 = dict(h, dLc=h["dLc"].flip(-1).contiguous(), dLo=h["dLo"].flip(-2).contiguous())
    RZ.set_deterministic(False)
    _bwd(h2, fw, not sum_shared)
    RZ.set_deterministic(True)
    _bwd(h2, fw, sum_shared)
    second = _bwd(h, fw, sum_shared)
    torch.cuda.synchronize()
    _same(first, second, f"F={F} sum_shared={sum_shared}")
    assert float(first["dL_dmeans3D"].abs().sum()) > 0 and (F == 0 or float(first["dL_dfeatures"].abs().sum()) > 0)


PER_FRAME = ("dL_dmeans2D", "dL_dtransMat", "dL_dmeans3D", "dL_drotations")   # per frame in _headline's batch


@pytest.mark.parametrize("F", [0, 22])
@pytest.mark.parametrize("sum_shared", [False, True], ids=["per_frame_grads", "sum_shared"])
def test_batch_equals_single_frame_bits(F, sum_shared, dev, det):
    """Every (M,P,.) gradient of the batch -- all nine without frame sums; with SR_BATCH_SUM_SHARED the four that stay
    per frame -- equals the one-frame call on that frame."""
    h = _headline(dev, F=F, seed=3)
    fw = _fwd(h)
    batch = _bwd(h, fw, sum_shared)
    for f in range(h["M"]):
        one = _bwd(h, _fwd(h, f), False, f)
        keys = [k for k in one if one[k] is not None and (not sum_shared or k in PER_FRAME)]
        assert len(keys) == (4 if sum_shared else 8 + (F > 0))
        _same({k: one[k] for k in keys}, {k: batch[k][f:f + 1] for k in keys}, f"frame {f}")


def test_deterministic_close_to_default(dev):
    """Same terms, other summation order: the two modes agree to a few ulps of the gradient's magnitude."""
    from vidu4d_b200 import rasterizer as RZ
    h = _headline(dev, F=22, M=2, P=50_000, res=256, seed=5)
    fw = _fwd(h)
    ref = _bwd(h, fw, True)
    RZ.set_deterministic(True)
    try:
        got = _bwd(h, fw, True)
    finally:
        RZ.set_deterministic(False)
    for k in ref:
        if ref[k] is None:
            continue
        scale = float(ref[k].abs().max()) + 1e-30
        assert float((got[k] - ref[k]).abs().max()) <= 1e-4 * scale, k


def _kernels(fn):
    from vidu4d_b200 import _capi
    _capi.set_profiling(True)
    try:
        _capi.get_profile()
        fn()
        return set(_capi.get_profile())
    finally:
        _capi.set_profiling(False)


def test_trigger(dev):
    from vidu4d_b200 import _capi
    from vidu4d_b200 import rasterizer as RZ
    h = _headline(dev, F=8, M=2, P=20_000, res=128, seed=9)
    fw = _fwd(h)
    was = torch.are_deterministic_algorithms_enabled()
    det_names = {"det_zero", "composite_bwd_det", "feature_bwd_det", "det_gather", "surfel_bwd"}
    try:
        torch.use_deterministic_algorithms(False)
        RZ.set_deterministic(False)
        n0 = _capi.launch_count()
        default = _kernels(lambda: _bwd(h, fw, True))
        n_default = _capi.launch_count() - n0
        assert default == {"composite_bwd", "feature_bwd", "surfel_bwd"} and n_default == 3
        torch.use_deterministic_algorithms(True)
        n0 = _capi.launch_count()
        assert _kernels(lambda: _bwd(h, fw, True)) == det_names
        assert _capi.launch_count() - n0 == 5
        torch.use_deterministic_algorithms(False)
        RZ.set_deterministic(True)
        assert _kernels(lambda: _bwd(h, fw, True)) == det_names
    finally:
        torch.use_deterministic_algorithms(was)
        RZ.set_deterministic(False)


# ---- the oracle bounds of test_gpu_grad_bounds.py / test_gpu_feature_bounds.py, run through the deterministic path --
def _no_fallback(monkeypatch):
    """The accumulator term of the bound without pairs past the buffer: each slot sum is one add per tile touched."""
    from . import test_gpu_feature_bounds as FB
    from . import test_gpu_grad_bounds as GB

    def bounds(st, og, dec):
        from oracle import surfel_oracle as so
        adds = GB._np(dec["tiles_touched"]).astype(np.float64)
        B = og["bound"] + (adds[:, None] + GB.CHAIN) * og["asum"]
        return {k: GB.K * GB.U * v for k, v in so.chain_bound(st, B).items()}
    monkeypatch.setattr(GB, "_bounds", bounds)
    monkeypatch.setattr(FB, "_bounds", bounds)
    monkeypatch.setattr(FB, "_fallback_pairs", lambda dec, P: np.zeros(P))

    def total(fr, dec, m_feat, F, zero_features=False):
        """test_gpu_feature_bounds._total for this path: the feature pass adds each pair's geometry terms into the slot
        once (m_feat adds, not n_chunks m_feat), and forms one F-channel dL/dalpha sum per pair, so its unmodelled
        roundings are F u asum (SLACK = F instead of 8)."""
        from oracle import surfel_oracle as so
        st = fr["st"]
        acc, bnd, asm = (fr["og_c"][k].copy() for k in ("acc", "bound", "asum"))
        for og in fr["og_g"]:
            for dst, k in ((acc, "acc"), (bnd, "bound"), (asm, "asum")):
                a = og[k].copy()
                a[:, FB.C3] = 0.0
                dst += a
        ref = so.chain(st, acc)
        if zero_features:
            assert not any(og["acc"].any() for og in fr["og_g"])
            return ref, bounds(st, fr["og_c"], dec)
        adds = FB._np(dec["tiles_touched"]).astype(np.float64) + m_feat + GB.CHAIN + F
        return ref, {k: GB.K * GB.U * v for k, v in so.chain_bound(st, bnd + adds[:, None] * asm).items()}
    monkeypatch.setattr(FB, "_total", total)


GRAD_CASES = ([("golden", n) for n in ("id_deg3_64", "rigid_bg_96x64", "ragged_80x48_deg1", "precomp_init_70x50",
                                       "big_surfels_64", "near_cull_64", "single_32")]
              + [("constructed", n) for n in ("exact_lengths", "dense", "long_overflow")]
              + [("batch8", None), ("batch5", None)])


@pytest.mark.parametrize("kind,name", GRAD_CASES)
def test_grad_bounds_deterministic(kind, name, dev, det, monkeypatch):
    from . import test_gpu_grad_bounds as GB
    _no_fallback(monkeypatch)
    if kind == "golden":
        GB.test_golden(name, dev)
    elif kind == "constructed":
        GB.test_constructed_scene(name, dev)      # the dense cases overflow the pair buffer: they run in passes here
    elif kind == "batch8":
        GB.test_batch8_per_frame_positions(dev)
    else:
        GB.test_batch5_empty_and_two_surfel_frames(dev)


FEATURE_CASES = [("grid", ("id_deg3_64", 22)), ("grid", ("oracle_seed21_256", 32)), ("grid", ("rigid_bg_96x64", 7)),
                 ("long", ("long_lists_50k_32", 8)), ("long", ("long_lists_50k_32", 32)), ("long", ("warp_stop", 22)),
                 ("lowpass", None), ("bg", "3+F"), ("batch3", False), ("batch3", True)]


@pytest.mark.parametrize("kind,arg", FEATURE_CASES)
def test_feature_bounds_deterministic(kind, arg, dev, det, monkeypatch):
    from . import test_gpu_feature_bounds as FB
    _no_fallback(monkeypatch)
    if kind == "grid":
        FB.test_feature_width_grid(*arg, dev)
    elif kind == "long":
        FB.test_long_lists_and_early_stops(*arg, dev)
    elif kind == "lowpass":
        FB.test_lowpass_pairs(dev)
    elif kind == "bg":
        FB.test_background(arg, dev)
    else:
        FB.test_batch3(arg, dev)


# ---- capture and a Stage-3 training run ------------------------------------------------------------------------------
E2E_NF, E2E_P, E2E_W, E2E_H, E2E_STEPS = 4, 40000, 256, 192, 30


def _e2e(dev, seed=0):
    """A FlatSurfelModel with the registration feature, four orbit cameras and its targets: RGB, silhouette, 16 feature
    channels; the rendered features are [regist (16) | 6 fixed channels], F = 22, the Gaussian mask in channel 21."""
    from vidu4d_b200.renderer import make_camera, stack_cameras
    from vidu4d_b200.surfel_store import FlatSurfelModel
    from vidu4d_b200.synthetic import object_scene, orbit_view
    sc = object_scene(E2E_P, seed=seed, center=(0.0, 0.0, 0.0))
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    op = np.clip(sc.opacities, 1e-6, 1 - 1e-6)
    g = torch.Generator(device=dev).manual_seed(seed + 1)
    model = FlatSurfelModel(t(sc.means3D), t(sc.shs[:, :1]), t(sc.shs[:, 1:]), t(np.log(op / (1 - op))), t(np.log(sc.scales)),
                            t(sc.rotations), lrs={"xyz": 1e-5, "f_dc": 1e-3, "f_rest": 1e-4, "opacity": 1e-2, "scaling": 1e-3,
                                                  "rotation": 1e-3},
                            regist_feat=torch.randn((E2E_P, 16), device=dev, generator=g) * 0.1)
    cams = []
    for f in range(E2E_NF):
        R, tr = orbit_view(9 * f + 2, 64)
        cams.append(make_camera(E2E_W, E2E_H, 2 * np.arctan(0.5), 2 * np.arctan(0.375), R=R.T, T=tr, device=dev))
    data = dict(cams=stack_cameras(cams), bg=torch.zeros(3, device=dev),
                rgb=torch.rand((E2E_NF, 3, E2E_H, E2E_W), device=dev, generator=g),
                mask=(torch.rand((E2E_NF, E2E_H, E2E_W), device=dev, generator=g) > 0.5).float(),
                ftgt=torch.randn((E2E_NF, 16, E2E_H, E2E_W), device=dev, generator=g) * 0.3,
                det=torch.ones(E2E_NF, device=dev), w=torch.tensor([1e-2, 1e-2], device=dev))
    return model, data


def _e2e_loss(model, d):
    from vidu4d_b200.renderer import PipelineParams, render_loss_batch
    P = model.P
    extra = torch.arange(6 * P, device=model.flat.device, dtype=torch.float32).view(P, 6).remainder(7.0) * 0.05
    feats = torch.cat([model._regist_feat, extra], 1)
    out = render_loss_batch(d["cams"], model, PipelineParams(), d["bg"], d["rgb"], mask_gt=d["mask"], w_mask=0.1,
                            lambda_normal=0.05, lambda_dist=0.01, features=feats, feature_target=d["ftgt"],
                            is_detected=d["det"], gauss_mask_channel=21, feature_loss_weights=d["w"])
    out["loss"].backward()
    return out


def test_graphed_step_equals_eager(dev, det):
    from vidu4d_b200 import rasterizer as RZ
    from vidu4d_b200.graph import GraphedStep
    model, d = _e2e(dev, seed=4)

    def body():
        model.zero_grad_flat()
        _e2e_loss(model, d)
    try:
        body()
        torch.cuda.synchronize()
        eager = model.grad_flat.clone()
        assert float(eager.abs().max()) > 0
        step = GraphedStep(body, device=dev)
        for _ in range(2):
            step()
            torch.cuda.synchronize()
            n = int((model.grad_flat.view(torch.int32) != eager.view(torch.int32)).sum())
            assert n == 0, f"replay differs from the eager step in {n} of {eager.numel()} gradient elements"
    finally:
        RZ._pending.clear()
        RZ.set_sync_mode(True)


def test_two_training_runs_stay_bit_identical(dev, det):
    """Two runs, stepped in lockstep: after every step the same P and the same flat buffer (parameters), Adam state and
    densification statistics.  Each densification's gradient threshold is the 80th percentile of that run's own
    statistic, so decisions sit on the threshold, where one ulp of difference would flip them."""
    runs = [_e2e(dev, seed=2), _e2e(dev, seed=2)]
    grown = 0
    for step in range(E2E_STEPS):
        for model, d in runs:
            model.zero_grad_flat()
            out = _e2e_loss(model, d)
            model.add_densification_stats(out["viewspace_points"].grad, out["visibility_filter"], out["radii"])
            model.clip_grad_norm_(1.0)
            model.step()
            if step % 10 == 9:
                ratio = torch.nan_to_num(model.xyz_gradient_accum[:, 0] / model.denom[:, 0], nan=0.0)
                thr = float(torch.quantile(ratio[model.denom[:, 0] > 0], 0.8))
                P0 = model.P
                model.densify_and_prune(thr, 0.005, 0.55, None, generator=torch.Generator(device=dev).manual_seed(step))
                if model is runs[0][0]:
                    grown += model.P != P0
        a, b = runs[0][0], runs[1][0]
        torch.cuda.synchronize()
        assert a.P == b.P, f"step {step}: P {a.P} vs {b.P}"
        for name in ("flat", "exp_avg", "exp_avg_sq", "densify_stats"):
            x, y = getattr(a, name), getattr(b, name)
            n = int((x.view(torch.int32) != y.view(torch.int32)).sum())
            assert n == 0, f"step {step}: {name} differs in {n} of {x.numel()} elements"
    assert grown >= 2, f"only {grown} of the 3 densifications changed P"
