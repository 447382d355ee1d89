"""GPU tests of the optimizer step with its state on the device (include/surfel_optim.h, csrc/optim.cu;
FlatSurfelModel.clip_grad_norm_ / step): the group sums and norm against a float64 oracle, the clip coefficient against
torch's own expression, the Adam pass against sr_adam_flat bit for bit, the pair against torch.nn.utils.clip_grad_norm_
+ torch.optim.Adam, and a captured step whose replays advance the step count on their own."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

NAMES = ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation", "regist_feat")


@pytest.fixture(scope="module")
def dev(built):
    from vidu4d_b200 import _capi
    _capi.load()
    return torch.device("cuda:0")


def _model(P, dev, seed=0, regist=True):
    from vidu4d_b200.surfel_store import FlatSurfelModel
    from vidu4d_b200.synthetic import object_scene
    sc = object_scene(P, seed=seed, center=(0.0, 0.0, 0.0))
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    op = np.clip(sc.opacities, 1e-6, 1 - 1e-6)
    rf = torch.randn((P, 16), device=dev, generator=torch.Generator(device=dev).manual_seed(seed)) * 0.1 if regist else None
    return FlatSurfelModel(t(sc.means3D), t(sc.shs[:, :1]), t(sc.shs[:, 1:]), t(np.log(op / (1 - op))), t(np.log(sc.scales)),
                           t(sc.rotations), regist_feat=rf)


def _fill_grads(m, seed, scale=1.0):
    """Seeded gradients whose size differs by group (1e-4 .. 1e2), scaled by `scale`."""
    g = torch.Generator(device=m.flat.device).manual_seed(seed)
    off, total = m._offsets(m.P)
    for q, (a, b) in enumerate(zip(off, off[1:] + [total])):
        m.grad_flat[a:b].copy_(torch.randn((b - a,), device=m.flat.device, generator=g) * (10.0 ** (q - 4)) * scale)


def _grad_norm(m, grad_scale, extra_norms, max_norm):
    """sr_grad_norm_flat on m's gradient buffer: (total, coef, group sums of squares)."""
    from vidu4d_b200 import _capi
    dev, n = m.flat.device, len(m.groups)
    scratch = torch.empty((int(_capi.load().sr_grad_norm_scratch_bytes(n)),), dtype=torch.uint8, device=dev)
    total, coef = torch.empty((), device=dev), torch.empty((), device=dev)
    sums = torch.empty((n,), dtype=torch.float64, device=dev)
    _capi.call("sr_grad_norm_flat", dev, n, m._begin(), m.grad_flat, float(grad_scale), extra_norms,
               0 if extra_norms is None else extra_norms.numel(), float(max_norm), total, coef, sums, scratch, scratch.numel())
    return total, coef, sums


@pytest.mark.parametrize("P,regist", [(5003, False), (1, True), (300000, True)])
def test_group_sums_and_norm_match_float64(P, regist, dev):
    """Each group's sum of squares within 2 n u64 of a float64 oracle (both are sums of n exact non-negative squares);
    the norm within one fp32 ulp of the float64 norm (one rounding of a float64 value whose own error is ~1e-9 ulp).
    Bit-identical over repeated calls and on another stream.  P odd or 1: groups start inside a float4."""
    m = _model(P, dev, seed=P % 97, regist=regist)
    _fill_grads(m, seed=3)
    gs = 0.37
    extras = torch.tensor([0.5, 3.0, 1e-3], device=dev)
    total, coef, sums = _grad_norm(m, gs, extras, 5.0)
    off, tot = m._offsets(m.P)
    x = (m.grad_flat * gs).double()                     # the fp32 products, squared exactly in float64
    want = torch.stack([x[a:b].square().sum() for a, b in zip(off, off[1:] + [tot])])
    n = torch.tensor([b - a for a, b in zip(off, off[1:] + [tot])], dtype=torch.float64, device=dev)
    assert bool(((sums - want).abs() <= 2 * n * 2.0 ** -53 * want).all()), (sums, want)
    ref = float(torch.sqrt(want.sum() + extras.double().square().sum()))
    assert abs(float(total) - ref) <= float(np.spacing(np.float32(ref))), (float(total), ref)
    for _ in range(3):
        t2, c2, s2 = _grad_norm(m, gs, extras, 5.0)
        assert torch.equal(t2, total) and torch.equal(c2, coef) and torch.equal(s2, sums)
    side = torch.cuda.Stream(device=dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        t3, c3, s3 = _grad_norm(m, gs, extras, 5.0)
    torch.cuda.current_stream(dev).wait_stream(side)
    assert torch.equal(t3, total) and torch.equal(c3, coef) and torch.equal(s3, sums)


def test_coefficient_is_torch_expression_bit_for_bit(dev):
    """Given the same total, the coefficient equals torch's clamp(max_norm / (total + 1e-6), max=1) on a CUDA fp32 0-d
    tensor, bit for bit: totals over 80 decades, around max_norm, 0, Inf, NaN.  A zero gradient buffer and one extra norm
    T make the kernel's total exactly T (T^2 and its square root are exact in float64)."""
    m = _model(1, dev, regist=False)
    m.grad_flat.zero_()
    g = torch.Generator(device=dev).manual_seed(9)
    Ts = torch.cat([10.0 ** (torch.rand(400, device=dev, generator=g) * 80 - 40),
                    5.0 * (1 + (torch.rand(200, device=dev, generator=g) - 0.5) * 1e-5),
                    torch.tensor([0.0, 5.0, 5.0 - 1e-6, 4.999999, float("inf"), float("nan")], device=dev)]).float()
    for max_norm in (5.0, 0.1, 1.0):
        got_t, got_c = [], []
        for T in Ts:
            t, c, _ = _grad_norm(m, 1.0, T.reshape(1).clone(), max_norm)
            got_t.append(t)
            got_c.append(c)
        got_t, got_c = torch.stack(got_t), torch.stack(got_c)
        assert bool(((got_t == Ts) | (Ts.isnan() & got_t.isnan())).all())
        want = torch.stack([torch.clamp(max_norm / (T + 1e-6), max=1.0) for T in Ts])
        same = (got_c.view(torch.int32) == want.view(torch.int32)) | (want.isnan() & got_c.isnan())
        assert bool(same.all()), (max_norm, Ts[~same], got_c[~same], want[~same])


def test_step_matches_sr_adam_flat_bit_for_bit(dev):
    """Without a clip, step() gives the parameters and moments adam_step() gives at the same step numbers; with one,
    the same bits as grad_flat.mul_(grad_scale).mul_(coef) followed by adam_step().  Device counter = host counter."""
    a, b = _model(5003, dev, seed=2), _model(5003, dev, seed=2)
    gs = 0.3
    for k in range(8):
        clip = k % 2 == 1
        for m in (a, b):
            m.zero_grad_flat()
            _fill_grads(m, seed=10 + k)
        if clip:
            a.clip_grad_norm_(1e-2, grad_scale=gs)
            assert float(a.clip_coef) < 1.0
            a.step(grad_scale=gs)
            b.grad_flat.mul_(gs).mul_(a.clip_coef)
            b.adam_step(1.0)
        else:
            a.step(grad_scale=gs)
            b.grad_flat.mul_(gs)
            b.adam_step(1.0)
        assert int(a.device_step) == b.step_count == k + 1
        for x, y in ((a.flat, b.flat), (a.exp_avg, b.exp_avg), (a.exp_avg_sq, b.exp_avg_sq)):
            assert torch.equal(x, y), k


def test_step_without_surfels_still_counts(dev):
    from vidu4d_b200 import _capi
    buf = torch.zeros(4, device=dev)
    step = torch.tensor(41, dtype=torch.int64, device=dev)
    lr = torch.ones(2, device=dev)
    begin = (C.c_int64 * 3)(0, 0, 0)
    _capi.call("sr_adam_flat_state", dev, 2, begin, lr, 0.9, 0.999, 1e-15, step, 1.0, None, buf, buf, buf, buf)
    assert int(step) == 42 and float(buf.abs().sum()) == 0.0


def test_bias_corrections_equal_host_formula_to_step_100000(dev):
    """Every step 1..100 000: step() from a reset parameter buffer gives the bits adam_step() gives, so the device's bias
    corrections equal the host formula's.  Seven rates and varied moments make a different bc1 or sqrt_bc2 show; the
    parameters are reset each step so that an update never falls below half an ulp of them."""
    a, b = _model(16, dev, seed=5), _model(16, dev, seed=5)
    _fill_grads(a, seed=1)
    b.grad_flat.copy_(a.grad_flat)
    p0 = a.flat.clone()
    bad = torch.zeros((), dtype=torch.int64, device=dev)
    for t in range(1, 100001):
        a.flat.copy_(p0)
        b.flat.copy_(p0)
        a.step()
        b.adam_step()
        bad += (a.flat != b.flat).sum()
    assert int(a.device_step) == b.step_count == 100000
    assert int(bad) == 0


def test_clip_and_step_match_torch_clip_and_adam(dev):
    """clip_grad_norm_(5.0, extras) + step() against torch.nn.utils.clip_grad_norm_ + torch.optim.Adam (seven groups
    plus the extras, eps 1e-15) over ten steps, clipping on alternate steps, each step from torch's parameters and
    moments: the surfel moments bit for bit and each surfel parameter within the rounding of the fp32 rate
    (tests/optim_model.py rate_rounding_ok).  Where the totals differ in their last bits, so that torch's coefficient is
    not the kernel's, torch's Adam gets the kernel's coefficient."""
    from . import optim_model as om
    m = _model(5003, dev, seed=4)
    gen = torch.Generator(device=dev).manual_seed(2)
    extras = [torch.nn.Parameter(torch.rand(3, device=dev, generator=gen)),          # a learnable background
              torch.nn.Parameter(torch.randn((64, 32), device=dev, generator=gen)),
              torch.nn.Parameter(torch.randn(5, device=dev, generator=gen))]          # one without a gradient
    ref = [p.detach().clone().requires_grad_(True) for p in m.flat_params()]
    ref_x = [p.detach().clone().requires_grad_(True) for p in extras]
    opt_ref = torch.optim.Adam([{"params": [p], "lr": m.lrs[n]} for p, n in zip(ref, NAMES)]
                               + [{"params": [p], "lr": 1e-3} for p in ref_x], lr=0.0, eps=1e-15)
    opt_x = torch.optim.Adam([{"params": [p], "lr": 1e-3} for p in extras], lr=0.0, eps=1e-15)
    for step in range(10):
        scale = 1.0 if step % 2 == 0 else 1e-4
        m.zero_grad_flat()
        _fill_grads(m, seed=20 + step, scale=scale)
        with torch.no_grad():
            for p, r in zip(m.flat_params(), ref):
                p.copy_(r)
            if step:
                m.exp_avg.copy_(torch.cat([opt_ref.state[r]["exp_avg"].flatten() for r in ref]))
                m.exp_avg_sq.copy_(torch.cat([opt_ref.state[r]["exp_avg_sq"].flatten() for r in ref]))
        before = [r.detach().clone() for r in ref]
        for p, r in zip(m.flat_params(), ref):
            r.grad = p.grad.detach().clone()
        raw = [r.grad.clone() for r in ref]
        for i, (p, r) in enumerate(zip(extras, ref_x)):
            if i == 2:
                p.grad = r.grad = None
                continue
            gr = torch.randn(p.shape, device=dev, generator=gen) * scale
            p.grad, r.grad = gr.clone(), gr.clone()
        total = m.clip_grad_norm_(5.0, extras)
        total_ref = torch.nn.utils.clip_grad_norm_(ref + ref_x, 5.0)
        assert abs(float(total) - float(total_ref)) <= 1e-6 * float(total_ref), step
        assert (float(m.clip_coef) < 1.0) == (step % 2 == 0), (step, float(total))
        if not bool(torch.clamp(5.0 / (total_ref + 1e-6), max=1.0) == m.clip_coef):
            for r, g0 in zip(ref, raw):
                r.grad = g0 * m.clip_coef
        m.step()
        opt_x.step()
        opt_ref.step()
        off, tot = m._offsets(m.P)
        for p, r, n, b, a, e in zip(m.flat_params(), ref, NAMES, before, off, off[1:] + [tot]):
            assert torch.equal(m.exp_avg[a:e], opt_ref.state[r]["exp_avg"].flatten()), (step, n)
            assert torch.equal(m.exp_avg_sq[a:e], opt_ref.state[r]["exp_avg_sq"].flatten()), (step, n)
            assert om.rate_rounding_ok(p.detach().cpu().numpy(), r.detach().cpu().numpy(), b.cpu().numpy()).all(), (step, n)
        for p, r, n in zip(extras, ref_x, ("bkgd", "x", "no_grad")):
            p, r = p.detach(), r.detach()
            assert float((p - r).abs().max()) <= 1e-6 * float(r.abs().max()) + 1e-9, (step, n)
    assert int(m.device_step) == 10


def _scene(P, W, H, M, dev, seed=31):
    from vidu4d_b200.renderer import make_camera, stack_cameras
    from vidu4d_b200.synthetic import orbit_view
    cams = []
    for f in range(M):
        R, t = orbit_view(7 * f + 3, 64)
        cams.append(make_camera(W, H, 2 * np.arctan(0.5), 2 * np.arctan(0.5 * H / W), R=R.T, T=t, device=dev))
    return stack_cameras(cams)


def _close(a, b, tol):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).abs().max()) <= tol * float(b.abs().max()) + 1e-30


def test_graphed_step_advances_its_step_count(dev):
    """render_loss_batch -> backward -> clip_grad_norm_ -> step() as one CUDA graph.  Every replay matches an eager step
    from the same parameters and moments whose own device counter has advanced by itself (no rewinding): same loss and
    gradients, and the same update, which a bias correction frozen at capture would change by several percent.  The
    counter equals eager steps plus replays, survives densify_and_prune and reset_opacity, and the re-capture continues
    from it."""
    from vidu4d_b200 import rasterizer as RZ
    from vidu4d_b200.graph import GraphedStep
    from vidu4d_b200.renderer import PipelineParams, render_loss_batch
    M, P, W, H = 2, 20000, 96, 96
    bc = _scene(P, W, H, M, dev, seed=51)
    gen = torch.Generator(device=dev).manual_seed(6)
    rgb = torch.rand((M, 3, H, W), device=dev, generator=gen)
    mask = (torch.rand((M, H, W), device=dev, generator=gen) > 0.4).float()
    pipe, bg = PipelineParams(), torch.zeros(3, device=dev)
    mg, me = _model(P, dev, seed=7), _model(P, dev, seed=7)
    bkg, bke = (torch.nn.Parameter(torch.full((3,), 0.2, device=dev)) for _ in range(2))
    for b in (bkg, bke):
        b.grad = torch.zeros(3, device=dev)
    max_norm = [None]

    def body(m, bk, out):
        m.zero_grad_flat()
        bk.grad.zero_()
        res = render_loss_batch(bc, m, pipe, bg, rgb, mask_gt=mask, w_mask=0.1, learnable_bkgd=bk)
        res["loss"].backward()
        out[1].copy_(m.clip_grad_norm_(max_norm[0], [bk]))
        m.step()
        out[0].copy_(res["loss"].detach())

    def eager(m, bk, out, n=1):
        RZ.set_sync_mode(True)
        for _ in range(n):
            body(m, bk, out)
        RZ.set_sync_mode(False)

    og, oe = [torch.zeros((), device=dev), torch.zeros((), device=dev)], [torch.zeros((), device=dev), torch.zeros((), device=dev)]
    try:
        # a max_norm below the scene's gradient norm, so that every step clips
        max_norm[0] = float("inf")
        me.zero_grad_flat()
        render_loss_batch(bc, me, pipe, bg, rgb, mask_gt=mask, w_mask=0.1, learnable_bkgd=bke)["loss"].backward()
        max_norm[0] = 0.5 * float(me.clip_grad_norm_(float("inf"), [bke]))
        me.zero_grad_flat()
        assert max_norm[0] > 0

        step = GraphedStep(lambda: body(mg, bkg, og), key=lambda: (mg.P, mg.active_sh_degree), device=dev)
        step()
        eager(me, bke, oe, n=5)                        # as many eager bodies as the capture ran, plus its replay
        assert int(mg.device_step) == int(me.device_step) == 5 and step.captures == 1

        def replay_vs_eager():
            for a, b in ((me.flat, mg.flat), (me.exp_avg, mg.exp_avg), (me.exp_avg_sq, mg.exp_avg_sq)):
                a.copy_(b)
            before = mg.flat.clone()
            step()
            eager(me, bke, oe)
            assert int(mg.device_step) == int(me.device_step)
            assert float(mg.clip_coef) < 1.0 and float(me.clip_coef) < 1.0
            assert abs(float(og[0]) - float(oe[0])) <= 1e-5 * abs(float(oe[0]))
            assert abs(float(og[1]) - float(oe[1])) <= 1e-4 * float(oe[1])
            assert _close(mg.grad_flat, me.grad_flat, 1e-4) and _close(bkg.grad, bke.grad, 1e-4)
            off, total = mg._offsets(mg.P)
            for n, a, b in zip(NAMES, off, off[1:] + [total]):
                assert _close(mg.flat[a:b] - before[a:b], me.flat[a:b] - before[a:b], 1e-3), n
        for k in range(3):
            replay_vs_eager()
            assert int(mg.device_step) == 6 + k and step.captures == 1

        n0 = int(mg.device_step)
        for a, b in ((me.flat, mg.flat), (me.exp_avg, mg.exp_avg), (me.exp_avg_sq, mg.exp_avg_sq)):
            a.copy_(b)
        for m in (mg, me):
            m.xyz_gradient_accum += 1.0
            m.denom += 1.0
        mg.densify_and_prune(2e-4, 0.005, 1.0, None, generator=torch.Generator(device=dev).manual_seed(3))
        me.densify_and_prune(2e-4, 0.005, 1.0, None, generator=torch.Generator(device=dev).manual_seed(3))
        assert mg.P == me.P > P and int(mg.device_step) == int(me.device_step) == n0
        step()                                         # P changed: re-capture, continuing from the counter
        eager(me, bke, oe, n=5)
        assert step.captures == 2 and int(mg.device_step) == int(me.device_step) == n0 + 5
        replay_vs_eager()

        n1 = int(mg.device_step)
        mg.reset_opacity()
        me.reset_opacity()
        assert int(mg.device_step) == int(me.device_step) == n1
        replay_vs_eager()
        assert step.captures == 2 and int(mg.device_step) == n1 + 1
    finally:
        RZ.set_sync_mode(True)
        RZ._pending.clear()
