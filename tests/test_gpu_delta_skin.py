"""GPU tests of the fused delta-skinning MLP (csrc/skin_mlp.cu via vidu4d_b200.warp.delta_skin) against the reference's
fixtures (tests/golden/dskin_*.npz) and the kernels' chain with its rounding-error bound (tests/delta_skin_model.py,
pinned to the fixtures by tests/test_delta_skin_cpu.py): every element of delta, g_x, g_F and the five weight / bias
gradients within K u B + FLOOR, knife points (a ReLU decision within its own bound) masked on both sides."""
import numpy as np
import pytest
import torch

from . import delta_skin_model as dm
from .conftest import load_golden
from .test_delta_skin_cpu import CASES, LEAVES, frames

pytestmark = pytest.mark.gpu
NAMES = {"W1": "linear_1.0.weight", "b1": "linear_1.0.bias", "W2": "linear_2.0.weight", "b2": "linear_2.0.bias",
         "W3": "linear_final.weight", "b3": "linear_final.bias"}
KNIFE_MAX = 0.02            # largest fraction of knife points a case may mask


@pytest.fixture(scope="module")
def dev(built):
    from vidu4d_b200 import _capi
    _capi.load()
    return torch.device("cuda:0")


def make_mlp(g, dev):
    from vidu4d_b200.warp import DeltaSkinMLP
    B = g["in_W3"].shape[0]
    mlp = DeltaSkinMLP(B, g["in_W1"].shape[1] - 3 * B)
    mlp.load_state_dict({v: torch.from_numpy(np.asarray(g["in_" + k])) for k, v in NAMES.items()})
    return mlp.to(dev)


def run_op(g, dev, g_delta=None):
    """delta_skin on a fixture-shaped dict; backward of sum(delta * g_delta).  Returns delta, the leaves and the table."""
    from vidu4d_b200.warp import delta_skin, delta_skin_tables
    mlp = make_mlp(g, dev)
    t = {k: torch.tensor(g["in_" + k], device=dev, requires_grad=True) for k in ("points", "art_r", "art_d", "log_gauss", "cond")}
    delta = delta_skin(t["points"], (t["art_r"], t["art_d"]), t["log_gauss"], mlp, t["cond"])
    if g_delta is not None:
        (delta * torch.as_tensor(g_delta, device=dev).reshape(delta.shape)).sum().backward()
    t.update({k: mlp.get_parameter(v) for k, v in NAMES.items()})
    with torch.no_grad():
        F = delta_skin_tables((t["art_r"], t["art_d"]), t["log_gauss"], t["W1"], t["b1"], t["cond"])
    return delta, t, F


def random_case(seed, B, shape, per_frame, C=160):
    """A fixture-shaped dict of seeded inputs (make_delta_skin_golden.make_case's distributions, torch's default Linear
    initialisation), at any size."""
    from vidu4d_b200.warp import DeltaSkinMLP
    rng = np.random.default_rng(seed)
    M = shape[0] if len(shape) > 1 else 1
    lead = (M,) if per_frame else ()
    q = rng.normal(size=lead + (B, 4))
    q /= np.linalg.norm(q, axis=-1, keepdims=True)
    tr = np.concatenate((np.zeros(lead + (B, 1)), rng.normal(size=lead + (B, 3)) * 0.15), -1)
    tq, tt = torch.from_numpy(q), torch.from_numpy(tr)
    f = lambda a: np.asarray(a, np.float32)  # noqa: E731
    torch.manual_seed(seed)
    mlp = DeltaSkinMLP(B, C)
    g = {"in_points": f(rng.normal(size=tuple(shape) + (3,)) * 0.15), "in_art_r": f(q), "in_art_d": f(0.5 * dm._qmul(tt, tq).numpy()),
         "in_log_gauss": f(np.log(0.03) + 0.3 * rng.normal(size=(B, 3))), "in_cond": f(rng.normal(size=lead + (C,)) * 0.5),
         "in_w_delta": f(rng.normal(size=tuple(shape) + (B,)))}
    g.update({"in_" + k: mlp.get_parameter(v).detach().numpy() for k, v in NAMES.items()})
    return g


def check_bounds(g, dev, what):
    """Every element of every output of both kernels against the chain on the op's own fp32 table."""
    pts, gd = frames(g)
    delta, t, F = run_op(g, dev)
    o = dm.chain_frames(pts, F.cpu().numpy(), g["in_W2"], g["in_b2"], g["in_W3"], g["in_b3"])
    assert dm.within(delta.detach().cpu().numpy().reshape(o["delta"].v.shape), o["delta"]) <= 1.0, what
    keep = ~o["knife"]
    frac = 1.0 - keep.mean()
    print(f"{what}: {int((~keep).sum())} of {keep.size} points masked ({100 * frac:.2f}%)")
    assert frac <= KNIFE_MAX, (what, frac)
    gd = gd * keep[..., None]
    _, t, F = run_op(g, dev, gd)
    # g_F is the gradient the kernel hands to autograd for the table; recover it with a second backward on the table alone
    from vidu4d_b200.warp import _DeltaSkin
    Fl = F.clone().requires_grad_(True)
    M, n, B = gd.shape
    d = _DeltaSkin.apply(torch.tensor(pts, device=dev), Fl, t["W2"].detach(), t["b2"].detach(), t["W3"].detach(), t["b3"].detach(),
                         (M, n, B))
    (d * torch.tensor(gd, device=dev)).sum().backward()
    o = dm.chain_frames(pts, F.cpu().numpy(), g["in_W2"], g["in_b2"], g["in_W3"], g["in_b3"], gd)
    got = {"g_x": t["points"].grad, "g_F": Fl.grad, "g_W2": t["W2"].grad, "g_b2": t["b2"].grad, "g_W3": t["W3"].grad, "g_b3": t["b3"].grad}
    for k, v in got.items():
        assert dm.within(v.cpu().numpy().reshape(o[k].v.shape), o[k]) <= 1.0, (what, k)
    return keep


@pytest.mark.parametrize("case", CASES)
def test_fixture_values_and_bounds(case, dev):
    """delta against the reference's float64 and float32 values, then every output element under the bound."""
    g = load_golden(case)
    delta, _, _ = run_op(g, dev)
    d = delta.detach().cpu().numpy()
    pts, _ = frames(g)
    F64 = dm.fold_table(g["in_art_r"], g["in_art_d"], g["in_log_gauss"], g["in_W1"], g["in_b1"], g["in_cond"])
    o = dm.chain_frames(pts, F64, g["in_W2"], g["in_b2"], g["in_W3"], g["in_b3"])      # the fold's rounding counted
    assert dm.within((d - g["ref64_delta"]).reshape(o["delta"].v.shape) + o["delta"].v, o["delta"]) <= 1.0
    assert np.abs(d - g["ref_delta"]).max() <= 1e-5
    if case == "dskin_b25_clipped":
        assert not d.any()
    check_bounds(g, dev, case)


@pytest.mark.parametrize("case", CASES)
def test_fixture_gradients_through_the_fold(case, dev):
    """Autograd through the kernel and the torch-side fold against the reference's float64 gradients of every leaf, knife
    points masked on both sides (the float64 side through the unfolded model, which the CPU tests pin to the fixtures)."""
    g = load_golden(case)
    pts, gd = frames(g)
    F64 = dm.fold_table(g["in_art_r"], g["in_art_d"], g["in_log_gauss"], g["in_W1"], g["in_b1"], g["in_cond"])
    keep = ~dm.chain_frames(pts, F64, g["in_W2"], g["in_b2"], g["in_W3"], g["in_b3"])["knife"]
    gd = gd * keep[..., None]
    _, t, _ = run_op(g, dev, gd)
    t64 = {k: torch.from_numpy(g["in_" + k]).double().requires_grad_(True) for k in LEAVES}
    d = dm.unfolded(t64["points"], t64["art_r"], t64["art_d"], t64["log_gauss"], {k: t64[k] for k in dm.PARAMS}, t64["cond"])
    (d.reshape(gd.shape) * torch.from_numpy(gd).double()).sum().backward()
    for k in LEAVES:
        ref, got = t64[k].grad.numpy(), t[k].grad.cpu().numpy()
        if case == "dskin_b25_clipped":
            assert not got.any() and not ref.any(), k
        else:
            assert np.abs(got - ref).max() <= 1e-4 * np.abs(ref).max(), (case, k, np.abs(got - ref).max(), np.abs(ref).max())


@pytest.mark.parametrize("B,shape,per_frame", [(1, (700,), False), (16, (3, 300), True), (17, (2, 257), True), (33, (1000,), False),
                                               (48, (2, 16, 24), False), (49, (2, 129), True), (64, (900,), False),
                                               (25, (5, 128), True), (25, (2, 1500), False)])
def test_bounds_at_every_bone_group(B, shape, per_frame, dev):
    """Each NJ = ceil(B / 16) instance of the kernels at its edges, tiles that end on and off a multiple of 128."""
    check_bounds(random_case(300 + B, B, shape, per_frame), dev, f"B={B} {shape} per_frame={per_frame}")


def test_bit_identical_over_two_runs(dev):
    g = random_case(7, 25, (2, 40_000), True)
    outs = []
    for _ in range(2):
        delta, t, _ = run_op(g, dev, g["in_w_delta"])
        outs.append([delta.detach().clone()] + [t[k].grad.clone() for k in LEAVES])
    for a, b in zip(*outs):
        assert torch.equal(a, b)


def test_graphed_step_with_refilled_weights(dev):
    """forward + backward captured as one CUDA graph, replayed after the weights and the points change in place."""
    from vidu4d_b200 import rasterizer as RZ
    from vidu4d_b200.graph import GraphedStep
    from vidu4d_b200.warp import delta_skin
    g = random_case(8, 25, (2, 5000), True)
    mlp = make_mlp(g, dev)
    t = {k: torch.tensor(g["in_" + k], device=dev, requires_grad=True) for k in ("points", "art_r", "art_d", "log_gauss", "cond")}
    w = torch.tensor(g["in_w_delta"], device=dev)
    leaves = list(t.values()) + list(mlp.parameters())
    for v in leaves:
        v.grad = torch.zeros_like(v)
    out = torch.zeros_like(w)

    def body():
        for v in leaves:
            v.grad.zero_()
        d = delta_skin(t["points"], (t["art_r"], t["art_d"]), t["log_gauss"], mlp, t["cond"])
        (d * w).sum().backward()
        out.copy_(d.detach())
    step = GraphedStep(body, device=dev)
    try:
        step()
        for scale in (0.5, -0.75):
            with torch.no_grad():
                mlp.linear_2[0].weight.mul_(scale)
                mlp.linear_final.bias.add_(0.01)
                t["points"].mul_(0.9)
            step()
            torch.cuda.synchronize()
            got = [out.clone()] + [v.grad.clone() for v in leaves]
            body()
            torch.cuda.synchronize()
            for a, b in zip(got, [out] + [v.grad for v in leaves]):
                assert torch.equal(a, b)
        assert step.captures == 1
    finally:
        RZ.set_sync_mode(True)                 # GraphedStep leaves the rasterizer in no-sync mode
        RZ._pending.clear()


def test_composes_with_warp_and_cycle(dev):
    """bob_warp(delta=delta_skin(...)) and cycle_loss(delta=delta_skin(...)) end to end against the same chain with the
    torch model's delta: values and the gradients that flow through delta into the MLP and the points."""
    from tests.golden.make_cycle_golden import make_case
    from vidu4d_b200.warp import bob_warp, cycle_loss, delta_skin
    from .test_cycle_cpu import q2dq
    P, B, M = 3000, 25, 2
    inp = {k: v for k, v in make_case(31, P, B, M, False).items() if v is not None}
    g = random_case(32, B, (M, P), True)
    res = []
    for fused in (True, False):
        t = {k: v.to(dev).clone().requires_grad_(True) for k, v in inp.items()}
        mlp = make_mlp(g, dev)
        p = {k: mlp.get_parameter(v) for k, v in NAMES.items()}
        cond = torch.tensor(g["in_cond"], device=dev, requires_grad=True)
        rest, art, cam = q2dq(t["rest_q"], t["rest_t"]), q2dq(t["art_q"], t["art_t"]), (t["cam_q"], t["cam_t"])
        if fused:
            d_rest = delta_skin(t["xyz"], rest, t["log_gauss"], mlp, cond[0])
        else:
            d_rest = dm.unfolded(t["xyz"], rest[0], rest[1], t["log_gauss"], p, cond[0])
        xc, rc, ent = bob_warp(t["xyz"], t["rot"], rest, art, t["log_gauss"], cam, d_rest)
        # the cycle's points: the warped surfels back in object space at time t (cam_to_field)
        from vidu4d_b200.warp import _qconj, _qmul
        cq = t["cam_q"][:, None]
        v = xc - t["cam_t"][:, None]
        xyz_t = _qmul(_qmul(_qconj(cq), torch.cat((torch.zeros_like(v[..., :1]), v), -1)), cq)[..., 1:]
        d_t = delta_skin(xyz_t, art, t["log_gauss"], mlp, cond) if fused else dm.unfolded(xyz_t, art[0], art[1], t["log_gauss"], p, cond)
        out = cycle_loss(t["xyz"], xc, rest, art, t["log_gauss"], cam, d_t, weights=(0.01, 5e-1, 5e-4))
        loss = out["loss"] + 1e-3 * (xc.square().sum() + rc.square().sum()) / P + 1e-3 * ent.mean()
        loss.backward()
        res.append((loss.detach(), [t["xyz"].grad, t["log_gauss"].grad, t["art_q"].grad, cond.grad] + [v.grad for v in p.values()]))
    (la, ga), (lb, gb) = res
    assert abs(float(la) - float(lb)) <= 1e-5 * abs(float(lb))
    for a, b in zip(ga, gb):
        assert float((a - b).abs().max()) <= 2e-3 * float(b.abs().max()) + 1e-9, (float((a - b).abs().max()), float(b.abs().max()))


def test_peak_memory_300k_surfels_two_frames(dev):
    """Forward + backward at P = 300 K, M = 2, B = 25, per-frame tables: above the inputs the op holds its output delta,
    the upstream gradient and the product that makes it (two (M,P,B)), g_points, the scratch of the weight-gradient
    partials, and 8 MB of slack for the tables, the small gradients and the allocator's rounding -- no (M,P,64) activation,
    no (M,P,3B+C) input."""
    from vidu4d_b200 import _capi
    from vidu4d_b200.warp import delta_skin
    P, B, M = 300_000, 25, 2
    g = random_case(9, B, (M, P), True)
    mlp = make_mlp(g, dev)
    t = {k: torch.tensor(g["in_" + k], device=dev, requires_grad=True) for k in ("points", "art_r", "art_d", "log_gauss", "cond")}
    w = torch.tensor(g["in_w_delta"], device=dev)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    d = delta_skin(t["points"], (t["art_r"], t["art_d"]), t["log_gauss"], mlp, t["cond"])
    (d * w).sum().backward()
    torch.cuda.synchronize()
    scratch = int(_capi.load().sr_delta_skin_scratch_bytes(M, P, B))
    limit = 4 * (3 * M * P * B + M * P * 3) + scratch + (8 << 20)
    assert torch.cuda.max_memory_allocated() - base <= limit
    assert limit < 4 * M * P * (3 * B + 160)              # less than the reference's concatenated input alone
    assert t["points"].grad is not None and mlp.linear_1[0].weight.grad is not None
