"""GPU tests of Stage 3's fused deformation-cycle regulariser (csrc/cycle.cu via vidu4d_b200.warp.cycle_loss), chained
with the fused forward warp (bob_warp), against the reference fixtures (tests/golden/cycle_*.npz, fp32 autograd of the
reference's own code) and against the float64 model (tests/cycle_model.py, pinned to the fixtures by
tests/test_cycle_cpu.py).

Two knife edges separate an fp32 kernel from a float64 oracle; the oracle comparison masks them rather than loosening
its tolerance:
  * the cycle distance d = |x_cycled - x|: its gradient is the unit direction (x_cycled - x) / d.  The fp32 error of
    x_cycled - x is a few ulps of |x_cam| ~ 1, below 2e-7, so the direction's error is below 2e-7 / d.  Values with a
    float64 d below CYC_KNIFE = 2e-3 are masked: above it the direction is good to 1e-4.
  * the skinning entropy ent = log(sum_b exp(l_b - max)): in fp32 it is exactly 0 once every runner-up bone's
    exp(l_b - max) rounds away against 1 (< 2^-24 each); with at most 64 bones that cannot happen once the float64 value
    exceeds 64 * 2^-24, so values in the band 0 < ent < ENT_KNIFE = 128 * 2^-24 (~7.6e-6, a 2x margin) are masked.  A
    float64 value of exactly 0 is an fp32 0 as well.
A surfel with a masked value in any frame is dropped from the gradient and value comparison on both sides: all of the op's
work is per surfel, so this zeroes the upstream gradient of its values on both sides.  On the full set the counts may
differ from the oracle's by at most the number of masked values."""
import os

import numpy as np
import pytest
import torch

from .conftest import GOLDEN_DIR

pytestmark = pytest.mark.gpu
TOL = 1e-4
WEIGHTS = (0.01, 5e-3, 5e-4)
CYC_KNIFE = 2e-3
ENT_KNIFE = 128 * 2.0 ** -24
LEAVES = ("xyz", "rot", "rest_q", "rest_t", "log_gauss", "art_q", "art_t", "cam_q", "cam_t", "delta", "cdelta")


@pytest.fixture(scope="module")
def dev(built):
    from vidu4d_b200 import _capi
    _capi.load()
    return torch.device("cuda:0")


def _rel(a, b):
    a, b = (x.detach().double().cpu() if torch.is_tensor(x) else torch.as_tensor(np.asarray(x, np.float64)) for x in (a, b))
    return float((a - b).abs().max() / (b.abs().max() + 1e-30))


def run_kernel(t, weights=WEIGHTS, backward=True):
    """bob_warp -> cycle_loss on leaves t (see LEAVES); backward of the loss."""
    from vidu4d_b200.warp import bob_warp, cycle_loss
    from .test_cycle_cpu import q2dq
    rest, art = q2dq(t["rest_q"], t["rest_t"]), q2dq(t["art_q"], t["art_t"])
    cam = (t["cam_q"], t["cam_t"])
    xc, _, _ = bob_warp(t["xyz"], t["rot"], rest, art, t["log_gauss"], cam, t.get("delta"))
    out = cycle_loss(t["xyz"], xc, rest, art, t["log_gauss"], cam, t.get("cdelta"), weights=weights)
    if backward:
        out["loss"].backward()
    return out


def make_inputs(seed, P, B, M, with_delta):
    """The fixtures' inputs at any size (make_cycle_golden.make_case): Gaussian bones wide enough that most surfels blend
    several bones.  With the forward warp's narrow bones (scale 0.03) nearly every surfel follows one bone, its cycle is
    the identity up to rounding, and almost every value would sit on a knife edge."""
    from tests.golden.make_cycle_golden import make_case
    return {k: v for k, v in make_case(seed, P, B, M, with_delta).items() if v is not None}


def _leaves(inp, dev, dtype=torch.float32):
    return {k: v.to(device=dev, dtype=dtype).clone().requires_grad_(True) for k, v in inp.items()}


def _check_grads(t, ref, tol, what=""):
    big_t = max(float(ref["art_t"].abs().max()), float(ref["xyz"].abs().max()))
    for k, v in t.items():
        if k == "rot":
            assert v.grad is None or float(v.grad.abs().max()) == 0.0, (what, k)       # the cycle never reads rot
        elif k == "cam_t":
            # to camera space and back: field2cam's translation cancels, both sides hold rounding noise only
            assert float(v.grad.abs().max()) <= tol * big_t, (what, k)
        else:
            assert _rel(v.grad, ref[k]) <= tol, (what, k)


@pytest.mark.parametrize("name", ["cycle_b25_m3", "cycle_b7_m2_nodelta"])
def test_cycle_kernel_against_reference_fixture(name, dev):
    g = dict(np.load(os.path.join(GOLDEN_DIR, name + ".npz")))
    t = {k: torch.tensor(g["in_" + k], device=dev, requires_grad=True) for k in LEAVES if "in_" + k in g}
    out = run_kernel(t)
    counts = g["ref_counts"]
    assert np.array_equal(out["counts"].cpu().numpy(), counts)
    ref_terms = np.stack([g["ref_" + k].astype(np.float64).clip(min=0).sum(-1) for k in
                          ("reg_deform_cyc", "reg_delta_skin", "reg_skin_entropy")], -1)
    tot = counts.sum(0)
    ref_terms = ref_terms * np.where(tot > 0, np.array(WEIGHTS) / np.maximum(tot, 1), 0.0)
    assert abs(float(out["loss"].detach()) - float(g["ref_loss"][0])) <= TOL * float(g["ref_loss"][0])
    assert _rel(out["terms"], ref_terms) <= TOL
    ref = {k: torch.from_numpy(g["ref_grad_" + k]) for k in t if "ref_grad_" + k in g}
    _check_grads(t, ref, 3e-4, name)                     # the fixture itself is float32 autograd


def _oracle(inp, dev, weights=WEIGHTS):
    from .test_cycle_cpu import oracle_cycle
    t64 = {k: v.double().requires_grad_(True) for k, v in inp.items()}
    return t64, oracle_cycle(t64, weights)


@pytest.mark.parametrize("P,B,M,with_delta", [(30000, 25, 4, True), (5000, 40, 2, False), (777, 3, 9, True), (4000, 64, 3, True)])
def test_cycle_kernel_against_float64_oracle(P, B, M, with_delta, dev):
    inp = make_inputs(seed=100 + B, P=P, B=B, M=M, with_delta=with_delta)
    # ---- full set: the knife mask, and counts within the number of masked values
    with torch.no_grad():
        _, (_, _, cnt64, (cyc, dsk, ent)) = _oracle(inp, dev)
    knife_cyc = cyc < CYC_KNIFE
    knife_ent = (ent > 0) & (ent < ENT_KNIFE)
    out = run_kernel(_leaves(inp, dev), backward=False)
    n_masked = torch.stack((knife_cyc.sum(-1), torch.zeros_like(knife_cyc.sum(-1)), knife_ent.sum(-1)), -1)
    dc = (out["counts"].cpu().long() - cnt64.long()).abs()
    assert bool((dc <= n_masked).all()), (dc, n_masked)
    # ---- the surfels with no masked value in any frame: exact counts, values and gradients
    keep = ~(knife_cyc | knife_ent).any(0)
    assert int(keep.sum()) >= P // 5, int(keep.sum())
    sub = {k: (v[keep] if k in ("xyz", "rot", "delta") else v[:, keep] if k == "cdelta" else v) for k, v in inp.items()}
    t64, (loss64, terms64, cnt64s, _) = _oracle(sub, dev)
    loss64.backward()
    t = _leaves(sub, dev)
    out = run_kernel(t)
    assert torch.equal(out["counts"].cpu().long(), cnt64s.long())
    assert abs(float(out["loss"].detach()) - float(loss64.detach())) <= TOL * float(loss64.detach())
    assert _rel(out["terms"], terms64) <= TOL
    _check_grads(t, {k: v.grad for k, v in t64.items() if v.grad is not None}, TOL, (P, B, M))


def test_zero_weights_give_exactly_zero_gradients(dev):
    inp = make_inputs(seed=7, P=3000, B=25, M=2, with_delta=True)
    t = _leaves(inp, dev)
    out = run_kernel(t, weights=torch.zeros(3, device=dev))
    assert float(out["loss"]) == 0.0 and float(out["terms"].abs().sum()) == 0.0 and int(out["counts"].sum()) > 0
    for k, v in t.items():
        assert v.grad is None or float(v.grad.abs().max()) == 0.0, k


def test_single_bone_entropy_is_zero(dev):
    inp = make_inputs(seed=8, P=2000, B=1, M=3, with_delta=True)
    t = _leaves(inp, dev)
    out = run_kernel(t)
    assert float(out["terms"][:, 2].abs().max()) == 0.0 and int(out["counts"][:, 2].sum()) == 0
    assert int(out["counts"][:, 0].sum()) > 0
    for k, v in t.items():
        assert v.grad is None or bool(torch.isfinite(v.grad).all()), k


def test_no_delta_equals_zero_delta(dev):
    inp = make_inputs(seed=9, P=4000, B=25, M=2, with_delta=False)
    a = run_kernel(_leaves(inp, dev), backward=False)
    z = dict(inp)
    z["cdelta"] = torch.zeros((2, 4000, 25))
    b = run_kernel(_leaves(z, dev), backward=False)
    assert torch.equal(a["counts"], b["counts"]) and int(a["counts"][:, 1].sum()) == 0
    assert _rel(a["terms"], b["terms"]) <= 1e-6 and float(a["terms"][:, 1].abs().max()) == 0.0      # atomics' order only


def test_identity_articulation_and_camera_are_finite(dev):
    inp = make_inputs(seed=10, P=3000, B=25, M=2, with_delta=True)
    inp["art_q"] = inp["rest_q"][None].expand(2, -1, -1).clone()
    inp["art_t"] = inp["rest_t"][None].expand(2, -1, -1).clone()
    inp["cam_q"] = torch.tensor([[1.0, 0.0, 0.0, 0.0]] * 2)
    inp["cam_t"] = torch.zeros((2, 3))
    t = _leaves(inp, dev)
    out = run_kernel(t)
    assert bool(torch.isfinite(out["loss"])) and bool(torch.isfinite(out["terms"]).all())
    for k, v in t.items():
        assert v.grad is None or bool(torch.isfinite(v.grad).all()), k


def test_graphed_step_with_new_weights_matches_eager(dev):
    """warp + cycle + backward captured as one CUDA graph and replayed with the weights refilled in place."""
    from vidu4d_b200 import rasterizer as RZ
    from vidu4d_b200.graph import GraphedStep
    inp = make_inputs(seed=11, P=20000, B=25, M=2, with_delta=True)
    t = _leaves(inp, dev)
    for v in t.values():
        v.grad = torch.zeros_like(v)
    wg = torch.tensor(WEIGHTS, device=dev)
    loss_g = torch.zeros((), device=dev)

    def body():
        for v in t.values():
            v.grad.zero_()
        out = run_kernel(t, weights=wg)
        loss_g.copy_(out["loss"].detach())
    step = GraphedStep(body, device=dev)
    try:
        step()
        for wv in ((0.02, 1e-3, 1e-3), (0.0, 5e-3, 2e-3)):
            wg.copy_(torch.tensor(wv, device=dev))
            step()
            torch.cuda.synchronize()
            grads_g = {k: v.grad.clone() for k, v in t.items()}
            te = _leaves(inp, dev)
            out = run_kernel(te, weights=wv)
            assert abs(float(loss_g) - float(out["loss"])) <= 1e-6 * abs(float(out["loss"])), wv
            for k, v in te.items():
                if v.grad is not None and k != "cam_t":            # cam_t: rounding noise only (see _check_grads)
                    assert _rel(grads_g[k], v.grad) <= 1e-5, (wv, k)
        assert step.captures == 1
    finally:
        RZ.set_sync_mode(True)                 # GraphedStep leaves the rasterizer in no-sync mode
        RZ._pending.clear()


def test_peak_memory_300k_surfels_two_frames(dev):
    """warp + cycle + backward at P = 300 K, M = 2, B = 25 with delta holds no (M,P,B,4) temporaries.  The limit is what
    the two ops must hold: bob_warp's outputs xyz_cam (M,P,3), rot_cam (M,P,4), skin_entropy (P,); the zero g_rot_cam
    (M,P,4) autograd hands its backward; g_xyz_cam (M,P,3), g_cdelta (M,P,B) and the cycle's g_xyz (P,3); bob_warp's
    g_xyz (P,3), g_rot (P,4), g_delta (P,B) and the summed leaf gradient of xyz (P,3); plus 16 MB of slack for the
    tables, their gradients and the allocator's rounding."""
    P, B, M = 300_000, 25, 2
    inp = make_inputs(seed=12, P=P, B=B, M=M, with_delta=True)
    t = _leaves(inp, dev)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    run_kernel(t)
    torch.cuda.synchronize()
    floats = M * P * 3 + M * P * 4 + P + M * P * 4 + M * P * 3 + M * P * B + P * 3 + P * 3 + P * 4 + P * B + P * 3
    assert torch.cuda.max_memory_allocated() - base <= 4 * floats + (16 << 20)
