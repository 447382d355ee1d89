"""GPU tests of Stage 3's fused feat_reproj loss (csrc/match.cu via vidu4d_b200.registration) against the float64 model
tests/reproj_model.py (pinned to the reference's own code by tests/test_reproj_cpu.py) and the reference fixtures.

The top-K sets: where the float64 gap between the K-th and (K+1)-th score exceeds EPS the kernel's set must be the
model's; elsewhere it must be a valid top-K within fp32 dot-product error (every chosen score within EPS of the K-th).
Outputs and gradients are then compared with the model evaluated on the kernel's own sets, within 1e-4 of each tensor's
max; counts are exact."""
import os

import numpy as np
import pytest
import torch

from .conftest import GOLDEN_DIR

pytestmark = pytest.mark.gpu
TOL = 1e-4
EPS = 1e-4          # fp32 error bound of a 16-term dot product of unit-scale features (~1e-5), with margin
LEAVES = ("regist_feat", "xyz", "logsigma", "rest_q", "rest_t", "log_gauss", "art_q", "art_t", "cam_q", "cam_t", "delta")


@pytest.fixture(scope="module")
def dev(built):
    from vidu4d_b200 import _capi
    _capi.load()
    return torch.device("cuda:0")


def _rel(a, b):
    a, b = (x.detach().double().cpu() if torch.is_tensor(x) else torch.as_tensor(np.asarray(x, np.float64)) for x in (a, b))
    return float((a - b).abs().max() / (b.abs().max() + 1e-30))


def make_inputs(seed, M, H, W, P, B, K, with_delta=True, num_candidates=2048):
    """Fixture-shaped inputs (numpy arrays under in_*) at any size."""
    from tests.golden.make_warp_golden import make_inputs as warp_inputs
    rng = np.random.default_rng(seed)
    g = {"in_" + k: v.numpy() for k, v in warp_inputs(seed, P, B, M, False).items() if v is not None and k != "rot"}
    g["in_feat_px"] = rng.normal(size=(M, H, W, 16)).astype(np.float32)
    g["in_regist_feat"] = rng.normal(size=(P, 16)).astype(np.float32)
    g["in_logsigma"] = np.array([np.log(2.0)], np.float32)
    f = np.array([[1.2 * W, 0, W / 2], [0, 1.2 * H, H / 2], [0, 0, 1]], np.float32)
    g["in_Kmat"] = np.stack([f + np.array([[0, 0, 0.5 * m], [0, 0, -0.3 * m], [0, 0, 0]], np.float32) for m in range(M)])
    ys, xs = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    hxy = np.stack([np.broadcast_to(xs, (M, H, W)), np.broadcast_to(ys, (M, H, W)), np.ones((M, H, W))], -1).astype(np.float32)
    g["in_hxy"] = hxy + np.concatenate([rng.normal(size=(M, H, W, 2)), np.zeros((M, H, W, 1))], -1).astype(np.float32)
    g["in_mask"] = (rng.random((M, H, W)) < 0.7).astype(np.float32)
    g["in_is_detected"] = np.ones(M, np.float32)
    if with_delta:
        g["in_delta"] = (np.maximum(rng.normal(size=(M, H, W, B)), 0.0) * 0.1).astype(np.float32)
    gen = torch.Generator().manual_seed(seed)
    g["in_cand"] = torch.randperm(M * P, generator=gen)[:min(num_candidates, M * P)].to(torch.int32).numpy()
    g["in_meta"] = np.array([K, 256], np.int32)
    g["in_weight"] = np.array([5e-2], np.float32)
    return g


def run_kernel(g, dev, weight=None):
    from vidu4d_b200.registration import global_match, reproj_loss
    from .reproj_model import q2dq
    t = {k: torch.tensor(g["in_" + k], device=dev).requires_grad_(True) for k in LEAVES if "in_" + k in g}
    d = lambda k: torch.tensor(g["in_" + k], device=dev)  # noqa: E731
    K, res = (int(v) for v in g["in_meta"])
    xyz_m, idx, prob = global_match(d("feat_px"), t["regist_feat"], t["xyz"], d("cand"), t["logsigma"], num_grad=K,
                                    return_topk=True)
    w = d("weight") if weight is None else weight
    out = reproj_loss(xyz_m, d("hxy"), d("Kmat"), q2dq(t["rest_q"], t["rest_t"]), q2dq(t["art_q"], t["art_t"]), t["log_gauss"],
                      (t["cam_q"], t["cam_t"]), d("mask"), d("is_detected"), weight=w, train_res=res, delta=t.get("delta"))
    out["loss"].backward()
    return t, xyz_m, idx, prob, out


def check_topk(score, idx, K, surf):
    """score (N,C) float64; idx (N,K) the kernel's positions; surf (C,) the surfel of each candidate.  Returns the fraction
    of pixels whose top-K set is unambiguous: a K-th / (K+1)-th gap above EPS, or an exact tie between two copies of one
    surfel (bit-identical scores: both orders pick the lower position)."""
    assert bool((idx >= 0).all())
    want = torch.sort(-score, dim=1, stable=True).indices
    srt = score.gather(1, want)
    sK = srt[:, K - 1]
    chosen = score.gather(1, idx.long())
    assert bool((chosen >= sK[:, None] - EPS).all())                                  # a valid top-K within fp32 error
    assert bool((torch.sort(idx, 1).values.diff(dim=1) != 0).all())                    # K distinct candidates
    assert bool((chosen.diff(dim=1) <= EPS).all())                                     # best first
    if score.shape[1] > K:
        clear = (sK - srt[:, K] > EPS) | (surf[want[:, K - 1]] == surf[want[:, K]])
    else:
        clear = torch.ones_like(sK, dtype=torch.bool)
    want = want[:, :K]
    assert torch.equal(torch.sort(idx[clear].long(), 1).values, torch.sort(want[clear], 1).values)
    return float(clear.double().mean())


def compare(g, dev, tol_delta=TOL):
    from .reproj_model import run_fixture
    t, xyz_m, idx, prob, out = run_kernel(g, dev)
    K = int(g["in_meta"][0])
    M, H, W = g["in_feat_px"].shape[:3]
    idx2 = idx.reshape(-1, K)
    tm, om = run_fixture(g, device=dev, order=idx2.long())
    surf = torch.from_numpy(g["in_cand"]).to(dev).long() % g["in_regist_feat"].shape[0]
    clear = check_topk(om["score"].detach(), idx2, K, surf)
    assert _rel(xyz_m, om["xyz_matched"]) <= TOL
    assert float((prob.reshape(-1, K).double() - om["prob"].detach()).abs().max()) <= TOL
    assert _rel(out["xy_reproj"], om["xy_reproj"]) <= TOL
    assert torch.equal(out["counts"].cpu().long(), om["counts"].cpu().long())
    assert abs(float(out["loss"].detach()) - float(om["loss"].detach())) <= TOL * abs(float(om["loss"].detach()))
    assert _rel(out["terms"], om["terms"]) <= TOL
    om["loss"].backward()
    for k, v in t.items():
        assert _rel(v.grad, tm[k].grad) <= (tol_delta if k == "delta" else TOL), k
    return t, out, clear


@pytest.mark.parametrize("name", ["reproj_ragged_48x40", "reproj_dup_nodelta_24x20", "reproj_undetected_k4_20x16",
                                  "reproj_empty_mask_20x16"])
def test_kernels_against_model_and_reference_fixture(name, dev):
    g = dict(np.load(os.path.join(GOLDEN_DIR, name + ".npz")))
    t, out, clear = compare(g, dev)
    assert clear > 0.99
    assert _rel(out["xy_reproj"], g["ref_xy_reproj"]) <= TOL
    assert np.array_equal(out["counts"].cpu().numpy(), g["ref_counts"])
    assert abs(float(out["loss"].detach()) - float(g["ref_loss"][0])) <= TOL * float(g["ref_loss"][0])
    for k, v in t.items():
        assert _rel(v.grad, g["ref_grad_" + k]) <= 3e-4, k      # the fixture itself is float32 autograd


def test_kernels_against_model_256x256_two_frames_300k_surfels(dev):
    g = make_inputs(seed=5, M=2, H=256, W=256, P=300_000, B=25, K=8)
    # dL/ddelta is the fp32 softmax VJP w (gw - sum w gw), bob_warp_bwd's arithmetic; over 131 K points its worst
    # cancellation reaches ~1.03e-4 of the tensor's max, so that one tensor is held to 2e-4 here
    _, out, clear = compare(g, dev, tol_delta=2e-4)
    assert clear > 0.99 and int(out["counts"].sum()) > 0


def test_skipped_candidate_indices_and_k_below_8(dev):
    """Candidate indices outside [0, M*P) are never chosen; K = 3 with a ragged frame."""
    g = make_inputs(seed=6, M=3, H=13, W=29, P=700, B=9, K=3, num_candidates=600)
    g_bad = dict(g)
    cand = g["in_cand"].copy()
    cand[::7] = 3 * 700 + 5
    cand[3::11] = -2
    g_bad["in_cand"] = cand
    _, _, idx, _, _ = run_kernel(g_bad, dev)
    bad = torch.from_numpy((cand < 0) | (cand >= 3 * 700)).to(dev)
    assert not bool(bad[idx.reshape(-1, 3).long()].any())
    compare(g, dev)


def test_zero_weight_gives_exactly_zero_gradients(dev):
    g = make_inputs(seed=7, M=2, H=32, W=40, P=3000, B=25, K=8)
    t, _, _, _, out = run_kernel(g, dev, weight=torch.zeros(1, device=dev))
    assert float(out["loss"].detach()) == 0.0 and float(out["terms"].abs().sum()) == 0.0 and int(out["counts"].sum()) > 0
    for k, v in t.items():
        assert float(v.grad.abs().max()) == 0.0, k


def test_peak_memory_256x256_two_frames_300k_surfels(dev):
    """The fused forward + backward never holds anything the size of the (M*H*W, C) score matrix (1.07 GB here)."""
    g = make_inputs(seed=8, M=2, H=256, W=256, P=300_000, B=25, K=8)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    run_kernel(g, dev)
    torch.cuda.synchronize()
    assert torch.cuda.max_memory_allocated() - base < 128 << 20


def _flat_model(P, dev, seed):
    from vidu4d_b200.surfel_store import FlatSurfelModel
    gen = torch.Generator(device=dev).manual_seed(seed)
    r = lambda *s: torch.randn(s, device=dev, generator=gen)  # noqa: E731
    return FlatSurfelModel(r(P, 3) * 0.15, r(P, 1, 3), r(P, 15, 3) * 0.1, r(P, 1), r(P, 2) - 4.0, r(P, 4), regist_feat=r(P, 16))


def _step_inputs(M, H, W, P, B, dev, seed):
    g = make_inputs(seed=seed, M=M, H=H, W=W, P=P, B=B, K=8)
    d = {k[3:]: torch.tensor(v, device=dev) for k, v in g.items() if k.startswith("in_")}
    for k in ("logsigma", "rest_q", "rest_t", "log_gauss", "art_q", "art_t", "cam_q", "cam_t"):
        d[k].requires_grad_(True)
        d[k].grad = torch.zeros_like(d[k])
    return d


def _step(m, d, cand, w):
    from vidu4d_b200.registration import global_match, reproj_loss
    from .reproj_model import q2dq
    xyz_m = global_match(d["feat_px"], m._regist_feat, m._xyz, cand, d["logsigma"])
    out = reproj_loss(xyz_m, d["hxy"], d["Kmat"], q2dq(d["rest_q"], d["rest_t"]), q2dq(d["art_q"], d["art_t"]), d["log_gauss"],
                      (d["cam_q"], d["cam_t"]), d["mask"], d["is_detected"], weight=w, train_res=256, delta=d["delta"])
    out["loss"].backward()
    return out


def test_flat_store_receives_gradients_in_xyz_and_regist_feat_groups(dev):
    M, H, W, P, B = 2, 48, 64, 5003, 25
    m = _flat_model(P, dev, seed=1)
    d = _step_inputs(M, H, W, P, B, dev, seed=9)
    cand = torch.from_numpy(make_inputs(9, M, H, W, P, B, 8)["in_cand"]).to(dev)
    w = torch.tensor([5e-2], device=dev)
    m.zero_grad_flat()
    _step(m, d, cand, w)
    # the same step on detached copies of the two groups
    rf = m._regist_feat.detach().clone().requires_grad_(True)
    xyz = m._xyz.detach().clone().requires_grad_(True)
    from vidu4d_b200.registration import global_match, reproj_loss
    from .reproj_model import q2dq
    xyz_m = global_match(d["feat_px"], rf, xyz, cand, d["logsigma"].detach())
    reproj_loss(xyz_m, d["hxy"], d["Kmat"], q2dq(d["rest_q"].detach(), d["rest_t"].detach()),
                q2dq(d["art_q"].detach(), d["art_t"].detach()), d["log_gauss"].detach(), (d["cam_q"].detach(), d["cam_t"].detach()),
                d["mask"], d["is_detected"], weight=w, train_res=256, delta=d["delta"])["loss"].backward()
    off, total = m._offsets(P)
    names = [n for n, _ in m.groups]
    for n, a, b in zip(names, off, off[1:] + [total]):
        gsl = m.grad_flat[a:b]
        if n == "xyz":
            assert _rel(gsl, xyz.grad.reshape(-1)) <= 1e-5 and float(gsl.abs().max()) > 0
        elif n == "regist_feat":
            assert _rel(gsl, rf.grad.reshape(-1)) <= 1e-5 and float(gsl.abs().max()) > 0
        else:
            assert float(gsl.abs().max()) == 0.0, n
    before = m.flat.clone()
    m.adam_step()
    moved = (m.flat != before)
    assert bool(moved[off[0]:off[1]].any()) and bool(moved[off[6]:].any()) and not bool(moved[off[1]:off[6]].any())


def test_graphed_step_with_new_candidates_and_weights_matches_eager(dev):
    """match + reproj + backward + FlatSurfelModel.adam_step as one CUDA graph, replayed with two candidate draws and two
    weights refilled in place; every replay is compared with an eager step from the same state."""
    from vidu4d_b200 import rasterizer as RZ
    from vidu4d_b200.graph import GraphedStep
    from vidu4d_b200.registration import draw_candidates
    M, H, W, P, B = 2, 64, 80, 20000, 25
    mg, me = _flat_model(P, dev, seed=2), _flat_model(P, dev, seed=2)
    d = _step_inputs(M, H, W, P, B, dev, seed=10)
    cand = draw_candidates(M, P, 2048, generator=torch.Generator().manual_seed(0), device=dev)
    wg = torch.tensor([5e-2], device=dev)
    loss_g = torch.zeros((), device=dev)

    def body(m, c, w, loss_out):
        m.zero_grad_flat()
        for k in ("logsigma", "art_q", "cam_t"):
            d[k].grad.zero_()
        out = _step(m, d, c, w)
        m.adam_step()
        loss_out.copy_(out["loss"].detach())
    step = GraphedStep(lambda: body(mg, cand, wg, loss_g), device=dev)
    try:
        _replay_and_compare(step, mg, me, d, cand, wg, loss_g, body, M, P, dev)
    finally:
        RZ.set_sync_mode(True)                 # GraphedStep leaves the rasterizer in no-sync mode
        RZ._pending.clear()


def _replay_and_compare(step, mg, me, d, cand, wg, loss_g, body, M, P, dev):
    from vidu4d_b200.registration import draw_candidates
    step()
    baked = mg.step_count
    for seed, wv in ((1, 5e-2), (2, 2e-1)):
        for a, b in ((me.flat, mg.flat), (me.exp_avg, mg.exp_avg), (me.exp_avg_sq, mg.exp_avg_sq)):
            a.copy_(b)
        cand.copy_(draw_candidates(M, P, 2048, generator=torch.Generator().manual_seed(seed), device=dev))
        wg.fill_(wv)
        step()
        grads_g = {k: d[k].grad.clone() for k in ("logsigma", "art_q", "cam_t")}
        me.step_count = baked - 1
        loss_e = torch.zeros((), device=dev)
        body(me, cand.clone(), torch.tensor([wv], device=dev), loss_e)
        assert abs(float(loss_g) - float(loss_e)) <= 1e-5 * abs(float(loss_e)), wv
        assert _rel(mg.grad_flat, me.grad_flat) <= 1e-5, wv
        assert _rel(mg.flat, me.flat) <= 1e-6, wv
        for k, v in grads_g.items():
            assert _rel(v, d[k].grad) <= 1e-5, (wv, k)
    assert step.captures == 1
