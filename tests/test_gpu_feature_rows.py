"""GPU tests of Stage 3's per-surfel feature rows (csrc/feature_rows.cu via vidu4d_b200.warp.feature_rows), alone and
chained with the fused forward warp (bob_warp) and the fused render + loss pass, against the reference fixtures
(tests/golden/frows_*.npz, fp32 autograd of the reference's own code) and the float64 model (tests/feature_rows_model.py,
pinned to the fixtures by tests/test_feature_rows_cpu.py).

Tolerances, each relative to the largest magnitude of the tensor compared (so a few ulps of the largest element):
  * flow / s: u = (Kx)[0:2] / (Kx)[2] is ~250 px, rounded to ~3e-5 each; the flow u' - u (up to s ~ 100 px) then carries
    ~1e-4 px of error, 1e-6 of s.  The normals are two quaternion rotations of a unit axis, a few ulps of 1; the density is
    exp(u) with |u| <= 100, relative error <= 100 * 2^-24 ~ 6e-6 of itself.  ROWS_TOL = 2e-5.
  * gradients: each is a short chain of the same quantities times the upstream weights (flow: g / s through K / z;
    normals: two quaternion VJPs; density: the score times (x - c) / 0.01^2, where x - c ~ 0.01 is a difference of
    values ~0.15, so ~1e-6 relative).  Sums over frames and over a CTA add a few ulps more; GRAD_TOL = 1e-4.
  * against the fp32 fixtures both sides carry their own fp32 rounding, and the chain through bob_warp adds the warp's
    (tests/test_gpu_warp.py uses 1e-4 for it): FIX_TOL = 3e-4.
The density's arg-max bone is a knife edge only if two bones score within fp32 rounding of each other; the seeded inputs
have none (a swap would show up as a 100% error in that surfel's centre gradient)."""
import os

import numpy as np
import pytest
import torch

from .conftest import GOLDEN_DIR

pytestmark = pytest.mark.gpu
ROWS_TOL = 2e-5
GRAD_TOL = 1e-4
FIX_TOL = 3e-4
CF = 16
WARP_LEAVES = ("xyz", "rot", "rest_q", "rest_t", "log_gauss", "art_q", "art_t", "cam_q", "cam_t", "delta")
CASES = ["frows_b25_m2", "frows_b7_m4_dup", "frows_b7_m2_eqscale", "frows_b7_m1"]


@pytest.fixture(scope="module")
def dev(built):
    from vidu4d_b200 import _capi
    _capi.load()
    return torch.device("cuda:0")


def _rel(a, b):
    a, b = (x.detach().double().cpu() if torch.is_tensor(x) else torch.as_tensor(np.asarray(x, np.float64)) for x in (a, b))
    return float((a - b).abs().max() / (b.abs().max() + 1e-30))


def _q2dq(q, t):
    from .test_feature_rows_cpu import q2dq
    return q2dq(q, t)


def _rows(t, scaling, Kmat, xc, rc):
    from vidu4d_b200.warp import feature_rows
    return feature_rows(t["regist"], t["xyz"], scaling, xc, rc, Kmat, (t["cam_q"], t["cam_t"]), _q2dq(t["rest_q"], t["rest_t"]),
                        t["logibeta"])


def _loss(out, w):
    return (out["rows"] * w["w_rows"]).sum() + out["flow_scale"] * w["w_s"][0] + (out["gauss_density"] * w["w_dens"]).sum()


def _weights(g, dev, dtype=torch.float32):
    return {k: torch.tensor(g[k], device=dev, dtype=dtype) for k in ("w_rows", "w_s", "w_dens")}


@pytest.mark.parametrize("name", CASES)
def test_rows_against_reference_fixture(name, dev):
    """The op alone on the reference warp's own xyz_cam / rot_cam, then chained behind bob_warp from the canonical leaves."""
    g = dict(np.load(os.path.join(GOLDEN_DIR, name + ".npz")))
    w = _weights(g, dev)
    scaling, Kmat = torch.tensor(g["in_scaling"], device=dev), torch.tensor(g["ref_Kmat"], device=dev)
    # ---- alone
    t = {k: torch.tensor(g["in_" + k], device=dev, requires_grad=True) for k in ("xyz", "regist", "logibeta", "rest_q", "rest_t",
                                                                                   "cam_q", "cam_t")}
    xc = torch.tensor(g["ref_xyz_cam"], device=dev, requires_grad=True)
    rc = torch.tensor(g["ref_rot_cam"], device=dev, requires_grad=True)
    out = _rows(t, scaling, Kmat, xc, rc)
    assert _rel(out["rows"], g["ref_rows"]) <= ROWS_TOL
    assert _rel(out["gauss_density"], g["ref_gauss_density"]) <= ROWS_TOL
    assert abs(float(out["flow_scale"].detach()) - float(g["ref_flow_scale"][0])) <= ROWS_TOL * float(g["ref_flow_scale"][0])
    _loss(out, w).backward()
    # (the fixture's xyz gradient includes the path through the warp: it is compared in the chained run below)
    for k, v in (("xyz_cam", xc), ("rot_cam", rc), ("regist", t["regist"]), ("logibeta", t["logibeta"])):
        assert _rel(v.grad, g["ref_grad_" + k]) <= FIX_TOL, (name, k)
    # ---- behind bob_warp: every leaf of the fixture chain
    from vidu4d_b200.warp import bob_warp
    t = {k: torch.tensor(g["in_" + k], device=dev, requires_grad=True) for k in WARP_LEAVES + ("regist", "logibeta")}
    xc, rc, _ = bob_warp(t["xyz"], t["rot"], _q2dq(t["rest_q"], t["rest_t"]), _q2dq(t["art_q"], t["art_t"]), t["log_gauss"],
                         (t["cam_q"], t["cam_t"]), t["delta"])
    out = _rows(t, scaling, Kmat, xc, rc)
    assert _rel(out["rows"], g["ref_rows"]) <= FIX_TOL
    _loss(out, w).backward()
    for k, v in t.items():
        assert _rel(v.grad, g["ref_grad_" + k]) <= FIX_TOL, (name, k)


def make_inputs(seed, P, B, M, dev, dup=False):
    """The fixtures' inputs at any size (make_feature_rows_golden.make_case), warped by the float64 oracle; returns fp32
    leaves for the op and the data tensors (scaling, Kmat)."""
    from tests.golden.make_feature_rows_golden import make_case
    from .test_feature_rows_cpu import oracle_rows
    inp = make_case(seed, P, B, M, dup=dup)
    M = int(inp["art_q"].shape[0])
    K = torch.linalg.inv(inp["Kinv"].double()).float()
    t64 = {k: inp[k].double() for k in WARP_LEAVES + ("regist", "logibeta")}
    with torch.no_grad():
        *_, xc, rc = oracle_rows(t64, inp["scaling"].double(), K.double())
    leaves = {"xyz": inp["xyz"], "regist": inp["regist"], "logibeta": inp["logibeta"], "rest_q": inp["rest_q"], "rest_t": inp["rest_t"],
              "cam_q": inp["cam_q"], "cam_t": inp["cam_t"], "xyz_cam": xc.float(), "rot_cam": rc.float()}
    rng = np.random.default_rng(seed + 7)
    Pn = inp["xyz"].shape[0]
    w = {"w_rows": rng.normal(size=(M, Pn, CF + 6)), "w_s": rng.normal(size=(1,)), "w_dens": rng.normal(size=(Pn, 1))}
    return leaves, inp["scaling"], K, w


def _run_kernel(leaves, scaling, K, w, dev):
    t = {k: v.to(dev).clone().requires_grad_(True) for k, v in leaves.items()}
    out = _rows(t, scaling.to(dev), K.to(dev), t["xyz_cam"], t["rot_cam"])
    _loss(out, {k: torch.tensor(v, device=dev, dtype=torch.float32) for k, v in w.items()}).backward()
    return t, out


def _run_oracle(leaves, scaling, K, w):
    from . import feature_rows_model as fm
    t = {k: v.double().requires_grad_(True) for k, v in leaves.items()}
    rows, s, dens, _ = fm.feature_rows(t["regist"], t["xyz"], scaling.double(), t["xyz_cam"], t["rot_cam"], K.double(),
                                       (t["cam_q"], t["cam_t"]), _q2dq(t["rest_q"], t["rest_t"]), t["logibeta"])
    out = {"rows": rows, "flow_scale": s, "gauss_density": dens}
    _loss(out, {k: torch.tensor(v, dtype=torch.float64) for k, v in w.items()}).backward()
    return t, out


@pytest.mark.parametrize("P,B,M", [(20000, 25, 2), (3001, 64, 8), (777, 1, 1), (5000, 25, 8), (4099, 64, 2)])
def test_rows_against_float64_oracle(P, B, M, dev):
    leaves, scaling, K, w = make_inputs(200 + B + M, P, B, M, dev)
    t, out = _run_kernel(leaves, scaling, K, w, dev)
    t64, out64 = _run_oracle(leaves, scaling, K, w)
    for k in ("rows", "gauss_density"):
        assert _rel(out[k], out64[k]) <= ROWS_TOL, k
    assert _rel(out["flow_scale"], out64["flow_scale"]) <= ROWS_TOL
    assert t["cam_t"].grad is None                                  # field2cam's translation is data here
    for k, v in t.items():
        if k != "cam_t":
            assert float(t64[k].grad.abs().max()) > 0 or k == "xyz_cam" and M == 1, k
            assert _rel(v.grad, t64[k].grad) <= GRAD_TOL, (P, B, M, k)
    if M == 1:
        assert float(out["rows"][..., CF:CF + 2].abs().max()) == 0.0 and float(out["flow_scale"]) == np.float32(1e-6)
        assert float(t["xyz_cam"].grad.abs().max()) == 0.0


def test_flow_scale_gradient_splits_over_tied_elements_as_torch(dev):
    """Duplicated surfels: the flow's max and min are each held by two bit-identical elements, and max = -min.  With
    the loss s alone, only the four tied (frame, surfel) pairs get a gradient, G / 2 / 2 each, through their projection."""
    leaves, scaling, K, _ = make_inputs(31, 3000, 7, 4, dev, dup=True)
    M, P = leaves["xyz_cam"].shape[:2]
    w = {"w_rows": np.zeros((M, P, CF + 6)), "w_s": np.array([1.3]), "w_dens": np.zeros((P, 1))}
    t, out = _run_kernel(leaves, scaling, K, w, dev)
    t64, out64 = _run_oracle(leaves, scaling, K, w)
    g, g64 = t["xyz_cam"].grad, t64["xyz_cam"].grad
    hit = g.abs().sum(-1).cpu() > 0
    assert int(hit.sum()) == 4 and torch.equal(hit, g64.abs().sum(-1) > 0)
    assert _rel(g, g64) <= GRAD_TOL
    # the same, with the rows' share: every element gets g / s, and dL/ds gains -sum(g * flow) / s^2
    leaves, scaling, K, w = make_inputs(32, 3000, 7, 4, dev, dup=True)
    t, _ = _run_kernel(leaves, scaling, K, w, dev)
    t64, _ = _run_oracle(leaves, scaling, K, w)
    assert _rel(t["xyz_cam"].grad, t64["xyz_cam"].grad) <= GRAD_TOL


def test_empty_and_ragged_sizes(dev):
    from vidu4d_b200.warp import feature_rows
    z = lambda *s: torch.zeros(s, device=dev, requires_grad=True)  # noqa: E731
    M, B = 2, 5
    rest = (torch.tensor([[1.0, 0, 0, 0]] * B, device=dev), torch.zeros((B, 4), device=dev))
    out = feature_rows(z(0, CF), z(0, 3), torch.ones((0, 2), device=dev), z(M, 0, 3), z(M, 0, 4), torch.eye(3, device=dev).repeat(M, 1, 1),
                       (z(M, 4), torch.zeros((M, 3), device=dev)), rest, z(1))
    assert out["rows"].shape == (M, 0, CF + 6) and out["gauss_density"].shape == (0, 1)
    assert float(out["flow_scale"]) == np.float32(1e-6)
    (out["rows"].sum() + out["flow_scale"]).backward()
    for P in (1, 255, 257):                                          # around one 256-thread block
        leaves, scaling, K, w = make_inputs(40 + P, P, 25, 2, dev)
        t, out = _run_kernel(leaves, scaling, K, w, dev)
        t64, out64 = _run_oracle(leaves, scaling, K, w)
        assert _rel(out["rows"], out64["rows"]) <= ROWS_TOL, P
        for k, v in t.items():
            if k != "cam_t":
                assert _rel(v.grad, t64[k].grad) <= GRAD_TOL, (P, k)


def test_regist_feat_view_of_flat_store_with_odd_p(dev):
    """A FlatSurfelModel group with odd P starts 8-byte but not 16-byte aligned: the rows and the gradient it receives
    equal those of a fresh copy, bit for bit."""
    from vidu4d_b200.surfel_store import FlatSurfelModel
    P = 5003
    gen = torch.Generator(device=dev).manual_seed(5)
    r = lambda *s: torch.randn(s, device=dev, generator=gen)  # noqa: E731
    m = FlatSurfelModel(r(P, 3) * 0.15, r(P, 1, 3), r(P, 15, 3) * 0.1, r(P, 1), r(P, 2) - 4.0, r(P, 4), regist_feat=r(P, CF))
    assert m._regist_feat.data_ptr() % 8 == 0 and m._regist_feat.data_ptr() % 16 != 0
    leaves, _, K, w = make_inputs(50, P, 25, 2, dev)
    leaves = {k: v.to(dev) for k, v in leaves.items()}
    leaves["xyz"] = m._xyz.detach().clone()
    wt = {k: torch.tensor(v, device=dev, dtype=torch.float32) for k, v in w.items()}
    res = []
    for view in (True, False):
        m.zero_grad_flat()
        regist = m._regist_feat if view else m._regist_feat.detach().clone().requires_grad_(True)
        t = dict(leaves, regist=regist)
        out = _rows(t, m.get_scaling.detach(), K.to(dev), t["xyz_cam"], t["rot_cam"])
        _loss(out, wt).backward()
        res.append((out["rows"].detach().clone(), regist.grad.clone()))
    assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][1], res[1][1])
    assert float(res[0][1].abs().max()) > 0


def test_invalid_shapes_raise_before_device_work(dev):
    from vidu4d_b200 import _capi
    from vidu4d_b200.warp import feature_rows
    leaves, scaling, K, _ = make_inputs(60, 500, 7, 2, dev)
    t = {k: v.to(dev) for k, v in leaves.items()}
    rest = _q2dq(t["rest_q"], t["rest_t"])
    torch.cuda.synchronize()
    n0 = _capi.launch_count()
    odd = lambda x: torch.cat([x, x[:1]])  # noqa: E731
    with pytest.raises(RuntimeError, match="M must be 1 or even"):
        feature_rows(t["regist"], t["xyz"], scaling.to(dev), odd(t["xyz_cam"]), odd(t["rot_cam"]), odd(K.to(dev)),
                     (odd(t["cam_q"]), odd(t["cam_t"])), rest, t["logibeta"])
    with pytest.raises(RuntimeError, match="regist_feat must be"):
        feature_rows(torch.zeros((500, 27), device=dev), t["xyz"], scaling.to(dev), t["xyz_cam"], t["rot_cam"], K.to(dev),
                     (t["cam_q"], t["cam_t"]), rest, t["logibeta"])
    with pytest.raises(RuntimeError, match="rest_articulation must be"):
        feature_rows(t["regist"], t["xyz"], scaling.to(dev), t["xyz_cam"], t["rot_cam"], K.to(dev), (t["cam_q"], t["cam_t"]),
                     (torch.zeros((65, 4), device=dev),) * 2, t["logibeta"])
    assert _capi.launch_count() == n0


def test_rows_are_bit_identical_run_to_run_and_graph_replay_equals_eager(dev):
    from vidu4d_b200 import rasterizer as RZ
    from vidu4d_b200.graph import GraphedStep
    leaves, scaling, K, w = make_inputs(70, 30000, 25, 2, dev)
    scaling, K = scaling.to(dev), K.to(dev)
    wt = {k: torch.tensor(v, device=dev, dtype=torch.float32) for k, v in w.items()}
    t = {k: v.to(dev).clone().requires_grad_(True) for k, v in leaves.items()}
    with torch.no_grad():                      # no autograd graph may outlive the eager runs into the capture
        a = _rows(t, scaling, K, t["xyz_cam"], t["rot_cam"])
        b = _rows(t, scaling, K, t["xyz_cam"], t["rot_cam"])
    for k in ("rows", "flow_scale", "gauss_density"):
        assert torch.equal(a[k], b[k]), k
    for v in t.values():
        v.grad = torch.zeros_like(v)
    rows_g = torch.zeros_like(a["rows"])

    def body():
        for v in t.values():
            v.grad.zero_()
        out = _rows(t, scaling, K, t["xyz_cam"], t["rot_cam"])
        _loss(out, wt).backward()
        rows_g.copy_(out["rows"].detach())
    step = GraphedStep(body, device=dev)
    try:
        for shift in (0.0, 0.01):
            with torch.no_grad():
                t["xyz_cam"].add_(shift)
            step()
            torch.cuda.synchronize()
            grads_g = {k: v.grad.clone() for k, v in t.items()}
            te = {k: v.detach().clone().requires_grad_(True) for k, v in t.items()}
            out = _rows(te, scaling, K, te["xyz_cam"], te["rot_cam"])
            _loss(out, wt).backward()
            assert torch.equal(rows_g, out["rows"]), shift
            for k, v in te.items():
                if k != "cam_t":
                    assert _rel(grads_g[k], v.grad) <= 1e-6, (shift, k)     # atomics' order only
        assert step.captures == 1
    finally:
        RZ.set_sync_mode(True)                 # GraphedStep leaves the rasterizer in no-sync mode
        RZ._pending.clear()


def test_end_to_end_warp_rows_render_loss_matches_torch_rows(dev):
    """bob_warp -> feature_rows -> render_loss_batch(features=rows, feature_target, gauss_mask_channel=Cf+5) plus the
    caller's loss on the flow planes times s, backward; against the same chain with the rows built by the reference's
    statements in fp32 torch on the GPU (tests/feature_rows_model.py in float32)."""
    from vidu4d_b200.renderer import PipelineParams, make_camera, render_loss_batch, stack_cameras
    from vidu4d_b200.synthetic import SurfelCloud, object_scene
    from vidu4d_b200.warp import bob_warp, feature_rows
    from tests.golden.make_warp_golden import make_inputs as warp_inputs
    from . import feature_rows_model as fm
    M, P, B, W, H = 2, 40000, 25, 128, 128
    fov = 2 * np.arctan(0.5)
    bc = stack_cameras([make_camera(W, H, fov, fov, device=dev) for _ in range(M)])
    scene = object_scene(P, seed=5, center=(0.0, 0.0, 0.0))
    inp = warp_inputs(8, P, B, M, True)
    inp["xyz"] = torch.tensor(np.asarray(scene.means3D), dtype=torch.float32)
    inp["rest_t"] = inp["xyz"][torch.randperm(P, generator=torch.Generator().manual_seed(1))[:B]].clone()
    inp["art_t"] = inp["rest_t"][None] + 0.01 * torch.randn((M, B, 3), generator=torch.Generator().manual_seed(2))
    inp["log_gauss"] = torch.full((B, 3), float(np.log(0.1)))
    gen = torch.Generator(device=dev).manual_seed(3)
    regist0 = torch.randn((P, CF), device=dev, generator=gen) * 0.3
    ftgt = torch.randn((M, CF, H, W), device=dev, generator=gen) * 0.3
    rgb = torch.rand((M, 3, H, W), device=dev, generator=gen)
    f = W / 2 / np.tan(fov / 2)
    Kmat = torch.tensor([[f, 0, W / 2], [0, f, H / 2], [0, 0, 1]], device=dev, dtype=torch.float32).repeat(M, 1, 1)
    wts = torch.tensor([1e-2, 4e-3], device=dev)
    pipe, bg = PipelineParams(), torch.zeros(3, device=dev)

    def run(fused):
        cloud = SurfelCloud(scene, dev)
        t = {k: v.to(dev).clone().requires_grad_(True) for k, v in inp.items() if k in WARP_LEAVES}
        t["regist"] = regist0.clone().requires_grad_(True)
        t["logibeta"] = torch.tensor([4.6], device=dev, requires_grad=True)
        rest, art = _q2dq(t["rest_q"], t["rest_t"]), _q2dq(t["art_q"], t["art_t"])
        cam = (t["cam_q"], t["cam_t"])
        xc, rc, _ = bob_warp(t["xyz"], t["rot"], rest, art, t["log_gauss"], cam, t["delta"])
        scaling = cloud.get_scaling.detach()
        if fused:
            o = feature_rows(t["regist"], t["xyz"], scaling, xc, rc, Kmat, cam, rest, t["logibeta"])
            rows, s = o["rows"], o["flow_scale"]
        else:
            rows, s, _, _ = fm.feature_rows(t["regist"], t["xyz"], scaling, xc, rc, Kmat, cam, rest, t["logibeta"])
        out = render_loss_batch(bc, cloud, pipe, bg, rgb, mask_gt=torch.ones((M, H, W), device=dev), means3D=xc, rotations=rc,
                                features=rows, feature_target=ftgt, gauss_mask_channel=CF + 5, feature_loss_weights=wts)
        flow = out["features"][:, CF:CF + 2] * s                      # the caller's flow planes (deformable_gaussian.py:1193)
        loss = out["loss"] + 1e-4 * flow.square().mean() + 1e-2 * out["features"][:, CF + 2:CF + 5].square().mean()
        loss.backward()
        return float(loss), {k: v.grad for k, v in t.items()}, out
    loss_f, g_f, out_f = run(True)
    loss_t, g_t, _ = run(False)
    assert float((out_f["allmap"][:, 1] > 0.5).float().mean()) > 0.05         # the warped object is on screen
    assert abs(loss_f - loss_t) <= 1e-5 * abs(loss_t)
    for k in ("xyz", "rot", "regist", "logibeta", "rest_q", "rest_t", "art_q", "art_t", "cam_q", "cam_t", "log_gauss"):
        assert float(g_t[k].abs().max()) > 0, k
        assert _rel(g_f[k], g_t[k]) <= 1e-3, k
