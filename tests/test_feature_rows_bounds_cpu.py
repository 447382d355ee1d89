"""The restated feature rows and their bound (tests/feature_rows_bounds.py), on the CPU: the model's float64 values and
gradients equal the float64 autograd of tests/feature_rows_model.py on the same fp32 inputs (on the committed frows_*.npz
fixtures and on seeded scenes, the routing of dL/ds over tied flow extremes included); its fp32 shadow lies within
K u B + FLOOR of its value for every element; the shadow's flows, s and tie counts equal a separate plain-float32
evaluation of the projection (the values the GPU must reproduce bit for bit); the density knife rule is sharp; and the
bound is not vacuous."""
import os

import numpy as np
import pytest
import torch

from oracle import warp_oracle as wo

from . import feature_rows_bounds as fb
from . import feature_rows_model as fm
from .conftest import GOLDEN_DIR

FIXTURES = ("frows_b25_m2", "frows_b7_m4_dup", "frows_b7_m2_eqscale", "frows_b7_m1")
SEEDED = {
    "m8_cf15": dict(seed=1, P=300, M=8, B=25, Cf=15),
    "m1_cf0": dict(seed=2, P=257, M=1, B=7, Cf=0, g_density=False),
    "dup_b64": dict(seed=3, P=400, M=2, B=64, Cf=16, dup=True, eq_scale=0.5),
    "single_max": dict(seed=4, P=300, M=4, B=7, Cf=1, single_max=True, g_s=False),
    "static": dict(seed=5, P=200, M=4, B=7, Cf=2, static=True),
    "far_sub": dict(seed=6, P=300, M=2, B=7, Cf=3, far=0.3, sub=0.3),
    "bone_dup": dict(seed=7, P=300, M=2, B=5, Cf=4, bone_dup=True),
}
# tol / max|value| ceilings: the cross-thread sums (acc, g_beta, g_cam_q, g_centres), charged (levels) u sum|t| over
# terms that cancel, and the flow chain (differences of ~250 px projections) carry the largest relative bounds
CEIL = dict(flow_ch=1e-4, normal=1e-5, density=1e-5, s=1e-4, acc=1e-2, g_xyz_cam=1e-3, g_rot_cam=1e-5, g_cam_q=1e-3,
            g_regist=1e-5, g_xyz=1e-4, g_centres=1e-3, g_beta=1e-2)


def fixture_scene(name):
    g = dict(np.load(os.path.join(GOLDEN_DIR, name + ".npz")))
    from .test_feature_rows_cpu import q2dq
    rq, rt = torch.tensor(g["in_rest_q"], dtype=torch.float64), torch.tensor(g["in_rest_t"], dtype=torch.float64)
    _, cen = wo.dq_to_qt(*q2dq(rq, rt))
    M, P = g["ref_xyz_cam"].shape[:2]
    f32 = lambda a: np.ascontiguousarray(a, np.float32)  # noqa: E731
    return dict(P=P, M=M, B=rq.shape[0], Cf=g["in_regist"].shape[1], regist=f32(g["in_regist"]), xyz=f32(g["in_xyz"]),
                scaling=f32(g["in_scaling"]), xyz_cam=f32(g["ref_xyz_cam"]), rot_cam=f32(g["ref_rot_cam"]),
                Kmat=f32(g["ref_Kmat"]), cam_q=f32(g["in_cam_q"]), centres=f32(cen.numpy()),
                beta=f32(np.exp(g["in_logibeta"].astype(np.float64))), g_rows=f32(g["w_rows"]), g_s=f32(g["w_s"][0]),
                g_density=f32(g["w_dens"][:, 0]))


SCENES = {**{n: (lambda n=n: fixture_scene(n)) for n in FIXTURES},
          **{n: (lambda kw=kw: fb.scene(**kw)) for n, kw in SEEDED.items()}}


def autograd(s):
    """tests/feature_rows_model.py in float64 at the kernels' inputs: the rest bones as identity rotations with the
    centres as translations, logibeta = log(beta); backward from sum(rows g_rows) + s g_s + sum(density g_density)."""
    from .test_feature_rows_cpu import q2dq
    t = lambda a: torch.tensor(np.asarray(a, np.float64), requires_grad=True)  # noqa: E731
    d = lambda a: torch.tensor(np.asarray(a, np.float64))  # noqa: E731
    regist, xyz, xc, rc, cq, cen = (t(s[k]) for k in ("regist", "xyz", "xyz_cam", "rot_cam", "cam_q", "centres"))
    lb = t(np.log(np.float64(s["beta"][0]))[None])
    rq = d(np.tile([1.0, 0.0, 0.0, 0.0], (s["B"], 1)))
    rows, sv, dens, flow = fm.feature_rows(regist, xyz, d(s["scaling"]), xc, rc, d(s["Kmat"]), (cq, torch.zeros(s["M"], 3)),
                                           q2dq(rq, cen), lb)
    loss = (rows * d(s["g_rows"])).sum() + (dens[:, 0] * d(s["g_density"])).sum() if s["g_density"] is not None else \
        (rows * d(s["g_rows"])).sum()
    if s["g_s"] is not None:
        loss = loss + sv * float(np.reshape(s["g_s"], ()))
    loss.backward()
    n = lambda x: x.detach().numpy()  # noqa: E731
    return dict(rows=n(rows), s=float(sv.detach()), density=n(dens)[:, 0], flow=n(flow), g_regist=n(regist.grad), g_xyz=n(xyz.grad),
                g_xyz_cam=n(xc.grad), g_rot_cam=n(rc.grad), g_cam_q=n(cq.grad), g_centres=n(cen.grad),
                g_beta=float(lb.grad[0]) / float(s["beta"][0]))


def _close(a, b, what, rel=1e-12):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    if b.size:
        assert np.abs(a - b).max() <= rel * max(np.abs(b).max(), 1e-300), (what, float(np.abs(a - b).max()), float(np.abs(b).max()))


@pytest.fixture(scope="module", params=list(SCENES))
def case(request):
    s = SCENES[request.param]()
    return request.param, s, fb.model(s)


def test_model_equals_float64_autograd(case):
    name, s, m = case
    ref = autograd(s)
    Cf = s["Cf"]
    # the shadow's tie set (data for the routing) is the float64 one in these scenes
    mx = np.abs(ref["flow"]).max()
    assert np.array_equal(m["hi_m"], ref["flow"] == mx) and np.array_equal(m["lo_m"], ref["flow"] == -mx), name
    _close(m["flow"].v, ref["flow"], "flow")
    _close(m["flow_ch"].v, ref["rows"][..., Cf:Cf + 2], "flow / s")
    _close(m["normal"].v, ref["rows"][..., Cf + 2:Cf + 5], "normal")
    _close(m["density"].v, ref["density"], "density")
    _close(m["density"].v[None].repeat(s["M"], 0), ref["rows"][..., Cf + 5], "density channel")
    _close(m["s"].v, ref["s"], "s")
    for k in ("g_regist", "g_xyz", "g_xyz_cam", "g_rot_cam", "g_cam_q", "g_centres", "g_beta"):
        _close(m[k].v, ref[k], k)
    # no projection knife; density knives only among subnormal scores (a few subnormal ulps apart), where fp32 cannot
    # tell the bones apart
    assert not m["pknife"].any() and (m["score"].v[m["dknife"]] < fb.TINY).all()


def _within(e, what, mask=None):
    assert e.f is not None, what
    tol = fb.K * fb.U * e.b + fb.FLOOR
    ok = np.abs(e.f.astype(np.float64) - e.v) <= tol
    if mask is not None:
        ok |= mask
    assert ok.all(), (what, float((np.abs(e.f - e.v) / tol).max()))


def test_fp32_shadow_within_its_bound(case):
    name, s, m = case
    for k in ("flow_ch", "normal", "s", "acc", "g_rot_cam", "g_cam_q", "g_regist", "g_centres", "g_beta"):
        _within(m[k], k)
    _within(m["density"], "density", m["dknife"])
    _within(m["g_xyz"], "g_xyz", m["dknife"][:, None])
    _within(m["g_xyz_cam"], "g_xyz_cam", m["g_xyz_cam_mask"][..., None])


def test_shadow_flow_scale_and_counts_are_plain_float32(case):
    """The values the GPU must reproduce bit for bit: a separate float32 evaluation of the projection gives the same flows,
    max |flow|, s, tie counts and flow channels as the model's shadow."""
    name, s, m = case
    f = fb.flow_f32(s["Kmat"], s["xyz_cam"])
    assert f.dtype == np.float32 and np.array_equal(f.view(np.uint32), m["flow"].f.view(np.uint32))
    sm = np.abs(f).max()
    s32 = np.float32(sm) + np.float32(1e-6)
    assert m["sm"].view(np.uint32) == sm.view(np.uint32) and np.float32(m["s"].f) == s32
    assert (m["hi"], m["lo"]) == (int((f == sm).sum()), int((f == -sm).sum()))
    assert np.array_equal(m["flow_ch"].f, f / s32)


def test_bound_is_not_vacuous(case):
    name, s, m = case
    for k, ceil in CEIL.items():
        e = m[k]
        mx = np.abs(e.v).max() if e.v.size else 0.0
        if mx == 0:
            continue
        tol = (fb.K * fb.U * e.b + fb.FLOOR).max()
        assert tol / mx <= ceil, (name, k, tol / mx)


def test_scene_edges():
    """The options of fb.scene reach their edges in the model: ties at both extremes, one holder of the max, the static
    pair, underflowed and subnormal scores, the exact bone tie."""
    m = fb.model(fb.scene(**SEEDED["dup_b64"]))
    assert m["hi"] == m["lo"] == 2
    s = fb.scene(**SEEDED["single_max"])
    m = fb.model(s)
    ch = np.abs(m["flow_ch"].f)
    assert m["hi"] == m["lo"] == 1 and ch[:, s["P"] // 2].max() == 1 and np.delete(ch, s["P"] // 2, 1).max() < 0.2
    s = fb.scene(**SEEDED["static"])
    m = fb.model(s)
    assert m["sm"] == 0 and m["hi"] == m["lo"] == 2 * s["M"] * s["P"] and np.float32(m["s"].f) == np.float32(1e-6)
    m = fb.model(fb.scene(**SEEDED["far_sub"]))
    d = m["score"].f
    assert (d == 0).sum() > 50 and ((d > 0) & (d < fb.TINY)).sum() > 50
    s = fb.scene(**SEEDED["bone_dup"])
    m = fb.model(s)
    assert (m["arg"] != 1).all() and (m["arg"] == 0).any() and (m["g_centres"].v[1] == 0).all()
    assert not m["dknife"].any()


def test_density_knife_rule_is_sharp():
    """Two bones whose r2 to a surfel are 1 ulp apart make it a knife surfel; exactly duplicated bones (an exact tie)
    do not.  The bone-knife scene flags some surfels, and the knife terms widen both candidates' g_centres bounds."""
    s = fb.scene(11, 64, 2, 3, 2)
    x = np.float32(0.01)
    s["xyz"][:] = 0.0
    s["xyz"][:, 0] = x
    s["centres"][:] = (5.0, 5.0, 5.0)
    s["centres"][0] = 0.0
    s["centres"][1] = (2 * x, 0.0, 0.0)
    m = fb.model(s)
    assert not m["dknife"].any() and (m["arg"] == 0).all()            # r2 bit-identical: an exact tie
    r2 = lambda c: np.float32(np.float32(x - c[0]) ** 2) + np.float32(np.float32(-c[1]) ** 2)  # noqa: E731
    for k in range(1, 200):                                              # bone 1 nudged off-axis until r2 is 1 ulp up
        c = np.array([2 * x, k * 1e-7], np.float32)
        if r2(c) == np.nextafter(r2(np.zeros(2, np.float32)), np.float32(1)):
            break
    else:
        raise AssertionError("no offset gives r2 one ulp apart")
    s["centres"][1, :2] = c
    m = fb.model(s)
    assert m["dknife"].all()
    s = fb.scene(12, 512, 2, 7, 2, bone_knife=True)
    m = fb.model(s)
    assert m["dknife"].sum() > 10 and set(np.unique(m["arg"][m["dknife"]])) <= {0, 1}
