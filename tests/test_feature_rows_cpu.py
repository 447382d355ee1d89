"""CPU tests of Stage 3's per-surfel feature rows (csrc/feature_rows.cu, vidu4d_b200.warp.feature_rows): the float64 model
(tests/feature_rows_model.py) against fixtures made by the reference's own code (tests/golden/frows_*.npz,
tests/golden/make_feature_rows_golden.py), the reference quirks it records, and argument validation through the C ABI and
the Python entry (every bad call is rejected before any CUDA work)."""
import numpy as np
import pytest
import torch

from oracle import warp_oracle as wo

from . import feature_rows_model as fm

CASES = ["frows_b25_m2", "frows_b7_m4_dup", "frows_b7_m2_eqscale", "frows_b7_m1"]
LEAVES = ("xyz", "rot", "rest_q", "rest_t", "log_gauss", "art_q", "art_t", "cam_q", "cam_t", "delta", "regist", "logibeta")


def q2dq(q, tr):
    """quaternion_translation_to_dual_quaternion (quat_transform.py:294-301): q_d = 0.5 * t (x) q."""
    t4 = torch.cat((torch.zeros_like(tr[..., :1]), tr), -1)
    return q, 0.5 * wo.qmul(t4, q)


def oracle_rows(t, scaling, Kmat):
    """The fixtures' chain in the oracle: forward warp of the canonical surfels (warp_oracle.bob_warp), then the rows.
    Returns rows, s, gauss_density, flow and the warp's xyz_cam, rot_cam."""
    rest = q2dq(t["rest_q"], t["rest_t"])
    art = q2dq(t["art_q"], t["art_t"])
    M = t["art_q"].shape[0]
    rest_m = (rest[0][None].expand(M, -1, -1), rest[1][None].expand(M, -1, -1))
    se3 = wo.dq_mul(art, wo.dq_inverse(rest_m))
    xc, rc, _ = wo.bob_warp(t["xyz"], t["rot"], rest, torch.exp(-t["log_gauss"]), se3, (t["cam_q"], t["cam_t"]), t.get("delta"))
    rows, s, dens, f = fm.feature_rows(t["regist"], t["xyz"], scaling, xc, rc, Kmat, (t["cam_q"], t["cam_t"]), rest, t["logibeta"])
    return rows, s, dens, f, xc, rc


def loss_of(rows, s, dens, g):
    return (rows * torch.from_numpy(g["w_rows"])).sum() + s * float(g["w_s"][0]) + (dens * torch.from_numpy(g["w_dens"])).sum()


def _leaves(g, dtype=torch.float64):
    return {k: torch.tensor(g["in_" + k], dtype=dtype, requires_grad=True) for k in LEAVES if "in_" + k in g}


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / (np.abs(b).max() + 1e-30))


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_reference_fixture(name):
    from .conftest import load_golden
    g = load_golden(name)
    t = _leaves(g)
    scaling = torch.from_numpy(g["in_scaling"]).double()
    rows, s, dens, f, xc, rc = oracle_rows(t, scaling, torch.from_numpy(g["ref64_Kmat"]))
    for k, v in (("rows", rows), ("gauss_density", dens), ("flow", f), ("xyz_cam", xc), ("rot_cam", rc)):
        assert _rel(v.detach(), g["ref64_" + k]) <= 1e-12, k
        # the float32 run of the same chain: flows are differences of projections ~ K x / z ~ 250 px
        assert _rel(v.detach(), g["ref_" + k]) <= 2e-5, k
    assert abs(float(s.detach()) - float(g["ref64_flow_scale"][0])) <= 1e-12 * float(s.detach())
    xc.retain_grad(); rc.retain_grad()
    loss_of(rows, s, dens, g).backward()
    for k, v in list(t.items()) + [("xyz_cam", xc), ("rot_cam", rc)]:
        assert _rel(v.grad, g["ref64_grad_" + k]) <= 1e-9, k
        assert _rel(v.grad, g["ref_grad_" + k]) <= 2e-3, k                   # the reference ran in float32


def test_single_frame_pairs_with_itself():
    """M = 1: flip_pair returns the frame itself, so the flow is exactly 0 and s = 1e-6; every flow value ties for both
    the max and the min, and the flow passes no gradient to xyz_cam."""
    from .conftest import load_golden
    g = load_golden("frows_b7_m1")
    assert float(np.abs(g["ref64_flow"]).max()) == 0.0 and float(np.abs(g["ref_flow"]).max()) == 0.0
    assert float(g["ref64_flow_scale"][0]) == 1e-6
    xc = torch.tensor(g["ref64_xyz_cam"], requires_grad=True)
    f = fm.flow(xc, torch.from_numpy(g["ref64_Kmat"]))
    s = torch.max(f.max(), torch.abs(f.min())) + 1e-6
    (f / s).sum().backward()
    assert float(xc.grad.abs().max()) == 0.0


def test_duplicated_surfels_tie_at_the_flow_extremes():
    """Clone densification's bit-identical copies: the max and the min of the flow are each held by two elements, and
    max(flow) = -min(flow) exactly (frame 2k+1's flow is minus frame 2k's), so torch.maximum splits dL/ds in half."""
    from .conftest import load_golden
    g = load_golden("frows_b7_m4_dup")
    for tag in ("ref", "ref64"):
        f = g[tag + "_flow"]
        assert (f == f.max()).sum() == 2 and (f == f.min()).sum() == 2 and f.max() == -f.min(), tag
    # the split, checked on the oracle: only the tied elements get dL/ds beyond the rows' share
    f = torch.tensor(g["ref64_flow"], requires_grad=True)
    s = torch.max(f.max(), torch.abs(f.min())) + 1e-6
    s.backward()
    gm = f.grad.numpy()
    fv = g["ref64_flow"]
    assert np.all(gm[fv == fv.max()] == 0.25) and np.all(gm[fv == fv.min()] == -0.25)
    assert np.all(gm[(fv != fv.max()) & (fv != fv.min())] == 0.0)


def test_equal_tangent_scales_take_the_first_axis():
    """Reference quirk 1: the axis is the arg-min of the two tangent scales, e_x on a tie; the normal is never e_z."""
    from .conftest import load_golden
    g = load_golden("frows_b7_m2_eqscale")
    sc = g["in_scaling"]
    tie = sc[:, 0] == sc[:, 1]
    assert tie.sum() == len(sc) // 2
    rc, cq = torch.from_numpy(g["ref64_rot_cam"]), torch.tensor(g["in_cam_q"], dtype=torch.float64)
    ex = wo.qapply(cq[:, None], wo.qapply(rc, torch.tensor([1.0, 0, 0], dtype=torch.float64).expand_as(rc[..., 1:])))
    n = g["ref64_rows"][..., 16 + 2:16 + 5]
    assert np.allclose(n[:, tie], ex.numpy()[:, tie], rtol=0, atol=1e-12)


def test_odd_frame_count_is_rejected():
    with pytest.raises(ValueError, match="M must be 1 or even"):
        fm.flow(torch.zeros((3, 5, 3), dtype=torch.float64), torch.eye(3, dtype=torch.float64).expand(3, 3, 3))


def _rows_args(P=100, M=2, B=25, Cf=16, null=None, backward=False):
    d = 4096
    names = ["xyz", "scaling", "xyz_cam", "rot_cam", "Kmat", "cam_q", "centres", "beta"]
    names = (["regist"] + names + ["rows", "density", "flow_scale", "aux"] if not backward else
             names + ["flow_scale", "aux", "g_rows", "g_density", "g_flow_scale", "g_regist", "g_xyz", "g_xyz_cam", "g_rot_cam",
                      "g_tables"])
    ptrs = {k: d for k in names}
    if null:
        ptrs[null] = None
    return [P, M, B, Cf] + list(ptrs.values()) + [None]


def test_c_abi_rejects_bad_feature_rows_arguments(built):
    from vidu4d_b200 import _capi
    lib = _capi.load()
    for bwd, fn in ((False, lib.sr_feature_rows_forward), (True, lib.sr_feature_rows_backward)):
        a = lambda **k: _rows_args(backward=bwd, **k)  # noqa: E731
        nulls = ("xyz", "scaling", "xyz_cam", "rot_cam", "Kmat", "cam_q", "centres", "beta", "flow_scale", "aux")
        nulls += ("g_rows", "g_regist", "g_xyz", "g_xyz_cam", "g_rot_cam", "g_tables") if bwd else ("regist", "rows", "density")
        for null in nulls:
            assert fn(*a(null=null)) == -1 and b"NULL" in lib.sr_last_error(), (bwd, null)
        assert fn(*a(P=-1)) == -1 and b"P must be >= 0" in lib.sr_last_error()
        for M in (0, 3, 5, 1026):
            assert fn(*a(M=M)) == -1 and b"M must be 1 or even" in lib.sr_last_error(), M
        assert fn(*a(B=0)) == -1 and b"B must be in [1, 64]" in lib.sr_last_error()
        assert fn(*a(B=65)) == -1 and b"B must be in [1, 64]" in lib.sr_last_error()
        assert fn(*a(Cf=27)) == -1 and b"Cf must be in [0, 26]" in lib.sr_last_error()
        assert fn(*a(Cf=-1)) == -1 and b"Cf must be in [0, 26]" in lib.sr_last_error()


def test_python_rejects_bad_feature_rows_arguments():
    from vidu4d_b200.warp import _check_feature_rows
    P, M, B = 50, 2, 7
    z = torch.zeros
    base = dict(regist_feat=z((P, 16)), xyz=z((P, 3)), scaling=z((P, 2)), xyz_cam=z((M, P, 3)), rot_cam=z((M, P, 4)),
                Kmat=z((M, 3, 3)), field2cam=(z((M, 4)), z((M, 3))), rest_articulation=(z((B, 4)), z((B, 4))), logibeta=z(1))

    def chk(**kw):
        return _check_feature_rows(**{**base, **kw})
    for kw, msg in ((dict(xyz=z((P, 4))), "xyz must be \\(P,3\\)"), (dict(regist_feat=z((P, 27))), "regist_feat must be"),
                    (dict(regist_feat=z((P + 1, 16))), "regist_feat must be"), (dict(scaling=z((P, 3))), "scaling must be"),
                    (dict(xyz_cam=z((3, P, 3)), rot_cam=z((3, P, 4))), "M must be 1 or even"),
                    (dict(xyz_cam=z((M, P + 1, 3))), "xyz_cam must be"), (dict(rot_cam=z((M, P, 3))), "rot_cam must be"),
                    (dict(Kmat=z((M, 3, 4))), "Kmat must be"), (dict(field2cam=(z((M + 2, 4)), z((M, 3)))), "field2cam must be"),
                    (dict(rest_articulation=(z((65, 4)), z((65, 4)))), "rest_articulation must be"),
                    (dict(logibeta=z(2)), "logibeta must hold one value"),
                    (dict(xyz=z((P, 3), dtype=torch.float64)), "xyz must be float32"),
                    ({}, "regist_feat must be a CUDA tensor")):
        with pytest.raises(RuntimeError, match=msg):
            chk(**kw)
