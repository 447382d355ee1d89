"""CPU tests of Stage 3's fused deformation-cycle regulariser (csrc/cycle.cu, vidu4d_b200.warp.cycle_loss): the float64
model (tests/cycle_model.py) against fixtures made by the reference's own code (tests/golden/cycle_*.npz,
tests/golden/make_cycle_golden.py), and argument validation through the C ABI and the Python entry (every bad call is
rejected before any CUDA work)."""
import numpy as np
import pytest
import torch

from oracle import warp_oracle as wo

from . import cycle_model as cm

CASES = ["cycle_b25_m3", "cycle_b7_m2_nodelta"]
LEAVES = ("xyz", "rot", "rest_q", "rest_t", "log_gauss", "art_q", "art_t", "cam_q", "cam_t", "delta", "cdelta")
TERMS = ("reg_deform_cyc", "reg_delta_skin", "reg_skin_entropy")
WEIGHTS = (0.01, 5e-3, 5e-4)


def q2dq(q, tr):
    """quaternion_translation_to_dual_quaternion (quat_transform.py:294-301): q_d = 0.5 * t (x) q."""
    t4 = torch.cat((torch.zeros_like(tr[..., :1]), tr), -1)
    return q, 0.5 * wo.qmul(t4, q)


def oracle_cycle(t, weights=WEIGHTS):
    """The fixtures' chain in the oracle: forward warp of the canonical surfels (warp_oracle.bob_warp), then cycle_loss
    with the backward warp.  t: leaves as in LEAVES (delta (P,B) of the forward warp, cdelta (M,P,B) of the backward)."""
    rest = q2dq(t["rest_q"], t["rest_t"])
    art = q2dq(t["art_q"], t["art_t"])
    M = t["art_q"].shape[0]
    rest_m = (rest[0][None].expand(M, -1, -1), rest[1][None].expand(M, -1, -1))
    se3 = wo.dq_mul(art, wo.dq_inverse(rest_m))
    ig = torch.exp(-t["log_gauss"])
    xc, _, _ = wo.bob_warp(t["xyz"], t["rot"], rest, ig, se3, (t["cam_q"], t["cam_t"]), t.get("delta"))
    return cm.cycle_loss(t["xyz"], xc, rest, art, ig, (t["cam_q"], t["cam_t"]), t.get("cdelta"), weights)


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
    loss, terms, counts, vals = oracle_cycle(t)
    for k, v in zip(TERMS, vals):
        assert _rel(v.detach(), g["ref64_" + k]) <= 1e-9, k
        assert _rel(v.detach(), g["ref_" + k]) <= 2e-5, k            # the float32 run of the same chain
    assert np.array_equal(counts.numpy(), g["ref64_counts"]) and np.array_equal(counts.numpy(), g["ref_counts"])
    assert abs(float(loss.detach()) - float(g["ref64_loss"][0])) <= 1e-9 * float(g["ref64_loss"][0])
    assert abs(float(terms.sum().detach()) - float(loss.detach())) <= 1e-12 * float(loss.detach())
    loss.backward()
    big = max(float(np.abs(g[k]).max()) for k in g if k.startswith("ref64_grad_"))
    for k, v in t.items():
        if "ref64_grad_" + k not in g:
            assert v.grad is None or float(v.grad.abs().max()) == 0.0, k        # rot never reaches the cycle term
            continue
        if k == "cam_t":
            # camera space and back: the translation of field2cam cancels, its gradient is rounding noise only
            for gr in (v.grad.numpy(), g["ref64_grad_" + k], g["ref_grad_" + k]):
                assert np.abs(gr).max() <= 1e-5 * big, k
            continue
        assert _rel(v.grad, g["ref64_grad_" + k]) <= 1e-9, k
        assert _rel(v.grad, g["ref_grad_" + k]) <= 2e-4, k                    # the reference ran in float32
    # knife-edge-free by construction (make_cycle_golden.make_case): distances far above fp32 rounding, entropies far
    # above fp32's zero threshold, so the fixture's counts and gradient directions are exact yardsticks for the kernel
    assert float(vals[0].min()) > 1e-4 and float(vals[2].min()) > 1e-3
    if name == "cycle_b7_m2_nodelta":
        assert "in_cdelta" not in g and counts[:, 1].sum() == 0 and float(terms[:, 1].abs().sum()) == 0.0


def test_oracle_identity_cycle_and_single_bone():
    """Rest = t articulation and identity camera: the cycle is the identity map.  One bone: the entropy is exactly 0."""
    from .conftest import load_golden
    g = load_golden("cycle_b7_m2_nodelta")
    t = {k: v.detach() for k, v in _leaves(g).items()}
    M = t["art_q"].shape[0]
    rest = q2dq(t["rest_q"], t["rest_t"])
    art = (rest[0][None].expand(M, -1, -1), rest[1][None].expand(M, -1, -1))
    cam = (torch.tensor([[1.0, 0, 0, 0]] * M, dtype=torch.float64), torch.zeros((M, 3), dtype=torch.float64))
    xc = t["xyz"][None].expand(M, -1, -1)
    cyc, dsk, ent = cm.cycle_values(t["xyz"], xc, rest, art, torch.exp(-t["log_gauss"]), cam)
    assert float(cyc.max()) < 1e-12 and float(dsk.abs().max()) == 0.0
    one = (rest[0][:1], rest[1][:1])
    _, _, ent1 = cm.cycle_values(t["xyz"], xc, one, (art[0][:, :1], art[1][:, :1]), torch.exp(-t["log_gauss"][:1]), cam)
    assert float(ent1.abs().max()) == 0.0


def _cycle_args(P=100, B=25, M=2, null=None, backward=False):
    d = 4096
    names = ["xyz", "xyz_cam", "o2b_q", "o2b_t", "inv_gauss", "delta", "se3_r", "se3_d", "cam_q", "cam_t"]
    names += ["scale", "g_loss", "g_xyz_cam", "g_xyz", "g_delta", "g_tables"] if backward else ["weights", "terms", "counts",
                                                                                                "scale", "loss"]
    ptrs = {k: d for k in names}
    if null:
        ptrs[null] = None
    return [P, B, M] + list(ptrs.values()) + [None]


def test_c_abi_rejects_bad_cycle_arguments(built):
    from vidu4d_b200 import _capi
    lib = _capi.load()
    assert lib.sr_cycle_loss_table_floats(25, 2) == 2 * 25 * 15 + 25 * 3 + 2 * 7
    for bwd, fn in ((False, lib.sr_cycle_loss_forward), (True, lib.sr_cycle_loss_backward)):
        a = lambda **k: _cycle_args(backward=bwd, **k)  # noqa: E731
        for null in ("xyz", "xyz_cam", "o2b_q", "inv_gauss", "se3_d", "cam_t", "scale") + (("g_loss", "g_xyz_cam", "g_xyz", "g_tables")
                                                                                         if bwd else ("weights", "terms", "loss")):
            assert fn(*a(null=null)) == -1 and b"NULL" in lib.sr_last_error(), null
        assert fn(*a(P=-1)) == -1 and b"P must be >= 0" in lib.sr_last_error()
        assert fn(*a(M=0)) == -1 and b"M must be >= 1" in lib.sr_last_error()
        assert fn(*a(B=0)) == -1 and b"B must be in [1, 64]" in lib.sr_last_error()
        assert fn(*a(B=65)) == -1 and b"B must be in [1, 64]" in lib.sr_last_error()
        assert fn(*a(B=64, M=27)) == -1 and b"do not fit in shared memory" in lib.sr_last_error()
    assert lib.sr_cycle_loss_backward(*_cycle_args(backward=True, null="delta")) == -1
    assert b"g_delta without delta" in lib.sr_last_error()


def test_python_rejects_bad_cycle_arguments():
    from vidu4d_b200.warp import _check_cycle
    P, B, M = 50, 7, 3
    z = torch.zeros
    base = dict(xyz=z((P, 3)), xyz_cam=z((M, P, 3)), rest_articulation=(z((B, 4)), z((B, 4))),
                t_articulation=(z((M, B, 4)), z((M, B, 4))), log_gauss=z((B, 3)), field2cam=(z((M, 4)), z((M, 3))), delta=None,
                weights=(0.01, 5e-3, 5e-4))

    def chk(**kw):
        return _check_cycle(**{**base, **kw})
    for kw, msg in ((dict(xyz=z((P, 4))), "xyz must be \\(P,3\\)"), (dict(xyz_cam=z((M, P + 1, 3))), "xyz_cam must be"),
                    (dict(xyz_cam=z((P, 3))), "xyz_cam must be"), (dict(log_gauss=z((65, 3))), "log_gauss must be"),
                    (dict(log_gauss=z((B, 2))), "log_gauss must be"),
                    (dict(rest_articulation=(z((B + 1, 4)), z((B + 1, 4)))), "rest_articulation must be"),
                    (dict(t_articulation=(z((M + 1, B, 4)), z((M + 1, B, 4)))), "t_articulation must be"),
                    (dict(field2cam=(z((M, 4)), z((M, 4)))), "field2cam must be"),
                    (dict(delta=z((P, B))), "delta must be \\(M,P,B\\)"), (dict(weights=z(2)), "weights must be"),
                    (dict(weights=(1.0, 2.0)), "weights must be"), (dict(xyz=z((P, 3), dtype=torch.float64)), "xyz must be float32"),
                    ({}, "xyz must be a CUDA tensor")):
        with pytest.raises(RuntimeError, match=msg):
            chk(**kw)
    # B = 64 fits up to M = 26 frames; beyond that the caller splits the frames
    Mb = 27
    with pytest.raises(RuntimeError, match="do not fit in shared memory"):
        _check_cycle(z((P, 3), device="meta"), z((Mb, P, 3), device="meta"), (z((64, 4), device="meta"),) * 2,
                     (z((Mb, 64, 4), device="meta"),) * 2, z((64, 3), device="meta"), (z((Mb, 4), device="meta"), z((Mb, 3), device="meta")),
                     None, (0.01, 5e-3, 5e-4))
