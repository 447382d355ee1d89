"""CPU side of tests/test_gpu_render_bounds.py: the per-frame-camera post model (tests/post_bounds.py) against the float64
oracle, its negative controls, and the cases and camera rows the GPU file runs."""
import numpy as np
import pytest

from . import post_bounds as PB
from .test_gpu_loss_bounds import POST_KEYS, _frames, _wvts


def _planted(M, W, H, seed):
    am, _, _, _, planted = _frames(M, W, H, seed, False, False)
    return am, _wvts(M, seed).contiguous().numpy(), planted


@pytest.mark.parametrize("W,H,M,r", [(33, 17, 3, 0.37), (65, 9, 3, 0.0), (97, 17, 2, 1.0), (3, 3, 1, 0.37), (2, 3, 1, 0.0)])
def test_frame_camera_model_equals_oracle(W, H, M, r):
    """Every map of the model, rend_normal and surf_depth included, equals post_oracle.post_forward with camera_model's
    offset rays within 1/64 of the bound, on planted frames with each frame's own camera row; the offsets matter."""
    from oracle import post_oracle as po
    am, wvt, planted = _planted(M, W, H, W * 100 + H + M)
    rows = PB.frame_rows(M, W, H)
    assert planted
    for f in range(M):
        fw, own = PB.forward_model(am[f], PB.cam(wvt[f], W, H, rows[f]), r)
        ref = PB.oracle(am[f], wvt[f], W, H, rows[f], r)
        x = PB.ratios({k: [e.v for e in fw[k]] for k in POST_KEYS}, fw, own, ref)
        for k in POST_KEYS:
            assert x[k].max() <= PB.MODEL_REL, (W, H, f, k, float(x[k].max()))
        # the computed maps carry roundings; acc, rend_dist and the median are copies, exact
        rounded = ("rend_normal", "render_depth_expected") + (("surf_depth",) if r != 1.0 else ())     # r = 1: the median
        for k in rounded + (("surf_normal",) if W >= 3 and H >= 3 else ()):
            assert all(e.b.max() > 0 for e in fw[k]), (W, H, f, k, "no rounding")
        if W >= 3 and H >= 3:
            centred = po.post_forward(am[f], wvt[f], float(rows[f][0]), float(rows[f][1]), float(np.float32(r)))
            sn = fw["surf_normal"]
            diff = max(np.abs(centred["surf_normal"][c] - sn[c].v).max() / (PB.K * PB.U * sn[c].b.max() + PB.FLOOR)
                       for c in range(3))
            assert diff > 100, (W, H, f, "the offset rays change nothing", diff)


def test_model_check_passes_an_exact_kernel():
    """The oracle rounded to fp32 -- what a correct kernel may return -- passes check_frame."""
    W, H, M, r = 65, 17, 3, 0.37
    am, wvt, _ = _planted(M, W, H, 5)
    rows = PB.frame_rows(M, W, H)
    report = {}
    for f in range(M):
        ref = PB.oracle(am[f], wvt[f], W, H, rows[f], r)
        got = {k: np.asarray(ref[k], np.float32) for k in POST_KEYS}
        PB.check_frame(f"frame {f}", got, am[f], wvt[f], rows[f], r, report, ref=ref)
    assert set(report) == set(POST_KEYS) and max(report.values()) <= 1.0


@pytest.mark.parametrize("control", list(PB.CONTROLS))
def test_negative_controls_leave_the_bound_on_the_model(control):
    """Each camera mistake of the GPU file's negative controls, applied to the model alone on planted frames with the
    GPU file's rows and depth ratio, takes at least CONTROL_SHARE of the covered pixels out of the bound of a correct
    kernel's maps (the oracle rounded to fp32)."""
    from . import test_gpu_batch_bounds as BB
    from .test_gpu_render_bounds import RATIO, T_
    W, H = BB.W, BB.H
    M = 3
    am, wvt, _ = _planted(M, W, H, 11)
    rows = BB._rows(T_, True)[[0, 1, T_ - 1]]
    got = [{k: np.asarray(v, np.float32) for k, v in PB.oracle(am[f], wvt[f], W, H, rows[f], RATIO).items()}
           for f in range(M)]
    bad, live = PB.control_failures(control, got, am, wvt, rows, RATIO)
    assert live > 0.9 * (M - (control == "row0_tangents")) * (W - 2) * (H - 2)
    assert bad >= PB.CONTROL_SHARE * live, (control, bad, live)


def test_cases_cover_the_block_edges_and_every_option():
    g = PB.GRID
    assert any(W % 32 and W > 32 for W, *_ in g) and any(H % 8 and H > 8 for _, H, *_ in g)
    assert any(W % 32 == 1 and W > 32 for W, *_ in g) and (1, 1) in [(W, H) for W, H, *_ in g]
    assert any(W < 3 for W, *_ in g) and any(H < 3 for _, H, *_ in g) and any(W % 2 and H % 2 and W > 3 for W, H, *_ in g)
    combos = {(p, r, b) for _, _, _, p, r, b in g}
    assert combos == {(p, r, b) for p in ("table", "scalar") for r in (0.0, 0.37, 1.0) for b in (False, True)}
    assert {(M, p) for _, _, M, p, _, _ in g} == {(M, p) for M in (1, 3, 257) for p in ("table", "scalar")}
    assert {M for _, _, M, *_ in g if M < 257} == {1, 3}
    assert {r for _, _, M, _, r, _ in g if M == 3} == {0.0, 0.37, 1.0}


@pytest.mark.parametrize("W,H,M", [(W, H, M) for W, H, M, *_ in PB.GRID if M > 1])
def test_table_rows_differ_on_every_frame(W, H, M):
    """Both tangents differ on every row of the tables the new tests use, stay positive, and the offsets are non-integer
    and of either sign."""
    from . import test_gpu_batch_bounds as BB
    from .test_gpu_render_bounds import T_
    for rows in (PB.frame_rows(M, W, H), BB._rows(T_, True)):
        n = rows.shape[0]
        assert len(set(rows[:, 0].tolist())) == n and len(set(rows[:, 1].tolist())) == n
        assert (rows[:, :2] > 0).all()
        assert (rows[:, 2:] != np.round(rows[:, 2:])).all()
        assert (rows[:, 2] > 0).any() and (rows[:, 2] < 0).any() and (rows[:, 3] > 0).any() and (rows[:, 3] < 0).any()
    np.testing.assert_array_equal(PB.frame_rows(3, W, H), PB._table(3, W, H))
