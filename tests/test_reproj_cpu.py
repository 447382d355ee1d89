"""CPU tests of Stage 3's fused feat_reproj loss (csrc/match.cu, vidu4d_b200.registration): the float64 model
(tests/reproj_model.py) against fixtures made by the reference's own code (tests/golden/reproj_*.npz), and argument
validation through the C ABI and the Python entries (every bad call is rejected before any CUDA work)."""
import numpy as np
import pytest
import torch

CASES = ["reproj_ragged_48x40", "reproj_dup_nodelta_24x20", "reproj_undetected_k4_20x16", "reproj_empty_mask_20x16"]


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / (np.abs(b).max() + 1e-30))


@pytest.mark.parametrize("name", CASES)
def test_model_matches_reference_fixture(name):
    from .conftest import load_golden
    from .reproj_model import run_fixture
    g = load_golden(name)
    t, out = run_fixture(g)
    assert _rel(out["xyz_matched"].detach(), g["ref_xyz_matched"]) <= 1e-5
    assert _rel(out["xy_reproj"].detach(), g["ref_xy_reproj"]) <= 1e-5
    assert abs(float(out["loss"].detach()) - float(g["ref_loss"][0])) <= 1e-5 * abs(float(g["ref_loss"][0]))
    assert np.array_equal(out["counts"].numpy(), g["ref_counts"])
    out["loss"].backward()
    for k, v in t.items():
        ref = g["ref_grad_" + k]
        assert _rel(v.grad, ref) <= 2e-4, k              # the fixture itself is float32 autograd
    # the K-th and (K+1)-th scores of every pixel are apart, or belong to two copies of one surfel (same score, same xyz,
    # same gradient row): the chosen surfels are unambiguous
    K = int(g["in_meta"][0])
    sc = out["score"].detach()
    o = torch.sort(-sc, dim=1, stable=True).indices
    surf = torch.from_numpy(g["in_cand"]).long() % g["in_regist_feat"].shape[0]
    gap = sc.gather(1, o[:, K - 1:K]) - sc.gather(1, o[:, K:K + 1])
    assert bool(((gap > 1e-5) | (surf[o[:, K - 1:K]] == surf[o[:, K:K + 1]])).all())
    if name == "reproj_dup_nodelta_24x20":
        P = g["in_regist_feat"].shape[0]
        surf = g["in_cand"].astype(np.int64) % P
        assert len(g["in_cand"]) == 2048 and len(np.unique(surf)) < len(surf)      # both copies of some surfels drawn
        assert "in_delta" not in g
    if name == "reproj_undetected_k4_20x16":
        assert g["ref_counts"][0] == 0 and K == 4
    if name == "reproj_empty_mask_20x16":
        assert g["ref_counts"][1] == 0


def test_match_tie_rule_lower_position_first():
    """Equal scores: the lower candidate position comes first, as the kernel orders them."""
    from .reproj_model import global_match
    feat_px = torch.ones((1, 1, 1, 16), dtype=torch.float64)
    regist = torch.zeros((6, 16), dtype=torch.float64)
    regist[[1, 3, 4], 0] = 1.0                      # three equal best scores
    regist[5, 0] = 0.5
    cand = torch.tensor([5, 4, 3, 2, 1, 0], dtype=torch.int32)
    _, order, _, _ = global_match(feat_px, regist, torch.zeros((6, 3), dtype=torch.float64), cand, torch.zeros(1), 4)
    assert order[0].tolist() == [1, 2, 4, 0]


def _match_args(M=2, H=8, W=8, P=100, C=64, K=8, null=None):
    d = 4096
    ptrs = dict(feat_px=d, regist_feat=d, xyz=d, cand=d, logsigma=d, xyz_matched=d, top_idx=d, top_prob=d, top_score=d)
    if null:
        ptrs[null] = None
    return [M, H, W, P, C, K] + list(ptrs.values()) + [None]


def _match_bwd_args(M=2, H=8, W=8, P=100, C=64, K=8, null=None):
    d = 4096
    ptrs = dict(feat_px=d, xyz=d, cand=d, logsigma=d, top_idx=d, top_prob=d, top_score=d, g_xyz_matched=d, g_cand=d,
                g_regist_feat=d, g_xyz=d, g_logsigma=d)
    if null:
        ptrs[null] = None
    return [M, H, W, P, C, K] + list(ptrs.values()) + [None]


def test_c_abi_rejects_bad_match_arguments(built):
    from vidu4d_b200 import _capi
    lib = _capi.load()
    for fn, args, nulls in ((lib.sr_global_match_forward, _match_args, ("feat_px", "regist_feat", "cand", "logsigma", "top_score")),
                            (lib.sr_global_match_backward, _match_bwd_args, ("feat_px", "top_idx", "g_cand", "g_regist_feat",
                                                                             "g_logsigma"))):
        for null in nulls:
            assert fn(*args(null=null)) == -1 and b"NULL" in lib.sr_last_error(), null
        for bad in (dict(M=0), dict(H=0), dict(W=0), dict(P=0)):
            assert fn(*args(**bad)) == -1 and b"must be >= 1" in lib.sr_last_error(), bad
        assert fn(*args(C=0)) == -1 and b"C must be in [1, M*P]" in lib.sr_last_error()
        assert fn(*args(P=10, C=21)) == -1 and b"C must be in [1, M*P]" in lib.sr_last_error()
        assert fn(*args(K=0)) == -1 and b"K must be in [1, min(8, C = 64)]" in lib.sr_last_error()
        assert fn(*args(K=9)) == -1 and b"K must be in" in lib.sr_last_error()
        assert fn(*args(C=3, K=4)) == -1 and b"K must be in [1, min(8, C = 3)]" in lib.sr_last_error()


def _reproj_args(M=2, H=8, W=8, B=25, hd=3, res=256.0, null=None, backward=False):
    d = 4096
    names = ["xyz_matched", "o2b_q", "o2b_t", "inv_gauss", "delta", "se3_r", "se3_d", "cam_q", "cam_t", "Kmat", "hxy", "mask",
             "is_detected"]
    names += ["scale", "g_loss", "g_xyz_matched", "g_delta", "g_tables"] if backward else ["weight", "xy_reproj", "terms", "counts",
                                                                                          "scale", "loss"]
    ptrs = {k: d for k in names}
    if null:
        ptrs[null] = None
    return [M, H, W, B, hd] + ([] if backward else [res]) + list(ptrs.values()) + [None]


def test_c_abi_rejects_bad_reproj_arguments(built):
    from vidu4d_b200 import _capi
    lib = _capi.load()
    for bwd, fn in ((False, lib.sr_reproj_loss_forward), (True, lib.sr_reproj_loss_backward)):
        a = lambda **k: _reproj_args(backward=bwd, **k)  # noqa: E731
        for null in ("xyz_matched", "o2b_q", "se3_d", "cam_t", "Kmat", "hxy", "mask") + (("g_loss", "g_tables") if bwd else ("weight", "loss")):
            assert fn(*a(null=null)) == -1 and b"NULL" in lib.sr_last_error(), null
        for bad in (dict(M=0), dict(H=0), dict(W=0)):
            assert fn(*a(**bad)) == -1 and b"must be >= 1" in lib.sr_last_error(), bad
        assert fn(*a(B=0)) == -1 and b"B must be in [1, 64]" in lib.sr_last_error()
        assert fn(*a(B=65)) == -1 and b"B must be in [1, 64]" in lib.sr_last_error()
        assert fn(*a(hd=4)) == -1 and b"hxy_dim must be 2 or 3" in lib.sr_last_error()
    assert lib.sr_reproj_loss_forward(*_reproj_args(res=0.0)) == -1 and b"train_res" in lib.sr_last_error()
    assert lib.sr_reproj_loss_backward(*_reproj_args(backward=True, null="delta")) == -1
    assert b"g_delta without delta" in lib.sr_last_error()


def test_python_rejects_bad_match_arguments():
    from vidu4d_b200.registration import _check_match, draw_candidates
    M, H, W, P = 2, 6, 5, 40
    fp, rf, xyz = torch.zeros((M, H, W, 16)), torch.zeros((P, 16)), torch.zeros((P, 3))
    cand, ls = draw_candidates(M, P, 50), torch.zeros(1)
    assert cand.dtype == torch.int32 and cand.shape == (50,) and len(set(cand.tolist())) == 50 and int(cand.max()) < M * P
    assert draw_candidates(M, P, 2048).shape == (M * P,)

    def chk(feat_px=fp, regist_feat=rf, xyz_=xyz, cand_=cand, logsigma=ls, k=8):
        return _check_match(feat_px, regist_feat, xyz_, cand_, logsigma, k)
    with pytest.raises(RuntimeError, match="feat_px must be \\(M,H,W,16\\)"):
        chk(feat_px=torch.zeros((M, H, W, 22)))
    with pytest.raises(RuntimeError, match="feat_px must be"):
        chk(feat_px=torch.zeros((M * H * W, 16)))
    with pytest.raises(RuntimeError, match="regist_feat must be \\(P,16\\)"):
        chk(regist_feat=torch.zeros((P, 8)))
    with pytest.raises(RuntimeError, match="xyz must be \\(P,3\\)"):
        chk(xyz_=torch.zeros((P + 1, 3)))
    with pytest.raises(RuntimeError, match="cand must be"):
        chk(cand_=cand.long())
    with pytest.raises(RuntimeError, match="cand must be"):
        chk(cand_=torch.zeros((M * P + 1,), dtype=torch.int32))
    with pytest.raises(RuntimeError, match="logsigma must hold one value"):
        chk(logsigma=torch.zeros(2))
    for k in (0, 9, 2.0, True):
        with pytest.raises(RuntimeError, match="num_grad must be"):
            chk(k=k)
    with pytest.raises(RuntimeError, match="num_grad must be an int in \\[1, min\\(8, C = 3\\)\\]"):
        chk(cand_=cand[:3], k=4)
    with pytest.raises(RuntimeError, match="regist_feat must be float32"):
        chk(regist_feat=rf.double())
    with pytest.raises(RuntimeError, match="feat_px must be a CUDA tensor"):
        chk()


def test_python_rejects_bad_reproj_arguments():
    from vidu4d_b200.registration import _check_reproj
    M, H, W, B = 2, 6, 5, 7
    z = torch.zeros
    base = dict(xyz_m=z((M, H, W, 3)), hxy=z((M, H, W, 3)), Kmat=z((M, 3, 3)), rest_articulation=(z((B, 4)), z((B, 4))),
                t_articulation=(z((M, B, 4)), z((M, B, 4))), log_gauss=z((B, 3)), field2cam=(z((M, 4)), z((M, 3))),
                mask=z((M, H, W)), is_detected=z(M), weight=0.05, train_res=256, delta=None)

    def chk(**kw):
        return _check_reproj(**{**base, **kw})
    for kw, msg in ((dict(xyz_m=z((M, H, W, 2))), "xyz_matched must be"), (dict(hxy=z((M, H, W, 4))), "hxy must be"),
                    (dict(hxy=z((M, H, W + 1, 2))), "hxy must be"), (dict(Kmat=z((M, 4, 4))), "Kmat must be"),
                    (dict(mask=z((M, H, W, 2))), "mask_fg must be"), (dict(is_detected=z(M + 1)), "is_detected must be"),
                    (dict(log_gauss=z((65, 3))), "log_gauss must be"),
                    (dict(t_articulation=(z((M + 1, B, 4)), z((M + 1, B, 4)))), "t_articulation must be"),
                    (dict(field2cam=(z((M, 4)), z((M, 4)))), "field2cam must be"),
                    (dict(delta=z((M, H, W, B + 1))), "delta must be"), (dict(weight=z(2)), "weight must be"),
                    (dict(train_res=0), "train_res must be > 0"), ({}, "xyz_matched must be a CUDA tensor")):
        with pytest.raises(RuntimeError, match=msg):
            chk(**kw)
