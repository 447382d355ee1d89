"""CPU tests of the fused feature-plane losses (csrc/loss.cu, sr_feature_loss_batch): the float64 model
(tests/feature_loss_model.py) against fixtures made by the reference's own loss code (tests/golden/featloss_*.npz), and
argument validation through the C ABI and the Python entry (every bad call is rejected before any CUDA work)."""
import ctypes as C

import numpy as np
import pytest
import torch

CASES = ["featloss_ragged_48x40", "featloss_undetected_36x20", "featloss_empty_mask_36x20", "featloss_no_gauss_36x20"]


@pytest.mark.parametrize("name", CASES)
def test_model_matches_reference_fixture(name):
    from .conftest import load_golden
    from .feature_loss_model import feature_losses
    g = load_golden(name)
    gm = int(g["in_gauss_mask_channel"][0])
    terms, counts, grad = feature_losses(g["in_features"], g["in_target"], g["in_mask"], g["in_is_detected"],
                                         g["in_alpha"], gm, g["in_weights"].astype(np.float64))
    ref = g["ref_terms"]
    for k in range(2):
        assert abs(terms[:, k].sum() - ref[k]) <= 1e-6 * abs(ref[k]), (k, terms[:, k].sum(), ref[k])
    assert np.array_equal(counts.sum(0), g["ref_counts"])
    rg = g["ref_grad_features"].astype(np.float64)
    M, F = rg.shape[:2]
    for m in range(M):
        for c in range(F):
            assert np.abs(grad[m, c] - rg[m, c]).max() <= 1e-6 * np.abs(rg[m, c]).max(), (m, c)
    if name == "featloss_undetected_36x20":
        assert counts[0, 0] == 0 and np.abs(grad[0, :16]).max() == 0 and counts[0, 1] > 0
    if name == "featloss_empty_mask_36x20":
        assert counts[1, 0] == 0 and np.abs(grad[1, :16]).max() == 0
    if name == "featloss_no_gauss_36x20":
        assert ref[1] == 0 and np.abs(grad[:, 16:]).max() == 0


def test_flat_store_regist_feat_group_layout_on_cpu():
    """regist_feat is a seventh group after the six, whose layout and values do not change; its parameter and gradient are
    views of the flat buffers, FlatGrads reduces it, and its learning rate defaults to feature_lr = 0.0025."""
    from vidu4d_b200 import distributed as D
    from vidu4d_b200.surfel_store import FlatSurfelModel
    P = 257
    g = torch.Generator().manual_seed(0)
    ts = [torch.randn((P, k), generator=g) for k in (3, 3, 45, 1, 2, 4)]
    rf = torch.randn((P, 16), generator=g)
    a = FlatSurfelModel(*ts)
    b = FlatSurfelModel(*ts, regist_feat=rf)
    assert [n for n, _ in b.groups] == ["xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation", "regist_feat"]
    assert b._offsets(P)[0][:6] == a._offsets(P)[0] and torch.equal(b.flat[:a.flat.numel()], a.flat)
    assert torch.equal(b._regist_feat.detach(), rf) and b._regist_feat.data_ptr() == b.flat[P * 58:].data_ptr()
    assert b._regist_feat.grad.data_ptr() == b.grad_flat[P * 58:].data_ptr()
    assert len(b.flat_params()) == 7 and b.flat_params()[6] is b._regist_feat and b.lrs["regist_feat"] == 2.5e-3
    assert len(a.flat_params()) == 6 and not hasattr(a, "_regist_feat")
    assert D.FlatGrads(b.flat_params()).flat.numel() == P * 74
    assert FlatSurfelModel(*ts, lrs={**a.lrs, "regist_feat": 1e-3}, regist_feat=rf).lrs["regist_feat"] == 1e-3


def _args(M=2, F=22, Cf=16, gm=21, target=True, mask=True, null=None):
    """sr_feature_loss_batch arguments with dummy (never dereferenced) pointers; `null` names one pointer set to NULL."""
    d = 4096
    ptrs = dict(features=d, target=d if target else None, mask_gt=d if mask else None, is_detected=None, allmap=d,
                weights=d, feature_terms=d, counts=d, dL_dfeatures=d)
    if null:
        ptrs[null] = None
    return [M, 48, 40, F, Cf, gm] + list(ptrs.values()) + [None]


def test_c_abi_rejects_bad_feature_loss_arguments(built):
    from vidu4d_b200 import _capi
    lib = _capi.load()
    fn = lib.sr_feature_loss_batch
    for null in ("features", "allmap", "weights", "feature_terms", "counts", "dL_dfeatures"):
        assert fn(*_args(null=null)) == -1 and b"must not be NULL" in lib.sr_last_error(), null
    assert fn(*_args(mask=False)) == -1 and b"needs mask_gt" in lib.sr_last_error()
    assert fn(*_args(Cf=23)) == -1 and b"Cf must be in [1, F = 22]" in lib.sr_last_error()
    assert fn(*_args(Cf=0)) == -1 and b"Cf must be in [1, F = 22]" in lib.sr_last_error()
    assert fn(*_args(target=False)) == -1 and b"Cf must be 0 without a target" in lib.sr_last_error()
    assert fn(*_args(gm=22)) == -1 and b"gauss_mask_channel must be -1 or in [0, F = 22)" in lib.sr_last_error()
    assert fn(*_args(gm=-2)) == -1 and b"gauss_mask_channel" in lib.sr_last_error()
    assert fn(*_args(gm=15)) == -1 and b"inside the feature target" in lib.sr_last_error()
    assert fn(*_args(target=False, Cf=0, gm=-1)) == -1 and b"no term" in lib.sr_last_error()
    assert fn(*_args(M=0)) == -1 and b"must be positive" in lib.sr_last_error()
    assert fn(*_args(F=0, Cf=0, target=False, gm=-1)) == -1 and b"F must be >= 1" in lib.sr_last_error()


def test_python_rejects_bad_feature_loss_arguments():
    from vidu4d_b200.renderer import _check_feature_losses
    M, H, W = 2, 40, 48
    feat, tgt, mask = torch.zeros((100, 22)), torch.zeros((M, 16, H, W)), torch.zeros((M, H, W))

    def chk(features=feat, target=tgt, mask_gt=mask, det=None, gm=21, wts=None):
        return _check_feature_losses(M, H, W, features, target, mask_gt, det, gm, wts)
    with pytest.raises(RuntimeError, match="need features="):
        chk(features=None)
    with pytest.raises(RuntimeError, match="needs mask_gt"):
        chk(mask_gt=None)
    for bad in ((M, 16, H, W + 1), (M + 1, 16, H, W), (M, 23, H, W), (M, 0, H, W), (M, 16, H * W)):
        with pytest.raises(RuntimeError, match="feature_target must be"):
            chk(target=torch.zeros(bad))
    for gm in (22, 15, -1):
        with pytest.raises(RuntimeError, match="gauss_mask_channel must be in"):
            chk(gm=gm)
    with pytest.raises(RuntimeError, match="gauss_mask_channel must be in \\[Cf, F\\) = \\[0, 22\\)"):
        chk(target=None, gm=22)
    with pytest.raises(RuntimeError, match="is_detected must be"):
        chk(det=torch.ones(M + 1))
    with pytest.raises(RuntimeError, match="feature_loss_weights must be"):
        chk(wts=torch.ones(3))
    with pytest.raises(RuntimeError, match="feature_loss_weights must be"):
        chk(wts=torch.ones(2, dtype=torch.float64))
    with pytest.raises(RuntimeError, match="features must be a CUDA tensor"):
        chk()
