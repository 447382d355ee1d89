"""CPU pinning of the feature-loss restatement and its rounding-error bound (tests/feature_loss_bounds.py): its float64
value equals the reference-pinned model (tests/feature_loss_model.py) far inside the bound, its fp32 shadow -- with and
without the FMA contraction of the channel sum -- lies inside it, and five plausible kernel mistakes planted in the
shadow fall outside it on a clear share of elements."""
import numpy as np
import pytest

from . import feature_loss_bounds as fb
from .feature_loss_model import feature_losses

FIXTURES = ["featloss_ragged_48x40", "featloss_undetected_36x20", "featloss_empty_mask_36x20", "featloss_no_gauss_36x20"]


def _fixture(name):
    from .conftest import load_golden
    g = load_golden(name)
    gm = int(g["in_gauss_mask_channel"][0])
    return (g["in_features"], g["in_target"], g["in_mask"], g["in_is_detected"], g["in_alpha"], gm,
            g["in_weights"].astype(np.float32))


def _case(name):
    if name in fb.CONFIGS:
        feat, target, mask, det, alpha, gm, _ = fb.config_inputs(name)
        return feat, target, mask, det, alpha, gm, fb.WEIGHTS
    return _fixture(name)


CASES = FIXTURES + list(fb.CONFIGS)


@pytest.mark.parametrize("name", CASES)
def test_restatement_value_matches_model(name):
    """The bound is evaluated on the expression it bounds: the float64 value equals feature_losses() to 1e-3 of the
    bound, planes and terms, when both scale with the model's own counts."""
    feat, target, mask, det, alpha, gm, w = _case(name)
    rt, rc, rg = feature_losses(feat, target, mask, det, alpha, gm, w.astype(np.float64))
    px = fb.pixel_terms(feat, target, mask, det, alpha, gm)
    _, tm, g = fb.scaled(px, rc, w, gm)
    for k, e in tm.items():
        tol = fb.K * fb.U * e.b + fb.FLOOR
        # the model's weights are the fp32 weights' float64 values: rt uses the same
        assert np.all(np.abs(e.v - rt[:, k]) <= 1e-3 * tol), (name, k, e.v, rt[:, k])
    for c, e in g.items():
        tol = fb.K * fb.U * e.b + fb.FLOOR
        assert np.all(np.abs(e.v - rg[:, c]) <= 1e-3 * tol), (name, c)
    for c in set(range(feat.shape[1])) - set(g):
        assert (rg[:, c] == 0).all()


@pytest.mark.parametrize("fma", [False, True])
@pytest.mark.parametrize("name", CASES)
def test_shadow_within_bound(name, fma):
    feat, target, mask, det, alpha, gm, w = _case(name)
    px = fb.pixel_terms(feat, target, mask, det, alpha, gm)
    terms, counts, grad = fb.shadow(feat, target, mask, det, alpha, gm, w, fma=fma)
    rep = fb.check(name, terms, counts, grad, px, w, gm, feat.shape[1])
    assert rep
    if name == "nothing_positive":
        assert (counts == 0).all() and (terms == 0).all() and (grad == 0).all()


def test_planted_pixels_reach_their_edges():
    """Each plant sits on a block seam and on the border, the underflowing ones are knife pixels, and the subnormal
    Gaussian-mask value is not."""
    feat, target, mask, det, alpha, gm, planted = fb.config_inputs("f22_det_0_half")
    c = fb.CONFIGS["f22_det_0_half"]
    H, W = c["H"], c["W"]
    kinds = {}
    for kind, f, y, x in planted:
        kinds.setdefault(kind, []).append((f, y, x))
        assert (x % 32 in (0, 31) or y % 8 in (0, 7)) or x == W - 1, (kind, y, x)
    assert set(kinds) == set(fb.PLANTS) and all(len(v) == 2 for v in kinds.values())
    px = fb.pixel_terms(feat, target, mask, det, alpha, gm)
    f, y, x = kinds["mask_1e-30"][0]
    if det[f] > 0:
        assert px["knife"][0][f, y, x] and np.float32(px["v"][0].v[f, y, x]) == 0
    f, y, x = kinds["d_1e-20"][0]
    assert not px["knife"][1][f, y, x] and 0 < px["v"][1].v[f, y, x] < np.finfo(np.float32).tiny
    f, y, x = kinds["d_1e-20"][1]
    assert px["knife"][1][f, y, x]
    assert px["knife"][0].sum() + px["knife"][1].sum() <= 4


def _share_outside(name, mutate):
    feat, target, mask, det, alpha, gm, w = _case(name)
    px = fb.pixel_terms(feat, target, mask, det, alpha, gm)
    _, counts, _ = fb.shadow(feat, target, mask, det, alpha, gm, w)
    terms, _, grad = fb.shadow(feat, target, mask, det, alpha, gm, w, mutate=mutate)
    _, tm, g = fb.scaled(px, counts, w, gm)
    shares = {}
    for c, e in g.items():
        key = "gm" if c == gm else "feat"
        kn = px["knife"][1 if c == gm else 0]
        r = fb.ratio(grad[:, c], e, skip=kn)
        live = (e.v != 0) & ~kn
        a, n = shares.get(key, (0, 0))
        shares[key] = (a + int((r[live] > 1).sum()), n + int(live.sum()))
    for k, e in tm.items():
        r = fb.ratio(terms[:, k], e)
        shares[f"terms{k}"] = (int((r > 1).sum()), r.size)
    return {k: a / max(n, 1) for k, (a, n) in shares.items()}


@pytest.mark.parametrize("mutate", fb.MUTATIONS)
@pytest.mark.parametrize("name", ["f22_det_0_half", "featloss_ragged_48x40"])
def test_bound_is_not_vacuous(name, mutate):
    """Each mistake puts at least a quarter of the elements of the tensor it touches outside the bound."""
    if mutate == "no_is_detected" and name == "featloss_ragged_48x40":
        pytest.skip("every frame of this fixture is detected")
    shares = _share_outside(name, mutate)
    assert max(shares.values()) >= 0.25, (name, mutate, shares)
