"""CPU: the float64 model of the radius outlier filter (tests/outlier_model.py) against scipy's KD-tree, and the host side
of sr_radius_outlier_mask (argument validation, scratch sizing) through the C ABI."""
import ctypes as C

import numpy as np
import pytest

from .outlier_model import keep_and_capped, radius_counts

SR_EINVAL = -1


def _points_clear_of_radius(rng, P, r, spread):
    """Random float32 points with no pair whose float64 distance lies within 1e-9 of r (so < and <= agree)."""
    x = (rng.random((P, 3)) * spread).astype(np.float32)
    while True:
        d = np.sqrt(((x[:, None, :].astype(np.float64) - x[None, :, :]) ** 2).sum(-1))
        bad = np.abs(d - r) < 1e-9
        if not bad.any():
            return x
        i = np.nonzero(bad.any(1))[0]
        x[i] = (rng.random((len(i), 3)) * spread).astype(np.float32)


@pytest.mark.parametrize("P,r,spread", [(1500, 0.05, 1.0), (800, 0.3, 1.0), (1200, 0.01, 0.2)])
def test_model_matches_kdtree(P, r, spread):
    from scipy.spatial import cKDTree
    rng = np.random.default_rng(P)
    x = _points_clear_of_radius(rng, P, r, spread)
    x[:40] = x[40:80]                          # clone-style duplicates: distance 0, counted both ways
    got = radius_counts(x, r)
    # cKDTree's ball query counts d <= r; with no distance within 1e-9 of r that is the same set as d2 < r2
    want = cKDTree(x.astype(np.float64)).query_ball_point(x.astype(np.float64), r, return_length=True)
    assert np.array_equal(got, want)
    assert got.min() >= 1 and got.max() > 5    # the point itself is counted; some points have company


def test_model_non_finite_and_exact_radius():
    x = np.array([[0, 0, 0], [3, 4, 0], [np.nan, 0, 0], [np.inf, 0, 0], [0, -np.inf, 1], [0, 0, 0]], dtype=np.float32) / 1024
    c = radius_counts(x, 5 / 1024)              # (0,0,0)-(3,4,0)/1024 is at exactly r: not a neighbour
    assert c.tolist() == [2, 1, 0, 0, 0, 2]
    c = radius_counts(x, np.nextafter(5 / 1024, 1.0))
    assert c.tolist() == [3, 3, 0, 0, 0, 3]
    keep, capped = keep_and_capped(c, 0)
    assert keep.tolist() == [True, True, False, False, False, True] and capped.tolist() == [1, 1, 0, 0, 0, 1]


def test_invalid_arguments_return_einval(built):
    from vidu4d_b200 import _capi
    lib = _capi.load()
    p = C.c_void_p(16)                           # never dereferenced: every call below fails validation first
    nbytes = lib.sr_radius_outlier_scratch_bytes(10)
    ok = dict(P=10, points=p, radius=0.004, nb=20, keep=p, counts=None, scratch=p, nbytes=nbytes)

    def call(**kw):
        a = {**ok, **kw}
        return lib.sr_radius_outlier_mask(a["P"], a["points"], a["radius"], a["nb"], a["keep"], a["counts"], a["scratch"],
                                          a["nbytes"], None)
    for bad in (dict(P=-1), dict(nb=-1), dict(radius=0.0), dict(radius=-1e-3), dict(radius=float("nan")),
                dict(radius=float("inf")), dict(nbytes=nbytes - 1), dict(points=None), dict(keep=None), dict(scratch=None)):
        assert call(**bad) == SR_EINVAL, bad
        assert lib.sr_last_error()
    # P = 0 is a no-op: nothing is read, nothing is launched
    assert call(P=0, points=None, keep=None, scratch=None, nbytes=0) == 0


def test_scratch_size_monotone_in_P(built):
    from vidu4d_b200 import _capi
    lib = _capi.load()
    assert lib.sr_radius_outlier_scratch_bytes(0) == 0
    assert lib.sr_radius_outlier_scratch_bytes(-5) == 0
    prev = 0
    for P in (1, 2, 3, 255, 256, 257, 10_000, 200_000, 300_000, 1_000_000, 2**31 - 1):
        b = lib.sr_radius_outlier_scratch_bytes(P)
        assert b >= prev and b % 256 == 0              # sub-arrays are 256-byte aligned: small P share a size
        # keys, indices (both double-buffered), sorted points and the sort's temporaries: at most 48 bytes per point + 2 MB
        assert b <= 48 * P + (2 << 20), (P, b)
        prev = b
    assert lib.sr_radius_outlier_scratch_bytes(300_000) > lib.sr_radius_outlier_scratch_bytes(200_000)
