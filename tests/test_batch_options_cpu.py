"""tests/batch_options.py without a GPU: the covering array covers every level and every valid pair of levels, is the
same on every build, stays small; the tolerance composition reduces to the existing single-option ones."""
import itertools
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from . import batch_options as BO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_every_valid_pair_is_covered():
    covered = set().union(*(BO.pairs_of(c) for c in BO.CASES))
    missing = BO.all_pairs() - covered
    assert not missing, sorted(missing, key=repr)[:8]
    for c in BO.CASES:
        assert tuple(c) == BO.NAMES and BO.valid(c), c
    for n, levels in BO.FACTORS.items():
        assert {c[n] for c in BO.CASES} == set(levels), n
    print(f"\n{len(BO.CASES)} cases cover all {len(BO.all_pairs())} valid pairs")


def test_invalid_pairs_are_the_documented_ones():
    """Left out: feature options without features (and with features, no feature option left unset), and an SH degree
    with colors_precomp (and SH colours without one)."""
    bad = set()
    for a, b in itertools.combinations(BO.NAMES, 2):
        for la in BO.FACTORS[a]:
            for lb in BO.FACTORS[b]:
                if not BO.valid({a: la, b: lb}):
                    bad.add(frozenset((a, b)))
    assert bad == {frozenset(p) for p in (("colour", "sh"), ("features", "planes"), ("features", "background"),
                                          ("planes", "background"))}


def test_edge_cases_in_the_array():
    # M = 1 with sum_shared: sr_backward ignores the flag; it must stay in the array
    assert any(c["M"] == 1 and c["sum_shared"] for c in BO.CASES)
    assert any(c["M"] == 5 and c["camera"] == "table_offsets" and c["features"] for c in BO.CASES)


def test_array_is_deterministic_and_small():
    assert BO.covering_array() == BO.CASES
    code = "from tests import batch_options as b; print([b.case_id(c) for c in b.CASES])"
    env = dict(os.environ, PYTHONHASHSEED="12345")
    got = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True, check=True)
    assert got.stdout.strip() == str([BO.case_id(c) for c in BO.CASES])
    assert len(BO.CASES) <= 30, len(BO.CASES)
    assert len({BO.case_id(c) for c in BO.CASES}) == len(BO.CASES)


# ------------------------------------------------------------------------------------------------ frame_reference
def _state():
    from oracle import surfel_oracle as so
    from .test_oracle_bounds_cpu import _scene
    inp, st = _scene(P=2000, W=72, H=56, seed=9)
    so.composite_ext(st)
    return inp, st


def _groups(st, F, seed):
    """Feature groups of 3 channels composited on st's records, each a colour run (test_gpu_feature_bounds)."""
    from oracle import surfel_oracle as so
    rng = np.random.default_rng(seed)
    n = (F + 2) // 3
    feat = np.zeros((st.P, 3 * n), np.float32)
    feat[:, :F] = rng.standard_normal((st.P, F))
    inp = st._inputs
    out = []
    for k in range(n):
        sg, _ = so.from_records(inp["means3D"], inp["opacities"], inp["scales"], inp["rotations"], None,
                                np.ascontiguousarray(feat[:, 3 * k:3 * k + 3]), sh_degree=0, W=st.W, H=st.H,
                                tanfovx=inp["tanfovx"], tanfovy=inp["tanfovy"], bg=np.zeros(3, np.float32),
                                viewmatrix=inp["viewmatrix"], projmatrix=inp["projmatrix"], campos=inp["campos"],
                                transMat=st.transMat, means2D=st.means2D, normal_opacity=st.normal_opacity, rgb=st.rgb,
                                radii=st.radii, clamped=st.clamped, point_list=st.point_list, ranges=st.ranges)
        out.append((sg, 3))
    return out


def _same(a, b):
    for k in a:
        assert np.array_equal(np.asarray(a[k]), np.asarray(b[k])), k


def test_reference_with_features_and_zero_offsets_is_the_feature_tests(monkeypatch):
    from oracle import surfel_oracle as so
    from . import test_gpu_feature_bounds as FB
    inp, st = _state()
    F = 7
    fr = dict(st=st, groups=_groups(st, F, 3), F=F)
    rng = np.random.default_rng(4)
    dLf = rng.standard_normal((F, st.H, st.W)).astype(np.float32)
    FB._oracle_bwd(fr, inp["dL_dcolor"], inp["dL_dallmap"], dLf)
    tiles = rng.integers(1, 5, st.P).astype(np.float64)
    fallback = rng.integers(0, 3, st.P)
    m = rng.integers(0, 50, st.P)
    monkeypatch.setattr(FB, "_fallback_pairs", lambda dec, P: fallback)
    ref, tol = FB._total(fr, {"tiles_touched": torch.from_numpy(tiles)}, m, F)
    adds = tiles + fallback + FB._chunks(F)[0] * m + FB.CHAIN + FB.SLACK
    for off in (None, (0.0, 0.0)):
        mine, mtol = BO.frame_reference(st, fr["og_c"], fr["og_g"], adds, off)
        _same(ref, mine)
        _same(tol, mtol)
    assert any(np.abs(v).max() > 0 for v in so.chain(st, fr["og_g"][0]["acc"]).values())


def test_reference_without_features_is_the_off_centre_tests():
    from oracle import surfel_oracle as so
    from . import camera_model as cm
    inp, st = _state()
    og = so.backward(st, inp["dL_dcolor"], inp["dL_dallmap"], bounds=True)
    adds = np.full(st.P, 3.0) + 32
    for ox, oy in ((7.25, -3.5), (-11.75, 5.125)):
        B = og["bound"] + adds[:, None] * og["asum"]
        B = cm.offset_bound_sums(st, B, og["acc"], og["dL_dtransMat"], ox, oy)
        tol = {k: BO.K * BO.U * v for k, v in so.chain_bound(st, B).items()}
        ref = dict(og, **cm.offset_chain(st, og["acc"], og["dL_dtransMat"], ox, oy))
        mine, mtol = BO.frame_reference(st, og, [], adds, (ox, oy))
        _same({k: ref[k] for k in mine}, mine)
        _same(tol, mtol)
    # and with zero offsets, test_gpu_grad_bounds._bounds' composition on the centred chain
    mine, mtol = BO.frame_reference(st, og, [], adds, (0.0, 0.0))
    _same({k: og[k] for k in mine if k in og}, mine)
    _same({k: BO.K * BO.U * v for k, v in so.chain_bound(st, og["bound"] + adds[:, None] * og["asum"]).items()}, mtol)


@pytest.mark.parametrize("off", [(0.0, 0.0), (9.5, -4.25)])
def test_offsets_compose_with_features(off):
    """The new composition: the (offset) chain of the combined accumulator is, within the combined tolerance, the
    colour run's plus the chain of the groups' non-colour accumulators alone (the chain is linear in the accumulator,
    each evaluation rounds in fp32); its bound dominates the colour-only one; non-zero offsets change the result."""
    from oracle import surfel_oracle as so
    from . import camera_model as cm
    from . import test_gpu_feature_bounds as FB
    inp, st = _state()
    F = 7
    fr = dict(st=st, groups=_groups(st, F, 5), F=F)
    FB._oracle_bwd(fr, inp["dL_dcolor"], inp["dL_dallmap"],
                   np.random.default_rng(6).standard_normal((F, st.H, st.W)).astype(np.float32))
    adds = np.full(st.P, 40.0)
    ref, tol = BO.frame_reference(st, fr["og_c"], fr["og_g"], adds, off)
    ref_c, tol_c = BO.frame_reference(st, fr["og_c"], [], adds, off)
    g_acc = sum(np.array(og["acc"], np.float64, copy=True) for og in fr["og_g"])
    g_acc[:, BO.C3] = 0.0
    tm_g = so.chain(st, g_acc)["dL_dtransMat"]
    ref_g = cm.offset_chain(st, g_acc, tm_g, *off) if any(off) else so.chain(st, g_acc)
    assert any(np.abs(ref_g[k]).max() > 0 for k in ref_g)
    for k in tol:
        err = np.abs(ref[k].astype(np.float64) - (ref_c[k].astype(np.float64) + ref_g[k]))
        assert (err <= tol[k] + 1e-38).all(), (k, float((err / (tol[k] + 1e-38)).max()))
        assert (tol[k] >= tol_c[k]).all(), k
    if any(off):
        centred, _ = BO.frame_reference(st, fr["og_c"], fr["og_g"], adds, None)
        assert not np.array_equal(centred["dL_dmeans3D"], ref["dL_dmeans3D"])
