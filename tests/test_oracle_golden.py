"""CPU: pin the oracle (oracle/surfel_oracle.c) to outputs of the UNMODIFIED reference extension.

The fixtures in tests/golden/*.npz were produced by tests/golden/make_golden.py from the reference extension compiled
for sm_100a (oracle/_ref/_C.so) (the reference has no tests or golden vectors of its own for this path, SURVEY.md section 4).
Integer / index work must be bit-exact; float buffers within 1e-4 (north_star tolerance), in practice ~1e-6.
"""
import numpy as np
import pytest

from .conftest import GOLDEN_CASES, load_golden, oracle_forward_from_golden

TOL = 1e-4


@pytest.fixture(scope="module", params=GOLDEN_CASES)
def case(request, built):
    g = load_golden(request.param)
    st = oracle_forward_from_golden(g)
    return request.param, g, st


def test_binning_bit_exact(case):
    name, g, st = case
    assert st.num_rendered == int(g["ref_num_rendered"][0])
    np.testing.assert_array_equal(st.radii, g["ref_radii"])
    np.testing.assert_array_equal(st.tiles_touched.astype(np.int64), g["ref_geom_tiles_touched"].astype(np.int64))
    vis = g["ref_radii"] > 0
    # sort keys = (tile << 32 | depth bits): bit-exact, hence so are the view-space depths
    np.testing.assert_array_equal(st.depths[vis].view(np.int32), g["ref_geom_depths"][vis].view(np.int32))
    np.testing.assert_array_equal(st.keys_unsorted.astype(np.int64), g["ref_bin_keys_unsorted"])
    np.testing.assert_array_equal(st.keys.astype(np.int64), g["ref_bin_keys"])
    np.testing.assert_array_equal(st.point_list.astype(np.int64), g["ref_bin_point_list"].astype(np.int64))
    np.testing.assert_array_equal(st.ranges.astype(np.int64), g["ref_img_ranges"].astype(np.int64))


def test_contributor_counts_exact(case):
    name, g, st = case
    nc = g["ref_img_n_contrib"].astype(np.int64) & 0xFFFFFFFF
    np.testing.assert_array_equal(st.n_contrib.astype(np.int64), nc)


def test_projected_geometry(case):
    name, g, st = case
    vis = g["ref_radii"] > 0
    # T matrices / box centres / normals: the oracle follows the reference's FMA map; the only source of
    # difference is rsqrtf (MUFU.RSQ on the GPU, 1/sqrtf here): a couple of ulp
    # (the box centre divides by d = Tw.x^2+Tw.y^2-Tw.z^2, which is ill-conditioned for the one giant surfel of
    #  `single_32`: allow 5e-5 there)
    for mine, ref, tol in ((st.transMat, g["ref_geom_transMat"], 2e-6), (st.means2D, g["ref_geom_means2D"], 5e-5),
                           (st.normal_opacity[:, :3], g["ref_geom_normal_opacity"][:, :3], 2e-6)):
        a, b = mine[vis], ref[vis]
        assert np.abs(a - b).max() <= tol * max(1.0, np.abs(b).max())
    if g["in_meta"][4] == 0:
        assert np.abs(st.rgb[vis] - g["ref_geom_rgb"][vis]).max() < 5e-6
        np.testing.assert_array_equal(st.clamped[vis].astype(bool), g["ref_geom_clamped"][vis].astype(bool))


def test_rendered_buffers(case):
    name, g, st = case
    for mine, ref, what in ((st.color, g["ref_color"], "color"), (st.allmap, g["ref_allmap"], "allmap"),
                            (st.final_T, g["ref_img_final_T"], "final_T")):
        err = np.abs(mine - ref)
        assert err.max() <= TOL * max(1.0, np.abs(ref).max()), (name, what, err.max())


def test_gradients(case):
    from oracle import surfel_oracle as so
    name, g, st = case
    og = so.backward(st, g["in_dL_dcolor"], g["in_dL_dallmap"])
    for k in ("dL_dmeans2D", "dL_dcolors", "dL_dopacity", "dL_dmeans3D", "dL_dtransMat", "dL_dsh", "dL_dscales",
              "dL_drotations"):
        ref = g["ref_grad_" + k]
        if ref.size == 0:
            continue
        mine = og[k].reshape(ref.shape)
        scale = np.abs(ref).max() + 1e-30
        assert np.abs(mine - ref).max() / scale <= TOL, (name, k, np.abs(mine - ref).max() / scale)


def test_mark_visible(built):
    from oracle import surfel_oracle as so
    g = load_golden("near_cull_64")
    vis = so.mark_visible(g["in_means3D"], g["in_viewmatrix"])
    z = g["in_means3D"] @ g["in_viewmatrix"].reshape(4, 4)[:3, 2] + g["in_viewmatrix"].reshape(4, 4)[3, 2]
    clear = np.abs(z - 0.2) > 1e-5
    np.testing.assert_array_equal(vis[clear], (z > 0.2)[clear])
    # every surfel the reference rendered is in front of the near plane
    assert vis[g["ref_radii"] > 0].all()


def test_empty_and_degenerate(built):
    from oracle import surfel_oracle as so
    kw = dict(sh_degree=0, W=32, H=32, tanfovx=0.5, tanfovy=0.5, bg=(0.5, 0.25, 0.125))
    # P = 0: the reference short-circuits (rasterize_points.cu:106)
    st = so.forward(np.zeros((0, 3)), np.zeros((0, 1)), np.zeros((0, 2)), np.zeros((0, 4)), colors_precomp=np.zeros((0, 3)), **kw)
    assert st.num_rendered == 0 and st.radii.shape == (0,)
    # all surfels behind the near plane -> nothing binned, background everywhere
    P = 10
    m = np.zeros((P, 3), np.float32); m[:, 2] = 0.1
    q = np.tile(np.array([1, 0, 0, 0], np.float32), (P, 1))
    st = so.forward(m, np.full((P, 1), 0.9), np.full((P, 2), 0.05), q, colors_precomp=np.full((P, 3), 0.5), **kw)
    assert st.num_rendered == 0 and (st.radii == 0).all()
    np.testing.assert_allclose(st.color[:, 5, 5], [0.5, 0.25, 0.125])
    assert (st.allmap == 0).all()
    # exactly-one-of (SHs | colours): same exception text as the reference
    with pytest.raises(Exception, match="excatly one of either SHs or precomputed colors"):
        so.forward(m, np.full((P, 1), 0.9), np.full((P, 2), 0.05), q, **kw)
