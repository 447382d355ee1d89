"""The CPU oracle's knife mask, rounding-error bound sums and per-surfel chain (oracle/surfel_oracle.c), which
tests/test_gpu_grad_bounds.py builds its per-element bounds from.  No GPU."""
import numpy as np
import pytest

from oracle import surfel_oracle as so

GRADS = ("dL_dmeans2D", "dL_dcolors", "dL_dopacity", "dL_dmeans3D", "dL_dtransMat", "dL_dsh", "dL_dscales", "dL_drotations",
         "dL_dnormal")
U = 2.0 ** -24
K = 2.0
THR = np.float32(1.0 / 255.0)


def _facing_records(W, H, mx, my, sigma, opac, order=None, seed=0):
    """Hand-built records of surfels that face the camera: transMat rows Tu = (-1, 0, mx / s), Tv = (0, -1, my / s),
    Tw = (0, 0, 1 / s), so that at pixel centre (x, y) k = x Tw - Tu = (1, 0, (x - mx) / s), l = (0, 1, (y - my) / s),
    p_z = 1, rho3d = |(x, y) - (mx, my)|^2 / s^2, the depth is 1 / s, and at the surfel's centre G = exp(0) = 1 exactly:
    alpha = opacity.  All surfels in the one 16 x 16 tile, in list order `order`."""
    rng = np.random.default_rng(seed)
    mx, my, sigma, opac = (np.atleast_1d(np.asarray(v, np.float64)) for v in (mx, my, sigma, opac))
    P = mx.size
    T = np.zeros((P, 9), np.float32)
    T[:, 0], T[:, 2] = -1.0, mx / sigma
    T[:, 4], T[:, 5] = -1.0, my / sigma
    T[:, 8] = 1.0 / sigma
    no = np.zeros((P, 4), np.float32)
    no[:, 2] = -1.0
    no[:, 3] = opac.astype(np.float32)
    rgb = rng.uniform(0.1, 1.0, (P, 3)).astype(np.float32)
    pl = np.arange(P, dtype=np.uint32) if order is None else np.asarray(order, np.uint32)
    tiles = ((W + 15) // 16) * ((H + 15) // 16)
    ranges = np.zeros((tiles, 2), np.uint32)
    ranges[0] = (0, pl.size)
    return dict(means3D=rng.normal(size=(P, 3)).astype(np.float32) + np.float32([0, 0, 3]), opacities=no[:, 3],
                scales=np.full((P, 2), 0.1, np.float32), rotations=np.tile(np.float32([1, 0, 0, 0]), (P, 1)),
                colors_precomp=rgb, sh_degree=0, W=W, H=H, tanfovx=0.5, tanfovy=0.5, bg=(0.0, 0.0, 0.0),
                viewmatrix=np.eye(4, dtype=np.float32), campos=np.zeros(3, np.float32),
                transMat=T, means2D=np.stack([mx, my], 1).astype(np.float32), normal_opacity=no, rgb=rgb,
                radii=np.full(P, 3, np.int32), clamped=np.zeros((P, 3), np.uint8), point_list=pl, ranges=ranges)


def _signs():
    # a broad surfel over the whole tile (sigma 4: depth 0.25, alpha ~ 0.07 at 8 px) behind a point-like one centred on
    # pixel (5, 5) whose alpha there is its opacity
    return dict(mx=[8.0, 5.5], my=[8.0, 5.5], sigma=[4.0, 1.0])


def test_knife_mask_flags_alpha_one_ulp_either_side_of_the_threshold():
    for o in (np.nextafter(THR, np.float32(1)), np.nextafter(THR, np.float32(0))):
        st, ext = so.from_records(**_facing_records(16, 16, opac=[0.5, o], **_signs()))
        assert ext["knife"][5, 5], o
        # with alpha = opacity just above the threshold the point contributes at its centre, just below it does not
        assert st.n_contrib[0][5, 5] == (2 if o >= THR else 1)
    # far from every threshold: alpha = 0.5 at the centre, T = 1 before it and 0.5 * (1 - alpha_broad) after
    st, ext = so.from_records(**_facing_records(16, 16, opac=[0.5, 0.5], **_signs()))
    assert not ext["knife"].any()
    assert st.n_contrib[0][5, 5] == 2


def _upstream(H, W, seed, knife=None):
    rng = np.random.default_rng(seed)
    dc = rng.normal(size=(3, H, W)).astype(np.float32)
    do = rng.normal(size=(8, H, W)).astype(np.float32)
    if knife is not None:
        dc *= ~knife
        do *= ~knife
    return dc, do


def _tolerance(st, g):
    B = g["bound"] + (1 + 32) * g["asum"]           # one tile: one cross-tile rounding; the chain's own roundings
    return {k: K * U * v for k, v in so.chain_bound(st, B).items()}


def test_masking_the_knife_pixel_removes_it_exactly():
    """Opacity 1 ulp above / below 1/255 flips the point's contribution at its centre.  With that pixel's upstream
    gradient zeroed, the two states' gradients agree within the bound everywhere; without, they do not."""
    up, down = np.nextafter(THR, np.float32(1)), np.nextafter(THR, np.float32(0))
    sa, ea = so.from_records(**_facing_records(16, 16, opac=[0.5, up], **_signs()))
    sb, eb = so.from_records(**_facing_records(16, 16, opac=[0.5, down], **_signs()))
    assert ea["knife"][5, 5] and eb["knife"][5, 5]
    mask = ea["knife"] | eb["knife"]
    dc, do = _upstream(16, 16, 3, mask)
    ga, gb = so.backward(sa, dc, do, bounds=True), so.backward(sb, dc, do, bounds=True)
    tol = _tolerance(sa, ga)
    for k in GRADS:
        assert (np.abs(ga[k].astype(np.float64) - gb[k]) <= tol[k] + 1e-38).all(), k
    dc, do = _upstream(16, 16, 3)
    ga, gb = so.backward(sa, dc, do, bounds=True), so.backward(sb, dc, do, bounds=True)
    tol = _tolerance(sa, ga)
    assert any((np.abs(ga[k].astype(np.float64) - gb[k]) > tol[k] + 1e-38).any() for k in GRADS)


def _scene(P=3000, W=96, H=80, seed=5, rigid=False):
    """build_case's scene; rigid=True moves the camera by a generic rotation (far from symmetric, unlike build_case's
    rigid view), so that a transposed view matrix anywhere in the chain shows."""
    from tests.golden.make_golden import build_case
    inp = build_case(P, W, H, seed)
    if rigid:
        from vidu4d_b200.synthetic import Scene, projection_matrix, random_rotation, rigid_view
        sc = Scene(means3D=inp["means3D"], scales=inp["scales"], rotations=inp["rotations"], opacities=inp["opacities"],
                   shs=inp["shs"])
        sc, vm, cp = rigid_view(sc, random_rotation(np.random.default_rng(1)), np.array([0.1, -0.05, 0.2]))
        inp.update(means3D=sc.means3D, rotations=sc.rotations, viewmatrix=vm.astype(np.float32), campos=cp,
                   projmatrix=(vm.astype(np.float64) @ projection_matrix(0.5, 0.5)).astype(np.float32))
    st = so.forward(inp["means3D"], inp["opacities"], inp["scales"], inp["rotations"], shs=inp["shs"], sh_degree=3, W=W, H=H,
                    tanfovx=0.5, tanfovy=0.5, bg=inp["bg"], viewmatrix=inp["viewmatrix"], projmatrix=inp["projmatrix"],
                    campos=inp["campos"])
    return inp, st


def test_bound_sums_dominate_the_accumulators():
    inp, st = _scene()
    so.composite_ext(st)
    g = so.backward(st, inp["dL_dcolor"], inp["dL_dallmap"], bounds=True)
    acc = np.abs(g["acc"])
    assert (g["asum"] >= acc * (1 - 1e-5)).all()
    assert (g["bound"] >= 32 * g["asum"]).all()            # every weight is at least the per-term roundings
    assert (g["asum"][st.radii > 0] > 0).any()


def test_bound_sums_equal_the_accumulators_for_single_pairs():
    """Point-like surfels 3 px apart, each the only contributor of one pixel, and one upstream plane: every accumulator
    element has a single, cancellation-free term, so its magnitude sum equals it."""
    xs = np.arange(4) * 3 + 2.3
    mx, my = np.repeat(xs, 4), np.tile(xs, 4)
    st, ext = so.from_records(**_facing_records(16, 16, mx, my, sigma=0.3, opac=np.full(16, 0.006), seed=4))
    # walk_S sums 1 / (1 - alpha) over a pixel's contributors: one contributor each at 16 pixels, none elsewhere
    assert (ext["walk_S"] < 1.5).all() and (ext["walk_S"] > 0).sum() == 16
    assert sorted(st.n_contrib[0][st.n_contrib[0] > 0].tolist()) == list(range(1, 17))
    dc = np.zeros((3, 16, 16), np.float32)
    dc[0] = np.random.default_rng(6).normal(size=(16, 16))
    g = so.backward(st, dc, np.zeros((8, 16, 16), np.float32), bounds=True)
    np.testing.assert_allclose(g["asum"], np.abs(g["acc"]), rtol=1e-5, atol=0)
    assert (g["acc"][:, so.ACC_OPAC] != 0).all() and (g["acc"][:, so.ACC_M2D] != 0).all()


@pytest.mark.parametrize("rigid", [False, True], ids=["identity_view", "rigid_view"])
def test_chain_reproduces_backward_bit_for_bit_and_is_linear(rigid):
    """On a rigid view as well: with the identity view matrix |W| = |W^T| would hide a transposed W^T shadow."""
    inp, st = _scene(rigid=rigid)
    vm = np.asarray(inp["viewmatrix"], np.float64)[:3, :3]
    assert rigid == (np.abs(vm - vm.T).max() > 0.5)
    so.composite_ext(st)
    g = so.backward(st, inp["dL_dcolor"], inp["dL_dallmap"], bounds=True)
    c = so.chain(st, g["acc"])
    for k in GRADS:
        assert c[k].tobytes() == g[k].tobytes(), k
    rng = np.random.default_rng(9)
    a, b = rng.normal(size=g["acc"].shape), rng.normal(size=g["acc"].shape)
    ca, cb, cab = so.chain(st, a), so.chain(st, b), so.chain(st, a - 3 * b)
    ba = so.chain_bound(st, np.abs(a))
    for k in GRADS:
        lin = ca[k].astype(np.float64) - 3 * cb[k]
        scale = np.abs(ca[k]).max() + 3 * np.abs(cb[k]).max() + 1e-30
        assert np.abs(lin - cab[k]).max() <= 1e-5 * scale, k
        # |chain(a)| <= the chain on absolute values (up to fp32 rounding)
        assert (np.abs(ca[k]) <= ba[k] * (1 + 1e-5) + 1e-30).all(), k
    # ... which dominates the Jacobian entry by entry: sum_j |chain(e_j)| |a_j| <= chain_bound(|a|)
    jb = {k: np.zeros_like(v) for k, v in ba.items()}
    for j in range(so.NACC):
        e = np.zeros_like(a)
        e[:, j] = 1.0
        cj = so.chain(st, e)
        for k in GRADS:
            jb[k] += np.abs(cj[k].astype(np.float64)) * np.abs(a[:, j]).reshape((-1,) + (1,) * (cj[k].ndim - 1))
    for k in GRADS:
        assert (jb[k] <= ba[k] * (1 + 1e-5) + 1e-30).all(), k


def test_new_options_leave_every_output_unchanged():
    inp, st = _scene()
    plain = so.backward(st, inp["dL_dcolor"], inp["dL_dallmap"])
    planes = [st.color.copy(), st.allmap.copy(), st.final_T.copy(), st.n_contrib.copy()]
    ext = so.composite_ext(st)                              # the composite again, with every optional output
    for a, b in zip(planes, [st.color, st.allmap, st.final_T, st.n_contrib]):
        assert a.tobytes() == b.tobytes()
    assert ext["fbound"].shape == (14, 80, 96)
    assert ((ext["walk_S"] >= 1) == (st.n_contrib[0] > 0)).all() and ((ext["walk_S"] == 0) == (st.n_contrib[0] == 0)).all()
    bound = so.backward(st, inp["dL_dcolor"], inp["dL_dallmap"], bounds=True)
    for k in GRADS:
        assert plain[k].tobytes() == bound[k].tobytes(), k
    # the composite from the forward's own records = the forward
    rs, _ = so.from_records(inp["means3D"], inp["opacities"], inp["scales"], inp["rotations"], shs=inp["shs"], sh_degree=3,
                            W=96, H=80, tanfovx=0.5, tanfovy=0.5, bg=inp["bg"], viewmatrix=inp["viewmatrix"],
                            projmatrix=inp["projmatrix"], campos=inp["campos"], transMat=st.transMat, means2D=st.means2D,
                            normal_opacity=st.normal_opacity, rgb=st.rgb, radii=st.radii, clamped=st.clamped,
                            point_list=st.point_list, ranges=st.ranges)
    for a, b in zip(planes, [rs.color, rs.allmap, rs.final_T, rs.n_contrib]):
        assert a.tobytes() == b.tobytes()
    again = so.backward(rs, inp["dL_dcolor"], inp["dL_dallmap"])
    for k in GRADS:
        assert plain[k].tobytes() == again[k].tobytes(), k


def test_bounds_need_the_composite_walk():
    inp, st = _scene(P=500, W=32, H=32)
    with pytest.raises(ValueError, match="composite_ext"):
        so.backward(st, inp["dL_dcolor"], inp["dL_dallmap"], bounds=True)
