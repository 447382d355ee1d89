"""Every buffer the binning stage writes, bit for bit against tests/binning_model.py, at the edges where it can go wrong.

For every case and every frame: num_rendered and the overflow bit, tiles_touched, point_offsets, the sorted keys and
point list, the tile ranges, every field of every instance record (as int32 bits), the 64 sort control words (pass
count, skip vector, ping/pong parity, tickets handed out) and the tile order's two properties (a permutation; buckets
never rise).  The model reads only the GPU's own per-surfel records (centres, radii, depths), which
tests/test_gpu_preprocess_bounds.py pins to the inputs.

Each case asserts, from the GPU's own buffers, that it reaches the edge it exists for and prints it: key width and
pass count (5, 6 and 7 passes; 1-bit and 8-bit last passes), skip vectors that flip the ping/pong parity, R at the
edges of the 384-key warp, the 3072-key sort tile and the 4096-key histogram block, a sort of over 1000 sort tiles,
emission at the 32/33-tile boundary of the cooperative path, clamped rectangles, ties, R = capacity, an overflowed
frame inside a batch, and scratch buffers full of 0xFF before the forward.

Scenes are built directly for an identity camera with tan(fov / 2) = 0.5, so the focal lengths are W and H pixels, the
depth key is the surfel's z bit for bit and a face-on surfel's centre lands where it is put.  Small face-on surfels
(radius 3 px) centred in a tile's interior touch exactly that tile."""
import numpy as np
import pytest
import torch

from . import binning_model as bm

pytestmark = pytest.mark.gpu

F32 = np.float32
TAN = 0.5
NEAR = 0.1                          # a surfel at this depth is culled (near plane 0.2): it emits nothing


@pytest.fixture(scope="module")
def dev(built):
    from vidu4d_b200 import _capi, rasterizer as RZ
    _capi.load()
    RZ.set_sync_mode(True)          # every case reads num_rendered back and decodes the buffers it sized
    return torch.device("cuda:0")


def _np(x):
    return x.detach().cpu().numpy()


# ------------------------------------------------------------------------------------------------ scenes
def place(u, v, z, W, H, foot=0.05):
    """Face-on surfels whose projected centres are the pixel positions (u, v) at depths z, footprint `foot` px (radius
    3 px below a footprint of 0.7 px).  Returns (means (n, 3), scales (n, 2))."""
    u, v, z = (np.broadcast_to(np.asarray(a, np.float64), np.broadcast(u, v, z).shape) for a in (u, v, z))
    means = np.stack([(u - W / 2) * z / W, (v - H / 2) * z / H, z], 1)
    s = np.asarray(foot, np.float64) * z / W
    return means.astype(F32), np.stack([s, s], 1).astype(F32)


def tile_centre(t, W):
    gx = (W + 15) // 16
    t = np.asarray(t)
    return (t % gx) * 16 + 8.0, (t // gx) * 16 + 8.0


def one_tile_each(tiles, z, W, H):
    """One small surfel centred in each of `tiles` (tile ids), at depths z."""
    u, v = tile_centre(tiles, W)
    return place(u, v, z, W, H)


def z_of_bits(bits):
    return np.asarray(bits, np.uint32).view(F32)


def footprint_for_radius(r):
    """The footprint (px) of a face-on surfel at z = 1 whose radius comes out as r: 3 e = r - 1/2, far from ceil's edges."""
    return (np.asarray(r, np.float64) - 0.5) / 3.0


# ------------------------------------------------------------------------------------------------ the forward
def _cams(M, dev):
    from vidu4d_b200.synthetic import projection_matrix
    vm = torch.eye(4, device=dev)
    pm = torch.from_numpy(projection_matrix(TAN, TAN).astype(F32)).to(dev)
    return vm.repeat(M, 1, 1).contiguous(), pm.repeat(M, 1, 1).contiguous(), torch.zeros((M, 3), device=dev)


def forward(dev, W, H, means, scales, rotations=None, opacities=None):
    """One batched forward of M frames (means (P, 3) or (M, P, 3), scales (P, 2) or (M, P, 2)).  Returns a dict: M, P,
    W, H, the per-frame num_rendered and overflow flags, radii (M, P) and the three scratch buffers, colour and allmap."""
    from vidu4d_b200 import rasterizer as RZ
    means, scales = np.asarray(means, F32), np.asarray(scales, F32)
    M = 1 if means.ndim == 2 else means.shape[0]
    P = means.shape[-2]
    rng = np.random.default_rng(P)
    if rotations is None:
        rotations = np.tile(np.array([1, 0, 0, 0], F32), (P, 1))
    if opacities is None:
        opacities = np.full((P, 1), 0.5, F32)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)     # noqa: E731
    vms, pms, cps = _cams(M, dev)
    e = torch.empty((0,), device=dev)
    bg = torch.tensor([0.1, 0.2, 0.3], device=dev)
    nr, color, allmap, radii, gb, bb, ib = RZ._C.rasterize_gaussians_batch(
        bg, t(means), t(rng.uniform(0, 1, (P, 3)).astype(F32)), t(opacities), t(scales), t(rotations), 1.0, vms, pms, TAN,
        TAN, H, W, e, 0, cps)[:7]
    if nr == -1:                                    # nosync: the status words of this call are the last pending ones
        torch.cuda.synchronize()
        words = RZ._pending[-1][0].tolist()
        nr, over = [r for r, _ in words], [bool(s & 1) for _, s in words]
    else:
        over = [False] * M
    return dict(M=M, P=P, W=W, H=H, nr=list(nr), over=over, radii=radii.view(M, P), bufs=(gb, bb, ib), color=color,
                allmap=allmap)


# ------------------------------------------------------------------------------------------------ the checks
def _u32(x):
    return np.ascontiguousarray(_np(x)).view(np.uint32)


def _same(name, what, gpu, model):
    gpu, model = np.asarray(gpu), np.asarray(model)
    assert gpu.shape == model.shape, (name, what, gpu.shape, model.shape)
    bad = np.argwhere(gpu != model)
    if bad.size:
        i = tuple(bad[0])
        raise AssertionError(f"{name}: {what} differs from the model at {i} ({len(bad)} elements differ): "
                             f"GPU {int(gpu[i]):#x}, model {int(model[i]):#x}")


def check_frame(name, r, f):
    """Frame f of forward()'s result against the model, every buffer; returns the edge report (npass, skip vector,
    R, sort tiles the passes ran, last pass's width) and the model's prediction, with the centres and radii it read."""
    from vidu4d_b200 import debug as dbg, rasterizer as RZ
    M, P, W, H = r["M"], r["P"], r["W"], r["H"]
    gb, bb, ib = (b.view(M, -1)[f] for b in r["bufs"])
    R, over = int(r["nr"][f]), r["over"][f]
    cap = RZ._capacity_from_bytes(int(bb.numel()), W, H)
    dec = dbg.decode(gb, bb, ib, P, W, H, 0 if over else R)
    rec = _np(dec["surfel_rec"]).reshape(P, 20)
    radii = _np(r["radii"][f]).astype(np.int64)
    m = bm.predict(rec[:, 9], rec[:, 10], radii, _np(dec["depths"]), W, H, cap)
    m.update(centre=(rec[:, 9], rec[:, 10]), radii=radii)
    name = f"{name} frame {f}"
    assert (R, over) == (m["R"], m["overflow"]), (name, "num_rendered / overflow", (R, over), (m["R"], m["overflow"]))
    _same(name, "tiles_touched", _u32(dec["tiles_touched"]), m["tiles_touched"])
    _same(name, "point_offsets", _u32(dec["point_offsets"]), m["point_offsets"])
    ctl = _u32(dec["sort_ctl"])
    _same(name, "sort_ctl", ctl, m["sort_ctl"])
    rg = _u32(dec["ranges"]).reshape(-1, 2)
    _same(name, "ranges", rg, m["ranges"])
    if not over:
        _same(name, "keys", np.ascontiguousarray(_np(dec["keys"])).view(np.uint64), m["keys"])
        _same(name, "point_list", _u32(dec["point_list"]), m["point_list"])
        for a in range(0, R, 1 << 20):             # in slices of 1 M instances (80 MB each)
            b = min(R, a + (1 << 20))
            inst = _u32(dec["inst_rec"][a:b]).reshape(b - a, 20)
            lo, hi = bm.inst_records(rec, m["point_list"][a:b], m["keys"][a:b], m["grid"][0])
            _same(name, f"inst_rec[{a}:]", np.where(inst == hi, lo, inst), lo)
    msg = bm.check_tile_order(_u32(dec["tile_order"]), rg)
    assert msg is None, (name, "tile_order", msg)
    npass = int(ctl[bm.CTL_NPASS])
    plan = bm.pass_plan(bm.key_bits(rg.shape[0]))
    rep = dict(npass=npass, skip=tuple(int(v) for v in ctl[bm.CTL_SKIP:bm.CTL_SKIP + npass]), R=R,
               sort_tiles=int(ctl[bm.CTL_TILE_COUNTER:bm.CTL_TILE_COUNTER + npass].max()), last_bits=plan[-1][1],
               overflow=over, cap=cap)
    print(f"\n[{name}] {W}x{H}: R {R} (capacity {cap}{', overflowed' if over else ''}), {npass} passes "
          f"(last {rep['last_bits']} bit{'s' if rep['last_bits'] > 1 else ''}), skip {''.join(map(str, rep['skip']))}, "
          f"{rep['sort_tiles']} sort tiles")
    return rep, m


def check_all(name, r):
    return [check_frame(name, r, f)[0] for f in range(r["M"])]


# ------------------------------------------------------------------------------------------------ key widths
PASS_CASES = {
    # image: (passes, last pass's width, skip vector): random depths in [1.5, 4) run every depth byte
    (16, 16): (5, 1, (0, 0, 0, 0, 1)),
    (240, 272): (5, 8, (0, 0, 0, 0, 0)),
    (256, 256): (6, 1, (0, 0, 0, 0, 0, 1)),
    (4080, 4112): (6, 8, (0, 0, 0, 0, 0, 0)),
    (4096, 4096): (7, 1, (0, 0, 0, 0, 0, 0, 1)),
}


@pytest.mark.parametrize("W,H", list(PASS_CASES))
def test_key_width_and_pass_count(W, H, dev):
    """One small surfel on the first tile, the last tile and up to 20000 tiles between, in random order and depth."""
    rng = np.random.default_rng(W * 7 + H)
    tiles = ((W + 15) // 16) * ((H + 15) // 16)
    t = np.concatenate([[0, tiles - 1], rng.integers(0, tiles, min(20000, 4 * tiles))])
    rng.shuffle(t)
    r = forward(dev, W, H, *one_tile_each(t, rng.uniform(1.5, 4.0, t.size), W, H))
    rep, = check_all(f"passes {W}x{H}", r)
    npass, last, skip = PASS_CASES[(W, H)]
    assert (rep["npass"], rep["last_bits"], rep["skip"], rep["R"]) == (npass, last, skip, t.size), rep


# ------------------------------------------------------------------------------------------------ skip patterns
def _skip_scene(pattern, rng):
    """(W, H, tiles, depths, expected skip vector) of a skip pattern."""
    n = 256
    if pattern == "all_skipped":                 # one tile, one depth: the result is the emission order
        return 16, 16, np.zeros(n, int), np.full(n, 2.0, F32), (1, 1, 1, 1, 1)
    if pattern == "depth_byte0":
        return 16, 16, np.zeros(n, int), F32(2.0) + rng.permutation(n).astype(F32) * F32(2.0 ** -22), (0, 1, 1, 1, 1)
    if pattern == "depth_byte1":
        return 16, 16, np.zeros(n, int), F32(2.0) + rng.permutation(n).astype(F32) * F32(2.0 ** -14), (1, 0, 1, 1, 1)
    if pattern == "exponent_bytes":
        return 16, 16, np.zeros(n, int), rng.choice(np.array([2, 4, 8, 16], F32), n), (1, 1, 0, 0, 1)
    if pattern == "top_tile_byte_constant":      # 65535 tiles, all surfels on tiles 0 .. 255: the 8-bit top pass skips
        return 4080, 4112, rng.integers(0, 256, n), np.full(n, 2.0, F32), (1, 1, 1, 1, 0, 1)
    if pattern == "alternating_run_skip":        # bytes 0, 2 and the low tile byte vary: src 0 1 1 0 0 1, sorted in pong
        bits = 0x40000000 | (rng.integers(0, 3, n) << 20) | rng.integers(0, 256, n)
        return 256, 256, rng.integers(0, 256, n), z_of_bits(bits), (0, 1, 0, 1, 0, 1)
    if pattern == "alternating_skip_run":        # bytes 1 and 3 vary, one tile: src 0 0 1 1 0 0, sorted back in ping
        bits = np.where(rng.random(n) < 0.5, 0x3F000000, 0x40000000) | (rng.integers(0, 256, n) << 8)
        return 256, 256, np.full(n, 37), z_of_bits(bits), (1, 0, 1, 0, 1, 1)
    if pattern == "all_but_one_share_digit":     # the one key that differs in byte 0 sorts first but is emitted last
        bits = np.full(n, 0x40000010)
        bits[-1] = 0x40000001
        return 16, 16, np.zeros(n, int), z_of_bits(bits), (0, 1, 1, 1, 1)
    raise KeyError(pattern)


SKIP_PATTERNS = ("all_skipped", "depth_byte0", "depth_byte1", "exponent_bytes", "top_tile_byte_constant",
                 "alternating_run_skip", "alternating_skip_run", "all_but_one_share_digit")


@pytest.mark.parametrize("pattern", SKIP_PATTERNS)
def test_skip_pattern(pattern, dev):
    W, H, tiles, z, skip = _skip_scene(pattern, np.random.default_rng(len(pattern)))
    r = forward(dev, W, H, *one_tile_each(tiles, z, W, H))
    rep, m = check_frame(f"skip {pattern}", r, 0)
    assert rep["skip"] == skip and rep["R"] == tiles.size, rep
    if pattern == "all_skipped":
        assert np.array_equal(m["point_list"], np.arange(tiles.size))
    if pattern == "all_but_one_share_digit":
        assert m["point_list"][0] == tiles.size - 1


# ------------------------------------------------------------------------------------------------ R edges
R_EDGES = (0, 1, 383, 384, 385, 3071, 3072, 3073, 4095, 4096, 4097, 6144)


def test_instance_count_edges(dev):
    """One frame per R of R_EDGES in one batch (128 x 128, 64 tiles): R visible one-tile surfels, the rest culled."""
    W = H = 128
    P, M = max(R_EDGES) + 5, len(R_EDGES)
    rng = np.random.default_rng(11)
    means, scales = np.empty((M, P, 3), F32), np.empty((M, P, 2), F32)
    for f, R in enumerate(R_EDGES):
        z = rng.uniform(1.5, 4.0, P)
        z[rng.permutation(P)[R:]] = NEAR
        means[f], scales[f] = one_tile_each(rng.integers(0, 64, P), z, W, H)
    reps = check_all("R edges", forward(dev, W, H, means, scales))
    assert [rp["R"] for rp in reps] == list(R_EDGES)
    # a lone key shares every digit with itself: R = 1 skips every pass like R = 0
    assert [rp["sort_tiles"] for rp in reps] == [-(-R // bm.SORT_TILE) if R > 1 else 0 for R in R_EDGES]


# ------------------------------------------------------------------------------------------------ emission
def _row_scene(lefts, radii, W, z=1.0):
    """Face-on surfels at depths z on a one-tile-row image whose rectangles are the given radii, centred so that the
    rectangle's left tile is `lefts` (x0 = floor((u - r) / 16) with u - r 4 px into that tile)."""
    r = np.asarray(radii, np.float64)
    u = np.asarray(lefts) * 16 + 4.0 + r
    return place(u, np.full(u.shape, 8.0), z, W, 16, footprint_for_radius(r))


def _width(radius, W):
    x0, _, x1, _ = bm.tile_rect(np.asarray(4.0 + radius, F32), np.float32(8), np.asarray(radius), (W + 15) // 16, 1)
    return int(x1 - x0)


def _radius_for_width(widths, W):
    """The smallest radius giving each rectangle width of _row_scene."""
    found = {}
    for w in np.unique(widths):
        found[w] = next(r for r in range(3, 16 * int(w)) if _width(r, W) == w)
    return np.array([found[w] for w in np.asarray(widths).reshape(-1)])


def test_cooperative_emission_boundary_and_ties(dev):
    """A one-row image (80 tiles): per warp, surfels touching 31, 32, 33 and 40 tiles, big ones at lanes 0 and 31 of
    every warp and in between, small ones around them; 48 surfels with one and the same 33-tile rectangle and depth (ties
    on the cooperative path) and 300 with one tile and one depth (ties on the per-thread path)."""
    W = 80 * 16
    rng = np.random.default_rng(21)
    P = 32 * 24
    widths = rng.choice([1, 2, 5, 31, 32, 33, 40], P)
    widths[0::32] = np.tile([32, 33], P // 64)
    widths[31::32] = np.tile([33, 32], P // 64)
    radii = _radius_for_width(widths, W)
    means, scales = _row_scene(rng.integers(0, 80 - widths + 1), radii, W, rng.uniform(1.5, 4.0, P))
    # ties: surfels 100 .. 147 share a 33-tile rectangle and a depth; 300 of the others share tile 7 and a depth
    tie_big = np.arange(100, 148)
    means[tie_big], scales[tie_big] = _row_scene(np.full(48, 3), _radius_for_width(np.full(48, 33), W), W, 2.5)
    tie_small = np.setdiff1d(rng.permutation(P), np.concatenate([tie_big, np.arange(0, P, 32), np.arange(31, P, 32)]))[:300]
    means[tie_small], scales[tie_small] = place(np.full(300, 7 * 16 + 8.0), np.full(300, 8.0), 1.75, W, 16)
    _, m = check_frame("emission", forward(dev, W, 16, means, scales), 0)
    tt = m["tiles_touched"].astype(np.int64)
    for lane in (0, 31):
        assert set(tt[lane::32]) == {32, 33}, (lane, sorted(set(tt[lane::32])))
    assert (tt[tie_big] == 33).all() and (tt[tie_small] == 1).all()
    assert {31, 32, 33, 40} <= set(tt)
    # equal keys keep ascending surfel ids, on both emission paths
    same = m["keys"][1:] == m["keys"][:-1]
    pl = m["point_list"].astype(np.int64)
    assert (pl[1:][same] > pl[:-1][same]).all()
    big_runs = np.isin(pl[1:], tie_big) & same
    small_runs = np.isin(pl[1:], tie_small) & same
    print(f"[emission] tied neighbours: cooperative path {int(big_runs.sum())}, per-thread path {int(small_runs.sum())}")
    assert big_runs.sum() >= 33 * 47 and small_runs.sum() >= 299


def test_clamped_rectangles(dev):
    """A 13 x 9 tile grid (200 x 136): big surfels centred beyond every edge and corner and on them, so that their
    rectangles clamp at each side, and one that covers the whole grid."""
    W, H = 200, 136
    rng = np.random.default_rng(31)
    u = np.concatenate([rng.uniform(-60, W + 60, 200), [-30, W + 30, W / 2, W / 2, -10, W + 10, -10, W + 10, W / 2]])
    v = np.concatenate([rng.uniform(-60, H + 60, 200), [H / 2, H / 2, -30, H + 30, -10, -10, H + 10, H + 10, H / 2]])
    foot = np.concatenate([rng.uniform(5, 40, 200), np.full(8, 20.0), [300.0]])
    means, scales = place(u, v, rng.uniform(1.5, 4.0, u.size), W, H, foot)
    _, m = check_frame("clamped", forward(dev, W, H, means, scales), 0)
    gx, gy = m["grid"]
    x0, y0, x1, y1 = m["rect"]
    vis = m["tiles_touched"] > 0
    (cx, cy), rad = m["centre"], m["radii"]
    clamped = dict(left=vis & (x0 == 0) & (cx - rad <= -16), right=vis & (x1 == gx) & (cx + rad + 15 >= 16 * gx + 16),
                   top=vis & (y0 == 0) & (cy - rad <= -16), bottom=vis & (y1 == gy) & (cy + rad + 15 >= 16 * gy + 16))
    n = {k: int(v.sum()) for k, v in clamped.items()}
    whole = int((m["tiles_touched"] == gx * gy).sum())
    print(f"[clamped] rectangles clamped per side {n}; covering the whole grid {whole}")
    assert min(n.values()) >= 3 and whole >= 1, (n, whole)


# ------------------------------------------------------------------------------------------------ long sorts, batches
def test_long_lookback_single_frame(dev):
    """512 x 512, 75 K surfels of 1 to ~150 tiles: R > 3.1 M, over 1000 sort tiles chained by look-back per pass."""
    W = H = 512
    rng = np.random.default_rng(41)
    n = 75_000
    means, scales = place(rng.uniform(0, W, n), rng.uniform(0, H, n), rng.uniform(1.5, 4.0, n), W, H,
                          rng.uniform(0.3, 30.0, n))
    rep, = check_all("long look-back", forward(dev, W, H, means, scales))
    assert rep["R"] >= 3_100_000 and rep["sort_tiles"] >= 1000, rep


def test_stage3_batch_per_frame_positions(dev):
    """The flagship Stage-3 batch: 8 frames of 300 K surfels at 512 x 512, every surfel moved along its ray per frame."""
    from vidu4d_b200.synthetic import object_scene
    sc = object_scene(300_000, seed=5)
    rng = np.random.default_rng(51)
    means = np.stack([sc.means3D * (1 + 1e-3 * f * rng.normal(size=(sc.means3D.shape[0], 1))).astype(F32)
                      for f in range(8)])
    reps = check_all("stage-3 batch", forward(dev, 512, 512, means, sc.scales, sc.rotations, sc.opacities))
    assert all(rp["R"] > 0 for rp in reps)


def _mixed_batch(rng, W, H, Rs, big_frames=()):
    """Per-frame positions: frame f has Rs[f] visible one-tile surfels (the rest culled), or, in big_frames, 40 K
    surfels visible with footprints of 6 to 24 px (about 2 M instances on 512 x 512)."""
    M = len(Rs)
    P = max([r for f, r in enumerate(Rs) if f not in big_frames] + [40_000 if big_frames else 0])
    tiles = ((W + 15) // 16) * ((H + 15) // 16)
    means, scales = np.empty((M, P, 3), F32), np.empty((M, P, 2), F32)
    for f, R in enumerate(Rs):
        if f in big_frames:
            means[f], scales[f] = place(rng.uniform(0, W, P), rng.uniform(0, H, P), rng.uniform(1.5, 4.0, P), W, H,
                                        rng.uniform(6, 24, P))
            continue
        z = rng.uniform(1.5, 4.0, P)
        z[rng.permutation(P)[R:]] = NEAR
        means[f], scales[f] = one_tile_each(rng.integers(0, tiles, P), z, W, H)
    return means, scales


def test_mixed_batch(dev):
    """M = 8 frames interleaved in one sort grid: R = 0, 1, 3072 and over a million next to each other."""
    rng = np.random.default_rng(61)
    Rs = (3072, 0, None, 1, 383, 0, 6144, 3073)
    means, scales = _mixed_batch(rng, 512, 512, Rs, big_frames=(2,))
    reps = check_all("mixed batch", forward(dev, 512, 512, means, scales))
    got = [rp["R"] for rp in reps]
    assert [g for f, g in enumerate(got) if f != 2] == [r for f, r in enumerate(Rs) if f != 2] and got[2] > 1_000_000, got


# ------------------------------------------------------------------------------------------------ capacity
@pytest.fixture
def capacity(monkeypatch):
    """Pins the instance buffer's capacity (a multiple of 256) for the forwards of one test."""
    from vidu4d_b200 import rasterizer as RZ
    box = {}
    monkeypatch.setattr(RZ, "_pick_capacity", lambda key, P: box["cap"])
    return box


def test_capacity_exactly_full(dev, capacity):
    W = H = 128
    capacity["cap"] = 4096
    rng = np.random.default_rng(71)
    rep, = check_all("R = capacity", forward(dev, W, H, *one_tile_each(rng.integers(0, 64, 4096), rng.uniform(1.5, 4, 4096),
                                                                        W, H)))
    assert rep["R"] == rep["cap"] == 4096 and rep["sort_tiles"] == 2


def test_overflowed_frame_inside_batch(dev, capacity):
    """Nosync mode, capacity 4096: the middle frame of five (R = 4097) is abandoned -- overflow bit set, ranges all
    zero, every pass skipped -- while its neighbours (R = 4096, 1, 4095, 0) match the model exactly; check_overflow
    raises."""
    from vidu4d_b200 import _capi, rasterizer as RZ
    W = H = 128
    capacity["cap"] = 4096
    rng = np.random.default_rng(81)
    means, scales = _mixed_batch(rng, W, H, (4096, 1, 4097, 4095, 0))
    key = (dev.index, W, H)
    had = RZ._cap_hint.get(key)
    try:
        RZ.set_sync_mode(False)
        RZ._cap_hint[key] = 4096                    # a hint makes the forward skip the read-back
        r = forward(dev, W, H, means, scales)
        reps = check_all("overflow batch", r)
        with pytest.raises(_capi.SurfelRasterError, match="overflow"):
            RZ.check_overflow()
    finally:
        RZ.set_sync_mode(True)
        RZ._pending.clear()
        if had is None:
            RZ._cap_hint.pop(key, None)
        else:
            RZ._cap_hint[key] = had
    assert [rp["R"] for rp in reps] == [4096, 1, 4097, 4095, 0] and [rp["overflow"] for rp in reps] == [0, 0, 1, 0, 0]
    assert reps[2]["skip"] == (1,) * reps[2]["npass"]


# ------------------------------------------------------------------------------------------------ stale scratch
@pytest.fixture
def stale_scratch(monkeypatch):
    """Fills the geometry, binning and image buffers of every sr_forward with 0xFF before the call."""
    from vidu4d_b200 import _capi
    call = _capi.call

    def filled(name, device, *args):
        if name == "sr_forward":
            for buf in args[22:25]:                 # geom, binning, image (rasterizer._forward's argument order)
                assert buf.dtype == torch.uint8
                buf.fill_(0xFF)
        return call(name, device, *args)
    monkeypatch.setattr(_capi, "call", filled)


def _stale_scenes():
    rng = np.random.default_rng(91)
    mixed = _mixed_batch(rng, 512, 512, (0, 3072, 1, 40_000), big_frames=(3,))
    W = 80 * 16
    radii = _radius_for_width(rng.choice([1, 31, 32, 33, 60], 256), W)
    return {"mixed": (512, 512) + mixed, "row": (W, 16) + _row_scene(rng.integers(0, 20, 256), radii, W)}


@pytest.mark.parametrize("scene", ["mixed", "row"])
def test_stale_scratch_gives_the_same_bits(scene, dev, request):
    """The same forward on fresh buffers and on buffers full of 0xFF: both match the model, and every output plane is
    bit-identical."""
    W, H, means, scales = _stale_scenes()[scene]
    clean = forward(dev, W, H, means, scales)
    check_all(f"stale {scene} clean", clean)
    request.getfixturevalue("stale_scratch")
    dirty = forward(dev, W, H, means, scales)
    check_all(f"stale {scene} 0xFF", dirty)
    assert torch.equal(clean["color"].view(torch.int32), dirty["color"].view(torch.int32))
    assert torch.equal(clean["allmap"].view(torch.int32), dirty["allmap"].view(torch.int32))
    assert torch.equal(clean["radii"], dirty["radii"]) and clean["nr"] == dirty["nr"]
