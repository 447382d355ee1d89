"""The composite forward's cull rectangle and rho cut never drop a contributing pair, at grazing, near-parabolic,
sub-pixel, threshold-opacity and off-image surfels (tests/cull_model.py's classes), mixed into ordinary clouds.

Each case
  * pins the model to the GPU: every visible surfel's surfel_rec[18:20] equals cull_model's packed box, and every
    instance's cull word (inst_rec[19]) equals the model's word for its (surfel, tile), bit for bit.  Where the GPU's
    double or logf rounding could decide a value, the model names each value the kernel may produce;
  * compares blended pairs per pixel: the GPU's (the population count of its contribution masks) with the CPU oracle's,
    which composites every pair of the tile's list without culling.  They must be equal at every pixel outside the
    oracle's knife mask, so a dropped pair fails here even where T barely moves;
  * holds every forward plane, every element of the composite backward's accumulators (dL/dcolours, dL/dopacity) and
    the cloud surfels' every gradient element to the rounding-error bound of tests/test_gpu_grad_bounds.py.  The
    per-surfel chain (dL/dT through dL/drotations) of the adversarial surfels is not held to it: at a grazing surfel of
    opacity 1e3, dL/drotations lay 255 times outside that bound, whose 32 roundings do not model the conditioning of a
    near-edge-on projection;
  * asserts from the GPU's own buffers that it reaches its edges: grazing surfels blended within a pixel of their
    rectangle's edge, a pair blended at opacity exactly f32(1/255), and surfels centred outside the image contributing.
It prints, per class, the smallest headroom of the GPU's blended pairs: distance in pixels to the padded box's edge, and
cut - rho."""
import numpy as np
import pytest
import torch

from . import cull_model as cm
from . import test_gpu_grad_bounds as gb
from .test_gpu_grad_bounds import (ACC_LEVEL, CHAIN, GRADS, K, U, _bounds, _check_forward, _check_grad, _check_knife,
                                   _fallback_pairs, _np, _oracle_frame, _print)

pytestmark = pytest.mark.gpu

TAN = cm.TAN
NEAR_EDGE = 1.0           # px: a blended pair this close to its rectangle's edge reaches it
MIN_GRAZING_NEAR = 5      # grazing surfels with such a pair, per case

# Knife pixels measured per case on an H100, under tests/test_gpu_grad_bounds.py's cap (at most 4 x + 8).  A pair at
# opacity f32(1/255) centred on its pixel has alpha exactly at the threshold: each such pixel is a knife edge.
KNIFE_MEASURED = {"cull_mix_72x52": 13, "cull_mix_200x116": 18, "cull_mix_37x23": 7, "cull_batch4": 35,
                  "cull off-centre": 6}
gb.KNIFE_MEASURED.update(KNIFE_MEASURED)


@pytest.fixture(scope="module")
def dev(built):
    from vidu4d_b200 import _capi, rasterizer as RZ
    _capi.load()
    RZ.set_sync_mode(True)          # every case reads num_rendered back and decodes the buffers it sized
    return torch.device("cuda:0")


# ------------------------------------------------------------------------------------------------ scenes
def _cloud(rng, n, W, H, ppx, ppy):
    """An ordinary cloud: random orientations, footprints of 1 .. 12 px, depths 1.5 .. 4, opacities 0.05 .. 1."""
    z = rng.uniform(1.5, 4.0, n)
    u, v = rng.uniform(0, W, n), rng.uniform(0, H, n)
    means = np.stack([(u - ppx) * z * 2 * TAN / W, (v - ppy) * z * 2 * TAN / H, z], 1)
    q = rng.normal(size=(n, 4))
    s = rng.uniform(1, 12, (n, 2)) * z[:, None] * 2 * TAN / W
    return dict(means=means.astype(np.float32), scales=s.astype(np.float32),
                rotations=(q / np.linalg.norm(q, axis=1, keepdims=True)).astype(np.float32),
                opacities=rng.uniform(0.05, 1.0, n).astype(np.float32))


def _mix(seed, W, H, n_cloud, n_class, ox=0.0, oy=0.0):
    """Cloud + n_class surfels of every class, shuffled; returns the parts and each surfel's class index (-1: cloud)."""
    rng = np.random.default_rng(seed)
    ppx, ppy = W / 2 + ox, H / 2 + oy
    parts = [_cloud(rng, n_cloud, W, H, ppx, ppy)] + [cm.adversarial(rng, c, n_class, W, H, ppx, ppy) for c in cm.CLASSES]
    label = np.concatenate([np.full(len(p["opacities"]), k - 1) for k, p in enumerate(parts)])
    perm = rng.permutation(label.size)
    cat = {k: np.concatenate([p[k] for p in parts])[perm] for k in parts[0]}
    return cat, label[perm]


def scene_single(seed, W, H, n_cloud, n_class):
    """One frame for the identity camera in build_case's format (colours precomputed), and the class labels."""
    from vidu4d_b200.synthetic import projection_matrix
    s, label = _mix(seed, W, H, n_cloud, n_class)
    P = label.size
    rng = np.random.default_rng(seed + 1)
    inp = dict(means3D=s["means"], scales=s["scales"], rotations=s["rotations"], opacities=s["opacities"].reshape(P, 1),
               shs=np.zeros((0,), np.float32), colors_precomp=rng.uniform(0, 1, (P, 3)).astype(np.float32),
               viewmatrix=np.eye(4, dtype=np.float32), projmatrix=projection_matrix(TAN, TAN).astype(np.float32),
               campos=np.zeros(3, np.float32), bg=np.array([0.1, 0.2, 0.3], np.float32),
               dL_dcolor=rng.normal(size=(3, H, W)).astype(np.float32),
               dL_dallmap=rng.normal(size=(8, H, W)).astype(np.float32),
               meta=np.array([P, W, H, 0, 1], np.int64), tanfov=np.array([TAN, TAN], np.float32))
    return inp, label


def _batch_scene(seed, W, H, n_cloud, n_class, ox=0.0, oy=0.0):
    """A synthetic.Scene (SH degree 3, random DC colour) of _mix's surfels, and the labels."""
    from vidu4d_b200.synthetic import Scene
    s, label = _mix(seed, W, H, n_cloud, n_class, ox, oy)
    P = label.size
    rng = np.random.default_rng(seed + 1)
    shs = np.zeros((P, 16, 3), np.float32)
    shs[:, 0] = rng.uniform(-1.5, 1.5, (P, 3))
    return Scene(means3D=s["means"], scales=s["scales"], rotations=s["rotations"],
                 opacities=s["opacities"].reshape(P, 1), shs=shs), label


def _identity_cams(M, dev):
    from vidu4d_b200.synthetic import projection_matrix
    vm = torch.eye(4, device=dev)
    pm = torch.from_numpy(projection_matrix(TAN, TAN).astype(np.float32)).to(dev)
    return vm.repeat(M, 1, 1).contiguous(), pm.repeat(M, 1, 1).contiguous(), torch.zeros((M, 3), device=dev)


# ------------------------------------------------------------------------------------------------ checks
def _u32(x):
    return np.ascontiguousarray(_np(x)).view(np.uint32)


def _blended_pairs(dec, W, H):
    """(px, py, instance) of every pair the GPU blended, from its contribution masks (debug._lane_counts' rows)."""
    rg = _np(dec["ranges"]).astype(np.int64)
    sl = _np(dec["sub_last"]).astype(np.int64)
    masks = _u32(dec["contrib_masks"])
    tiles_x = (W + 15) // 16
    nb = (np.minimum(sl, (rg[:, 1] - rg[:, 0])[:, None]) + 31) >> 5
    t, w = np.nonzero(nb)
    reps = nb[t, w]
    t, w = np.repeat(t, reps), np.repeat(w, reps)
    s = np.arange(t.size) - np.repeat(np.cumsum(reps) - reps, reps)
    words = masks[(rg[t, 0] >> 5) + t + s, w]                               # (k, 32 lanes)
    bits = (words[:, :, None] >> np.arange(32, dtype=np.uint32)) & 1        # (k, lane, bit)
    k, lane, j = np.nonzero(bits)
    px = (t[k] % tiles_x) * 16 + (w[k] & 1) * 8 + (lane & 7)
    py = (t[k] // tiles_x) * 16 + (w[k] >> 1) * 4 + (lane >> 3)
    return px, py, rg[t[k], 0] + 32 * s[k] + j


def _check_lists(name, dec, P, W, H):
    """The sorted list and tile ranges the CPU oracle will walk: every range inside the list, every id a surfel with a
    record (radius > 0).  A bad buffer then fails here instead of sending the oracle out of bounds."""
    R = int(dec["num_rendered"])
    pl = _u32(dec["point_list"]).astype(np.int64)
    rg = _u32(dec["ranges"]).astype(np.int64).reshape(-1, 2)
    radii = np.asarray(dec["radii"]).reshape(P)
    assert pl.size == R and rg.shape[0] == ((W + 15) // 16) * ((H + 15) // 16), (name, pl.size, R, rg.shape)
    assert ((rg[:, 0] <= rg[:, 1]) & (rg[:, 1] <= R)).all(), (name, "ranges", rg[(rg[:, 0] > rg[:, 1]) | (rg[:, 1] > R)][:4])
    assert ((pl >= 0) & (pl < P)).all(), (name, "point_list ids outside [0, P)", pl[(pl < 0) | (pl >= P)][:4])
    assert (radii[pl] > 0).all(), (name, "point_list names surfels without a record", np.unique(pl[radii[pl] <= 0])[:4])


def _check_cull(name, dec, ext, P, W, H, label, edges=True):
    """Pins, per-pixel counts, headroom and (edges) the edges reached, of one frame; returns the per-class headroom."""
    from vidu4d_b200 import debug as dbg
    rec = _np(dec["surfel_rec"]).reshape(P, 20)
    radii = np.asarray(dec["radii"]).reshape(P)
    vis = radii > 0
    gbx, gby = rec[:, 18].view(np.uint32), rec[:, 19].view(np.uint32)
    BX, BY, box, amb = cm.cull_candidates(rec[:, :9], rec[:, 9], rec[:, 10], rec[:, 11], W, H)
    ok = cm.match_bbox(gbx, gby, BX, BY)
    bad = np.nonzero(vis & ~ok)[0]
    assert bad.size == 0, (name, "surfel_rec[18:20] differs from cull_bbox", bad[:4].tolist(),
                           [(hex(gbx[i]), hex(gby[i]), [hex(v) for v in BX[i]], [hex(v) for v in BY[i]]) for i in bad[:2]])
    # every instance's cull word: the GPU's own (pinned) box narrowed to its tile, and the model's rho bits
    R = int(dec["num_rendered"])
    inst = _np(dec["inst_rec"]).reshape(R, 20)
    sid = inst[:, 18].view(np.uint32).astype(np.int64)
    word = inst[:, 19].view(np.uint32)
    tile = (_np(dec["keys"]).view(np.uint64) >> np.uint64(32)).astype(np.int64)
    assert (_u32(dec["point_list"]).astype(np.int64) == sid).all(), name
    lo, hi = cm.rho_cut_words(rec[:, 11])
    tiles_x = (W + 15) // 16
    w_lo = cm.cull_word(gbx[sid], gby[sid], tile, tiles_x, lo[sid])
    w_hi = cm.cull_word(gbx[sid], gby[sid], tile, tiles_x, hi[sid])
    bad = np.nonzero((word != w_lo) & (word != w_hi))[0]
    assert bad.size == 0, (name, "inst_rec[19] differs from the model's cull word", bad[:4].tolist(),
                           [(hex(word[i]), hex(w_lo[i]), float(rec[sid[i], 11])) for i in bad[:4]])
    n_amb = int((amb & vis).sum() + ((lo != hi) & vis).sum())
    # blended pairs per pixel against the uncut oracle
    mine, outside = dbg.contributing_pairs_per_pixel(dec, W, H)
    mine = _np(mine)
    assert outside == 0, (name, "pairs recorded for pixels outside the image", outside)
    keep = ~ext["knife"]
    diff = np.argwhere((mine != ext["nblend"].astype(np.int64)) & keep)
    assert diff.size == 0, (name, "blended pairs per pixel differ from the uncut oracle at", diff[:6].tolist(),
                            [(int(mine[y, x]), int(ext["nblend"][y, x])) for y, x in diff[:6]])
    # the GPU's blended pairs under the model: inside the box, rho within the cut; headroom and edges
    px, py, ins = _blended_pairs(dec, W, H)
    assert px.size == int(mine.sum()), name
    s = sid[ins]
    ev = cm.pair_eval(rec[s, :12], px[:, None], py[:, None])
    rho = ev["rho"][:, 0]
    c, d, b = px + 0.5, py + 0.5, box[:, s]
    marg = np.minimum(np.minimum(c - b[0], b[1] - c), np.minimum(d - b[2], b[3] - d))
    cut = cm.rho_cut_value(lo[s]) - rho
    assert (marg >= 0).all() and (cut >= 0).all(), (name, float(marg.min()), float(cut.min()))
    cls = label[s]
    head = {}
    for k, nm in enumerate(cm.CLASSES):
        m = cls == k
        head[nm] = (int(m.sum()), float(marg[m].min()) if m.any() else np.inf, float(cut[m].min()) if m.any() else np.inf)
    grazing_near = np.unique(s[(cls == cm.CLASSES.index("grazing")) & (marg < NEAR_EDGE)]).size
    at_threshold = int((rec[s, 11] == cm.INV255).sum())
    cx, cy = rec[s, 9], rec[s, 10]
    off = np.unique(s[(cx < 0) | (cx > W) | (cy < 0) | (cy > H)]).size
    print(f"\n[{name}] knife {int(ext['knife'].sum())}; ambiguous model values {n_amb}; grazing surfels near their edge "
          f"{grazing_near}; pairs at f32(1/255) {at_threshold}; off-image surfels contributing {off}; headroom "
          + ", ".join(f"{k}: {n} pairs, {r:.3g} px, cut {u:.3g}" for k, (n, r, u) in head.items()))
    if edges:
        assert grazing_near >= MIN_GRAZING_NEAR and at_threshold >= 1 and off >= 1, (name, grazing_near, at_threshold, off)
    return head


# ------------------------------------------------------------------------------------------------ the device's expf
def test_device_expf_never_exceeds_one_below_zero(dev):
    """cull_bbox drops surfels with opacity < 1/255 on alpha = opacity expf(power) <= opacity, i.e. expf(x) <= 1 for
    x <= 0, and cull_model's "may blend" relies on it too.  Checked on the device's expf (torch.exp, the libdevice
    expf without fast math) at 2^22 arguments from -1e-45 to -1e-3, and at the 2^16 floats nearest below zero."""
    x = -torch.logspace(-45, -3, 1 << 22, dtype=torch.float64, device=dev).float()
    tiny = -torch.arange(1, 1 << 16, dtype=torch.int32, device=dev).view(torch.float32).abs()
    for v in (x, tiny, torch.zeros(1, device=dev)):
        assert float(torch.exp(v).max()) <= 1.0


# ------------------------------------------------------------------------------------------------ single frames
SINGLE = {
    "cull_mix_72x52": (dict(seed=301, W=72, H=52, n_cloud=1500, n_class=120)),
    "cull_mix_200x116": (dict(seed=302, W=200, H=116, n_cloud=6000, n_class=300)),
    "cull_mix_37x23": (dict(seed=303, W=37, H=23, n_cloud=400, n_class=80)),
}


def _check_grads(name, st, og, tol, mine, label, report):
    """test_gpu_grad_bounds._check_all's element-wise checks: the accumulator-level tensors for every surfel, the
    per-surfel chain's outputs for the cloud's surfels."""
    cloud = label < 0
    for k in GRADS:
        if og[k].size == 0:
            assert mine[k].numel() == 0, (name, k)
        elif k in ACC_LEVEL:
            _check_grad(name, k, mine[k], og[k], tol[k], report)
        else:
            sel = torch.from_numpy(cloud).to(mine[k].device)
            _check_grad(name, k, mine[k].reshape(og[k].shape)[sel], og[k][cloud], np.asarray(tol[k]).reshape(og[k].shape)[cloud],
                        report)


@pytest.mark.parametrize("name", list(SINGLE))
def test_single_frame(name, dev):
    """One frame: GPU forward, oracle composite from its records, the cull checks, masked upstream gradients, both
    backwards (test_gpu_grad_bounds._run_single with _check_grads)."""
    from oracle import surfel_oracle as so
    from vidu4d_b200 import rasterizer as R
    from .test_gpu_parity import _run_ours
    kw = SINGLE[name]
    inp, label = scene_single(**kw)
    P, W, H = label.size, kw["W"], kw["H"]
    r = _run_ours(inp, dev, with_grads=False)
    r["radii"] = _np(r["radii"])
    _check_lists(name, r, P, W, H)
    st, ext = _oracle_frame(r, P, W, H, inp["means3D"], inp["opacities"], inp["scales"], inp["rotations"], None,
                            inp["colors_precomp"], 0, inp["bg"], inp["viewmatrix"], inp["projmatrix"], inp["campos"])
    fwd = _check_forward(name, st, ext, _np(r["color"]), _np(r["allmap"]), r, W, H)
    _check_knife(name, int(ext["knife"].sum()))
    _check_cull(name, r, ext, P, W, H, label)
    keep = (~ext["knife"]).astype(np.float32)
    dLc, dLo = inp["dL_dcolor"] * keep, inp["dL_dallmap"] * keep
    t = {k: torch.from_numpy(np.ascontiguousarray(v)).to(dev) for k, v in inp.items() if k != "meta"}
    e = torch.empty((0,), device=dev)
    gb_, bb, ib = r["bufs"]
    g = R._C.rasterize_gaussians_backward(t["bg"], t["means3D"], torch.from_numpy(r["radii"]).to(dev), t["colors_precomp"],
                                          t["scales"], t["rotations"], 1.0, e, t["viewmatrix"], t["projmatrix"], TAN, TAN,
                                          torch.from_numpy(dLc).to(dev), torch.from_numpy(dLo).to(dev), e, 0, t["campos"],
                                          gb_, r["num_rendered"], bb, ib, False)
    og = so.backward(st, dLc, dLo, bounds=True)
    report = {}
    _check_grads(name, st, og, _bounds(st, og, r), dict(zip(GRADS, g)), label, report)
    _print(name, int(ext["knife"].sum()), fwd, report)


# ------------------------------------------------------------------------------------------------ batches
def _oracle_from_dec(so, dec, sc, means, W, H, tx, ty):
    P = sc.opacities.shape[0]
    rec = _np(dec["surfel_rec"]).reshape(P, 20)
    cl = _np(dec["clamped"]).astype(np.uint8).reshape(P)
    return so.from_records(_np(means), sc.opacities, sc.scales, sc.rotations, shs=sc.shs, sh_degree=3, W=W, H=H,
                           tanfovx=tx, tanfovy=ty, bg=np.array([0.2, 0.1, 0.4], np.float32),
                           viewmatrix=np.eye(4, dtype=np.float32), projmatrix=np.eye(4, dtype=np.float32),
                           campos=np.zeros(3, np.float32), transMat=rec[:, 0:9], means2D=rec[:, 9:11],
                           normal_opacity=rec[:, [12, 13, 14, 11]], rgb=rec[:, 15:18], radii=dec["radii"],
                           clamped=(cl[:, None] >> np.arange(3)) & 1, point_list=_u32(dec["point_list"]),
                           ranges=_u32(dec["ranges"]))


def _run_batch(name, dev, sc, label, means, W, H, rows, edge_frames):
    """M frames through the batched entry points, per-frame intrinsics rows (tan_fovx, tan_fovy, cx_off, cy_off) from a
    device table; per frame the forward planes, the cull checks (edges asserted in edge_frames), and the gradients
    (_check_grads) with the offsets' terms in the chain (tests/camera_model.py), as test_gpu_cameras' off-centre test."""
    from oracle import surfel_oracle as so
    from vidu4d_b200 import debug as dbg, rasterizer as RZ
    from . import camera_model as cmo
    M, P = means.shape[0], label.size
    t = sc.to_torch(dev)
    vms, pms, cps = _identity_cams(M, dev)
    table = torch.tensor(rows, device=dev)
    g = torch.Generator(device=dev).manual_seed(M * 1000 + W)
    dLc = torch.randn((M, 3, H, W), device=dev, generator=g)
    dLo = 0.1 * torch.randn((M, 8, H, W), device=dev, generator=g)
    bg = torch.tensor([0.2, 0.1, 0.4], device=dev)
    e = torch.empty((0,), device=dev)
    nan = float("nan")
    nr, color, allmap, radii, gbuf, bb, ib = RZ._C.rasterize_gaussians_batch(
        bg, means, e, t["opacities"], t["scales"], t["rotations"], 1.0, vms, pms, nan, nan, H, W, t["shs"], 3, cps,
        intrinsics=table)[:7]
    frames = []
    for f, (tx, ty, ox, oy) in enumerate(rows):
        dec = dbg.decode(gbuf.view(M, -1)[f], bb.view(M, -1)[f], ib.view(M, -1)[f], P, W, H, nr[f])
        dec["radii"] = _np(radii[f])
        dec["num_rendered"] = nr[f]
        _check_lists(f"{name} frame {f}", dec, P, W, H)
        st, ext = _oracle_from_dec(so, dec, sc, means[f], W, H, tx, ty)
        fwd = _check_forward(f"{name} frame {f}", st, ext, _np(color[f]), _np(allmap[f]), dec, W, H)
        _check_cull(f"{name} frame {f}", dec, ext, P, W, H, label, edges=f in edge_frames)
        keep = torch.from_numpy((~ext["knife"]).astype(np.float32)).to(dev)
        dLc[f] *= keep
        dLo[f] *= keep
        og = so.backward(st, _np(dLc[f]), _np(dLo[f]), bounds=True)
        adds = _np(dec["tiles_touched"]).astype(np.float64) + _fallback_pairs(dec, P)
        B = og["bound"] + (adds[:, None] + CHAIN) * og["asum"]
        B = cmo.offset_bound_sums(st, B, og["acc"], og["dL_dtransMat"], ox, oy)
        tol = {k: K * U * v for k, v in so.chain_bound(st, B).items()}
        og = dict(og, **cmo.offset_chain(st, og["acc"], og["dL_dtransMat"], ox, oy))
        frames.append((st, ext, og, tol, fwd))
    _check_knife(name, sum(int(fr[1]["knife"].sum()) for fr in frames))
    gr = dict(zip(GRADS, RZ._C.rasterize_gaussians_backward_batch(
        bg, means, radii, e, t["scales"], t["rotations"], 1.0, vms, pms, nan, nan, dLc, dLo, t["shs"], 3, cps, gbuf, bb, ib,
        intrinsics=table)))
    report = {}
    for f, (st, _, og, tol, _) in enumerate(frames):
        _check_grads(f"{name} frame {f}", st, og, tol, {k: gr[k][f] for k in GRADS}, label, report)
    _print(name, sum(int(fr[1]["knife"].sum()) for fr in frames), max(fr[4] for fr in frames), report)


def test_batch_per_frame_positions(dev):
    """Four frames of the centred identity camera, each surfel moved a little along its view ray per frame (its grazing
    angle and Dc move with it)."""
    M, W, H = 4, 104, 72
    sc, label = _batch_scene(311, W, H, 3000, 200)
    g = torch.Generator(device=dev).manual_seed(312)
    base = torch.from_numpy(sc.means3D).to(dev)
    means = torch.stack([base * (1 + 1e-3 * f * torch.randn((base.shape[0], 1), device=dev, generator=g))
                         for f in range(M)]).contiguous()
    _run_batch("cull_batch4", dev, sc, label, means, W, H, [(TAN, TAN, 0.0, 0.0)] * M, edge_frames=range(M))


def test_batch_off_centre_principal_points(dev):
    """Three frames with principal points up to 0.9 W off the image centre, read from the intrinsics table: T carries
    the offset.  The adversarial surfels are placed for frame 0's offsets, so the edges are asserted there; frames 1 and
    2 see them through the other principal points."""
    M, W, H = 3, 88, 61
    rows = [(TAN, TAN, 40.25, -27.5), (TAN, TAN, -79.0, 13.125), (TAN, TAN, 0.5, 54.75)]
    sc, label = _batch_scene(321, W, H, 2500, 400, ox=rows[0][2], oy=rows[0][3])
    means = torch.from_numpy(sc.means3D).to(dev)[None].repeat(M, 1, 1).contiguous()
    _run_batch("cull off-centre", dev, sc, label, means, W, H, rows, edge_frames=(0,))
