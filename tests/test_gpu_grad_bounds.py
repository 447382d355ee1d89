"""Every rasterizer gradient element against the CPU oracle, under an a-priori rounding-error bound.

The oracle (oracle/surfel_oracle.c) composites from the GPU's own per-surfel records, sorted list and tile ranges, so the
only inputs of a pair's arithmetic that differ between the two sides are exp() and what depends on it.  It returns

  * a knife mask: pixels where some pair's expf-dependent decision (alpha < 1/255, T (1 - alpha) < 1e-4, T > 0.5) lies
    within the error margin of its threshold.  Those pixels may legitimately walk differently on the two sides.  Their
    upstream gradients are set to zero on both sides; every pixel's share of every gradient is linear in its own
    upstream gradient, so they then contribute exactly nothing to either;
  * per pixel and plane, and per surfel and accumulator, bound sums  B = sum over terms of w |t|  in units of
    u = 2^-24, with |t| the term evaluated on absolute values (no cancellation) and w the term's roundings plus the
    error its transmittance and recursions carry into it, plus, for the accumulators, the roundings of a sequential
    per-tile sum over the tile's 256 pixels (see so_acc in the oracle).

Outside the knife mask every discrete decision must agree, so n_contrib must be identical there.  Each float output must
satisfy  |gpu - oracle| <= K u B' + FLOOR,  where for the gradients B' is B pushed through the per-surfel chain
(oracle.chain_bound: the chain evaluated on absolute values, which dominates |d out / d acc| and is what the chain's own
roundings are relative to) after adding
  * the reductions into the accumulator: the kernel adds a surfel's per-tile totals, and one by one each of its pairs
    that fall past the 4,608-slot pair buffer of a chunk, with fp32 atomics in no fixed order.  m such adds cost at most
    m u sum |t|, with m = tiles touched + the surfel's pairs past the buffer (_fallback_pairs reproduces the kernel's
    slot assignment from the GPU's contribution masks);
  * the chain's own roundings: about 30 on its longest path (AABB vjp, K^T, W^T, the rotation, the quaternion vjp, an
    SH polynomial and the direction normalisation), CHAIN u sum |t| with CHAIN = 32 since sum |t| >= |acc|.
Summed frames (sum_shared) add M u sum_f |oracle_f| for the kernel's sequential frame sum.

K = 2: the weights bound the rounding error of ONE fp32 evaluation (the expf and reciprocal differences between the two
sides are already in the weights, see the oracle's error analysis), and the two sides are two evaluations whose errors
may have opposite signs.  The oracle's double sums only make its own share smaller.  FLOOR is the smallest normal
float: where a bound is 0 every term is exactly 0 on both sides.

Each case asserts from the GPU's own buffers that it reaches its edge and that the knife mask stays within a few times
its measured size, and prints the knife pixels and, per tensor, the largest err / (K u B') -- the headroom.  The
accumulator-level tensors are checked first and dL/dSH also from the GPU's own dL/dcolors, so that a failure says
whether the composite backward or the per-surfel backward went wrong.
"""
import numpy as np
import pytest
import torch

from .conftest import GOLDEN_CASES, load_golden

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
K = 2.0
FLOOR = float(np.finfo(np.float32).tiny)
CHAIN = 32
TAN = 0.5
CH = 256                 # instances per chunk of the composite backward
BWD_CAP = 4608           # pair-buffer slots of the composite backward (composite_tile.cu BWD_CAP)
GRADS = ("dL_dmeans2D", "dL_dcolors", "dL_dopacity", "dL_dmeans3D", "dL_dtransMat", "dL_dsh", "dL_dscales", "dL_drotations")
FWD_PLANES = [("color", i) for i in range(3)] + [("allmap", i) for i in range(8)] + [("final_T", i) for i in range(3)]


@pytest.fixture(scope="module")
def dev(built):
    from vidu4d_b200 import _capi
    _capi.load()
    return torch.device("cuda:0")


def _np(x):
    return x.detach().cpu().numpy()


# ------------------------------------------------------------------------------------------------ oracle side
def _oracle_frame(dec, P, W, H, means3D, opacities, scales, rotations, shs, colors, deg, bg, vm, pm, cp, tan=(TAN, TAN)):
    """The oracle's state composited from one frame's decoded GPU buffers, and its knife mask / bounds."""
    from oracle import surfel_oracle as so
    rec = _np(dec["surfel_rec"]).reshape(P, 20)
    cl = _np(dec["clamped"]).astype(np.uint8).reshape(P)
    radii = dec["radii"]
    return so.from_records(means3D, opacities, scales, rotations, shs=shs, colors_precomp=colors, sh_degree=deg, W=W, H=H,
                           tanfovx=tan[0], tanfovy=tan[1], bg=bg, viewmatrix=vm, projmatrix=pm, campos=cp,
                           transMat=rec[:, 0:9], means2D=rec[:, 9:11], normal_opacity=rec[:, [12, 13, 14, 11]],
                           rgb=rec[:, 15:18], radii=radii, clamped=(cl[:, None] >> np.arange(3)) & 1,
                           point_list=_np(dec["point_list"]).view(np.uint32), ranges=_np(dec["ranges"]).view(np.uint32))


def _check_forward(name, st, ext, color, allmap, dec, W, H):
    """n_contrib identical outside the knife mask (the median plane only in non-empty tiles, 0 in empty ones); every
    float plane within its per-pixel bound there."""
    ok = ~ext["knife"]
    nc = _np(dec["n_contrib"]).view(np.uint32)
    rg = _np(dec["ranges"]).astype(np.int64)
    ys, xs = np.mgrid[0:H, 0:W]
    nonempty = (rg[:, 1] - rg[:, 0])[(ys // 16) * ((W + 15) // 16) + xs // 16] > 0
    bad0 = (nc[0] != st.n_contrib[0]) & ok
    bad1 = (nc[1] != st.n_contrib[1]) & ok & nonempty
    assert not bad0.any() and not bad1.any(), (name, "n_contrib disagrees at pixels no knife edge explains",
                                               np.argwhere(bad0 | bad1)[:8].tolist())
    assert (nc[1][~nonempty] == 0).all(), name
    mine = {"color": color, "allmap": allmap, "final_T": _np(dec["final_T"])}
    ref = {"color": st.color, "allmap": st.allmap, "final_T": st.final_T}
    worst = 0.0
    for k, (plane, i) in enumerate(FWD_PLANES):
        err = np.abs(mine[plane][i].astype(np.float64) - ref[plane][i])
        tol = K * U * ext["fbound"][k] + FLOOR
        r = np.where(ok, err / tol, 0.0)
        assert r.max() <= 1.0, (name, f"{plane}[{i}]", float(r.max()), np.argwhere(r > 1)[:4].tolist())
        worst = max(worst, float(r.max()))
    return worst


def _fallback_pairs(dec, P):
    """Per surfel, how many of its pairs the composite backward reduces into its accumulator one by one, past the pair
    buffer.  Reproduces the kernel's slot assignment from the GPU's contribution masks: per (tile, 256-instance chunk),
    the CTA's 256 pixels (8 x 4 sub-tile w, lane) take consecutive slots in thread order w * 32 + lane, a pixel's own
    pairs back to front (highest instance first); slots from BWD_CAP on go out directly.  So a pixel whose slots end
    f past the buffer sends its f lowest contributing instances of the chunk."""
    rg = _np(dec["ranges"]).astype(np.int64)
    sl = _np(dec["sub_last"]).astype(np.int64)
    masks = _np(dec["contrib_masks"]).view(np.uint32)                      # (rows, 8, 32)
    pl = _np(dec["point_list"]).view(np.uint32)
    rlen = rg[:, 1] - rg[:, 0]
    nb = (np.minimum(sl, rlen[:, None]) + 31) >> 5                        # live stages per sub-tile
    nch = (np.minimum(rlen, sl.max(1)) + CH - 1) // CH                     # chunks the CTA streams
    t = np.repeat(np.arange(rg.shape[0]), nch)
    c = np.arange(t.size) - np.repeat(np.cumsum(nch) - nch, nch)
    counts = np.zeros(P, np.int64)
    if t.size == 0:
        return counts
    g = c[:, None] * (CH // 32) + np.arange(CH // 32)                        # (tc, 8 stages) global stage index
    rows = np.minimum((rg[t, 0] >> 5)[:, None] + t[:, None] + g, masks.shape[0] - 1)
    words = masks[rows]                                                     # (tc, stage, w, lane)
    words = np.where((g[:, :, None] < nb[t][:, None, :])[..., None], words, 0).transpose(0, 2, 3, 1)  # (tc, w, lane, st)
    npix = np.bitwise_count(words).sum(-1).reshape(t.size, 256).astype(np.int64)
    end = np.cumsum(npix, 1)                                                # slot after each pixel's last pair
    f = np.clip(end - BWD_CAP, 0, npix)
    tc_i, p_i = np.nonzero(f)
    if tc_i.size == 0:
        return counts
    w8 = words.reshape(t.size, 256, CH // 32)[tc_i, p_i]                     # (K, 8) stage words of those pixels
    bits = ((w8[:, :, None] >> np.arange(32, dtype=np.uint32)) & 1).reshape(-1, CH).astype(np.int64)   # position st*32+j
    take = (bits == 1) & (np.cumsum(bits, 1) <= f[tc_i, p_i][:, None])
    k, pos = np.nonzero(take)
    inst = rg[t[tc_i[k]], 0] + c[tc_i[k]] * CH + pos
    counts += np.bincount(pl[inst].astype(np.int64), minlength=P)
    assert counts.sum() == f.sum()
    return counts


def _bounds(st, og, dec):
    """K u B' per output element: the oracle's bound sums plus the reductions into the accumulator in arbitrary order
    (one per tile touched and one per pair past the pair buffer) and the chain's roundings, pushed through the chain on
    absolute values."""
    from oracle import surfel_oracle as so
    adds = _np(dec["tiles_touched"]).astype(np.float64) + _fallback_pairs(dec, st.P)
    B = og["bound"] + (adds[:, None] + CHAIN) * og["asum"]
    return {k: K * U * v for k, v in so.chain_bound(st, B).items()}


def _check_grad(name, k, mine, ref, tol, report):
    """Asserts |mine - ref| <= tol + FLOOR element by element; records the largest ratio under report[k]."""
    ref = np.asarray(ref, np.float64)
    if ref.size == 0:
        assert mine.numel() == 0, (name, k)
        return
    m_ = _np(mine).astype(np.float64).reshape(ref.shape)
    t_ = np.asarray(tol, np.float64).reshape(ref.shape) + FLOOR
    ratio = np.abs(m_ - ref) / t_
    i = int(np.argmax(ratio))
    report[k] = max(report.get(k, 0.0), float(ratio.flat[i]))
    assert ratio.flat[i] <= 1.0, (name, k, "element", np.unravel_index(i, ref.shape), "gpu", m_.flat[i], "oracle",
                                  ref.flat[i], "tolerance", t_.flat[i])


ACC_LEVEL = ("dL_dcolors", "dL_dopacity")      # the composite backward's accumulators themselves, before the chain


def _check_all(name, st, og, tol, mine, report):
    """Every gradient tensor of one frame, ordered so that a failure says where it arose: the accumulator-level tensors
    (the composite backward alone), then dL/dSH from the oracle's chain fed the GPU's own dL/dcolors (the per-surfel
    backward alone: dL/dSH depends on nothing else), then the rest end to end."""
    from oracle import surfel_oracle as so
    for k in ACC_LEVEL:
        _check_grad(name + " [composite backward]", k, mine[k], og[k], tol[k], report)
    if og["dL_dsh"].size:
        acc = np.zeros((st.P, so.NACC), np.float32)
        acc[:, so.ACC_COLOR:so.ACC_COLOR + 3] = _np(mine["dL_dcolors"]).reshape(st.P, 3)
        own = so.chain(st, acc)["dL_dsh"]
        ctol = K * U * CHAIN * so.chain_bound(st, np.abs(acc.astype(np.float64)))["dL_dsh"]
        _check_grad(name + " [per-surfel backward, GPU accumulators]", "dL_dsh", mine["dL_dsh"], own, ctol, {})
    for k in GRADS:
        if k not in ACC_LEVEL:
            _check_grad(name, k, mine[k], og[k], tol[k], report)


# Masked (knife-edge) pixels measured per case on an H100; a case may mask at most 4 times as many plus 8.  The mask takes
# pixels out of every comparison, so a margin that grew by mistake could otherwise hide most of an image.
KNIFE_MEASURED = {"golden precomp_init_70x50": 1, "oracle_seed21_256": 2, "oracle_seed22_200x120": 1, "c2_100k_512": 11,
                  "headline_300k_512": 18, "long_lists_50k_32": 1, "dense": 9, "long_overflow": 56, "sh M=1 deg=0": 1,
                  "batch8": 9, "batch5": 2}


def _check_knife(name, n):
    assert n <= 4 * KNIFE_MEASURED.get(name, 0) + 8, (name, "knife pixels", n)


def _print(name, knife, fwd, report):
    print(f"\n[{name}] knife pixels {knife}; forward err/bound {fwd:.3g}; "
          + ", ".join(f"{k} {v:.3g}" for k, v in report.items()))


# ------------------------------------------------------------------------------------------------ single frames
def _run_single(name, inp, dev):
    """GPU forward, oracle composite from its records, masked upstream gradients, both backwards, every check."""
    from oracle import surfel_oracle as so
    from vidu4d_b200 import rasterizer as R
    from .test_gpu_parity import _run_ours
    P, W, H, deg, pre = [int(v) for v in inp["meta"]]
    tan = (float(inp["tanfov"][0]), float(inp["tanfov"][1]))              # as _run_ours passes them to the forward
    r = _run_ours(inp, dev, with_grads=False)
    r["radii"] = _np(r["radii"])
    shs = None if pre else inp["shs"]
    col = inp["colors_precomp"] if pre else None
    st, ext = _oracle_frame(r, P, W, H, inp["means3D"], inp["opacities"], inp["scales"], inp["rotations"], shs, col, deg,
                            inp["bg"], inp["viewmatrix"], inp["projmatrix"], inp["campos"], tan)
    fwd = _check_forward(name, st, ext, _np(r["color"]), _np(r["allmap"]), r, W, H)
    _check_knife(name, int(ext["knife"].sum()))
    keep = (~ext["knife"]).astype(np.float32)
    dLc = inp["dL_dcolor"] * keep
    dLo = inp["dL_dallmap"] * keep
    t = {k: torch.from_numpy(np.ascontiguousarray(v)).to(dev) for k, v in inp.items() if k != "meta"}
    e = torch.empty((0,), device=dev)
    gb, bb, ib = r["bufs"]
    g = R._C.rasterize_gaussians_backward(t["bg"], t["means3D"], torch.from_numpy(r["radii"]).to(dev),
                                          t["colors_precomp"] if pre else e, t["scales"], t["rotations"], 1.0, e,
                                          t["viewmatrix"], t["projmatrix"], tan[0], tan[1],
                                          torch.from_numpy(dLc).to(dev), torch.from_numpy(dLo).to(dev),
                                          e if pre else t["shs"], deg, t["campos"], gb, r["num_rendered"], bb, ib, False)
    mine = dict(zip(GRADS, g))
    og = so.backward(st, dLc, dLo, bounds=True)
    report = {}
    _check_all(name, st, og, _bounds(st, og, r), mine, report)
    _print(name, int(ext["knife"].sum()), fwd, report)
    return r, ext, report


def _chunk_pairs(dec):
    """{(tile, chunk): contributing pairs} from the GPU's live contribution masks."""
    from .test_gpu_variants import _frame, _chunk_pairs as cp
    fr = _frame(dec, dec["num_rendered"], None, None, None)
    return cp({"exact": fr})


def _lengths(dec):
    rg = _np(dec["ranges"]).astype(np.int64)
    return rg[:, 1] - rg[:, 0]


@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_golden(name, dev):
    g = load_golden(name)
    r, _, _ = _run_single(f"golden {name}", {k[3:]: v for k, v in g.items() if k.startswith("in_")}, dev)
    assert r["num_rendered"] == int(g["ref_num_rendered"][0])


BUILT = {
    "oracle_seed21_256": (dict(P=20000, W=256, H=256, seed=21, rigid=False, bg=(0.3, 0.1, 0.6)), None),
    "oracle_seed22_200x120": (dict(P=8000, W=200, H=120, seed=22, rigid=True, bg=(0.3, 0.1, 0.6)), None),
    "c2_100k_512": (dict(P=100_000, W=512, H=512, seed=31, rigid=True), "big"),
    "headline_300k_512": (dict(P=300_000, W=512, H=512, seed=41), "big"),
    "ragged_72x52": (dict(P=6000, W=72, H=52, seed=81), "ragged"),
    "ragged_200x116": (dict(P=12000, W=200, H=116, seed=82, center=(0.25, 0.2, 0.8)), "ragged"),
    "long_lists_50k_32": (dict(P=50000, W=32, H=32, seed=72), "long"),
}


@pytest.mark.parametrize("name", list(BUILT))
def test_built_scene(name, dev):
    from tests.golden.make_golden import build_case
    kw, edge = BUILT[name]
    r, _, _ = _run_single(name, build_case(**kw), dev)
    ln = _lengths(r)
    if edge == "big":
        assert r["num_rendered"] > kw["P"]
    elif edge == "ragged":
        W, H = kw["W"], kw["H"]
        tx = (W + 15) // 16
        outside = [t for t in range(len(ln)) if ln[t] > 0 and ((t % tx) * 16 + 8 >= W or (t // tx) * 16 + 4 >= H)]
        assert W % 16 == 8 and H % 16 == 4 and outside, "no busy tile reaches past the image edge"
    elif edge == "long":
        assert ln.min() > 32 * CH


def scene_long_overflow():
    """9,000 large faint surfels over a 32 x 32 image: 9,000 instances in each of the 4 tiles, and every pixel walks about
    750 of them before T falls below 1e-4, so each of a tile's first three chunks has far more than 4,608 contributing
    pairs and the backward sends the excess through its per-pair path, chunk after chunk."""
    from .test_gpu_variants import _facing_case
    rng = np.random.default_rng(109)
    n = 9000
    return _facing_case(32, 32, 16 + rng.uniform(-2, 2, n), 16 + rng.uniform(-2, 2, n), rng.uniform(0.5, 5.0, n),
                        np.full(n, 48.0), rng.uniform(0.01, 0.015, n), seed=110)


@pytest.mark.parametrize("name", ["exact_lengths", "dense", "long_overflow"])
def test_constructed_scene(name, dev):
    from .test_gpu_variants import CONSTRUCTED, DENSE_N, EXACT_LENGTHS
    inp = scene_long_overflow() if name == "long_overflow" else CONSTRUCTED[name]()
    r, _, _ = _run_single(name, inp, dev)
    pairs = _chunk_pairs(r)
    # _bounds counts each surfel's pairs past the pair buffer pixel by pixel; their total must be the chunks' excess
    assert _fallback_pairs(r, int(inp["meta"][0])).sum() == sum(max(0, n - BWD_CAP) for n in pairs.values())
    if name == "long_overflow":
        over = [c for c in pairs.values() if c > BWD_CAP]
        assert _lengths(r).min() > 32 * CH and len(over) >= 8, sorted(pairs.values())[-8:]
    elif name == "exact_lengths":
        assert _lengths(r).tolist() == list(EXACT_LENGTHS) + [0]        # 1, 255, 256, 257, 769 among them
    else:
        counts = sorted(pairs.values())
        # chunk 0 of each tile: 256 x 256 pairs, past the buffer; chunk 1: 16 x 256 = 4,096, just under it
        assert max(counts) == CH * CH and (DENSE_N - CH) * 256 in counts and (DENSE_N - CH) * 256 < BWD_CAP, counts


@pytest.mark.parametrize("M,deg", [(1, 0), (4, 1), (9, 2), (16, 1), (16, 3)])
def test_sh_coefficient_counts(M, deg, dev):
    from tests.golden.make_golden import build_case
    inp = build_case(3000, 96, 80, 80 + M, sh_degree=deg)
    inp["shs"] = np.ascontiguousarray(inp["shs"][:, :M])
    inp["meta"][3] = deg
    _run_single(f"sh M={M} deg={deg}", inp, dev)


# ------------------------------------------------------------------------------------------------ batches
def _batch(name, dev, sc, means, cams, W, H, seed):
    """M frames with per-frame positions through the batched entry points; sum_shared off (frame by frame) and on
    (shared inputs' gradients against the sum of the oracle's frames, with the bounds summed)."""
    from oracle import surfel_oracle as so
    from vidu4d_b200 import debug as dbg, rasterizer as R
    C = R._C
    t = sc.to_torch(dev)
    M, P = int(means.shape[0]), int(t["opacities"].shape[0])
    vms, pms, cps = cams
    bg = torch.tensor([0.2, 0.1, 0.4], device=dev)
    e = torch.empty((0,), device=dev)
    nr, color, allmap, radii, gb, bb, ib = C.rasterize_gaussians_batch(bg, means, e, t["opacities"], t["scales"], t["rotations"],
                                                                       1.0, vms, pms, TAN, TAN, H, W, t["shs"], 3, cps)
    g = torch.Generator(device=dev).manual_seed(seed)
    dLc = torch.randn((M, 3, H, W), device=dev, generator=g)
    dLo = 0.1 * torch.randn((M, 8, H, W), device=dev, generator=g)
    frames, decs = [], []
    for f in range(M):
        dec = dbg.decode(gb.view(M, -1)[f], bb.view(M, -1)[f], ib.view(M, -1)[f], P, W, H, nr[f])
        dec["radii"] = _np(radii[f])
        dec["num_rendered"] = nr[f]
        st, ext = _oracle_frame(dec, P, W, H, _np(means[f]), sc.opacities, sc.scales, sc.rotations, sc.shs, None, 3,
                                _np(bg), _np(vms[f]), _np(pms[f]), _np(cps[f]))
        fwd = _check_forward(f"{name} frame {f}", st, ext, _np(color[f]), _np(allmap[f]), dec, W, H)
        keep = torch.from_numpy((~ext["knife"]).astype(np.float32)).to(dev)
        dLc[f] *= keep
        dLo[f] *= keep
        og = so.backward(st, _np(dLc[f]), _np(dLo[f]), bounds=True)
        frames.append((st, ext, og, _bounds(st, og, dec), fwd))
        decs.append(dec)
    for sum_shared in (False, True):
        gr = dict(zip(GRADS, C.rasterize_gaussians_backward_batch(bg, means, radii, e, t["scales"], t["rotations"], 1.0, vms,
                                                                  pms, TAN, TAN, dLc, dLo, t["shs"], 3, cps, gb, bb, ib,
                                                                  sum_shared=sum_shared)))
        report = {}
        if not sum_shared:
            _check_knife(name, sum(int(fr[1]["knife"].sum()) for fr in frames))
        per_frame = [k for k in GRADS if gr[k].dim() == frames[0][2][k].ndim + 1]
        summed = [k for k in GRADS if k not in per_frame]
        assert summed == ([] if not sum_shared else ["dL_dcolors", "dL_dopacity", "dL_dsh", "dL_dscales", "dL_drotations"]), summed
        for f, (st, _, og, tol, _) in enumerate(frames):
            if not sum_shared:
                _check_all(f"{name} frame {f}", st, og, tol, {k: gr[k][f] for k in GRADS}, report)
                continue
            for k in per_frame:
                _check_grad(f"{name} sum_shared=True frame {f}", k, gr[k][f], og[k], tol[k], report)
        for k in summed:
            ref = sum(fr[2][k].astype(np.float64) for fr in frames)
            tol = sum(fr[3][k] for fr in frames) + M * U * sum(np.abs(fr[2][k].astype(np.float64)) for fr in frames)
            _check_grad(f"{name} sum_shared=True", k, gr[k], ref, tol, report)
        _print(f"{name} sum_shared={sum_shared}", sum(int(fr[1]["knife"].sum()) for fr in frames),
               max(fr[4] for fr in frames), report)
    return decs


def test_batch8_per_frame_positions(dev):
    from vidu4d_b200.synthetic import object_scene
    from .test_gpu_batch import _cams
    sc = object_scene(20000, seed=8, center=(0.0, 0.0, 0.0))
    g = torch.Generator(device=dev).manual_seed(88)
    base = torch.from_numpy(sc.means3D).to(dev)
    means = torch.stack([base + 0.002 * f * torch.randn(base.shape, device=dev, generator=g) for f in range(8)]).contiguous()
    decs = _batch("batch8", dev, sc, means, _cams(8, dev), 128, 96, seed=8)
    nr = [int(d["num_rendered"]) for d in decs]
    assert min(nr) > 0 and len(set(nr)) > 1, nr


def test_batch5_empty_and_two_surfel_frames(dev):
    from vidu4d_b200.synthetic import object_scene
    from .test_gpu_batch import _cams
    sc = object_scene(20000, seed=5, center=(0.0, 0.0, 0.0))
    cams = _cams(5, dev)
    base = torch.from_numpy(sc.means3D).to(dev)
    cp = cams[2]
    means = base[None].repeat(5, 1, 1)
    means[0] = 2 * cp[0]                                             # frame 0: everything 1 behind its camera
    means[1] = 2 * cp[1]                                             # frame 1: all but the two surfels nearest its camera
    near = torch.topk(base @ cp[1] / cp[1].norm(), 2).indices
    means[1, near] = base[near]
    decs = _batch("batch5", dev, sc, means.contiguous(), cams, 120, 88, seed=55)
    assert int(decs[0]["num_rendered"]) == 0
    assert int((decs[1]["radii"] > 0).sum()) == 2 and int(decs[1]["num_rendered"]) >= 2
