"""Every element of the feature pass (composite_feat.cu) against the CPU oracle, under an a-priori rounding-error bound.

A feature plane is composited with exactly the colour's contributors, weights and FMA order, so the colour oracle
(oracle/surfel_oracle.c) is the feature pass's oracle too: the F channels are split into groups of 3 (the last one
zero-padded), and each group runs through the oracle as a colour -- composited from the GPU's own decoded records as in
test_gpu_grad_bounds.py, with colours_precomp = the group's feature columns, bg = the group's 3 feature background values
(zeros for a 3-value background), dL/dcolour = the group's upstream gradient and dL/dallmap = 0.  The knife mask depends
on geometry only, so it is the colour run's; every group's mask must equal it, and the feature upstream gradients are
masked with it too.  Checked, outside the mask:

  * the feature planes: within K u fbound of the group's composite, and bit for bit a colour render of the same values;
  * dL/dfeatures: each group's colour accumulator, element by element, within
        K u (bound + (m_feat + SLACK) asum)                                                   (colour slots)
    m_feat = the surfel's contributing pairs: the backward reduces  T alpha dL/dplane  into dL/dfeatures once per pair and
    channel (each channel belongs to one chunk), m_feat fp32 adds in no fixed order, and m adds into one slot cost at most
    m u sum |t| over everything added.  When the frames of a batch share one dL/dfeatures row (shared features under
    sum_shared) every frame's pairs add into it: m_feat is summed over the frames, and so are bound and asum;
  * every gradient tensor, end to end: the total accumulator is the colour run's plus every group's with the group's
    colour slots zeroed (the feature pass adds only to dT, dopacity and the low-pass dmean2D; its dL/dz is 0), pushed
    through the oracle's per-surfel chain of the colour state.  Its bound is
        B = bound_c + sum_g bound_g + (m_c + n_chunks m_feat + CHAIN + SLACK) (asum_c + sum_g asum_g)
    through oracle.chain_bound, with m_c = tiles touched + pairs past the colour backward's pair buffer (as in _bounds)
    and n_chunks = ceil(F / 8): each of a pair's chunks reduces its own share of dL/dalpha into the same slots.  The
    accumulator-level dL/dopacity is checked first, so a failure says whether the composite or the chain went wrong.

SLACK, in units of u times asum, is what the 3-channel oracle does not model:

  * the 8-channel sums.  A CTA owns FC = 8 channels and forms, per pair, dL/dalpha = T sum_c (x_c - behind_c) g_c and,
    per pixel, bg_dot = sum_c bg_c g_c over its 8 channels; the oracle forms both over 3.  In a recursive fp32 sum of n
    products each term meets at most n roundings (its product and n - 1 additions), so at most FC = 8 here; counting all
    8 as unmodelled is conservative (the oracle's SO_CB already pays for its own 3-channel sums).  Each term of
    dL/dalpha lies in one of the two sums, so the relative error they add to dL/dalpha is at most 8 u times the sum of
    its terms' magnitudes, and not 16.  dT, dopacity and the low-pass dmean2D of a pair are dL/dalpha times factors the
    oracle already bounds, and their |t| in asum are linear in the same magnitudes: FC u asum covers the sums.
  * dout * features_grad_scale: the kernel multiplies each upstream value by the scale once, an fp32 product of two fp32
    numbers.  The oracle is fed that product correctly rounded to fp32 (the double product is exact, so rounding it once
    gives the same bits), so both sides start from the same upstream values and the scale's rounding costs nothing,
    whether or not the scale is a power of two.  A features_grad_scale of 0 makes every dL/dalpha and every reduced value
    +-0, which leaves every accumulator slot bit for bit unchanged: then the geometry must meet the colour-only bound
    (_bounds) and dL/dfeatures must be exactly 0.

So SLACK = FC.

K = 2, FLOOR and CHAIN are test_gpu_grad_bounds.py's.  Summed frames (sum_shared) add M u sum_f |oracle_f| for the
per-surfel kernel's sequential frame sum, as there.

Each case asserts from the GPU's buffers or the oracle state that it reaches its edge (its load width and chunking, its
low-pass share, its background, its early-stopping sub-tiles, ...), prints its knife pixels and the largest err /
tolerance per tensor, and keeps its knife mask within a few times the size measured on an H100 (KNIFE_MEASURED).
"""
import numpy as np
import pytest
import torch

from .conftest import load_golden
from .test_gpu_grad_bounds import (CHAIN, FLOOR, GRADS, K, U, _bounds, _check_all, _check_forward, _check_grad,
                                   _fallback_pairs, _oracle_frame, _print)

pytestmark = pytest.mark.gpu

FC = 8                   # SR_FEAT_CHUNK: channels per CTA of the feature pass, gridDim.y = ceil(F / FC)
FEATURES_MAX = 32        # SR_FEAT_MAX
SLACK = FC               # see the module docstring
CH = 256                 # instances per chunk of the composite backward
TAN = 0.5
C3 = slice(15, 18)       # oracle.surfel_oracle.ACC_COLOR .. + 3
F_GRID = (1, 2, 3, 4, 7, 8, 9, 16, 20, 22, 30, 31, 32)

# Masked (knife-edge) pixels per scene (batch3: over its 3 frames), measured on an H100; a case may mask at most 4 times
# as many plus 8.  The mask depends on the geometry only, so every feature width of a scene masks the same pixels.
# cta_stop's opaque front surfels clamp alpha at 0.99, so T (1 - alpha) after the second one is 0.01^2, on the 1e-4
# stopping threshold, at most of the pixels they cover: the case checks the other 3,500.
KNIFE_MEASURED = {"id_deg3_64": 0, "oracle_seed21_256": 2, "rigid_bg_96x64": 0, "lowpass_64": 1,
                  "long_lists_50k_32": 1, "warp_stop": 1, "cta_stop": 593, "c2_100k_512": 11, "batch3": 3}


@pytest.fixture(scope="module")
def dev(built):
    from vidu4d_b200 import _capi
    _capi.load()
    return torch.device("cuda:0")


def _np(x):
    return x.detach().cpu().numpy()


def feature_vec(F, addrs):
    """Floats per vector access of a feature row, as api.cu's feature_vec picks it: 4 or 2 when F is a multiple and every
    address (features, their frame stride in bytes, and in the backward dL/dfeatures) is 16- or 8-byte aligned, else 1."""
    for v in (4, 2):
        if F % v == 0 and all(a % (4 * v) == 0 for a in addrs):
            return v
    return 1


def _chunks(F):
    """(number of FC-channel chunks, live channels of the last one)."""
    n = (F + FC - 1) // FC
    return n, F - FC * (n - 1)


def _check_knife(scene, n):
    assert n <= 4 * KNIFE_MEASURED[scene] + 8, (scene, "knife pixels", n)


# ------------------------------------------------------------------------------------------------ pairs
def _stage_words(dec):
    """The live contribution-mask words: (tile, stage, first instance, words (n, 8 sub-tiles, 32 lanes)), with the words
    of a sub-tile past its deepest contributor zeroed (the kernels read stage s of sub-tile w for
    s < ceil(min(sub_last, len) / 32))."""
    rg = _np(dec["ranges"]).astype(np.int64)
    sl = _np(dec["sub_last"]).astype(np.int64)
    masks = _np(dec["contrib_masks"]).view(np.uint32)
    nb = (np.minimum(sl, (rg[:, 1] - rg[:, 0])[:, None]) + 31) >> 5            # (tiles, 8)
    n = nb.max(1)
    t = np.repeat(np.arange(rg.shape[0]), n)
    b = np.arange(t.size) - np.repeat(np.cumsum(n) - n, n)
    words = masks[(rg[t, 0] >> 5) + t + b]                                     # (rows, 8, 32)
    words = np.where((b[:, None] < nb[t])[..., None], words, 0)
    return t, b, rg[t, 0] + 32 * b, words


def _pair_counts(dec, P):
    """Per surfel, its contributing (pixel, surfel) pairs, from the GPU's contribution masks: bit j of a stage word is the
    stage's j-th instance."""
    from vidu4d_b200 import debug as dbg
    rg = _np(dec["ranges"]).astype(np.int64)
    t, _, first, words = _stage_words(dec)
    w = words.reshape(words.shape[0], -1)
    cnt = np.stack([((w >> np.uint32(j)) & np.uint32(1)).sum(1, dtype=np.int64) for j in range(32)], 1)   # (rows, 32)
    inst = first[:, None] + np.arange(32)
    live = cnt > 0
    assert (inst[live] < rg[t, 1][:, None].repeat(32, 1)[live]).all(), "a contribution bit past the tile's list"
    pl = _np(dec["point_list"]).view(np.uint32).astype(np.int64)
    m = np.bincount(pl[inst[live]], weights=cnt[live], minlength=P).astype(np.int64)
    assert m.sum() == dbg.contributing_pairs(dec)
    return m


def _pair_list(dec, W):
    """Every contributing pair as (instance, pixel x, pixel y) -- for small scenes."""
    t, _, first, words = _stage_words(dec)
    i, w, lane = np.nonzero(words)
    bits = (words[i, w, lane][:, None] >> np.arange(32, dtype=np.uint32)) & 1
    k, j = np.nonzero(bits)
    i, w, lane = i[k], w[k], lane[k]
    tx = (W + 15) // 16
    x = (t[i] % tx) * 16 + (w & 1) * 8 + lane % 8
    y = (t[i] // tx) * 16 + (w >> 1) * 4 + lane // 8
    return first[i] + j, x, y


def _lowpass_pairs(st, dec):
    """(low-pass pairs, all pairs): the rho3d > rho2d test of tests/feature_model.py's _walk, on the oracle state's
    records, over the pairs the GPU's masks say contributed."""
    inst, x, y = _pair_list(dec, st.W)
    sid = st.point_list[inst].astype(np.int64)
    Tm = st.transMat[sid].astype(np.float64)
    px, py = x + 0.5, y + 0.5
    k = px[:, None] * Tm[:, 6:9] - Tm[:, 0:3]
    l_ = py[:, None] * Tm[:, 6:9] - Tm[:, 3:6]
    p = np.cross(k, l_)
    with np.errstate(divide="ignore", invalid="ignore"):
        sx, sy = p[:, 0] / p[:, 2], p[:, 1] / p[:, 2]
    rho3d = sx * sx + sy * sy
    dx, dy = st.means2D[sid, 0] - px, st.means2D[sid, 1] - py
    rho2d = 2 * (dx * dx + dy * dy)
    return int((rho3d > rho2d).sum()), int(inst.size)


# ------------------------------------------------------------------------------------------------ GPU side
def _scene(inp, dev):
    """The inputs of a case in build_case's format as contiguous float32 CUDA tensors (what rasterizer._forward takes)."""
    P, W, H, deg, pre = [int(v) for v in inp["meta"]]
    t = lambda k, *s: torch.from_numpy(np.ascontiguousarray(inp[k], np.float32)).to(dev).reshape(*s)  # noqa: E731
    return dict(P=P, W=W, H=H, deg=deg, means3D=t("means3D", P, 3), opac=t("opacities", P, 1), scales=t("scales", P, 2),
                rots=t("rotations", P, 4), sh=None if pre else t("shs", P, -1, 3),
                col=t("colors_precomp", P, 3) if pre else None, vm=t("viewmatrix", 4, 4), pm=t("projmatrix", 4, 4),
                cp=t("campos", 3), tan=(float(inp["tanfov"][0]), float(inp["tanfov"][1])))


def _forward(s, bg, feat):
    """One frame through rasterizer._forward (below _f32c, so a misaligned features view reaches the kernels as is)."""
    from vidu4d_b200 import debug as dbg, rasterizer as R
    nr, color, allmap, radii, gb, bb, ib, _ = R._forward(
        1, False, {}, bg, s["means3D"], s["sh"], s["col"], s["opac"], s["scales"], s["rots"], feat, s["vm"], s["pm"],
        s["cp"], s["H"], s["W"], s["deg"], s["tan"][0], s["tan"][1], 1.0, False, False)
    dec = dbg.decode(gb, bb, ib, s["P"], s["W"], s["H"], nr[0])
    dec["radii"] = _np(radii)
    dec["num_rendered"] = nr[0]
    return color, allmap, radii, (gb, bb, ib), dec


def _backward(s, bg, feat, radii, bufs, dLc, dLo, dLf, fgs=None):
    from vidu4d_b200 import rasterizer as R
    g = R._backward(1, False, {}, bg, s["means3D"], s["sh"], s["col"], s["scales"], s["rots"], feat, s["vm"], s["pm"],
                    s["cp"], radii, dLc, dLf, dLo, *bufs, s["deg"], s["tan"][0], s["tan"][1], 1.0, False,
                    features_grad_scale=fgs)
    return dict(zip(GRADS + ("dL_dfeatures",), g))


def _colour_render(s, cols, bg3):
    """The GPU's colour planes of the scene with precomputed colours cols (P,3) over bg3."""
    from vidu4d_b200 import rasterizer as R
    return R._forward(1, False, {}, bg3, s["means3D"], None, cols, s["opac"], s["scales"], s["rots"], None, s["vm"],
                      s["pm"], s["cp"], s["H"], s["W"], 0, s["tan"][0], s["tan"][1], 1.0, False, False)[1]


# ------------------------------------------------------------------------------------------------ oracle side
def _groups(feat, bgf):
    """[(columns (P,3), background (3,), live channels)] of the features in groups of 3, the last zero-padded."""
    P, F = feat.shape
    n = (F + 2) // 3
    fp = np.zeros((P, 3 * n), np.float32)
    fp[:, :F] = feat
    bp = np.zeros(3 * n, np.float32)
    if bgf is not None:
        bp[:F] = bgf
    return [(np.ascontiguousarray(fp[:, 3 * k:3 * k + 3]), bp[3 * k:3 * k + 3].copy(), min(3, F - 3 * k)) for k in range(n)]


def _oracle_fwd(name, dec, inp, means3D, feat, bgf, color, allmap, dev=None, s=None, off=None):
    """The colour oracle and one oracle per feature group, composited from this frame's GPU records; checks n_contrib,
    the colour/allmap planes and every feature plane within its bound outside the knife mask, every group's mask equal to
    the colour's, and (given the scene s) every feature plane bit for bit a colour render of the same values.  off: the
    principal-point offsets of the frame's camera-table row, for the records' check."""
    P, W, H, deg, pre = [int(v) for v in inp["meta"]]
    tan = (float(inp["tanfov"][0]), float(inp["tanfov"][1]))
    geo = (means3D, inp["opacities"], inp["scales"], inp["rotations"])
    st, ext = _oracle_frame(dec, P, W, H, *geo, None if pre else inp["shs"], inp["colors_precomp"] if pre else None, deg,
                            inp["bg"], inp["viewmatrix"], inp["projmatrix"], inp["campos"], tan, off=off, name=name)
    fwd = _check_forward(name, st, ext, _np(color[:3]), _np(allmap), dec, W, H)
    ok = ~ext["knife"]
    planes = _np(color[3:])
    groups = []
    for k, (cols, b3, n) in enumerate(_groups(feat, bgf)):
        # the records hold the colour forward's rgb, not the group's: their geometry only
        sg, eg = _oracle_frame(dec, P, W, H, *geo, None, cols, 0, b3, inp["viewmatrix"], inp["projmatrix"], inp["campos"], tan,
                               off=off, records=None, name=f"{name} group {k}")
        assert np.array_equal(eg["knife"], ext["knife"]), (name, "group", k, "knife mask differs from the colour's")
        for c in range(n):
            err = np.abs(planes[3 * k + c].astype(np.float64) - sg.color[c])
            r = np.where(ok, err / (K * U * eg["fbound"][c] + FLOOR), 0.0)
            assert r.max() <= 1.0, (name, f"feature plane {3 * k + c}", float(r.max()), np.argwhere(r > 1)[:4].tolist())
            fwd = max(fwd, float(r.max()))
        if s is not None:
            oc = _colour_render(s, torch.from_numpy(cols).to(dev), torch.from_numpy(b3).to(dev))
            assert torch.equal(color[3 + 3 * k:3 + 3 * k + n], oc[:n]), (name, "group", k, "not a colour render's bits")
        groups.append((sg, n))
    return dict(st=st, ext=ext, groups=groups, fwd=fwd, knife=int(ext["knife"].sum()))


def _oracle_bwd(fr, dLc, dLo, dLf):
    """The colour run's and every group's accumulators and bound sums, for upstream gradients already masked (and
    scaled: dLf is what the kernel multiplies out, fl(dout * features_grad_scale))."""
    from oracle import surfel_oracle as so
    H, W = dLc.shape[-2:]
    fr["og_c"] = so.backward(fr["st"], dLc, dLo, bounds=True)
    F = dLf.shape[0]
    pad = np.zeros((3 * len(fr["groups"]), H, W), np.float32)
    pad[:F] = dLf
    zo = np.zeros((8, H, W), np.float32)
    fr["og_g"] = [so.backward(sg, pad[3 * k:3 * k + 3], zo, bounds=True) for k, (sg, _) in enumerate(fr["groups"])]


def _dfeat_ref(frames, m_feat):
    """dL/dfeatures of the summed frames' groups and its tolerance; m_feat is the number of adds into each slot."""
    ref = sum(np.concatenate([og["acc"][:, C3] for og in fr["og_g"]], 1) for fr in frames)
    bnd = sum(np.concatenate([og["bound"][:, C3] for og in fr["og_g"]], 1) for fr in frames)
    asm = sum(np.concatenate([og["asum"][:, C3] for og in fr["og_g"]], 1) for fr in frames)
    F = frames[0]["F"]
    return ref[:, :F], (K * U * (bnd + (m_feat + SLACK)[:, None] * asm))[:, :F]


def _total(fr, dec, m_feat, F, zero_features=False):
    """The oracle's gradients from the total accumulator (colour + every group's non-colour slots) and their
    tolerances, see the module docstring; zero_features: the feature pass adds only +-0, so the colour-only bound."""
    from oracle import surfel_oracle as so
    st = fr["st"]
    acc, bnd, asm = (fr["og_c"][k].copy() for k in ("acc", "bound", "asum"))
    for og in fr["og_g"]:
        for dst, k in ((acc, "acc"), (bnd, "bound"), (asm, "asum")):
            a = og[k].copy()
            a[:, C3] = 0.0
            dst += a
    ref = so.chain(st, acc)
    if zero_features:
        assert not any(og["acc"].any() for og in fr["og_g"])
        return ref, _bounds(st, fr["og_c"], dec)
    adds = (_np(dec["tiles_touched"]).astype(np.float64) + _fallback_pairs(dec, st.P) + _chunks(F)[0] * m_feat
            + CHAIN + SLACK)
    return ref, {k: K * U * v for k, v in so.chain_bound(st, bnd + adds[:, None] * asm).items()}


def _check_frame(name, fr, dec, mine, report, zero_features=False):
    """dL/dfeatures, then every gradient tensor (accumulator level first) of one frame."""
    F = fr["F"]
    m = _pair_counts(dec, fr["st"].P)
    ref, tol = _dfeat_ref([fr], m)
    if zero_features:
        assert int(torch.count_nonzero(mine["dL_dfeatures"])) == 0, (name, "dL/dfeatures not exactly 0")
    _check_grad(name + " [feature backward]", "dL_dfeatures", mine["dL_dfeatures"], ref, tol, report)
    ref, tol = _total(fr, dec, m, F, zero_features)
    _check_all(name, fr["st"], ref, tol, mine, report)
    return m


# ------------------------------------------------------------------------------------------------ single frames
def _features(P, F, seed, bg="3+F"):
    rng = np.random.default_rng(seed)
    feat = rng.standard_normal((P, F)).astype(np.float32)
    bgf = rng.uniform(0.2, 1.0, F).astype(np.float32) if bg == "3+F" else None
    return feat, bgf, rng


def _run(name, scene, inp, dev, F, seed, bg="3+F", fgs=None, offset=None, colour_bg=None):
    """One frame with F feature channels: GPU forward and backward, the oracle on its records, every check.  offset: the
    features are a contiguous view that many floats into its storage; fgs: features_grad_scale.  Returns what the edge
    assertions need."""
    P, W, H = (int(v) for v in inp["meta"][:3])
    if colour_bg is not None:
        inp = dict(inp, bg=np.asarray(colour_bg, np.float32))
    s = _scene(inp, dev)
    feat, bgf, rng = _features(P, F, seed, bg)
    bg_t = torch.from_numpy(inp["bg"].reshape(3) if bgf is None else np.concatenate([inp["bg"].reshape(3), bgf])).to(dev)
    ft = torch.from_numpy(feat).to(dev)
    if offset is not None:
        store = torch.zeros(P * F + offset, device=dev)
        ft = store[offset:].view(P, F)
        ft.copy_(torch.from_numpy(feat))
    color, allmap, radii, bufs, dec = _forward(s, bg_t, ft)
    fr = _oracle_fwd(name, dec, inp, inp["means3D"], feat, bgf, color, allmap, dev, s)
    fr["F"] = F
    _check_knife(scene, fr["knife"])
    keep = (~fr["ext"]["knife"]).astype(np.float32)
    dLc = inp["dL_dcolor"] * keep
    dLo = inp["dL_dallmap"] * keep
    dLf = rng.standard_normal((F, H, W)).astype(np.float32) * keep
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    mine = _backward(s, bg_t, ft, radii, bufs, t(dLc), t(dLo), t(dLf), None if fgs is None else torch.tensor(fgs, device=dev))
    scaled = dLf if fgs is None else (dLf.astype(np.float64) * np.float64(np.float32(fgs))).astype(np.float32)
    _oracle_bwd(fr, dLc, dLo, scaled)
    report = {}
    m = _check_frame(name, fr, dec, mine, report, zero_features=fgs == 0)
    _print(name, fr["knife"], fr["fwd"], report)
    v = feature_vec(F, (ft.data_ptr(), 0, mine["dL_dfeatures"].data_ptr()))
    return dict(dec=dec, fr=fr, color=color, mine=mine, m=m, vec=v, feat=ft, bgf=bgf)


def _inputs(scene):
    from tests.golden.make_golden import build_case
    from .test_gpu_variants import CONSTRUCTED
    if scene in ("id_deg3_64", "rigid_bg_96x64"):
        return {k[3:]: v for k, v in load_golden(scene).items() if k.startswith("in_")}
    if scene in CONSTRUCTED:
        return CONSTRUCTED[scene]()
    if scene == "lowpass_64":
        return scene_lowpass()
    return build_case(**BUILT[scene])


BUILT = {"oracle_seed21_256": dict(P=20000, W=256, H=256, seed=21, rigid=False, bg=(0.3, 0.1, 0.6)),
         "long_lists_50k_32": dict(P=50000, W=32, H=32, seed=72),
         "c2_100k_512": dict(P=100_000, W=512, H=512, seed=31, rigid=True)}


def _expected_vec(F):
    """The load width of F features at an aligned address (torch allocations are 512-byte aligned)."""
    return feature_vec(F, (0, 0, 0))


def test_grid_reaches_every_load_width_and_chunking():
    """The F grid below reaches V = 4, 2 and 1 each with a single chunk, with several chunks the last of which is partial,
    and with the 4 chunks of FEATURES_MAX."""
    want = {4: {"single": (4, 8), "partial": (20,), "four": (32,)},
            2: {"single": (2,), "partial": (22,), "four": (30,)},
            1: {"single": (1, 3, 7), "partial": (9,), "four": (31,)}}
    for v, kinds in want.items():
        for kind, fs in kinds.items():
            for F in fs:
                n, last = _chunks(F)
                assert F in F_GRID and _expected_vec(F) == v, (F, v)
                assert {"single": n == 1, "partial": n > 1 and last < FC, "four": n == 4}[kind], (F, kind, n, last)
    assert max(F_GRID) == FEATURES_MAX and _chunks(FEATURES_MAX) == (4, FC)
    # feature_vec's alignment rule: an F that is a multiple of 4 drops to 2 and 1 floats at 8- and 4-byte offsets
    assert [feature_vec(16, (a, 0, 0)) for a in (0, 8, 4)] == [4, 2, 1]


# every feature width on the 64 x 64 scene; on the 256 x 256 one (the CPU oracle's time grows with its pairs) one width
# per load width, with 1, 3 and 4 chunks
GRID = [("id_deg3_64", F) for F in F_GRID] + [("oracle_seed21_256", F) for F in (8, 22, 32)]


@pytest.mark.parametrize("scene,F", GRID)
def test_feature_width_grid(scene, F, dev):
    r = _run(f"{scene} F={F}", scene, _inputs(scene), dev, F, seed=1000 + F)
    # the case reaches its load width and chunking: the kernels' feature_vec sees these addresses
    assert r["vec"] == _expected_vec(F), (F, r["vec"])
    assert r["color"].shape[0] == 3 + F and r["m"].sum() > 0


def test_same_features_at_three_load_widths(dev):
    """F = 16 as a contiguous view 0, 2 and 1 floats into its storage: V = 4, 2 and 1.  The planes are bit-identical;
    each backward is within the bound (its reductions run in another order, so not bit for bit)."""
    scene, F = "id_deg3_64", 16
    inp = _inputs(scene)
    planes, vecs = [], []
    for off in (0, 2, 1):
        r = _run(f"{scene} F={F} storage offset {off}", scene, inp, dev, F, seed=77, offset=off)
        assert r["feat"].storage_offset() == off and r["feat"].is_contiguous()
        vecs.append(r["vec"])
        planes.append(r["color"][3:].clone())
    assert vecs == [4, 2, 1], vecs
    assert torch.equal(planes[0], planes[1]) and torch.equal(planes[0], planes[2])


def scene_lowpass():
    """2,000 sub-pixel surfels (footprint 0.2 - 0.5 px: rho3d > rho2d at every pixel centre, the low-pass branch) among
    1,000 faint ones of 1 - 2.5 px (the 3D branch), facing the camera over a 64 x 64 image."""
    from .test_gpu_variants import _facing_case
    rng = np.random.default_rng(201)
    a, b = 2000, 1000
    px = rng.uniform(0, 64, a + b)
    py = rng.uniform(0, 64, a + b)
    z = rng.uniform(1.0, 5.0, a + b)
    sigma = np.concatenate([rng.uniform(0.2, 0.5, a), rng.uniform(1.0, 2.5, b)])
    opac = np.concatenate([rng.uniform(0.3, 0.9, a), rng.uniform(0.05, 0.3, b)])
    return _facing_case(64, 64, px, py, z, sigma, opac, seed=202)


def test_lowpass_pairs(dev):
    r = _run("lowpass_64 F=8", "lowpass_64", _inputs("lowpass_64"), dev, 8, seed=203)
    low, total = _lowpass_pairs(r["fr"]["st"], r["dec"])
    assert total == r["m"].sum()
    print(f"[lowpass_64] low-pass pairs {low} of {total}")
    assert low >= 0.25 * total and low > 5000, (low, total)


@pytest.mark.parametrize("bg", ["3", "3+F"])
def test_background(bg, dev):
    """A non-zero colour background with a 3-value background (zero feature background, bg_dot = 0) and with 3+F values;
    the scene leaves many pixels with a large final T, where the background term dominates dL/dalpha."""
    scene, F = "rigid_bg_96x64", 11
    r = _run(f"{scene} bg={bg} F={F}", scene, _inputs(scene), dev, F, seed=300, bg=bg, colour_bg=(0.3, 0.1, 0.6))
    Tf = _np(r["dec"]["final_T"][0])
    empty = _np(r["dec"]["n_contrib"][0]) == 0
    assert (Tf > 0.5).mean() > 0.1 and empty.any(), ((Tf > 0.5).mean(), int(empty.sum()))
    # pixels nothing reaches show the feature background itself: 0, or the 3+F background's tail
    planes = _np(r["color"][3:])[:, empty]
    want = np.zeros(F, np.float32) if r["bgf"] is None else r["bgf"]
    assert np.array_equal(planes, np.repeat(want[:, None], planes.shape[1], 1))
    assert np.array_equal(_np(r["color"][:3])[:, empty], np.repeat(np.float32([[0.3], [0.1], [0.6]]), empty.sum(), 1))


@pytest.mark.parametrize("scale", [0.37, 0.0])
def test_features_grad_scale(scale, dev):
    scene, F = "id_deg3_64", 22
    r = _run(f"{scene} features_grad_scale={scale} F={F}", scene, _inputs(scene), dev, F, seed=400, fgs=scale)
    if scale:
        assert np.frexp(np.float32(scale))[0] != 0.5, "a power of two scales exactly"
    else:
        assert int(torch.count_nonzero(r["mine"]["dL_dfeatures"])) == 0


@pytest.mark.parametrize("scene,F", [("long_lists_50k_32", 8), ("long_lists_50k_32", 32), ("warp_stop", 22),
                                     ("cta_stop", 22)])
def test_long_lists_and_early_stops(scene, F, dev):
    """Lists far longer than the 2-stage ring (it wraps many times), and sub-tiles whose walk stops (sub_last) short of
    the tile's list while another goes deep."""
    r = _run(f"{scene} F={F}", scene, _inputs(scene), dev, F, seed=500 + F)
    rg = _np(r["dec"]["ranges"]).astype(np.int64)
    ln = rg[:, 1] - rg[:, 0]
    sl = _np(r["dec"]["sub_last"]).astype(np.int64)
    if scene == "long_lists_50k_32":
        # every tile's deepest sub-tile walks more than 64 stages of 32 records through the 2-stage ring
        assert ln.min() > 32 * CH and (np.minimum(sl, ln[:, None]).max(1) > 64 * 32).all(), (ln.tolist(), sl.tolist())
    elif scene == "warp_stop":
        assert any(any(0 < v <= CH for v in sl[t]) and sl[t].max() > 2 * CH and ln[t] > 3 * CH
                   for t in range(len(ln))), (ln.tolist(), sl.tolist())
    else:
        assert ln[0] == 1208 and sl[0].max() + 2 * CH < ln[0], (ln.tolist(), sl.tolist())


def test_c2_production_size(dev):
    scene, F = "c2_100k_512", 22
    r = _run(f"{scene} F={F}", scene, _inputs(scene), dev, F, seed=600)
    assert int(r["dec"]["num_rendered"]) > BUILT[scene]["P"]


# ------------------------------------------------------------------------------------------------ batches
@pytest.mark.parametrize("shared", [False, True], ids=["per_frame_features", "shared_features"])
def test_batch3(shared, dev):
    """3 frames with per-frame positions and per-frame (M,P,F) or shared (P,F) features through the batched entry points,
    sum_shared off (frame by frame) and on (shared inputs' gradients -- and shared features' dL/dfeatures -- against the
    sum of the oracle's frames)."""
    from vidu4d_b200 import debug as dbg, rasterizer as R
    from vidu4d_b200.synthetic import object_scene
    from .test_gpu_batch import _cams
    C = R._C
    M, P, W, H, F = 3, 8000, 112, 80, 12
    sc = object_scene(P, seed=13, center=(0.0, 0.0, 0.0))
    t = sc.to_torch(dev)
    g = torch.Generator(device=dev).manual_seed(131)
    base = t["means3D"]
    means = torch.stack([base + 0.002 * f * torch.randn(base.shape, device=dev, generator=g) for f in range(M)]).contiguous()
    vms, pms, cps = _cams(M, dev)
    rng = np.random.default_rng(132)
    feat = rng.standard_normal((P, F) if shared else (M, P, F)).astype(np.float32)
    bgc = np.float32([0.2, 0.1, 0.4])
    bgf = rng.uniform(0.2, 1.0, F).astype(np.float32)
    bg = torch.from_numpy(np.concatenate([bgc, bgf])).to(dev)
    e = torch.empty((0,), device=dev)
    nr, color, allmap, radii, gb, bb, ib, _ = C.rasterize_gaussians_batch(
        bg, means, e, t["opacities"], t["scales"], t["rotations"], 1.0, vms, pms, TAN, TAN, H, W, t["shs"], 3, cps,
        features=torch.from_numpy(feat).to(dev))
    dLc = rng.standard_normal((M, 3, H, W)).astype(np.float32)
    dLo = 0.1 * rng.standard_normal((M, 8, H, W)).astype(np.float32)
    dLf = rng.standard_normal((M, F, H, W)).astype(np.float32)
    frames, decs = [], []
    for f in range(M):
        dec = dbg.decode(gb.view(M, -1)[f], bb.view(M, -1)[f], ib.view(M, -1)[f], P, W, H, nr[f])
        dec["radii"] = _np(radii[f])
        dec["num_rendered"] = nr[f]
        inp = dict(opacities=sc.opacities, scales=sc.scales, rotations=sc.rotations, shs=sc.shs,
                   colors_precomp=np.zeros(0, np.float32), bg=bgc, viewmatrix=_np(vms[f]), projmatrix=_np(pms[f]),
                   campos=_np(cps[f]), meta=np.array([P, W, H, 3, 0]), tanfov=np.float32([TAN, TAN]))
        fr = _oracle_fwd(f"batch3 frame {f}", dec, inp, _np(means[f]), feat if shared else feat[f], bgf, color[f], allmap[f])
        fr["F"] = F
        keep = (~fr["ext"]["knife"]).astype(np.float32)
        dLc[f] *= keep
        dLo[f] *= keep
        dLf[f] *= keep
        _oracle_bwd(fr, dLc[f], dLo[f], dLf[f])
        fr["m"] = _pair_counts(dec, P)
        frames.append(fr)
        decs.append(dec)
    assert min(nr) > 0 and len(set(nr)) > 1, nr
    knife = sum(fr["knife"] for fr in frames)
    _check_knife("batch3", knife)
    T = lambda a: torch.from_numpy(a).to(dev)  # noqa: E731
    for sum_shared in (False, True):
        gr = dict(zip(GRADS + ("dL_dfeatures",), C.rasterize_gaussians_backward_batch(
            bg, means, radii, e, t["scales"], t["rotations"], 1.0, vms, pms, TAN, TAN, T(dLc), T(dLo), t["shs"], 3, cps,
            gb, bb, ib, sum_shared=sum_shared, features=T(feat), dL_dout_features=T(dLf))))
        name = f"batch3 {'shared' if shared else 'per-frame'} features sum_shared={sum_shared}"
        report = {}
        totals = [_total(fr, dec, fr["m"], F) for fr, dec in zip(frames, decs)]
        per_frame = [k for k in GRADS if gr[k].dim() == totals[0][0][k].ndim + 1]
        summed = [k for k in GRADS if k not in per_frame]
        assert summed == ([] if not sum_shared else ["dL_dcolors", "dL_dopacity", "dL_dsh", "dL_dscales", "dL_drotations"])
        for f, (fr, (ref, tol)) in enumerate(zip(frames, totals)):
            if not sum_shared:
                _check_all(f"{name} frame {f}", fr["st"], ref, tol, {k: gr[k][f] for k in GRADS}, report)
            else:
                for k in per_frame:
                    _check_grad(f"{name} frame {f}", k, gr[k][f], ref[k], tol[k], report)
        for k in summed:
            ref = sum(r[k].astype(np.float64) for r, _ in totals)
            tol = sum(tl[k] for _, tl in totals) + M * U * sum(np.abs(r[k].astype(np.float64)) for r, _ in totals)
            _check_grad(f"{name} summed", k, gr[k], ref, tol, report)
        if shared and sum_shared:
            assert tuple(gr["dL_dfeatures"].shape) == (P, F)
            ref, tol = _dfeat_ref(frames, sum(fr["m"] for fr in frames))
            _check_grad(f"{name} summed [feature backward]", "dL_dfeatures", gr["dL_dfeatures"], ref, tol, report)
        else:
            assert tuple(gr["dL_dfeatures"].shape) == (M, P, F)
            for f, fr in enumerate(frames):
                ref, tol = _dfeat_ref([fr], fr["m"])
                _check_grad(f"{name} frame {f} [feature backward]", "dL_dfeatures", gr["dL_dfeatures"][f], ref, tol, report)
        _print(name, knife, max(fr["fwd"] for fr in frames), report)
