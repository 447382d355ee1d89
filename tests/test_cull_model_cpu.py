"""The composite's cull word (tests/cull_model.py) is conservative: no pair the uncut composite may blend falls outside
its surfel's cull rectangle or above its rho cut.

Seeded adversarial surfels of each class of cull_model.adversarial (grazing, near-parabolic, sub-pixel, off-image,
threshold-opacity) are evaluated against every pixel of ragged images, with centred and off-centre principal points up to
W away.  Each class prints its smallest headroom: the distance in pixels from a blended pair's pixel centre to the padded
box's edge, and cut - rho.  A few cull words are checked by hand.  No GPU."""
import functools

import numpy as np
import pytest

from . import cull_model as cm

# (W, H, principal point offset from the image centre)
CONFIGS = [(72, 52, (0.0, 0.0)), (37, 23, (-30.25, 17.5)), (61, 45, (55.5, -40.75))]
PER_CLASS = 400
CHUNK = 128


@functools.lru_cache(maxsize=None)
def _evaluate(cls):
    """Per config: blended pairs, pairs the cull word drops, smallest rectangle and cut headroom, and the pairs blended at
    each edge the class exists for."""
    out = []
    for k, (W, H, (ox, oy)) in enumerate(CONFIGS):
        rng = np.random.default_rng(1000 * k + cm.CLASSES.index(cls))
        ppx, ppy = W / 2 + ox, H / 2 + oy
        s = cm.adversarial(rng, cls, PER_CLASS, W, H, ppx, ppy)
        T, cxy = cm.trans_mat(s["means"], s["scales"], s["rotations"], W / (2 * cm.TAN), H / (2 * cm.TAN), ppx, ppy)
        keep = np.isfinite(cxy[0]) & np.isfinite(cxy[1])
        rec = cm.records(T, cxy, s["opacities"])[keep]
        bx, by, box = cm.cull_bbox(rec[:, :9], rec[:, 9], rec[:, 10], rec[:, 11], W, H)
        lo, _ = cm.rho_cut_words(rec[:, 11])                 # the smallest cut the kernel may encode
        ys, xs = np.mgrid[0:H, 0:W]
        xs, ys = xs.ravel(), ys.ravel()
        tiles_x = (W + cm.TILE - 1) // cm.TILE
        st = dict(pairs=0, dropped=0, rect=np.inf, cut=np.inf, thr=0, off=0)
        for i in range(0, len(rec), CHUNK):
            e = cm.pair_eval(rec[i:i + CHUNK], xs[None], ys[None])
            si, pi = np.nonzero(e["blend"])
            j = i + si
            rho = e["rho"][si, pi]
            w = cm.cull_word(bx[j], by[j], (ys[pi] // cm.TILE) * tiles_x + xs[pi] // cm.TILE, tiles_x, lo[j])
            st["pairs"] += si.size
            st["dropped"] += int((~cm.word_admits(w, xs[pi], ys[pi], rho)).sum())
            if si.size:
                c, d, b = xs[pi] + 0.5, ys[pi] + 0.5, box[:, j]
                m = np.minimum(np.minimum(c - b[0], b[1] - c), np.minimum(d - b[2], b[3] - d))
                st["rect"] = min(st["rect"], float(m.min()))
                st["cut"] = min(st["cut"], float((cm.rho_cut_value(lo[j]) - rho).min()))
                st["thr"] += int((rec[j, 11] == cm.INV255).sum())
                cx, cy = rec[j, 9], rec[j, 10]
                st["off"] += int(((cx < 0) | (cx > W) | (cy < 0) | (cy > H)).sum())
        out.append(st)
    return out


@pytest.mark.parametrize("cls", cm.CLASSES)
def test_cull_word_is_conservative(cls):
    res = _evaluate(cls)
    print(f"\n[{cls}] " + "; ".join(f"{W}x{H} pp+({ox},{oy}): {r['pairs']} pairs, rect headroom {r['rect']:.3g} px, "
                                     f"cut headroom {r['cut']:.3g}" for (W, H, (ox, oy)), r in zip(CONFIGS, res)))
    for (W, H, _), r in zip(CONFIGS, res):
        assert r["dropped"] == 0, (cls, W, H, r)
        assert r["pairs"] > 1000, (cls, W, H, r)
        assert r["rect"] >= 0 and r["cut"] >= 0, (cls, W, H, r)
    if cls == "threshold":
        # pairs at exactly f32(1/255): cut - rho is then about the 1e-4 margin (the product 255 opacity rounds to 1)
        assert all(r["thr"] > 0 for r in res) and min(r["cut"] for r in res) < 2e-4, res
    if cls == "offimage":
        assert all(r["off"] > 1000 for r in res), res


def test_grazing_angles_reach_the_hyperbola():
    """The grazing class spans both signs of Dc, and near-parabolic surfels sit on both sides of Dc = 0 within 1e-3."""
    for cls in ("grazing", "dc_zero"):
        rng = np.random.default_rng(7)
        s = cm.adversarial(rng, cls, PER_CLASS, 72, 52)
        T, cxy = cm.trans_mat(s["means"], s["scales"], s["rotations"], 72, 52, 36, 26)
        _, _, _, aux = cm._box(T, cxy[0], cxy[1], s["opacities"], 72, 52)
        live = ~aux["skip"]
        rel = aux["dc"][live] / (aux["c2"][live] * aux["a"][live] + aux["T"][live, 8] ** 2)
        assert (rel < 0).sum() > 20 and (rel > 0).sum() > 20, cls
        if cls == "dc_zero":
            assert (np.abs(rel) < 1e-3).sum() > 40, np.sort(np.abs(rel))[:8]


# ------------------------------------------------------------------------------------------------ hand-checked words
def _facing(ux, uy, a, b):
    """A surfel facing the camera with semi-axes a, b px (u = 1) centred on (ux, uy): T = ((a, 0, ux), (0, b, uy),
    (0, 0, 1)).  Its level set u^2 + v^2 <= c2 is the box ux +- a sqrt(c2), uy +- b sqrt(c2)."""
    return np.array([[a, 0, ux, 0, b, uy, 0, 0, 1]], np.float32)


def test_hand_checked_rectangle():
    # opacity 1: c2 = 2 ln 255 * 1.004 + 1e-3 = 11.12786, sqrt(c2) = 3.33584; x: 20.8 +- (2 * 3.33584 * 1.004 + 0.1)
    # = 20.8 +- 6.79838 -> [14.0016, 27.5984] -> pixels ceil(13.5016) = 14 .. floor(27.0984) = 27 (without the pad,
    # +- 6.65839 -> 14 .. 26); y: 10.5 +- 10.14756 -> pixels 0 .. 20 (without the pad 0 .. 19)
    bx, by, box = cm.cull_bbox(_facing(20.8, 10.5, 2, 3), [20.8], [10.5], [1.0], 64, 24)
    assert (int(bx[0]) & 0xffff, int(bx[0]) >> 16, int(by[0]) & 0xffff, int(by[0]) >> 16) == (14, 27, 0, 20)
    np.testing.assert_allclose(box[:, 0], [20.8 - 6.798375, 20.8 + 6.798375, 10.5 - 10.147563, 10.5 + 10.147563],
                               atol=1e-5)
    # in tile 1 (x 16..31) of a 4-tile-wide image: x0 = 0, x1 = 11, y0 = 0, y1 = 15, rho bits of opacity 1
    lo, hi = cm.rho_cut_words([1.0])
    assert int(cm.cull_word(bx, by, [1], 4, lo)[0]) == 0 | 11 << 4 | 0 << 8 | 15 << 12 | 1 << 16 | 0x41320000


def test_hand_checked_rectangle_clamped_at_the_right_edge():
    # W = 37: the box 36 +- 6.8 is clamped to pixel 36 = W - 1, which is x = 4 of the last tile column (32..36)
    bx, by, _ = cm.cull_bbox(_facing(36.0, 10.5, 2, 3), [36.0], [10.5], [1.0], 37, 20)
    assert (int(bx[0]) & 0xffff, int(bx[0]) >> 16, int(by[0]) & 0xffff, int(by[0]) >> 16) == (29, 36, 0, 19)
    assert int(cm.cull_word(bx, by, [2], 3, [0])[0]) == 0x1f040          # x0 0, x1 4, y0 0, y1 15, valid


def test_hand_checked_empty_rectangles():
    below = np.nextafter(cm.INV255, np.float32(0))
    bx, by, _ = cm.cull_bbox(_facing(20.8, 10.5, 2, 3), [20.8], [10.5], [below], 64, 24)
    assert int(bx[0]) == cm.EMPTY and int(by[0]) == cm.EMPTY               # alpha <= opacity < 1/255 everywhere
    assert int(cm.cull_word(bx, by, [0], 4, [0x41320000])[0]) == 0       # x0 = 1 > x1 = 0: no valid bit in tile 0
    assert int(cm.cull_word(bx, by, [3], 4, [0x41320000])[0]) == 0
    bx, by, _ = cm.cull_bbox(_facing(-20.0, 10.5, 2, 3), [-20.0], [10.5], [1.0], 64, 24)
    assert int(bx[0]) == cm.EMPTY                                          # wholly left of the image


def test_hand_checked_rho_cuts():
    lo, hi = cm.rho_cut_words(np.array([cm.INV255, 1.0, 1e3, np.nan, -1.0, 0.0], np.float32))
    assert lo.tolist() == hi.tolist()
    # f32(1/255): 255 * opacity rounds to 1, logf = 0, c2 = 1e-4f = 0x38d1b717 -> 0x38d20000 (1.0014e-4)
    # 1: c2 = 11.082627 = 0x41315271 -> 0x41320000 = 11.125;  1e3: 24.898136 = 0x41c72f62 -> 0x41c80000 = 25
    # NaN: no cut (+inf); negative: logf is NaN, no cut; 0: logf = -inf, c2 clamped to 0
    assert [hex(v) for v in lo] == ["0x38d20000", "0x41320000", "0x41c80000", "0x7f800000", "0x7f800000", "0x0"]
    bx, by, _ = cm.cull_bbox(_facing(20.8, 10.5, 2, 3), [20.8], [10.5], [np.nan], 64, 24)
    assert (int(bx[0]), int(by[0])) == (0 | 63 << 16, 0 | 23 << 16)      # NaN opacity: no cull, the whole image


def test_word_admits_decodes_the_rectangle_and_cut():
    w = np.uint32(2 | 5 << 4 | 3 << 8 | 9 << 12 | 1 << 16 | 0x41320000)
    px = np.array([18, 21, 17, 22, 18, 18, 18])
    py = np.array([3, 9, 3, 3, 2, 10, 3])
    rho = np.array([11.125, 0, 0, 0, 0, 0, np.nextafter(np.float32(11.125), np.float32(12))], np.float32)
    assert cm.word_admits(w, px, py, rho).tolist() == [True, True, False, False, False, False, False]
