"""TEST INFRASTRUCTURE -- the composite's cull word restated on the CPU, and what the uncut composite blends.

The composite forward skips a (pixel, instance) pair before blending it in two ways, both claimed never to change a
result:

  * the cull rectangle.  cull_bbox (csrc/preprocess.cu) pads, in double, the pixel box of the exact level set
    min(rho3d, rho2d) <= c2 of the fp32 homography T and stores it in surfel_rec floats 18/19 as x0 | x1 << 16 and
    y0 | y1 << 16 (x0 = 1 > x1 = 0: empty).  The sort (csrc/sort.cu) narrows it to a 4-bit tile-local rectangle in the
    instance record's cull word (float 19), and group_survivors drops every pixel outside it;
  * the rho cut.  cull_encode_rho_cut (composite_common.cuh) computes 2 logf(255 opacity) + 1e-4 in fp32, rounds it up
    to a 15-bit fp32 prefix and stores it in bits 17..31 of the same word; FwdPixel::blend skips a pair with rho > cut.

cull_bbox and rho_cut_words restate both.  The GPU evaluates cull_bbox's double arithmetic with its own contractions
and `log`, and logf to within 1 ulp, so where that rounding could decide an integer edge, the sign of Dc or a 15-bit
prefix, the restatement gives every value the kernel may produce (cull_candidates); everywhere else it gives one.

pair_eval is the uncut composite's per-pair arithmetic (composite_common.cuh pair_plane and FwdPixel::blend) in fp32
NumPy, in the kernel's operation order, pixel centres at i + 0.5.  A fused multiply-add is one float64 evaluation (the
product is exact there) rounded once to fp32; correctly rounded fp32 division stands for div2_rn, which is bit-identical
to it.  Its `blend` is "may blend": every test of blend() passes with expf anywhere within its 2-ulp error and at most
1 (cull_bbox relies on alpha <= opacity, i.e. expf(x) <= 1 for x <= 0; the GPU test checks that of the device's expf),
so it is a superset of what the GPU blends.  T's early stop is not modelled: it ends a pixel's walk, it never admits a pair.
"""
import numpy as np

F32 = np.float32
INV255 = F32(1.0 / 255.0)
TILE = 16
EMPTY = 1                      # x0 = 1 > x1 = 0
ULP53 = 2.0 ** -53
TAN = 0.5                      # the identity camera's tan(fov / 2) in the adversarial scenes


def _f(x):
    return np.asarray(x, F32)


def fm(a, b):
    return _f(a) * _f(b)


def fa(a, b):
    return _f(a) + _f(b)


def ff(a, b, c):
    """fmaf: the product is exact in float64, the sum rounded once there and once to fp32."""
    return (_f(a).astype(np.float64) * _f(b) + _f(c)).astype(F32)


# ------------------------------------------------------------------------------------------------ the rectangle
def _box(T, cx, cy, opac, W, H, nudge=None, flip=None):
    """cull_bbox in double; nudge (4, S) moves the unclamped edges x0, x1, y0, y1 before they are rounded to pixels and
    flip (S,) takes the other branch of `Dc < 0`.  Returns (bx, by, box (4, S) unclamped edges, aux)."""
    T = _f(T).reshape(-1, 9).astype(np.float64)
    op = _f(opac).reshape(-1)
    cx = _f(cx).reshape(-1).astype(np.float64)
    cy = _f(cy).reshape(-1).astype(np.float64)
    with np.errstate(all="ignore"):
        skip = op < INV255                                     # NaN falls through: no cull
        c2 = 2.0 * np.log(255.0 * op.astype(np.float64))
        c2 = c2 * 1.004 + 1e-3
        Twx, Twy, Twz = T[:, 6], T[:, 7], T[:, 8]
        a = Twx * Twx + Twy * Twy
        dc = c2 * a - Twz * Twz
        ell = dc < 0.0
        if flip is not None:
            ell = ell ^ flip
        inv = 1.0 / dc
        f0, f2 = c2 * inv, -inv
        pcx = f0 * (T[:, 0] * Twx + T[:, 1] * Twy) + f2 * (T[:, 2] * Twz)
        pcy = f0 * (T[:, 3] * Twx + T[:, 4] * Twy) + f2 * (T[:, 5] * Twz)
        qx = f0 * (T[:, 0] * T[:, 0] + T[:, 1] * T[:, 1]) + f2 * (T[:, 2] * T[:, 2])
        qy = f0 * (T[:, 3] * T[:, 3] + T[:, 4] * T[:, 4]) + f2 * (T[:, 5] * T[:, 5])
        ex0, ey0 = np.sqrt(np.fmax(0.0, pcx * pcx - qx)), np.sqrt(np.fmax(0.0, pcy * pcy - qy))
        ex, ey = ex0 * 1.004 + 0.1, ey0 * 1.004 + 0.1
        x0 = np.where(ell, pcx - ex, -1e30)
        x1 = np.where(ell, pcx + ex, 1e30)
        y0 = np.where(ell, pcy - ey, -1e30)
        y1 = np.where(ell, pcy + ey, 1e30)
        r2 = np.sqrt(0.5 * c2) + 0.1
        x0, x1 = np.fmin(x0, cx - r2), np.fmax(x1, cx + r2)
        y0, y1 = np.fmin(y0, cy - r2), np.fmax(y1, cy + r2)
        box = np.stack([x0, x1, y0, y1])
        if nudge is not None:
            x0, x1, y0, y1 = box + nudge
        fx0, fx1 = np.fmax(0.0, np.ceil(x0 - 0.5)), np.fmin(W - 1.0, np.floor(x1 - 0.5))
        fy0, fy1 = np.fmax(0.0, np.ceil(y0 - 0.5)), np.fmin(H - 1.0, np.floor(y1 - 0.5))
        empty = skip | ~(fx0 <= fx1) | ~(fy0 <= fy1)
    u = lambda v: np.where(empty, 0.0, v).astype(np.uint32)                          # noqa: E731
    bx = np.where(empty, np.uint32(EMPTY), u(fx0) | (u(fx1) << np.uint32(16))).astype(np.uint32)
    by = np.where(empty, np.uint32(EMPTY), u(fy0) | (u(fy1) << np.uint32(16))).astype(np.uint32)
    aux = dict(c2=c2, a=a, dc=dc, ell=ell & ~skip, skip=skip, pcx=pcx, pcy=pcy, qx=qx, qy=qy, ex0=ex0, ey0=ey0, T=T,
               cx=cx, cy=cy)
    return bx, by, box, aux


def cull_bbox(T, cx, cy, opac, W, H):
    """(bx, by, box): the kernel's two packed words for each surfel, and the padded box's unclamped edges (x0, x1, y0,
    y1) in pixel coordinates (pixel i spans [i, i + 1]); (-1e30, 1e30) where the level set is not a bounded ellipse."""
    bx, by, box, _ = _box(T, cx, cy, opac, W, H)
    return bx, by, box


def _edge_error(aux):
    """A first-order bound, with a safety factor of 16, on how far the GPU's double evaluation of each unclamped edge
    (its own contractions and `log`) can lie from this one's, and on |Dc|'s rounding."""
    T, c2, a, dc = aux["T"], aux["c2"], aux["a"], aux["dc"]
    with np.errstate(all="ignore"):
        dc_err = 8 * ULP53 * (np.abs(c2) * a + T[:, 8] ** 2)
        rel = 8 * ULP53 + dc_err / np.abs(dc)                 # relative error of f0 and f2
        tx = np.abs(c2 / dc) * (np.abs(T[:, 0] * T[:, 6]) + np.abs(T[:, 1] * T[:, 7])) + np.abs(T[:, 2] * T[:, 8] / dc)
        ty = np.abs(c2 / dc) * (np.abs(T[:, 3] * T[:, 6]) + np.abs(T[:, 4] * T[:, 7])) + np.abs(T[:, 5] * T[:, 8] / dc)
        qxa = np.abs(c2 / dc) * (T[:, 0] ** 2 + T[:, 1] ** 2) + T[:, 2] ** 2 / np.abs(dc)
        qya = np.abs(c2 / dc) * (T[:, 3] ** 2 + T[:, 4] ** 2) + T[:, 5] ** 2 / np.abs(dc)
        epx, epy = (rel + 4 * ULP53) * tx, (rel + 4 * ULP53) * ty
        e2x = 2 * np.abs(aux["pcx"]) * epx + (rel + 4 * ULP53) * qxa + 4 * ULP53 * aux["pcx"] ** 2
        e2y = 2 * np.abs(aux["pcy"]) * epy + (rel + 4 * ULP53) * qya + 4 * ULP53 * aux["pcy"] ** 2
        eex = np.where(aux["ex0"] > 0, np.fmin(e2x / (2 * aux["ex0"]), np.sqrt(e2x)), np.sqrt(e2x))
        eey = np.where(aux["ey0"] > 0, np.fmin(e2y / (2 * aux["ey0"]), np.sqrt(e2y)), np.sqrt(e2y))
        ell_x = np.where(aux["ell"], epx + 1.004 * eex, 0.0)
        ell_y = np.where(aux["ell"], epy + 1.004 * eey, 0.0)
        disc = 4 * ULP53 * (np.abs(aux["cx"]) + np.abs(aux["cy"]) + np.abs(c2) + 1)
        ex = 16 * (np.fmax(ell_x, disc) + 1e-12)
        ey = 16 * (np.fmax(ell_y, disc) + 1e-12)
    ex = np.where(np.isfinite(ex), ex, 1e300)
    ey = np.where(np.isfinite(ey), ey, 1e300)
    return ex, ey, (np.abs(dc) <= 16 * dc_err) & ~aux["skip"]


def cull_candidates(T, cx, cy, opac, W, H):
    """Every (bx, by) the kernel may write for each surfel: (bx, by) (S, 4) -- nominal, edges moved outwards, edges moved
    inwards by their rounding bound, and the other branch of Dc's sign where |Dc| is within its rounding.  A GPU field
    (x0, x1, y0 or y1) matches if it equals that field of any candidate.  Also returns the nominal box edges and the
    surfels where the candidates differ."""
    bx, by, box, aux = _box(T, cx, cy, opac, W, H)
    ex, ey, dc_amb = _edge_error(aux)
    e = np.stack([ex, ex, ey, ey])
    out = np.array([-1.0, 1.0, -1.0, 1.0])[:, None] * e
    bxo, byo, _, _ = _box(T, cx, cy, opac, W, H, nudge=out)
    bxi, byi, _, _ = _box(T, cx, cy, opac, W, H, nudge=-out)
    bxf, byf, _, _ = _box(T, cx, cy, opac, W, H, flip=dc_amb)
    BX, BY = np.stack([bx, bxo, bxi, bxf], 1), np.stack([by, byo, byi, byf], 1)
    amb = (BX != bx[:, None]).any(1) | (BY != by[:, None]).any(1)
    return BX, BY, box, amb


def match_bbox(gpu_bx, gpu_by, BX, BY):
    """Per surfel: every 16-bit field of the GPU's words equals that field of some candidate."""
    ok = np.ones(len(gpu_bx), bool)
    for g, C in ((np.asarray(gpu_bx, np.uint32), BX), (np.asarray(gpu_by, np.uint32), BY)):
        for sh in (0, 16):
            f = (g >> np.uint32(sh)) & np.uint32(0xffff)
            ok &= (((C >> np.uint32(sh)) & np.uint32(0xffff)) == f[:, None]).any(1)
    return ok


# ------------------------------------------------------------------------------------------------ the rho cut
def encode_rho_cut(c2):
    """cull_encode_rho_cut from its fp32 c2 = 2 logf(255 opacity) + 1e-4: +inf for NaN, else the next 15-bit prefix at
    or above max(c2, 0)."""
    c2 = _f(c2)
    bits = np.fmax(c2, F32(0)).view(np.uint32)
    w = (bits + np.uint32(0x1ffff)) & np.uint32(0xfffe0000)
    return np.where(np.isnan(c2), np.uint32(0x7f800000), w).astype(np.uint32)


def rho_cut_words(opac):
    """(lo, hi): the smallest and largest rho-cut bits (word & 0xfffe0000) the kernel may encode for each opacity.  The
    product 255 opacity is exact arithmetic here; logf is correctly rounded +- 1 ulp, its CUDA error bound."""
    p = fm(F32(255.0), _f(opac))
    with np.errstate(all="ignore"):
        l0 = np.log(p.astype(np.float64)).astype(F32)
        ws = [encode_rho_cut(fa(F32(2.0) * lv, F32(1e-4)))
              for lv in (np.nextafter(l0, F32(-np.inf)), l0, np.nextafter(l0, F32(np.inf)))]
    ws = np.stack(ws)
    return ws.min(0), ws.max(0)


def rho_cut_value(word):
    """The cut a word decodes to (cull_rho_cut: one AND)."""
    return (np.asarray(word, np.uint32) & np.uint32(0xfffe0000)).view(F32)


# ------------------------------------------------------------------------------------------------ the instance word
def cull_word(bx, by, tile, tiles_x, rho_word):
    """sort.cu's cull word of an instance of a surfel with packed box (bx, by) in tile `tile`: the box narrowed to the
    tile, 4 bits per edge, the valid bit and the rho-cut bits; 0 when the box misses the tile."""
    bx, by = np.asarray(bx, np.int64), np.asarray(by, np.int64)
    tile = np.asarray(tile, np.int64)
    tx, ty = (tile % tiles_x) * TILE, (tile // tiles_x) * TILE
    x0, x1 = np.maximum((bx & 0xffff) - tx, 0), np.minimum((bx >> 16) - tx, TILE - 1)
    y0, y1 = np.maximum((by & 0xffff) - ty, 0), np.minimum((by >> 16) - ty, TILE - 1)
    ok = (x0 <= x1) & (y0 <= y1)
    w = x0 | (x1 << 4) | (y0 << 8) | (y1 << 12) | (1 << 16) | np.asarray(rho_word, np.int64)
    return np.where(ok, w, 0).astype(np.uint32)


def word_admits(word, px, py, rho):
    """What the composite keeps of pair (pixel (px, py), rho) under a cull word: the pixel inside the word's tile-local
    rectangle (group_survivors) and rho <= the decoded cut (blend)."""
    w = np.asarray(word, np.int64)
    lx, ly = np.asarray(px) % TILE, np.asarray(py) % TILE
    inside = (((w >> 16) & 1) == 1) & ((w & 15) <= lx) & (lx <= ((w >> 4) & 15)) & (((w >> 8) & 15) <= ly) & \
        (ly <= ((w >> 12) & 15))
    return inside & ~(_f(rho) > rho_cut_value(w))


# ------------------------------------------------------------------------------------------------ the uncut composite
def pair_eval(rec, xs, ys):
    """One surfel per row of rec (S, 12: T[0..8], cx, cy, opacity, as surfel_rec floats 0..11) against the pixels (xs, ys)
    (broadcast against (S, 1)).  Returns blend (may blend: blend()'s tests with expf rounded up by 2 ulp), rho, rho3d,
    rho2d and depth."""
    r = _f(rec)
    c = lambda k: r[:, k:k + 1]                                                       # noqa: E731
    pixx = (np.asarray(xs).astype(F32) + F32(0.5))
    pixy = (np.asarray(ys).astype(F32) + F32(0.5))
    with np.errstate(all="ignore"):
        kx, ky, kz = ff(pixx, c(6), -c(0)), ff(pixx, c(7), -c(1)), ff(pixx, c(8), -c(2))
        lx, ly, lz = ff(pixy, c(6), -c(3)), ff(pixy, c(7), -c(4)), ff(pixy, c(8), -c(5))
        pz = ff(kx, ly, -fm(ky, lx))
        ppx, ppy = ff(ky, lz, -fm(kz, ly)), ff(kz, lx, -fm(kx, lz))
        sx, sy = ppx / pz, ppy / pz
        rho3d = ff(sx, sx, fm(sy, sy))
        dx, dy = fa(c(9), -pixx), fa(c(10), -pixy)
        q2 = ff(dx, dx, fm(dy, dy))
        rho2d = fa(q2, q2)
        rho = np.fmin(rho3d, rho2d)
        depth = np.where(rho3d <= rho2d, fa(c(8), ff(c(6), sx, fm(c(7), sy))), c(8))
        power = fm(rho, F32(-0.5))
        g = np.exp(power.astype(np.float64)).astype(F32)
        g = np.nextafter(np.nextafter(g, F32(np.inf)), F32(np.inf))               # expf within 2 ulp, rounded up,
        g = np.fmin(g, F32(1.0))                                                    # but never above expf(0) = 1
        alpha = np.fmin(F32(0.99), fm(c(11), g))
        blend = (pz != 0) & ~(depth < F32(0.2)) & ~(power > 0) & ~(alpha < INV255)
    return dict(blend=blend, rho=rho, rho3d=rho3d, rho2d=rho2d, depth=depth)


def trans_mat(means, scales, rotations, fx, fy, ppx, ppy):
    """The homography rows (S, 9) and the AABB centre (cx, cy) of surfels seen by the identity camera with focal lengths
    (fx, fy) and principal point (ppx, ppy), in float64 and then rounded to fp32 (the kernel's own rounding is not
    needed: the cull claims hold for whatever fp32 T it is given).  rotations (w, x, y, z): the tangent axes are the first
    two columns of the rotation matrix."""
    R = rot_columns(rotations)
    p = np.asarray(means, np.float64)
    s = np.asarray(scales, np.float64)
    M0, M1 = R[:, :, 0] * s[:, :1], R[:, :, 1] * s[:, 1:2]
    rows = []
    for v in (M0, M1, p):
        rows.append(fx * v[:, 0] + ppx * v[:, 2])
    for v in (M0, M1, p):
        rows.append(fy * v[:, 1] + ppy * v[:, 2])
    rows += [M0[:, 2], M1[:, 2], p[:, 2]]
    T = np.stack(rows, 1).astype(F32)
    return T, aabb_centre(T)


def aabb_centre(T):
    """computeAABB's centre (cxp, cyp) in the kernel's fp32 operations (preprocess.cu); NaN where d == 0."""
    T = _f(T)
    t = [T[:, k] for k in range(9)]
    with np.errstate(all="ignore"):
        d = ff(-t[8], t[8], ff(t[6], t[6], fm(t[7], t[7])))
        r = F32(1.0) / d
        cxp = ff(fm(t[2], t[8]), -r, ff(fm(t[1], t[7]), r, fm(fm(t[0], t[6]), r)))
        cyp = ff(fm(t[5], t[8]), -r, ff(fm(t[4], t[7]), r, fm(fm(t[3], t[6]), r)))
    return np.where(d != 0, cxp, np.nan).astype(F32), np.where(d != 0, cyp, np.nan).astype(F32)


def records(T, cxy, opac):
    """surfel_rec floats 0..11 (T, cx, cy, opacity) from trans_mat's output."""
    return np.concatenate([_f(T), _f(cxy[0])[:, None], _f(cxy[1])[:, None], _f(opac).reshape(-1, 1)], 1)


# ------------------------------------------------------------------------------------------------ adversarial surfels
def rot_columns(q):
    """(S, 3, 3) rotation matrices of unit-normalised quaternions (w, x, y, z)."""
    q = np.asarray(q, np.float64)
    q = q / np.linalg.norm(q, axis=1, keepdims=True)
    w, x, y, z = q.T
    return np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)], 1),
                     np.stack([2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)], 1),
                     np.stack([2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], 1)], 1)


def _quat(R):
    """Unit quaternions (w, x, y, z) of rotation matrices (S, 3, 3), by Shepperd's method: the largest of 4 w^2, 4 x^2,
    4 y^2, 4 z^2 (from the trace and the diagonal) is taken from the diagonal, the other three from the off-diagonal
    sums and differences divided by it.  Plain NumPy: the GPU test processes load no further compiled libraries."""
    R = np.asarray(R, np.float64)
    d0, d1, d2 = R[:, 0, 0], R[:, 1, 1], R[:, 2, 2]
    k = np.argmax(np.stack([d0, d1, d2, d0 + d1 + d2], 1), 1)
    s = np.sqrt(np.maximum(np.stack([1 + d0 - d1 - d2, 1 - d0 + d1 - d2, 1 - d0 - d1 + d2, 1 + d0 + d1 + d2], 1), 0))
    big = s[np.arange(len(k)), k]                                   # 2 |x|, 2 |y|, 2 |z| or 2 |w|
    dw = np.stack([R[:, 2, 1] - R[:, 1, 2], R[:, 0, 2] - R[:, 2, 0], R[:, 1, 0] - R[:, 0, 1]], 1)    # 4 w (x, y, z)
    sxy, sxz, syz = R[:, 0, 1] + R[:, 1, 0], R[:, 0, 2] + R[:, 2, 0], R[:, 1, 2] + R[:, 2, 1]       # 4 xy, 4 xz, 4 yz
    num = np.where((k == 3)[:, None], np.stack([big * big, dw[:, 0], dw[:, 1], dw[:, 2]], 1), 0.0)
    num = np.where((k == 0)[:, None], np.stack([dw[:, 0], big * big, sxy, sxz], 1), num)
    num = np.where((k == 1)[:, None], np.stack([dw[:, 1], sxy, big * big, syz], 1), num)
    num = np.where((k == 2)[:, None], np.stack([dw[:, 2], sxz, syz, big * big], 1), num)
    q = num / (2 * big[:, None])
    return q / np.linalg.norm(q, axis=1, keepdims=True)


def _unit(v):
    return v / np.linalg.norm(v, axis=1, keepdims=True)


def _frame_with_normal(rng, n):
    """Rotation matrices whose third column is n (S, 3) and whose tangent axes are turned at random about it."""
    a = _unit(np.cross(n, rng.normal(size=n.shape)))
    b = np.cross(n, a)
    phi = rng.uniform(0, 2 * np.pi, len(n))[:, None]
    t1 = np.cos(phi) * a + np.sin(phi) * b
    t2 = np.cross(n, t1)
    return np.stack([t1, t2, n], 2)


def _logu(rng, lo, hi, n):
    return np.exp(rng.uniform(np.log(lo), np.log(hi), n))


THRESHOLD_OPACITIES = np.array([np.nextafter(INV255, F32(0)), INV255, np.nextafter(INV255, F32(1)), 0.989, 0.99, 0.991,
                                1.0, 5.0, 1e3], F32)


def _opacities(rng, n):
    """Half from THRESHOLD_OPACITIES, half uniform in [1/255, 1]."""
    o = rng.uniform(1 / 255, 1, n).astype(F32)
    pick = rng.random(n) < 0.5
    o[pick] = rng.choice(THRESHOLD_OPACITIES, int(pick.sum()))
    return o


CLASSES = ("grazing", "dc_zero", "subpixel", "offimage", "threshold")


def adversarial(rng, cls, n, W, H, ppx=None, ppy=None, z_range=(0.25, 50.0)):
    """n surfels of one class for an identity camera (looking down +z) with tan(fov / 2) = TAN in both axes, so the focal
    lengths are W and H pixels, and principal point (ppx, ppy) (default the image centre).  Returns means (n, 3), scales
    (n, 2), rotations (n, 4) (w, x, y, z) and opacities (n,), all fp32:

      grazing    the surfel plane within 1e-7 .. 1e-1 rad of the view ray through its centre, either side;
      dc_zero    the level set's conic within a relative 1e-7 .. 1e-1 of a parabola (Dc = 0), either side;
      subpixel   scales 1e-4 .. 1 at depths 0.2 .. 50 (sub-pixel footprints: the low-pass disc decides);
      offimage   centred up to W (H) outside the image, big enough to reach in;
      threshold  opacities in THRESHOLD_OPACITIES only, centred within 1e-4 px of a pixel centre.
    Every class but `threshold` draws half its opacities from THRESHOLD_OPACITIES."""
    fx, fy = W / (2 * TAN), H / (2 * TAN)
    ppx = W / 2 if ppx is None else ppx
    ppy = H / 2 if ppy is None else ppy
    z = _logu(rng, z_range[0], z_range[1], n)
    u, v = rng.uniform(0, W, n), rng.uniform(0, H, n)
    op = _opacities(rng, n)
    foot = _logu(rng, 0.5, 30.0, n)                          # footprint in pixels
    aspect = _logu(rng, 0.3, 3.0, n)
    if cls == "offimage":
        side = rng.integers(0, 4, n)
        du, dv = rng.uniform(0, W, n), rng.uniform(0, H, n)
        u = np.where(side == 0, -du, np.where(side == 1, W + du, u))
        v = np.where(side == 2, -dv, np.where(side == 3, H + dv, v))
        dist = np.maximum(np.maximum(-u, u - W), np.maximum(-v, v - H)).clip(0)
        foot = (dist + rng.uniform(1, 8, n)) / 2.5
    elif cls == "threshold":
        u = rng.integers(0, W, n) + 0.5 + rng.uniform(-1e-4, 1e-4, n)
        v = rng.integers(0, H, n) + 0.5 + rng.uniform(-1e-4, 1e-4, n)
        op = rng.choice(THRESHOLD_OPACITIES, n)
        foot = _logu(rng, 0.3, 5.0, n)
    means = np.stack([(u - ppx) * z / fx, (v - ppy) * z / fy, z], 1)
    d = _unit(means)
    if cls == "grazing":
        e = _unit(np.cross(d, rng.normal(size=(n, 3))))
        eps = _logu(rng, 1e-7, 1e-1, n) * rng.choice([-1.0, 1.0], n)
        R = _frame_with_normal(rng, np.cos(eps)[:, None] * e + np.sin(eps)[:, None] * d)
    else:
        R = _frame_with_normal(rng, _unit(rng.normal(size=(n, 3))))
    s = foot * z / fx
    scales = np.stack([s * aspect, s / aspect], 1)
    if cls == "subpixel":
        scales = np.stack([_logu(rng, 1e-4, 1.0, n), _logu(rng, 1e-4, 1.0, n)], 1)
    elif cls == "dc_zero":
        # Dc = c2 ((s1 t1z)^2 + (s2 t2z)^2) - z^2 with the kernel's inflated c2: scale both axes to put it at eta z^2
        c2 = 2 * np.log(255 * op.astype(np.float64)) * 1.004 + 1e-3
        a0 = (aspect * R[:, 2, 0]) ** 2 + (R[:, 2, 1] / aspect) ** 2
        eta = _logu(rng, 1e-7, 1e-1, n) * rng.choice([-1.0, 1.0], n)
        s = z * np.sqrt((1 + eta) / (c2 * a0))
        scales = np.stack([s * aspect, s / aspect], 1)
    return dict(means=means.astype(F32), scales=scales.astype(F32), rotations=_quat(R).astype(F32), opacities=op)
