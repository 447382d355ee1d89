"""Every output element of the fused Stage-3 loss kernel (csrc/loss.cu, sr_render_loss_batch) and of the post-processing
kernels (csrc/postprocess.cu, sr_post_forward / sr_post_backward) against the float64 oracle (oracle/post_oracle.py), on
the same constructed fp32 inputs with no rasterizer in the loop, under an a-priori rounding-error bound.

The shapes are chosen for the kernels' 32 x 8 blocks: partial last blocks in x and in y, 1-column last blocks (W = 32k + 1),
odd W and H (cx = W / 2 a half-integer), images with no interior stencil (W or H < 3).  The content is a smooth depth
surface with planted degenerate pixels, each on a block seam and on the image border: alpha = 0 with depth 0 and with
depth > 0 (0/0 and d/0 under nan_to_num), NaN and +inf median depth, a stencil whose vertical difference is exactly zero
(the 1e12 branch of F.normalize's VJP), colour exactly equal to its target, vis2d of 0, -1 and 1e-30.  -inf in the median
plane is left out on purpose: nan_to_num turns it into -FLT_MAX, which overflows in the fp32 stencil while the float64
oracle stays finite; both sides follow torch, so the two legitimately differ there.

Bound.  |gpu - oracle| <= K u B + FLOOR with u = 2^-24, where B is a first-order running error bound of the kernel's own
expression: _E evaluates it in float64 on the same fp32 inputs and carries, per element, a bound on the absolute error of
the fp32 evaluation (each operation adds |a| err(b) + |b| err(a) for a product, err(a) / |b| + |a/b| err(b) / |b| for a
quotient, and so on, plus one rounding of its result unless that result is exact in fp32).  The loss terms and dL/dbkgd
add  (5 + 8 + blocks) u sum |t|  for the warp-shuffle, block and atomic sums.  K = 2 covers the terms of second order the
first-order bound leaves out; the oracle's own float64 error is far below it.  FLOOR is the smallest normal float: where
B is 0 every operation is exact on both sides.  The model's values must equal the oracle's far inside the bound, so the
bound is evaluated on the expression that is compared.

Knife elements are masked, counted and asserted to stay rare:
  * rgb: |colour + (1 - alpha) bk - target| within its rounding bound, so the sign may differ: there dL/dcolor must be
    one of -s, 0, +s, and the oracle's dL/dalpha and dL/dbkgd are re-evaluated at the GPU's sign;
  * stencil: the rounding bound of |n| = |dx x dy| is more than 1/64 of |n|, where normalising makes a first-order bound
    meaningless: that pixel's normal planes and its four neighbours' depth planes are not compared.  An exactly zero n is
    exact on both sides and is compared.
"""
import numpy as np
import pytest
import torch

from .error_bound import _E, _where
from .feature_loss_bounds import CONFIGS as FEATURE_CONFIGS

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
K = 2.0
FLOOR = float(np.finfo(np.float32).tiny)
KNIFE_REL = 2.0 ** -6
TANX, TANY = 0.5, 0.35
NAN = float("nan")


@pytest.fixture(scope="module")
def dev(built):
    from vidu4d_b200 import _capi
    _capi.load()
    return torch.device("cuda:0")


def _full(inner, H, W):
    """A stencil quantity on the interior [1:-1, 1:-1] embedded in exact zeros."""
    v, b = np.zeros((H, W)), np.zeros((H, W))
    if H >= 3 and W >= 3:
        v[1:-1, 1:-1], b[1:-1, 1:-1] = np.broadcast_to(inner.v, (H - 2, W - 2)), np.broadcast_to(inner.b, (H - 2, W - 2))
    return _E(v, b)


def _cam(wvt, W, H, tanx, tany, ox=0.0, oy=0.0):
    """post_common.cuh load_cam: R, the adjugate inverse A, fx, fy, cx = W * 0.5f + ox, cy = H * 0.5f + oy (tanx, tany,
    ox, oy: the fp32 values of a per-frame camera row, or the shared tangents with no offset)."""
    m = [_E(float(x)) for x in np.asarray(wvt, np.float32).reshape(16)]
    R = [m[i * 4 + j] for i in range(3) for j in range(3)]
    B = [m[j * 4 + i] for i in range(3) for j in range(3)]
    c0 = (B[4] * B[8] - B[5] * B[7], B[5] * B[6] - B[3] * B[8], B[3] * B[7] - B[4] * B[6])
    c1 = (B[7] * B[2] - B[8] * B[1], B[8] * B[0] - B[6] * B[2], B[6] * B[1] - B[7] * B[0])
    c2 = (B[1] * B[5] - B[2] * B[4], B[2] * B[3] - B[0] * B[5], B[0] * B[4] - B[1] * B[3])
    inv = _E(1.0) / (B[0] * c0[0] + B[1] * c0[1] + B[2] * c0[2])
    A = [c[k] * inv for k in range(3) for c in (c0, c1, c2)]
    fx = _E(float(W)) / _E(2.0 * float(np.float32(tanx)))
    fy = _E(float(H)) / _E(2.0 * float(np.float32(tany)))
    cx = _E(W * 0.5) + _E(float(np.float32(ox)))
    cy = _E(H * 0.5) + _E(float(np.float32(oy)))
    return dict(R=R, A=A, fx=fx, fy=fy, cx=cx, cy=cy)


def _ray(c, X, Y):
    """ray_dir: A (u, v, 1) with u = (x - cx) / fx, v = (y - cy) / fy; X and Y broadcast."""
    u = (_E(np.asarray(X, np.float64)) - c["cx"]) / c["fx"]
    v = (_E(np.asarray(Y, np.float64)) - c["cy"]) / c["fy"]
    A = c["A"]
    return [A[3 * k] * u + A[3 * k + 1] * v + A[3 * k + 2] for k in range(3)]


def _dot3(M, idx, x):
    return M[idx[0]] * x[0] + M[idx[1]] * x[1] + M[idx[2]] * x[2]


def _surf_depth(am, r):
    """loss_depth_kernel / post_fwd_kernel: surf_depth, the expected-depth quotient's finiteness, the median's."""
    with np.errstate(divide="ignore", invalid="ignore"):
        qfin = np.isfinite(am[0] / am[1])
    a, d0 = _E(am[1]), _E(am[0])
    ex = _where(qfin, d0 / _where(qfin, a, 1.0), 0.0)
    mfin = np.isfinite(am[5])
    med = _E(np.where(mfin, am[5], 0.0))
    sd = ex * (_E(1.0) - r) + r * med
    return sd, ex, med, qfin, mfin


def _stencils(c, sd, H, W):
    """The depth_to_normal stencils centred on the interior: dx, dy, n = dx x dy, |n|."""
    X, Y = np.arange(1, W - 1)[None], np.arange(1, H - 1)[:, None]
    ra, rb, re, rf = _ray(c, X, Y + 1), _ray(c, X, Y - 1), _ray(c, X + 1, Y), _ray(c, X - 1, Y)
    dD, dU, dR, dL = sd[2:, 1:-1], sd[:-2, 1:-1], sd[1:-1, 2:], sd[1:-1, :-2]
    dx = [dD * ra[k] - dU * rb[k] for k in range(3)]
    dy = [dR * re[k] - dL * rf[k] for k in range(3)]
    n = [dx[1] * dy[2] - dx[2] * dy[1], dx[2] * dy[0] - dx[0] * dy[2], dx[0] * dy[1] - dx[1] * dy[0]]
    ln = (n[0] * n[0] + n[1] * n[1] + n[2] * n[2]).sqrt()
    return dict(dx=dx, dy=dy, n=n, ln=ln)


def _stencil_vjp(st, g):
    """d normalize(n) / d (dx, dy) applied to g (both branches of F.normalize's VJP), as the kernels write it."""
    n, ln, dx, dy = st["n"], st["ln"], st["dx"], st["dy"]
    big = ln.v > 1e-12
    inv = _E(1.0) / _where(big, ln, 1.0)
    w = [n[k] * inv for k in range(3)]
    d = w[0] * g[0] + w[1] * g[1] + w[2] * g[2]
    eps = _E.const(1e12)
    gn = [_where(big, (g[k] - w[k] * d) * inv, g[k] * eps) for k in range(3)]
    gdx = [dy[1] * gn[2] - dy[2] * gn[1], dy[2] * gn[0] - dy[0] * gn[2], dy[0] * gn[1] - dy[1] * gn[0]]
    gdy = [gn[1] * dx[2] - gn[2] * dx[1], gn[2] * dx[0] - gn[0] * dx[2], gn[0] * dx[1] - gn[1] * dx[0]]
    return gdx, gdy


def _gather(gdx, gdy, H, W):
    """The depth gradient each pixel collects from the four stencils it takes part in: (+above - below) + left - right."""
    out = []
    for k in range(3):
        fx_, fy_ = _full(gdx[k], H, W), _full(gdy[k], H, W)
        z = _E(np.zeros((H, W)))

        def sh(e, dy_, dx_):
            v, b = np.zeros((H, W)), np.zeros((H, W))
            ys, yd = (slice(0, H - dy_), slice(dy_, H)) if dy_ >= 0 else (slice(-dy_, H), slice(0, H + dy_))
            xs, xd = (slice(0, W - dx_), slice(dx_, W)) if dx_ >= 0 else (slice(-dx_, W), slice(0, W + dx_))
            v[yd, xd], b[yd, xd] = e.v[ys, xs], e.b[ys, xs]
            return _E(v, b)
        out.append((((z + sh(fx_, 1, 0)) - sh(fx_, -1, 0)) + sh(fy_, 0, 1)) - sh(fy_, 0, -1))
    return out


def _stencil_knife(st, H, W):
    """(stencil knife mask on the interior embedded in the image, mask of the pixels whose depth gradient gathers one)."""
    ln = st["ln"]
    inner = ((ln.v > 0) & (U * ln.b > KNIFE_REL * ln.v)) | (np.abs(ln.v - 1e-12) <= K * U * ln.b)
    own = np.zeros((H, W), bool)
    if H >= 3 and W >= 3:
        own[1:-1, 1:-1] = inner
    nb = np.zeros((H, W), bool)
    nb[1:] |= own[:-1]
    nb[:-1] |= own[1:]
    nb[:, 1:] |= own[:, :-1]
    nb[:, :-1] |= own[:, 1:]
    return own, nb


def _loss_model(color, am, wvt, target, o, vis, mask, wt, bk, cam=(TANX, TANY, 0.0, 0.0)):
    """loss_grad_kernel's expressions for one frame as _E values: dL/dcolor, dL/dallmap planes 0..6, the per-pixel loss
    terms and dL/dbkgd parts, the rgb knife mask and the stencil knife masks.  cam: the frame's (tanx, tany, ox, oy)."""
    _, H, W = color.shape
    c = _cam(wvt, W, H, *cam)
    r = _E(float(np.float32(o["depth_ratio"])))
    invN = _E(1.0) / _E(float(H * W))
    sN = _E(float(np.float32(o["lambda_normal"]))) * invN
    a = _E(am[1])
    sd, _, _, qfin, mfin = _surf_depth(am, r)
    vv = np.ones((H, W)) if vis is None else (vis > 0).astype(np.float64)
    s_rgb = (_E(float(np.float32(o["w_rgb"]))) * invN) * _E.const(1.0 / 3.0)
    part = [_E(np.zeros((H, W))) for _ in range(7)]
    g_acc = _E(np.zeros((H, W)))
    gcol, rgb_knife = [], np.zeros((H, W), bool)
    for ch in range(3):
        bkc = _E(0.0 if bk is None else float(bk[ch]))
        col = _E(color[ch]) + (_E(1.0) - a) * bkc
        d = col - _E(target[ch])
        part[0] = part[0] + (d.abs() * _E(vv)) * s_rgb
        rgb_knife |= (np.abs(d.v) <= K * U * d.b) & (d.b > 0)
        gc = _E(np.sign(d.v) * vv) * s_rgb
        gcol.append(gc)
        part[4 + ch] = gc * (_E(1.0) - a)
        g_acc = g_acc - gc * bkc
    if mask is not None:
        w_e = _E(np.ones((H, W))) if wt is None else _E(wt)
        wm = _E(float(np.float32(o["w_mask"])))
        dm = a - _E(mask)
        part[1] = (((wm * dm) * dm) * w_e) * invN
        g_acc = g_acc + ((((wm * _E(2.0)) * dm) * w_e) * invN)
    n = [_E(am[2 + k]) for k in range(3)]
    R = c["R"]
    rn = [_dot3(R, (3 * k, 3 * k + 1, 3 * k + 2), n) for k in range(3)]
    sn = [_E(np.zeros((H, W)))] * 3
    gp = [_E(np.zeros((H, W)))] * 3
    own = nb = np.zeros((H, W), bool)
    if o["lambda_normal"] != 0 and H >= 3 and W >= 3:
        st = _stencils(c, sd, H, W)
        ai = a[1:-1, 1:-1]
        inv_s = ai / _where(st["ln"].v > 1e-12, st["ln"], _E.const(1e-12))
        sn = [_full(st["n"][k] * inv_s, H, W) for k in range(3)]
        ri = [_E(am[2 + k][1:-1, 1:-1]) for k in range(3)]
        sa = (-sN) * ai
        g = [sa * _dot3(R, (3 * k, 3 * k + 1, 3 * k + 2), ri) for k in range(3)]
        gp = _gather(*_stencil_vjp(st, g), H, W)
        own, nb = _stencil_knife(st, H, W)
    part[2] = sN * (_E(1.0) - _dot3(rn, (0, 1, 2), sn))
    if own.any():            # a knife stencil's unit normal may point anywhere: its term can move by 2 sN alpha |rn|
        rmag = np.sqrt(sum(x.v ** 2 for x in rn))
        part[2] = _E(part[2].v, part[2].b + np.where(own, 2.0 * sN.v * am[1] * rmag / U, 0.0))
    q = [(-sN) * sn[k] for k in range(3)]
    planes = {}
    for k in range(3):
        planes[2 + k] = _dot3(R, (k, 3 + k, 6 + k), q)
    ray = _ray(c, np.arange(W)[None], np.arange(H)[:, None])
    gsd = _dot3(gp, (0, 1, 2), ray)
    gex, gmed = gsd * (_E(1.0) - r), gsd * r
    planes[0] = _where(qfin, gex / a, 0.0)
    planes[1] = g_acc + _where(qfin, ((-gex) * _E(am[0])) / (a * a), 0.0)
    planes[5] = _where(mfin, gmed, 0.0)
    part[3] = (_E(float(np.float32(o["lambda_dist"]))) * _E(am[6])) * invN
    return dict(gcol=gcol, planes=planes, part=part, rgb_knife=rgb_knife, st_own=own, st_nb=nb)


def _post_model(am, wvt, r, wts):
    """post_fwd / post_normal / post_bwd kernels for one frame as _E values."""
    _, H, W = am.shape
    c = _cam(wvt, W, H, TANX, TANY)
    r = _E(float(np.float32(r)))
    a = _E(am[1])
    sd, ex, med, qfin, mfin = _surf_depth(am, r)
    R = c["R"]
    n = [_E(am[2 + k]) for k in range(3)]
    fw = {"acc": [a], "rend_normal": [_dot3(R, (3 * k, 3 * k + 1, 3 * k + 2), n) for k in range(3)],
          "rend_dist": [_E(am[6])], "render_depth_median": [med], "render_depth_expected": [ex], "surf_depth": [sd]}
    sn = [_E(np.zeros((H, W)))] * 3
    gp = [_E(np.zeros((H, W)))] * 3
    own = nb = np.zeros((H, W), bool)
    if H >= 3 and W >= 3:
        st = _stencils(c, sd, H, W)
        ai = a[1:-1, 1:-1]
        inv = _E(1.0) / _where(st["ln"].v > 1e-12, st["ln"], _E.const(1e-12))
        sn = [_full((st["n"][k] * inv) * ai, H, W) for k in range(3)]
        g = [_E(wts["surf_normal"][k][1:-1, 1:-1]) * ai for k in range(3)]
        gp = _gather(*_stencil_vjp(st, g), H, W)
        own, nb = _stencil_knife(st, H, W)
    fw["surf_normal"] = sn
    ray = _ray(c, np.arange(W)[None], np.arange(H)[:, None])
    gsd = ((_E(wts["surf_depth"][0]) + gp[0] * ray[0]) + gp[1] * ray[1]) + gp[2] * ray[2]
    gex = _E(wts["render_depth_expected"][0]) + gsd * (_E(1.0) - r)
    gmed = _E(wts["render_depth_median"][0]) + gsd * r
    g = [None] * 8
    g[0] = _where(qfin, gex / a, 0.0)
    g[1] = _E(wts["acc"][0]) + _where(qfin, ((-gex) * _E(am[0])) / (a * a), 0.0)
    grn = [_E(wts["rend_normal"][k]) for k in range(3)]
    for k in range(3):
        g[2 + k] = _dot3(R, (k, 3 + k, 6 + k), grn)
    g[5] = _where(mfin, gmed, 0.0)
    g[6] = _E(wts["rend_dist"][0])
    g[7] = _E(np.zeros((H, W)))
    return fw, g, own, nb


# ------------------------------------------------------------------------------------------------ inputs
KINDS = ("alpha0_depth0", "alpha0_depth_pos", "median_nan", "median_inf", "zero_dx", "rgb_equal", "vis_zero",
         "vis_negative", "vis_tiny")


def _wvts(M, seed):
    """M world_view_transforms (W2C transposed) that differ in rotation and translation, as one (M,2,4,4) upload holding
    view and projection matrices (bench.py's layout); returns the strided (M,4,4) view of the view matrices."""
    rng = np.random.default_rng(seed)
    out = np.zeros((M, 2, 4, 4), np.float32)
    for f in range(M):
        ang = 0.15 * (f + 1) + rng.uniform(-0.05, 0.05, 3)
        cx_, sx_ = np.cos(ang), np.sin(ang)
        Rx = np.array([[1, 0, 0], [0, cx_[0], -sx_[0]], [0, sx_[0], cx_[0]]])
        Ry = np.array([[cx_[1], 0, sx_[1]], [0, 1, 0], [-sx_[1], 0, cx_[1]]])
        Rz = np.array([[cx_[2], -sx_[2], 0], [sx_[2], cx_[2], 0], [0, 0, 1]])
        W2C = np.eye(4)
        W2C[:3, :3] = Rz @ Ry @ Rx
        W2C[:3, 3] = rng.uniform(-0.3, 0.3, 3) + [0, 0, 2.5]
        out[f, 0] = W2C.T
        out[f, 1] = rng.normal(size=(4, 4))
    return torch.from_numpy(out)[:, 0]


def _is_seam(y, x, W, H):
    """Inside the image, next to a block boundary: the first or last column of a 32-wide block, row of an 8-high one."""
    return (np.isin(x % 32, (0, 31)) & (0 < x) & (x < W - 1)) | (np.isin(y % 8, (0, 7)) & (0 < y) & (y < H - 1))


def _is_border(y, x, W, H):
    return (x == 0) | (x == W - 1) | (y == 0) | (y == H - 1)


def _frames(M, W, H, seed, with_vis, with_bk):
    """Smooth random depth surfaces, alpha in (0, 1], random normals, colours and targets, with the degenerate pixels
    planted; returns the arrays and the planted list [(kind, frame, y, x, site)] (site: "seam" or "border")."""
    rng = np.random.default_rng(seed)
    ys, xs = np.mgrid[0:H, 0:W].astype(np.float64)
    am = np.zeros((M, 8, H, W))
    for f in range(M):
        k = rng.uniform(0.05, 0.2, 4)
        depth = 2.0 + 0.4 * np.sin(k[0] * xs + k[1] * ys + f) + 0.2 * np.cos(k[2] * xs - k[3] * ys)
        alpha = rng.uniform(0.05, 1.0, (H, W))
        am[f, 1] = alpha
        am[f, 0] = alpha * depth
        am[f, 5] = depth + rng.normal(0, 0.02, (H, W))
        am[f, 2:5] = rng.normal(0, 1, (3, H, W))
        am[f, 6] = rng.uniform(0, 0.1, (H, W))
        am[f, 7] = rng.uniform(0, 1, (H, W))
    color = rng.uniform(0, 1, (M, 3, H, W))
    target = rng.uniform(0, 1, (M, 3, H, W))
    vis = (rng.uniform(size=(M, H, W)) > 0.15) * rng.uniform(0.5, 2.0, (M, H, W))
    am, color, target, vis = (x.astype(np.float32) for x in (am, color, target, vis))
    used = np.zeros((M, H, W), bool)
    planted = []

    def free(f, pix):
        return all(0 <= y < H and 0 <= x < W and not used[f, max(0, y - 1):y + 2, max(0, x - 1):x + 2].any()
                   for y, x in pix)

    iy, ix = np.mgrid[0:H, 0:W]

    def sites(kind, site):
        if kind == "zero_dx":        # the stencil centre: its up / down neighbours across a seam row or on the border row
            inner = (iy >= 1) & (iy <= H - 2) & (ix >= 1) & (ix <= W - 2)
            ok = inner & ((iy % 8 == 0) if site == "seam" else ((iy == 1) | (iy == H - 2)))
        elif site == "seam":
            ok = _is_seam(iy, ix, W, H) & ~_is_border(iy, ix, W, H)
        else:
            ok = _is_border(iy, ix, W, H)
        return [tuple(int(v) for v in p) for p in np.argwhere(ok)]

    kinds = [k for k in KINDS if with_vis or not k.startswith("vis")]
    for i, kind in enumerate(kinds):
        for site in ("seam", "border"):
            f = (i + (site == "border")) % M
            cand = sites(kind, site)
            rng.shuffle(cand)
            for y, x in cand:
                pix = [(y, x)] + ([(y - 1, x), (y + 1, x)] if kind == "zero_dx" else [])
                if not free(f, pix):
                    continue
                for py, px in pix:
                    used[f, py, px] = True
                if kind == "alpha0_depth0":
                    am[f, 0, y, x] = am[f, 1, y, x] = 0.0
                elif kind == "alpha0_depth_pos":
                    am[f, 1, y, x] = 0.0
                elif kind == "median_nan":
                    am[f, 5, y, x] = np.nan
                elif kind == "median_inf":
                    am[f, 5, y, x] = np.inf
                elif kind == "zero_dx":
                    for py in (y - 1, y + 1):
                        am[f, 0, py, x] = am[f, 1, py, x] = am[f, 5, py, x] = 0.0
                elif kind == "rgb_equal":
                    target[f, :, y, x] = color[f, :, y, x]
                    if with_bk:
                        am[f, 1, y, x] = 1.0          # (1 - alpha) bk = 0 exactly: equal after the composite too
                else:
                    vis[f, y, x] = {"vis_zero": 0.0, "vis_negative": -1.0, "vis_tiny": np.float32(1e-30)}[kind]
                planted.append((kind, f, y, x, site))
                break
    return am, color, target, vis, planted


# option combinations: the bench.py call, everything on with a learnable background, no normal term, a mask without
# weights; depth_ratio 0, 0.3 and 1 among them
OPTS = {
    "bench": dict(vis=False, mask=False, wt=False, bk=False, w_rgb=1.0, w_mask=0.0, lambda_normal=0.05, lambda_dist=0.01,
                  depth_ratio=0.0),
    "all_bkgd": dict(vis=True, mask=True, wt=True, bk=True, w_rgb=0.8, w_mask=0.1, lambda_normal=0.05, lambda_dist=100.0,
                     depth_ratio=0.3),
    "no_normal": dict(vis=True, mask=True, wt=True, bk=False, w_rgb=0.8, w_mask=0.1, lambda_normal=0.0, lambda_dist=0.01,
                      depth_ratio=0.3),
    "mask_no_wt": dict(vis=True, mask=True, wt=False, bk=True, w_rgb=1.0, w_mask=0.5, lambda_normal=0.05, lambda_dist=0.01,
                       depth_ratio=1.0),
    # every term, each frame with its own camera row (sr_render_loss_batch_cameras)
    "cameras": dict(vis=True, mask=True, wt=True, bk=True, w_rgb=0.8, w_mask=0.1, lambda_normal=0.05, lambda_dist=100.0,
                    depth_ratio=0.3, table=True),
}


def camera_rows(M, W, H):
    """(M,4) fp32 per-frame (tan_x, tan_y, cx_off, cy_off): both tangents differ from frame to frame, the offsets are
    non-integer, alternate in sign and move the principal point (W/2 + ox, H/2 + oy) by about a third of the image --
    across a 32-column block seam from W = 97 up, across an 8-row seam from H = 17 up."""
    f = np.arange(M)
    sgn = np.where(f % 2, -1.0, 1.0)
    rows = np.stack([0.5 - 0.021 * f, 0.35 + 0.017 * f, sgn * (0.34 * W + 0.625 + 0.25 * f),
                     -sgn * (0.34 * H + 0.3125 + 0.125 * f)], 1)
    return rows.astype(np.float32)


# ------------------------------------------------------------------------------------------------ GPU calls
def _loss_gpu(M, W, H, o, color, am, wvt, target, vis, mask, wt, bk, dev, table=None):
    """sr_render_loss_batch with the shared TANX / TANY, or sr_render_loss_batch_cameras with the (M,4) device `table`."""
    from vidu4d_b200 import _capi
    lib = _capi.load()
    ptr = lambda t: None if t is None else t.data_ptr()  # noqa: E731
    terms = torch.full((M, 4), NAN, device=dev)
    dLc = torch.full((M, 3, H, W), NAN, device=dev)
    dLa = torch.full((M, 8, H, W), NAN, device=dev)
    dLb = torch.full((M, 3), NAN, device=dev) if bk is not None else None
    sd = torch.full((M, H, W), NAN, device=dev)
    rest = (o["depth_ratio"], color.data_ptr(), am.data_ptr(), wvt.data_ptr(), target.data_ptr(), ptr(vis), ptr(mask),
            ptr(wt), ptr(bk), o["w_rgb"], o["w_mask"], o["lambda_normal"], o["lambda_dist"], terms.data_ptr(),
            dLc.data_ptr(), dLa.data_ptr(), ptr(dLb), sd.data_ptr(), torch.cuda.current_stream(dev).cuda_stream)
    if table is None:
        fn = "sr_render_loss_batch"
        rc = lib.sr_render_loss_batch(M, W, H, TANX, TANY, *rest)
    else:
        fn = "sr_render_loss_batch_cameras"
        rc = lib.sr_render_loss_batch_cameras(M, W, H, table.data_ptr(), *rest)
    _capi.check(rc, fn)
    torch.cuda.synchronize(dev)
    return terms, dLc, dLa, dLb, sd


POST_KEYS = ("acc", "rend_normal", "rend_dist", "render_depth_median", "render_depth_expected", "surf_depth", "surf_normal")
POST_CH = (1, 3, 1, 1, 1, 1, 3)


def _post_gpu(am_f, wvt_f, r, wts, dev):
    from vidu4d_b200 import _capi
    lib = _capi.load()
    _, H, W = am_f.shape
    s = torch.cuda.current_stream(dev).cuda_stream
    outs = [torch.full((c, H, W), NAN, device=dev) for c in POST_CH]
    rc = lib.sr_post_forward(W, H, TANX, TANY, r, am_f.data_ptr(), wvt_f.data_ptr(), *[t.data_ptr() for t in outs], s)
    _capi.check(rc, "sr_post_forward")
    g = torch.full((8, H, W), NAN, device=dev)
    w = [torch.from_numpy(wts[k]).to(dev) for k in POST_KEYS]
    rc = lib.sr_post_backward(W, H, TANX, TANY, r, am_f.data_ptr(), wvt_f.data_ptr(), outs[5].data_ptr(),
                              *[t.data_ptr() for t in w], g.data_ptr(), s)
    _capi.check(rc, "sr_post_backward")
    torch.cuda.synchronize(dev)
    return dict(zip(POST_KEYS, (t.cpu().numpy() for t in outs))), g.cpu().numpy()


# ------------------------------------------------------------------------------------------------ checks
def _cmp(name, what, mine, ref, e, report, skip=None, model_check=True):
    """|mine - ref| <= K u B + FLOOR element by element outside `skip`; the model's value agrees with the oracle's far
    inside the bound.  Records the headroom (largest err / (K u B)) under report[what]."""
    mine = np.atleast_1d(np.asarray(mine, np.float64))
    ref = np.broadcast_to(np.asarray(ref, np.float64), mine.shape)
    tol = K * U * np.broadcast_to(e.b, mine.shape) + FLOOR
    ok = np.ones(mine.shape, bool) if skip is None else ~np.broadcast_to(skip, mine.shape)
    if model_check:
        dm = np.abs(np.broadcast_to(e.v, mine.shape) - ref)
        bad = ok & ~(dm <= 1e-3 * tol)
        assert not bad.any(), (name, what, "bound model != oracle", np.argwhere(bad)[:4].tolist())
    err = np.abs(mine - ref)
    ratio = np.where(ok, err / tol, 0.0)
    ratio = np.where(np.isnan(mine) & ok, np.inf, ratio)
    i = int(np.argmax(ratio))
    report[what] = max(report.get(what, 0.0), float(ratio.flat[i]))
    assert ratio.flat[i] <= 1.0, (name, what, "element", np.unravel_index(i, mine.shape), "gpu", mine.flat[i], "oracle",
                                  ref.flat[i], "bound", tol.flat[i])


def _reached(H, W):
    """Pixels whose depth gradient some interior stencil reaches."""
    own = np.zeros((H, W), bool)
    if H >= 3 and W >= 3:
        own[1:-1, 1:-1] = True
    nb = np.zeros((H, W), bool)
    nb[1:] |= own[:-1]
    nb[:-1] |= own[1:]
    nb[:, 1:] |= own[:, :-1]
    nb[:, :-1] |= own[:, 1:]
    return nb


def _run(name, M, W, H, opt, seed, dev, post=True):
    from oracle import post_oracle as po
    from . import camera_model as cm
    o = dict(OPTS[opt])
    am, color, target, vis, planted = _frames(M, W, H, seed, o["vis"], o["bk"])
    mask = (np.random.default_rng(seed + 1).uniform(size=(M, H, W)) > 0.5).astype(np.float32) if o["mask"] else None
    wt = np.random.default_rng(seed + 2).uniform(0.5, 2.0, (M, H, W)).astype(np.float32) if o["wt"] else None
    bk = np.array([0.3, 0.5, 0.2], np.float32) if o["bk"] else None
    visn = vis if o["vis"] else None
    wview = _wvts(M, seed)
    assert not wview.is_contiguous() or M == 1
    wvt_np = wview.numpy().copy()
    T = lambda x: None if x is None else torch.from_numpy(np.ascontiguousarray(x)).to(dev)  # noqa: E731
    args = (T(color), T(am), wview.contiguous().to(dev), T(target), T(visn), T(mask), T(wt), T(bk))
    rows = camera_rows(M, W, H) if o.get("table") else None
    terms, dLc, dLa, dLb, sd = _loss_gpu(M, W, H, o, *args, dev, table=T(rows))
    # no atomics on image data: bit for bit the same planes on a second call
    _, dLc2, dLa2, _, _ = _loss_gpu(M, W, H, o, *args, dev, table=T(rows))
    assert torch.equal(dLc, dLc2) and torch.equal(dLa, dLa2), name
    terms, dLc, dLa, sd = terms.cpu().numpy(), dLc.cpu().numpy(), dLa.cpu().numpy(), sd.cpu().numpy()
    dLb = None if dLb is None else dLb.cpu().numpy()
    nblocks = ((W + 31) // 32) * ((H + 7) // 8)
    depth = 5 + 8 + nblocks
    report, knives = {}, {"rgb": 0, "stencil": 0}
    reached = _reached(H, W) if o["lambda_normal"] != 0 else np.zeros((H, W), bool)
    inv_n = np.float32(1.0) / np.float32(H * W)
    for f in range(M):
        tag = f"{name} frame {f}"
        mg = np.zeros((H, W), np.float32) if mask is None else mask[f]
        mw = np.ones((H, W), np.float32) if wt is None else wt[f]
        vf = np.ones((H, W), np.float32) if visn is None else visn[f]
        okw = dict(w_rgb=float(np.float32(o["w_rgb"])), w_mask=float(np.float32(o["w_mask"])) if mask is not None else 0.0,
                   lambda_normal=float(np.float32(o["lambda_normal"])), lambda_dist=float(np.float32(o["lambda_dist"])),
                   bkgd=bk)
        cam = (TANX, TANY, 0.0, 0.0) if rows is None else tuple(float(x) for x in rows[f])
        oargs = (color[f], am[f], wvt_np[f], float(np.float32(cam[0])), float(np.float32(cam[1])),
                 float(np.float32(o["depth_ratio"])), target[f], vf, mg, mw)
        if rows is None:
            _, ot = po.stage3_losses(*oargs, **okw)
            gr = po.stage3_losses_backward(*oargs, **okw)
        else:                   # the centred oracle with the ray grid's principal point moved (tests/camera_model.py)
            _, ot = cm.stage3_losses(cam[2], cam[3], *oargs, **okw)
            gr = cm.stage3_losses_backward(cam[2], cam[3], *oargs, **okw)
        gcol, gall = gr[0], gr[1].copy()
        mdl = _loss_model(color[f], am[f], wvt_np[f], target[f], o, visn[f] if visn is not None else None,
                          None if mask is None else mask[f], None if wt is None else wt[f], bk, cam=cam)
        # rgb knife pixels: the GPU's sign must be one of the three; the oracle is re-evaluated at it
        kn = mdl["rgb_knife"]
        knives["rgb"] += int(kn.sum())
        s32 = (np.float32(o["w_rgb"]) * inv_n) * (np.float32(1.0) / np.float32(3.0))
        if kn.any():
            assert np.isin(dLc[f][:, kn], np.array([-s32, 0, s32], np.float32)).all(), (tag, "rgb knife: not -s, 0 or s")
            delta = np.where(kn[None], dLc[f].astype(np.float64) - gcol, 0.0)
            gcol = gcol + delta
            if bk is not None:
                gall[1] -= (delta * bk[:, None, None].astype(np.float64)).sum(0)
                gr = gr[:2] + (gr[2] + (delta * (1.0 - am[f, 1].astype(np.float64))).sum((1, 2)),)
        for ch in range(3):
            _cmp(tag, "dL_dcolor", dLc[f, ch], gcol[ch], mdl["gcol"][ch], report, skip=kn, model_check=True)
        # stencil knives: the pixel's normal planes and its neighbours' depth planes
        own, nbk = mdl["st_own"], mdl["st_nb"]
        knives["stencil"] += int(own.sum())
        for p in (0, 1, 5):
            _cmp(tag, f"dL_dallmap[{p}]", dLa[f, p], gall[p], mdl["planes"][p], report, skip=nbk | (kn & (p == 1)))
        for p in (2, 3, 4):
            _cmp(tag, f"dL_dallmap[{p}]", dLa[f, p], gall[p], mdl["planes"][p], report, skip=own)
        if kn.any():            # plane 1 at rgb knives against the re-evaluated oracle; the bound adds the sign's terms
            e1 = mdl["planes"][1][kn]
            extra = 0.0 if bk is None else 4.0 * float(s32) * float(np.abs(bk).sum())
            _cmp(tag, "dL_dallmap[1]", dLa[f, 1][kn], gall[1][kn], _E(e1.v, e1.b + extra), report, model_check=False)
        # plane 6: the fp32 product lambda_dist * (1/N) bit for bit; plane 7: exactly 0
        assert (dLa[f, 6] == np.float32(o["lambda_dist"]) * inv_n).all(), tag
        assert (dLa[f, 7] == 0).all(), tag
        # pixels no stencil reaches: exactly zero stencil gradient
        assert (dLa[f, 0][~reached] == 0).all() and (dLa[f, 5][~reached] == 0).all(), tag
        for k, key in enumerate(("rgb", "mask", "normal", "dist")):
            t = mdl["part"][k]
            e = _E(t.v.sum(), t.b.sum() + depth * np.abs(t.v).sum())
            _cmp(tag, "loss_terms", terms[f, k], ot[key], e, report, model_check=False)
        if bk is not None:
            for ch in range(3):
                t = mdl["part"][4 + ch]
                t_v = np.where(kn, gcol[ch] * (1.0 - am[f, 1].astype(np.float64)), t.v)
                e = _E(t_v.sum(), t.b.sum() + 2.0 * np.abs(t_v[kn]).sum() + depth * np.abs(t_v).sum())
                _cmp(tag, "dL_dbkgd", dLb[f, ch], gr[2][ch], e, report, model_check=False)
        if post:
            rng = np.random.default_rng(seed + 10 + f)
            wts = {k: rng.normal(size=(c, H, W)).astype(np.float32) for k, c in zip(POST_KEYS, POST_CH)}
            pf, pg = _post_gpu(T(am[f]), T(wvt_np[f]), float(o["depth_ratio"]), wts, dev)
            # the loss kernel's surf_depth is the same expression as the post kernel's, bit for bit
            assert np.array_equal(sd[f], pf["surf_depth"][0], equal_nan=True), tag
            fw = po.post_forward(am[f], wvt_np[f], float(np.float32(TANX)), float(np.float32(TANY)),
                                 float(np.float32(o["depth_ratio"])))
            mfw, mg_, pown, pnb = _post_model(am[f], wvt_np[f], o["depth_ratio"], wts)
            knives["stencil"] += int(pown.sum())
            for k in POST_KEYS:
                for ch in range(pf[k].shape[0]):
                    _cmp(tag + " post", k, pf[k][ch], fw[k][ch], mfw[k][ch], report,
                         skip=pown if k == "surf_normal" else None)
            ga = po.post_backward(am[f], wvt_np[f], float(np.float32(TANX)), float(np.float32(TANY)),
                                  float(np.float32(o["depth_ratio"])), {k: wts[k] for k in POST_KEYS})
            for p in range(8):
                _cmp(tag + " post", f"g_allmap[{p}]", pg[p], ga[p], mg_[p], report, skip=pnb if p in (0, 1, 5) else None)
            assert (pg[7] == 0).all() and np.array_equal(pg[6], wts["rend_dist"][0]), tag
            if not (H >= 3 and W >= 3):
                assert (pf["surf_normal"] == 0).all(), tag
    print(f"\n[{name}] {opt} M={M} {W}x{H}: knife rgb {knives['rgb']} stencil {knives['stencil']} of {M * W * H} px; "
          + ", ".join(f"{k} {v:.3g}" for k, v in report.items()))
    # knife elements stay rare: a mask that grew by mistake could otherwise hide a broken block seam
    assert knives["rgb"] + knives["stencil"] <= 8 + 1e-4 * M * W * H, (name, knives)
    return dict(am=am, planted=planted, dLa=dLa, o=o, report=report)


def _check_reach(name, W, H, planted, o, dLa):
    """The planted pixels sit where they were meant to, and the 1e12 branch's gradient reaches the median plane."""
    kinds = {k for k in KINDS if o["vis"] or not k.startswith("vis")}
    for kind, f, y, x, site in planted:
        if kind == "zero_dx":
            assert 1 <= y <= H - 2 and 1 <= x <= W - 2, (name, kind)
            assert (site == "seam" and y % 8 == 0) or (site == "border" and y in (1, H - 2)), (name, kind, y)
        else:
            assert (_is_seam(y, x, W, H) if site == "seam" else _is_border(y, x, W, H)), (name, kind, site, y, x)
    if W >= 34 and H >= 10:        # room for every kind on a seam and on the border
        for site in ("seam", "border"):
            assert {p[0] for p in planted if p[4] == site} == kinds, (name, site)
    if o["lambda_normal"] != 0 and o["depth_ratio"] > 0:
        for kind, f, y, x, site in planted:
            if kind == "zero_dx":
                big = np.abs(dLa[f, 5, [y - 1, y + 1], x]).min()
                typical = np.median(np.abs(dLa[f, 5]))
                assert big > 1e3 * typical, (name, "the 1e12 branch did not reach the neighbours' median plane", big, typical)


W_GRID = (1, 2, 3, 31, 32, 33, 63, 65, 97)
H_GRID = (1, 2, 3, 7, 8, 9, 17)
BASE_OPTS = ("bench", "all_bkgd", "no_normal", "mask_no_wt")
GRID = [(W, H, 1 + 2 * ((i + j) % 2), BASE_OPTS[(i + 2 * j) % len(BASE_OPTS)])
        for i, W in enumerate(W_GRID) for j, H in enumerate(H_GRID)]
# the per-frame camera table on the same edges: no interior stencil, 1-column and partial last blocks, odd sizes
GRID += [(W, H, M, "cameras") for W, H, M in ((1, 8, 3), (2, 3, 1), (3, 3, 1), (31, 9, 3), (32, 2, 1), (33, 17, 1),
                                              (63, 7, 3), (65, 9, 1), (97, 17, 3))]


def test_grid_reaches_every_tile_edge():
    """The grid holds partial last blocks in x and y, 1-column last blocks, images with no interior stencil, odd sizes,
    and every option combination with a stencil-bearing image at a partial block."""
    assert any(W % 32 and W > 32 for W, _, _, _ in GRID) and any(H % 8 and H > 8 for _, H, _, _ in GRID)
    assert any(W % 32 == 1 and W > 32 for W, _, _, _ in GRID)
    assert any(W < 3 or H < 3 for W, H, _, _ in GRID) and any(W % 2 and H % 2 for W, H, _, _ in GRID)
    for opt in OPTS:
        assert any(o == opt and W > 32 and W % 32 and H > 8 and H % 8 for W, H, _, o in GRID), opt
        assert {M for W, H, M, o in GRID if o == opt} == {1, 3}, opt
    # the camera rows: both tangents differ between frames, non-integer offsets of either sign that carry the principal
    # point across a block seam in x and in y
    cams = [(W, H, M) for W, H, M, o in GRID if o == "cameras"]
    r = camera_rows(3, 97, 17)
    assert len(set(r[:, 0])) == 3 and len(set(r[:, 1])) == 3
    assert (r[:, 2:] != np.round(r[:, 2:])).all() and (r[:, 2] > 0).any() and (r[:, 2] < 0).any()
    x_cross = y_cross = False
    for W, H, M in cams:
        r = camera_rows(M, W, H)
        x_cross |= bool((np.floor(W / 2 / 32) != np.floor((W / 2 + r[:, 2]) / 32)).any() and W > 64)
        y_cross |= bool((np.floor(H / 2 / 8) != np.floor((H / 2 + r[:, 3]) / 8)).any() and H > 16)
    assert x_cross and y_cross


@pytest.mark.parametrize("W,H,M,opt", GRID)
def test_loss_and_post_kernels_elementwise(W, H, M, opt, dev):
    name = f"{W}x{H}"
    r = _run(name, M, W, H, opt, seed=W * 1000 + H, dev=dev)
    _check_reach(name, W, H, r["planted"], r["o"], r["dLa"])


@pytest.mark.parametrize("W,H,M,opt", [(1001, 563, 2, "all_bkgd"), (512, 512, 8, "bench"), (512, 512, 8, "cameras")])
def test_loss_kernel_large_reductions(W, H, M, opt, dev):
    """Thousands of blocks per frame: the loss terms' 7 fp32 atomics per block, against a bound that counts them."""
    name = f"{W}x{H}"
    r = _run(name, M, W, H, opt, seed=W + H, dev=dev, post=False)
    _check_reach(name, W, H, r["planted"], r["o"], r["dLa"])


# ------------------------------------------------------------------------------------------------ feature losses
@pytest.mark.parametrize("W", [1, 33, 97])
@pytest.mark.parametrize("H", [1, 9])
@pytest.mark.parametrize("M", [1, 3])
def test_feature_loss_kernel_at_tile_edges(W, H, M, dev):
    """sr_feature_loss_batch on the same 32 x 8 grid's edges against its restatement (tests/feature_loss_bounds.py):
    exact counts, every plane element and per-frame term under the rounding-error bound, untouched channels exactly 0,
    bitwise-deterministic planes."""
    from . import feature_loss_bounds as fb
    from .feature_loss_model import feature_losses
    from .test_gpu_feature_loss import _call, _inputs
    F, Cf, gm = 22, 16, 21
    feat, target, mask, det, allmap = _inputs(M, W, H, F, Cf, gm, dev, seed=W * 10 + H + M)
    w = torch.tensor([1e-2, 7e-3], device=dev)
    terms, counts, grad = _call(feat, target, mask, det, allmap, gm, w)
    n = lambda t: t.cpu().numpy()  # noqa: E731
    _, rc, _ = feature_losses(n(feat), n(target), n(mask), n(det), n(allmap[:, 1]), gm, [1e-2, 7e-3])
    assert np.array_equal(counts.cpu().numpy(), rc)
    px = fb.pixel_terms(n(feat), n(target), n(mask), n(det), n(allmap[:, 1]), gm)
    rep = fb.check(f"{W}x{H} M={M}", n(terms), n(counts), n(grad), px, n(w), gm, F)
    print(f"\n[feature {W}x{H} M={M}] " + ", ".join(f"{k} {v:.3g}" for k, v in rep.items()))
    assert torch.equal(_call(feat, target, mask, det, allmap, gm, w)[2], grad)


@pytest.mark.parametrize("name", list(FEATURE_CONFIGS))
def test_feature_loss_kernel_planted(name, dev):
    """The planted configurations of tests/feature_loss_bounds.py: features equal to the target, the Gaussian channel
    equal to alpha, masks of 0, 0.375 and 1e-30, |d| near 1e-20, on block seams and the image border; Cf = F, Cf = 1,
    the Gaussian-mask term alone, F = 32, frames undetected and at 0.5, a batch where nothing is positive."""
    from . import feature_loss_bounds as fb
    from .test_gpu_feature_loss import _call
    feat, target, mask, det, alpha, gm, planted = fb.config_inputs(name)
    M, F, H, W = feat.shape
    T = lambda x: None if x is None else torch.from_numpy(np.ascontiguousarray(x)).to(dev)  # noqa: E731
    allmap = torch.rand((M, 8, H, W), device=dev)
    allmap[:, 1] = T(alpha)
    w = T(fb.WEIGHTS)
    terms, counts, grad = _call(T(feat), T(target), T(mask), T(det), allmap, gm, w)
    n = lambda t: t.cpu().numpy()  # noqa: E731
    px = fb.pixel_terms(feat, target, mask, det, alpha, gm)
    rep = fb.check(name, n(terms), n(counts), n(grad), px, fb.WEIGHTS, gm, F)
    nk = sum(int(k.sum()) for k in px["knife"].values())
    print(f"\n[feature {name}] knife {nk} of {M * H * W} px; " + ", ".join(f"{k} {v:.3g}" for k, v in rep.items()))
    assert nk <= 4
    if fb.CONFIGS[name].get("empty"):
        assert int(counts.abs().sum()) == 0 and float(terms.abs().max()) == 0 and float(grad.abs().max()) == 0
