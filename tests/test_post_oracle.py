"""CPU tests pinning oracle/post_oracle.py (float64 NumPy restatement of the reference's render() post-processing and
Stage-3 image losses):
  (1) against fixtures produced by the REFERENCE's own code (tests/golden/make_post_golden.py executes the source text
      of gs/utils/point_utils.py and of render() lines 121-145 from the reference checkout on the CPU);
  (2) its hand-written vector-Jacobian products against central finite differences in float64.
"""
import os

import numpy as np
import pytest

from .conftest import GOLDEN_DIR
from oracle import post_oracle as po

POST_CASES = ["post_id_48x40", "post_rigid_56x36_r03"]
KEYS = ("acc", "rend_normal", "rend_dist", "render_depth_median", "render_depth_expected", "surf_depth", "surf_normal")


def _load(name):
    g = np.load(os.path.join(GOLDEN_DIR, name + ".npz"))
    return {k: g[k] for k in g.files}


@pytest.mark.parametrize("name", POST_CASES)
def test_post_oracle_matches_reference_outputs(name):
    g = _load(name)
    tanx, tany = [float(v) for v in g["in_tan"]]
    fw = po.post_forward(g["in_allmap"], g["in_wvt"], tanx, tany, float(g["in_depth_ratio"][0]))
    for k in KEYS:
        ref = g["ref_" + k].astype(np.float64)
        # the reference computes in float32; surf_normal normalises a cross product of central differences, which
        # amplifies float32 rounding where the surface is nearly flat in camera space
        tol = 2e-4 if k == "surf_normal" else 2e-6
        assert np.abs(fw[k] - ref).max() <= tol * max(1.0, np.abs(ref).max()), k


@pytest.mark.parametrize("name", POST_CASES)
def test_post_oracle_vjp_matches_reference_autograd(name):
    g = _load(name)
    tanx, tany = [float(v) for v in g["in_tan"]]
    grads = {k: g["w_" + k] for k in KEYS}
    ga = po.post_backward(g["in_allmap"], g["in_wvt"], tanx, tany, float(g["in_depth_ratio"][0]), grads)
    ref = g["ref_grad_allmap"].astype(np.float64)
    # autograd of 0/0 under nan_to_num yields NaN in the reference (div backward of a masked-out 0 gradient): the
    # rasterizer backward never reads those pixels' depth gradient (no contributor there); compare where finite
    fin = np.isfinite(ref)
    assert fin.mean() > 0.5
    scale = np.abs(ref[fin]).max()
    assert np.abs(ga[fin] - ref[fin]).max() <= 3e-4 * scale
    # the oracle (like the CUDA kernel) passes no gradient through the non-finite quotient: plane 0 gets 0, plane 1 only
    # the direct `acc` term
    assert not fin[0].all() and fin[2:].all()
    assert np.abs(ga[0][~fin[0]]).max(initial=0.0) == 0.0
    np.testing.assert_array_equal(ga[1][~fin[1]], grads["acc"][0].astype(np.float64)[~fin[1]])


def test_post_oracle_vjp_matches_finite_differences():
    g = _load("post_rigid_56x36_r03")
    tanx, tany = [float(v) for v in g["in_tan"]]
    rng = np.random.default_rng(0)
    am = g["in_allmap"].astype(np.float64)
    wts = {k: g["w_" + k].astype(np.float64) for k in KEYS}

    def f(a):
        fw = po.post_forward(a, g["in_wvt"], tanx, tany, 0.3)
        # alpha is DETACHED inside surf_normal (render():144): hold that factor at the unperturbed alpha
        with np.errstate(divide="ignore", invalid="ignore"):
            fw["surf_normal"] = np.where(a[1] > 0, fw["surf_normal"] / a[1] * am[1], 0.0)
        return sum((fw[k] * wts[k]).sum() for k in KEYS)
    ga = po.post_backward(am, g["in_wvt"], tanx, tany, 0.3, wts)
    cov = np.argwhere(am[1] > 0.2)
    for _ in range(40):
        y, x = cov[rng.integers(len(cov))]
        c = int(rng.integers(0, 7))
        h = 1e-6
        ap, an = am.copy(), am.copy()
        ap[c, y, x] += h; an[c, y, x] -= h
        fd = (f(ap) - f(an)) / (2 * h)
        assert abs(fd - ga[c, y, x]) <= 1e-5 * max(1.0, abs(fd)), (c, y, x, fd, ga[c, y, x])


def test_stage3_loss_oracle_gradients_match_finite_differences():
    g = _load("post_id_48x40")
    tanx, tany = [float(v) for v in g["in_tan"]]
    rng = np.random.default_rng(3)
    am = g["in_allmap"].astype(np.float64)
    H, W = am.shape[1:]
    color = rng.uniform(0, 1, size=(3, H, W))
    target = rng.uniform(0, 1, size=(3, H, W))
    vis = (rng.uniform(size=(H, W)) > 0.2).astype(np.float64)
    mask = (am[1] > 0.5).astype(np.float64)
    wt = po.mask_balance_wt(mask, vis)
    args = (g["in_wvt"], tanx, tany, 0.0, target, vis, mask, wt)
    kw = dict(w_rgb=0.8, w_mask=0.1, lambda_normal=0.05, lambda_dist=100.0)
    total, terms = po.stage3_losses(color, am, *args, **kw)
    assert np.isfinite(total) and set(terms) == {"rgb", "mask", "normal", "dist"}
    gc, ga = po.stage3_losses_backward(color, am, *args, **kw)
    cov = np.argwhere(am[1] > 0.2)
    for _ in range(30):
        y, x = cov[rng.integers(len(cov))]
        c = int(rng.choice([0, 2, 3, 4, 5, 6]))    # plane 1 (alpha) is detached inside surf_normal: checked below
        h = 1e-6
        ap, an = am.copy(), am.copy()
        ap[c, y, x] += h; an[c, y, x] -= h
        fd = (po.stage3_losses(color, ap, *args, **kw)[0] - po.stage3_losses(color, an, *args, **kw)[0]) / (2 * h)
        assert abs(fd - ga[c, y, x]) <= 1e-6 + 1e-4 * abs(fd), (c, y, x, fd, ga[c, y, x])
    kw0 = dict(kw, lambda_normal=0.0)              # without the normal term alpha is not detached anywhere
    ga0 = po.stage3_losses_backward(color, am, *args, **kw0)[1]
    for _ in range(10):
        y, x = cov[rng.integers(len(cov))]
        h = 1e-6
        ap, an = am.copy(), am.copy()
        ap[1, y, x] += h; an[1, y, x] -= h
        fd = (po.stage3_losses(color, ap, *args, **kw0)[0] - po.stage3_losses(color, an, *args, **kw0)[0]) / (2 * h)
        assert abs(fd - ga0[1, y, x]) <= 1e-6 + 1e-4 * abs(fd)
    for _ in range(10):
        y, x = cov[rng.integers(len(cov))]
        c = int(rng.integers(0, 3))
        h = 1e-7
        cp_, cn = color.copy(), color.copy()
        cp_[c, y, x] += h; cn[c, y, x] -= h
        fd = (po.stage3_losses(cp_, am, *args, **kw)[0] - po.stage3_losses(cn, am, *args, **kw)[0]) / (2 * h)
        assert abs(fd - gc[c, y, x]) <= 1e-9 + 1e-4 * abs(fd)


# ---- a float64 model of csrc/loss.cu's shared-memory tiling (32x8 tile + one-pixel ring, 80 ring threads, gather signs)
# against the oracle on ragged image sizes: the index logic of the kernel, checked where the GPU tests use block-aligned
# images.  The arithmetic is the oracle's; what is restated from the kernel is WHICH stencil lands in WHICH cell and who
# reads it.
def _loss_kernel_model(color, allmap, wvt, tanx, tany, depth_ratio, target, vis, mask_gt, mask_wt, w_rgb, w_mask, lam_n, lam_d):
    """Python restatement of csrc/loss.cu:loss_grad_kernel's indexing: 32x8 tiles, sg[6][10][34] ring, 80 ring threads."""
    _, H, W = color.shape
    N = H * W
    am = np.asarray(allmap, np.float64)
    # surf_depth as loss_depth_kernel
    med = po._nan_to_num00(am[5]); 
    with np.errstate(all='ignore'):
        ex = po._nan_to_num00((am[0] / am[1]))
    sd = ex * (1 - depth_ratio) + depth_ratio * med
    wv = np.asarray(wvt, np.float64)
    R = wv[:3, :3]                      # c.R[i*3+j] = m[i*4+j]
    B = wv[:3, :3].T                    # W2C rotation
    A = np.linalg.inv(B)
    fx, fy, cx, cy = W / (2 * tanx), H / (2 * tany), W * 0.5, H * 0.5
    sN = lam_n / N
    def ray(X, Y):
        u, v = (X - cx) / fx, (Y - cy) / fy
        return A @ np.array([u, v, 1.0])
    def stencil_eval(X, Y, scale):
        z = np.zeros(3)
        if not (1 <= X < W - 1 and 1 <= Y < H - 1): return z, z, z
        a_, b_, e_, f_ = ray(X, Y + 1), ray(X, Y - 1), ray(X + 1, Y), ray(X - 1, Y)
        dD, dU, dR, dL = sd[Y + 1, X], sd[Y - 1, X], sd[Y, X + 1], sd[Y, X - 1]
        dx = dD * a_ - dU * b_; dy = dR * e_ - dL * f_
        n = np.cross(dx, dy); ln = np.linalg.norm(n)
        a = am[1, Y, X]
        sn = n * (a / max(ln, 1e-12))
        g = scale * a * (R @ am[2:5, Y, X])
        if ln > 1e-12:
            w = n / ln; gn = (g - w * (w @ g)) / ln
        else:
            gn = g * 1e12
        gdx = np.cross(dy, gn)          # dy x gn
        gdy = np.cross(gn, dx)
        return sn, gdx, gdy
    g_allmap = np.zeros((8, H, W)); 
    for by in range((H + 7) // 8):
        for bx in range((W + 31) // 32):
            sg = np.full((6, 10, 34), np.nan)
            sn_own = {}
            for t in range(256):
                lx, ly = t & 31, t >> 5
                x, y = bx * 32 + lx, by * 8 + ly
                sn, gdx, gdy = stencil_eval(x, y, -sN)
                sn_own[t] = sn
                sg[0:3, ly + 1, lx + 1] = gdx; sg[3:6, ly + 1, lx + 1] = gdy
                if t < 80:
                    row = 0 if t < 32 else (9 if t < 64 else (t - 63 if t < 72 else t - 71))
                    col = t + 1 if t < 32 else (t - 31 if t < 64 else (0 if t < 72 else 33))
                    _, gdx, gdy = stencil_eval(bx * 32 + col - 1, by * 8 + row - 1, -sN)
                    sg[0:3, row, col] = gdx; sg[3:6, row, col] = gdy
            for t in range(256):
                lx, ly = t & 31, t >> 5
                x, y = bx * 32 + lx, by * 8 + ly
                if not (x < W and y < H): continue
                s = sn_own[t]
                q = -sN * s
                g_allmap[2:5, y, x] = R.T @ q
                gp = sg[0:3, ly, lx + 1] - sg[0:3, ly + 2, lx + 1] + sg[3:6, ly + 1, lx] - sg[3:6, ly + 1, lx + 2]
                assert np.isfinite(gp).all(), (bx, by, t)      # never reads an unwritten (corner) cell
                gsd = gp @ ray(x, y)
                gex, gmed = gsd * (1 - depth_ratio), gsd * depth_ratio
                a, d0, m5 = am[1, y, x], am[0, y, x], am[5, y, x]
                with np.errstate(all='ignore'):
                    qq = d0 / a
                qfin = np.isfinite(qq)
                g_allmap[0, y, x] = gex / a if qfin else 0.0
                g_acc = 0.0
                if mask_gt is not None:
                    g_acc += w_mask * 2 * (a - mask_gt[y, x]) * mask_wt[y, x] / N
                g_allmap[1, y, x] = g_acc + (-gex * d0 / (a * a) if qfin else 0.0)
                g_allmap[5, y, x] = gmed if np.isfinite(m5) else 0.0
                g_allmap[6, y, x] = lam_d / N
    return g_allmap



@pytest.mark.parametrize("W,H,depth_ratio", [(70, 50, 0.0), (33, 9, 0.3), (5, 3, 1.0)])
def test_loss_kernel_tiling_model_matches_oracle_on_ragged_sizes(W, H, depth_ratio):
    rng = np.random.default_rng(W * 131 + H)
    allmap = rng.uniform(0.2, 1.0, (8, H, W)); allmap[0] *= 3
    allmap[5] = allmap[0] / allmap[1] + rng.normal(0, .05, (H, W)); allmap[2:5] = rng.normal(0, 1, (3, H, W))
    color = rng.uniform(0, 1, (3, H, W)); target = rng.uniform(0, 1, (3, H, W))
    vis = (rng.uniform(0, 1, (H, W)) > .2).astype(float); mg = (rng.uniform(0, 1, (H, W)) > .5).astype(float)
    mw = rng.uniform(.5, 2, (H, W))
    c, s = np.cos(0.3), np.sin(0.3)
    W2C = np.eye(4); W2C[:3, :3] = np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]]); W2C[:3, 3] = [0.1, -0.2, 3.0]
    kw = dict(w_rgb=0.8, w_mask=0.1, lambda_normal=0.05, lambda_dist=100.0)
    _, ga = po.stage3_losses_backward(color, allmap, W2C.T, 0.5, 0.35, depth_ratio, target, vis, mg, mw, **kw)
    mine = _loss_kernel_model(color, allmap, W2C.T, 0.5, 0.35, depth_ratio, target, vis, mg, mw, 0.8, 0.1, 0.05, 100.0)
    assert np.abs(mine - ga).max() <= 1e-12 * np.abs(ga).max()
