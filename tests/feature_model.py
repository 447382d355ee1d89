"""float64 model of the feature-channel composite and its backward -- test infrastructure, imported by the feature tests only.

It restates, over a forward state of the C oracle (oracle/surfel_oracle.py: projected T matrices, centres, opacities,
sorted instance list, tile ranges), what vidu4d_b200/csrc/composite_feat.cu computes: per pixel, the colour's
front-to-back walk with the same tests (p.z == 0, depth < 0.2, alpha < 1/255, T < 1e-4 stops the pixel), and

    plane f = sum_i T_i alpha_i feat[i, f] + T_final bg_f                           (bg_f = 0 for a 3-value background)

Backward (for an upstream gradient G of the F planes):

    dL/dfeat[i, f]  = sum_pixels T_i alpha_i G_f
    dL/dalpha_i     = T_i sum_f (feat[i, f] - behind_f) G_f - T_final / (1 - alpha_i) sum_f bg_f G_f
    dL/dopacity_i  += dL/dalpha_i * G_i(pixel)          (alpha = opacity * exp(-rho / 2); the 0.99 clamp is not
                                                        differentiated, as in the rasterizer and the reference)

where behind_f is the alpha-composite of the contributors behind i.  Everything is vectorised over the 256 pixels of a
tile and evaluated in float64, so finite differences of `planes()` check `backward()` to many digits.
"""
from __future__ import annotations

import numpy as np


def _feature_bg(bg, F):
    bg = np.asarray(bg, dtype=np.float64).reshape(-1)
    if bg.size not in (3, 3 + F):
        raise ValueError(f"background must have 3 or 3+F = {3 + F} values")
    return np.zeros(F) if bg.size == 3 else bg[3:]


def _walk(st, opac, fn):
    """Calls fn(xs, ys, steps, T_final) per tile; steps = [(surfel id, ok mask, T before, alpha, G)] front to back."""
    W, H = st.W, st.H
    tx_n = (W + 15) // 16
    for t in range(st.ranges.shape[0]):
        r0, r1 = (int(v) for v in st.ranges[t])
        ys, xs = np.mgrid[(t // tx_n) * 16:(t // tx_n) * 16 + 16, (t % tx_n) * 16:(t % tx_n) * 16 + 16]
        keep = (xs < W) & (ys < H)
        xs, ys = xs[keep], ys[keep]
        px, py = xs + 0.5, ys + 0.5
        T = np.ones(px.shape)
        done = np.zeros(px.shape, bool)
        steps = []
        for i in range(r0, r1):
            sid = int(st.point_list[i])
            Tm = st.transMat[sid].astype(np.float64)
            Tu, Tv, Tw = Tm[0:3], Tm[3:6], Tm[6:9]
            k = px[None] * Tw[:, None] - Tu[:, None]
            l = py[None] * Tw[:, None] - Tv[:, None]
            p = np.cross(k, l, axis=0)
            with np.errstate(divide="ignore", invalid="ignore"):
                sx, sy = p[0] / p[2], p[1] / p[2]
            rho3d = sx * sx + sy * sy
            dx, dy = st.means2D[sid, 0] - px, st.means2D[sid, 1] - py
            rho2d = 2 * (dx * dx + dy * dy)
            rho = np.minimum(rho3d, rho2d)
            depth = np.where(rho3d <= rho2d, Tw[2] + Tw[0] * sx + Tw[1] * sy, Tw[2])
            G = np.exp(-0.5 * rho)
            alpha = np.minimum(0.99, opac[sid] * G)
            ok = (p[2] != 0) & (depth >= 0.2) & (alpha >= 1 / 255) & ~done
            test_T = T * (1 - alpha)
            stop = ok & (test_T < 1e-4)
            done |= stop
            ok &= ~stop
            if ok.any():
                steps.append((sid, ok, T.copy(), alpha, G))
            T = np.where(ok, test_T, T)
        fn(xs, ys, steps, T)


def planes(st, feat, bg, opac=None):
    """(F,H,W) float64 feature planes; feat (P,F); bg of 3 or 3+F values; opac (P,) overrides the state's opacities."""
    feat = np.asarray(feat, dtype=np.float64)
    F = feat.shape[1]
    bgf = _feature_bg(bg, F)
    opac = st.normal_opacity[:, 3].astype(np.float64) if opac is None else np.asarray(opac, dtype=np.float64)
    out = np.zeros((F, st.H, st.W))

    def tile(xs, ys, steps, T_final):
        C = np.zeros((F, xs.size))
        for sid, ok, T, alpha, _ in steps:
            C += np.where(ok, T * alpha, 0.0)[None] * feat[sid][:, None]
        out[:, ys, xs] = C + T_final[None] * bgf[:, None]
    _walk(st, opac, tile)
    return out


def backward(st, feat, bg, G):
    """dL/dfeatures (P,F) and the alpha term's dL/dopacity (P,) for L = sum(G * planes(st, feat, bg)), G (F,H,W)."""
    feat = np.asarray(feat, dtype=np.float64)
    P, F = feat.shape
    bgf = _feature_bg(bg, F)
    G = np.asarray(G, dtype=np.float64)
    opac = st.normal_opacity[:, 3].astype(np.float64)
    dfeat, dopac = np.zeros((P, F)), np.zeros(P)

    def tile(xs, ys, steps, T_final):
        g = G[:, ys, xs]
        bg_dot = (bgf[:, None] * g).sum(0)
        behind = np.zeros((F, xs.size))
        for sid, ok, T, alpha, Gs in reversed(steps):
            w = np.where(ok, T * alpha, 0.0)
            dfeat[sid] += (g * w[None]).sum(1)
            x = feat[sid][:, None]
            dalpha = T * ((x - behind) * g).sum(0) - T_final / (1 - alpha) * bg_dot
            dopac[sid] += np.where(ok, dalpha * Gs, 0.0).sum()
            behind = np.where(ok[None], alpha[None] * x + (1 - alpha[None]) * behind, behind)
    _walk(st, opac, tile)
    return dfeat, dopac
