"""TEST INFRASTRUCTURE -- the tracking kernel (csrc/track.cu track_kernel) restated in float64, with a first-order
rounding-error bound per output (tests/error_bound.py's _E, rot_matrix and w_mul as tests/preprocess_bounds.py states
them), and the anchor slot rule (composite_fwd.cu AnchorSlots) restated in numpy.

track() follows the kernel's operation tree for every (query, target frame): per non-empty slot k the scaled hit
coordinates u s_u and v s_v, the surface point mean + (u s_u) t_u + (v s_v) t_v, its weighted sum and the weight sum;
then X = sum / weight, the view transform, the quotients x / z and y / z and the pixel coordinates focal * q + c.  Every
written multiply and add is charged one rounding, so the bound holds whichever products the compiler contracts.
"""
import numpy as np

from .error_bound import _c, _E
from .preprocess_bounds import _fma, _rot, _w_mul, intrinsics

U = 2.0 ** -24
K_BOUND = 2.0                   # the kernel's result lies within K_BOUND u B of the float64 value
F32 = np.float32
NEAR = 0.2


def slot_rule(weights, K):
    """The anchor slots of one pixel: the indices (in walk order) of its K heaviest pairs, sorted by weight descending; a
    pair enters only if its weight is strictly larger than the last slot's, so among equal weights the earlier pair stays
    ahead.  Written as the insertion the kernel performs, one pair at a time."""
    slots = []
    for i, w in enumerate(weights):
        if len(slots) == K and not w > weights[slots[-1]]:
            continue
        pos = next((j for j, s in enumerate(slots) if w > weights[s]), len(slots))
        slots.insert(pos, i)
        del slots[K:]
    return slots


def slot_rule_sorted(weights, K):
    """The same slots by a stable sort on descending weight: the rule's closed form."""
    order = sorted(range(len(weights)), key=lambda i: -float(weights[i]))     # sorted() is stable
    return order[:K]


def track(ids, w, uv, queries, means, rots, scales, vms, W, H, tans=None, table=None):
    """float64 model of sr_track_pixels.  ids (S,K,H,W) int32, w (S,K,H,W), uv (S,K,2,H,W) float32; queries (N,3);
    means (T,P,3), rots (T,P,4), scales (P,2) float32; vms (T,16) the column-major view matrices; tans (tan_x, tan_y)
    or table (T,4) rows of surfel_camera.h.  Returns dict of xy (_E pair, (N,T) each), z (_E (N,T)), coverage (_E (N,)),
    valid (N,) bool (the kernel writes NaN where it is False)."""
    ids, w, uv = np.asarray(ids), np.asarray(w, F32), np.asarray(uv, F32)
    queries = np.asarray(queries, np.int64)
    S, K, Hh, Ww = ids.shape
    T, P = means.shape[0], means.shape[1]
    s, x, y = queries[:, 0], queries[:, 1], queries[:, 2]
    ok = (s >= 0) & (s < S) & (x >= 0) & (x < W) & (y >= 0) & (y < H)
    sc, xc, yc = np.where(ok, s, 0), np.where(ok, x, 0), np.where(ok, y, 0)
    sid = ids[sc, :, yc, xc]                                              # (N,K)
    sw_ = np.where(sid >= 0, w[sc, :, yc, xc], F32(0))
    su, sv = uv[sc, :, 0, yc, xc], uv[sc, :, 1, yc, xc]
    ok &= ~(sid >= P).any(axis=1)
    filled = sid >= 0
    gid = np.where(filled & (sid < P), sid, 0)
    out_xy, out_z = [], []
    cov = None
    for t in range(T):
        acc = [_c(np.zeros(len(queries))) for _ in range(3)]
        wsum = _c(np.zeros(len(queries)))
        for k in range(K):
            q = rots[t][gid[:, k]]
            R = _rot(q)
            scl = scales[gid[:, k]]
            wk = _E.leaf(np.where(filled[:, k], sw_[:, k], F32(0)))
            au = _E.leaf(su[:, k]) * _E.leaf(scl[:, 0])
            av = _E.leaf(sv[:, k]) * _E.leaf(scl[:, 1])
            mu = means[t][gid[:, k]]
            p = [_fma(av, R[3 + r], _fma(au, R[r], _E.leaf(mu[:, r]))) for r in range(3)]
            on = filled[:, k]
            for r in range(3):
                nxt = _fma(wk, p[r], acc[r])
                acc[r] = _E(np.where(on, nxt.v, acc[r].v), np.where(on, nxt.b, acc[r].b))
            nw = wsum + wk
            wsum = _E(np.where(on, nw.v, wsum.v), np.where(on, nw.b, wsum.b))
        cov = wsum
        X = [a / wsum for a in acc]
        m = [_E.leaf(np.full(len(queries), vms[t][i], F32)) for i in range(16)]
        p0 = _w_mul(m, X)
        v = [p0[r] + m[12 + r] for r in range(3)]
        fx, fy, cx, cy = intrinsics(W, H, tans if table is None else table[t][:2], None if table is None else table[t][2:])
        px = _fma(_c(np.float64(fx)), v[0] / v[2], _c(np.float64(cx)))
        py = _fma(_c(np.float64(fy)), v[1] / v[2], _c(np.float64(cy)))
        out_xy.append((px, py))
        out_z.append(v[2])
    valid = ok & (cov.v > 0)
    st = lambda es: _E(np.stack([e.v for e in es], 1), np.stack([e.b for e in es], 1))   # noqa: E731
    return {"x": st([p[0] for p in out_xy]), "y": st([p[1] for p in out_xy]), "z": st(out_z), "coverage": cov,
            "valid": valid}


def within(got, e, floor=1e-30):
    """|got - v| <= K_BOUND u b + floor, elementwise."""
    return np.abs(np.asarray(got, np.float64) - e.v) <= K_BOUND * U * e.b + floor
