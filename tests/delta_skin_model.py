"""TEST INFRASTRUCTURE -- the delta-skinning MLP (lab4d/nnutils/skinning.py:104-119) three ways.

  unfolded()      the reference's statements in torch, any dtype: get_bone_coords (transforms.py:9-25), / exp(log_gauss),
                  reshape to (…,3B), cat with the conditioning code expanded to every point, Linear -> ReLU -> Linear ->
                  ReLU -> Linear, relu * 0.1.  In float64 with autograd it is the oracle of every gradient; in float32 on
                  the GPU it is what tools/bench_skin_mlp.py times the fused op against.
  fold_table(), folded()   the first layer folded into one (64,4) table per frame, and the MLP on it, in float64 NumPy --
                  a restatement independent of vidu4d_b200.warp.delta_skin_tables.
  chain()         csrc/skin_mlp.cu restated operation for operation on tests/error_bound.py's running-error values, on
                  the kernel's own fp32 inputs (the fp32 table included), forward and backward, with the fixed-order
                  reduction of the weight gradients.  Every value carries its float64 value, its bound B (units of
                  u = 2^-24) and an fp32 shadow; the tests hold the GPU (and on the CPU the shadow) to
                  |x - value| <= K u B + FLOOR.

ReLU decisions are data: they are taken on the float64 values.  A point is a knife point when any of its 128 + B
pre-activations lies within its own bound of 0; the gradient checks zero the upstream gradient of such points on both
sides, which removes them from every gradient (all of a point's contributions are linear in its g_delta row).

The weight gradients are sums over points.  A thread of skin_mlp_bwd adds its points' terms one after the other (at most
n of them), then skin_mlp_reduce adds the CTAs' partial sums in float64 and rounds once: a term meets at most n + 1
roundings, so the sum's bound is sum B_i + (n + 1) sum |t_i|.  The shadow is one such order: all points in one thread.
"""
import numpy as np
import torch

from .error_bound import _E, _seqsum, _where

U = 2.0 ** -24
K = 2.0
FLOOR = float(np.finfo(np.float32).tiny)
WIDTH = 64
PARAMS = ("W1", "b1", "W2", "b2", "W3", "b3")


# ------------------------------------------------------------------------------------------------ the reference, in torch
def _qmul(a, b):
    aw, ax, ay, az = a.unbind(-1)
    bw, bx, by, bz = b.unbind(-1)
    return torch.stack((aw * bw - ax * bx - ay * by - az * bz, aw * bx + ax * bw + ay * bz - az * by,
                        aw * by - ax * bz + ay * bw + az * bx, aw * bz + ax * by - ay * bx + az * bw), -1)


def _qconj(q):
    return torch.cat((q[..., :1], -q[..., 1:]), -1)


def unfolded(points, art_r, art_d, log_gauss, p, cond):
    """points (N,3), (M,N,3) or (M,H,W,3); art_r, art_d (B,4) or (M,B,4); cond (C,) or (M,C); p: dict of PARAMS."""
    M = points.shape[0] if points.dim() > 2 else 1
    x = points.reshape(M, -1, 3)
    r, d = (a if a.dim() == 3 else a[None] for a in (art_r, art_d))
    q = _qconj(r)                                                      # dual_quaternion_inverse, then its (q, t)
    t = 2.0 * _qmul(_qconj(d), _qconj(q))[..., 1:]
    q, t = q[:, None], t[:, None]                                      # (Mb,1,B,·)
    x4 = torch.cat((torch.zeros_like(x[..., :1]), x), -1)[:, :, None]  # (M,N,1,4): the point as a pure quaternion
    xb = _qmul(_qmul(q, x4), _qconj(q))[..., 1:] + t                   # quaternion_apply + t, broadcast over frames
    xb = xb / log_gauss.exp()                                          # (M,N,B,3)
    c = (cond if cond.dim() == 2 else cond[None])[:, None].expand(M, x.shape[1], -1)
    h = torch.cat((xb.reshape(M, x.shape[1], -1), c), -1)              # (M,N,3B+C)
    h = torch.relu(torch.nn.functional.linear(h, p["W1"], p["b1"]))
    h = torch.relu(torch.nn.functional.linear(h, p["W2"], p["b2"]))
    y = torch.nn.functional.linear(h, p["W3"], p["b3"])
    return (torch.relu(y) * 0.1).reshape(tuple(points.shape[:-1]) + (y.shape[-1],))


# ------------------------------------------------------------------------------------------------ the fold, in float64
def fold_table(art_r, art_d, log_gauss, W1, b1, cond):
    """(Mt,64,4) float64: W1 [xyz_bone | cond] + b1 = F [x; 1].  NumPy arrays in, any float dtype."""
    r, d, lg, W1, b1, cond = (np.asarray(a, np.float64) for a in (art_r, art_d, log_gauss, W1, b1, cond))
    if r.ndim == 2:
        r, d = r[None], d[None]
    if cond.ndim == 1:
        cond = cond[None]
    B = lg.shape[0]
    tq = lambda a: torch.from_numpy(np.ascontiguousarray(a))  # noqa: E731
    q = _qconj(tq(r))
    t = (2.0 * _qmul(_qconj(tq(d)), _qconj(q))[..., 1:]).numpy()       # (Mb,B,3)
    eye = torch.eye(3, dtype=torch.float64)
    cols = []
    for c in range(3):                                                 # column c of R_b: q e_c q*
        e = torch.cat((torch.zeros(1, dtype=torch.float64), eye[c])).expand(q.shape)
        cols.append(_qmul(_qmul(q, e), _qconj(q))[..., 1:].numpy())
    R = np.stack(cols, -1)                                             # (Mb,B,3 (i),3 (c))
    Wx = W1[:, :3 * B].reshape(WIDTH, B, 3) / np.exp(lg)               # (64,B,3)
    A = np.einsum("jbi,fbic->fjc", Wx, R)
    c0 = np.einsum("jbi,fbi->fj", Wx, t)
    c1 = cond @ W1[:, 3 * B:].T + b1
    Mt = max(A.shape[0], c1.shape[0])
    return np.concatenate((np.broadcast_to(A, (Mt, WIDTH, 3)), np.broadcast_to(c0 + c1, (Mt, WIDTH))[..., None]), -1)


def folded(points, F, W2, b2, W3, b3):
    """delta in float64 from the folded table(s): points (…,3) as unfolded(); F (Mt,64,4)."""
    x = np.asarray(points, np.float64)
    M = x.shape[0] if x.ndim > 2 else 1
    x = x.reshape(M, -1, 3)
    F = np.broadcast_to(F, (M,) + F.shape[1:])
    h = np.maximum(np.einsum("mjc,mnc->mnj", F[..., :3], x) + F[:, None, :, 3], 0.0)
    h = np.maximum(h @ np.asarray(W2, np.float64).T + b2, 0.0)
    y = h @ np.asarray(W3, np.float64).T + b3
    return (np.maximum(y, 0.0) * 0.1).reshape(np.shape(points)[:-1] + (y.shape[-1],))


# ------------------------------------------------------------------------------------------------ the kernels' chain
def _matvec(W, h, init=None):
    """out[n,j] = init[j] + sum_k W[j,k] h[n,k], k ascending, one product and one add per term (an FMA rounds once: the
    two roundings charged still bound it)."""
    return _seqsum(W[None] * h[:, None, :], -1, init)


def _near_zero(e):
    """A '> 0' decision within its bound (an exact 0 with no error is the same decision on both sides)."""
    return (np.abs(e.v) <= K * U * e.b) & ~((e.v == 0) & (e.b == 0))


def _pointsum(t):
    """The fixed-order sum over the points (axis 0) of per-point terms: see the module docstring."""
    n = t.v.shape[0]
    f = None if t.f is None else np.add.accumulate(t.f, 0, dtype=np.float32)[-1]
    return _E(t.v.sum(0), t.b.sum(0) + (n + 1) * np.abs(t.v).sum(0), f)


def chain(points, F, W2, b2, W3, b3, g_delta=None):
    """One table's points through csrc/skin_mlp.cu.  points (n,3), W2 (64,64), b2 (64,), W3 (B,64), b3 (B,), g_delta (n,B)
    or None: fp32 arrays, the kernel's inputs.  F (64,4): the fp32 table the kernel reads, or fold_table()'s float64 one,
    whose rounding to fp32 then counts as part of the chain.  Returns a dict of running-error values: delta (n,B), knife
    (n,) bool, and with g_delta: g_x (n,3), g_F (64,4), g_W2, g_b2, g_W3, g_b3."""
    x, W2, b2, W3, b3 = (_E.leaf(a) for a in (points, W2, b2, W3, b3))
    # a float64 table is the exact fold: the kernel reads its fp32 rounding, one rounding per entry
    F = _E(F, np.abs(F), F.astype(np.float32)) if F.dtype == np.float64 else _E.leaf(F)
    pre1 = _seqsum(F[None, :, :3] * x[:, None, :], -1, F[:, 3])
    h1 = _where(pre1.v > 0, pre1, 0.0)
    pre2 = _matvec(W2, h1, b2)
    h2 = _where(pre2.v > 0, pre2, 0.0)
    y = _matvec(W3, h2, b3)
    tenth = _E.const(0.1)
    out = {"delta": tenth * _where(y.v > 0, y, 0.0),
           "knife": _near_zero(pre1).any(-1) | _near_zero(pre2).any(-1) | _near_zero(y).any(-1)}
    if g_delta is None:
        return out
    gy = _where(y.v > 0, tenth * _E.leaf(g_delta), 0.0)
    gh2 = _where(h2.v > 0, _seqsum(_T(W3)[None] * gy[:, None, :], -1), 0.0)          # sum_b W3[b,k] gy[n,b], b ascending
    gh1 = _where(h1.v > 0, _seqsum(_T(W2)[None] * gh2[:, None, :], -1), 0.0)
    x1 = _E(np.concatenate((x.v, np.ones_like(x.v[:, :1])), -1), None, np.concatenate((x.f, np.ones_like(x.f[:, :1])), -1))
    out.update(g_x=_seqsum(_T(F[:, :3])[None] * gh1[:, None, :], -1),
               g_W3=_pointsum(gy[:, :, None] * h2[:, None, :]), g_b3=_pointsum(gy),
               g_W2=_pointsum(gh2[:, :, None] * h1[:, None, :]), g_b2=_pointsum(gh2),
               g_F=_pointsum(gh1[:, :, None] * x1[:, None, :]))
    return out


def _T(e):
    return _E(e.v.T, e.b.T, None if e.f is None else e.f.T)


def chain_frames(points, F, W2, b2, W3, b3, g_delta=None):
    """chain() for points (M,n,3) and tables F (Mt,64,4): one table makes the frames one frame of M n points, as the
    kernel does; per-frame tables run frame by frame, g_F stacked, and the shared weights' gradients -- which the kernel
    sums over every frame's CTAs in one float64 pass -- summed with one rounding per frame charged."""
    M, n = points.shape[:2]
    B = W3.shape[0]
    if F.shape[0] == 1:
        o = chain(points.reshape(-1, 3), F[0], W2, b2, W3, b3, None if g_delta is None else g_delta.reshape(-1, B))
        o["delta"] = _E(o["delta"].v.reshape(M, n, B), o["delta"].b.reshape(M, n, B), o["delta"].f.reshape(M, n, B))
        o["knife"] = o["knife"].reshape(M, n)
        if g_delta is not None:
            o["g_x"] = _E(o["g_x"].v.reshape(M, n, 3), o["g_x"].b.reshape(M, n, 3), o["g_x"].f.reshape(M, n, 3))
            o["g_F"] = o["g_F"][None]
        return o
    per = [chain(points[m], F[m], W2, b2, W3, b3, None if g_delta is None else g_delta[m]) for m in range(M)]
    stack = lambda k: _E(np.stack([o[k].v for o in per]), np.stack([o[k].b for o in per]), np.stack([o[k].f for o in per]))  # noqa: E731
    out = {"delta": stack("delta"), "knife": np.stack([o["knife"] for o in per])}
    if g_delta is not None:
        out.update(g_x=stack("g_x"), g_F=stack("g_F"))
        for k in ("g_W2", "g_b2", "g_W3", "g_b3"):
            s = per[0][k]
            for o in per[1:]:
                s = s + o[k]
            out[k] = s
    return out


def within(x, e):
    """Largest |x - e.v| / (K u e.b + FLOOR) over the elements (<= 1 passes)."""
    return float((np.abs(np.asarray(x, np.float64) - e.v) / (K * U * e.b + FLOOR)).max())
