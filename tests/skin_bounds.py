"""TEST INFRASTRUCTURE -- the bob-skinning warp restated operation for operation, with its rounding-error bound.

The per-point chain of csrc/warp_common.cuh -- skin_weights, blend, the rsqrtf normalisation, x' = q x q* + t,
r' = q (x) r -- and its hand-written VJP (blend_vjp, and bob_warp_bwd_kernel's inline copy of skin_vjp) are restated
here in NumPy in the kernels' order, on the kernels' own fp32 inputs, as running-error values (tests/error_bound.py),
ending in bob_warp's (xyz_cam, rot_cam, entropy) (csrc/warp.cu).  Every value carries its float64 value, its bound B
(units of u = 2^-24) and an fp32 shadow evaluation; the tests hold the GPU (and, on the CPU, the shadow) to
|x - value| <= K u B + FLOOR.

Decisions are data.  The anchor is the first arg-max of the float64 logits; the sign of bone b is qdot(qa, r_b) > 0 in
float64.  A point is a knife point when a decision it depends on is within its own bound, or when a normalisation or
division is badly conditioned:
  * anchor: the top two logits differ by more than 0 and at most K u (B1 + B2) (an exact float64 tie is the same
    computation on both sides: both take the lower index);
  * sign: 0 < |qdot(qa, r_b)| <= K u B for a bone whose fp32 weight is not 0 (an exact 0 is -1 on both sides);
  * conditioning: u B > 1/64 of |QR|^2.

Reductions beyond one thread add (levels) u sum |t| to the bound of a sum of per-thread terms t.  Sums inside a thread
(gw over frames, g_xyz over frames and then bones, grot over frames, Z and QR over bones) are restated in order and need
nothing more.  The table gradients go through warp_common.cuh's butterfly32 / acc_table, then the CTA's flush: 5
butterfly or shuffle levels, then one shared-memory atomic per warp (4 warps in the 128-thread backward blocks), then
one global atomic per block in any order.  A term passing through a depth-5 tree, a chain of A = 4 adds and a chain of
NB adds (NB blocks) meets at most 5 + A + NB roundings.  The shadow of a reduction is one such order: a halving tree
over the 32 lanes, then the warps, then the blocks in order.
"""
import numpy as np

from .error_bound import _E, _c, _max, _seqsum, _where

U = 2.0 ** -24
K = 2.0
FLOOR = float(np.finfo(np.float32).tiny)
KNIFE_REL = 2.0 ** -6
ZERO = _E(0.0, None, np.float32(0.0))


# ------------------------------------------------------------------------------------------------ quaternion algebra
def qmul(a, b):
    aw, ax, ay, az = a
    bw, bx, by, bz = b
    return (((aw * bw - ax * bx) - ay * by) - az * bz, ((aw * bx + ax * bw) + ay * bz) - az * by,
            ((aw * by - ax * bz) + ay * bw) + az * bx, ((aw * bz + ax * by) - ay * bx) + az * bw)


def qconj(q):
    return (q[0], -q[1], -q[2], -q[3])


def qadd(a, b):
    return tuple(x + y for x, y in zip(a, b))


def qscale(a, s):
    return tuple(x * s for x in a)


def qdot(a, b):
    return ((a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]) + a[3] * b[3]


def pure(v):
    return (ZERO, v[0], v[1], v[2])


def qrot(q, v):
    """q v q* (warp_common.cuh qrot)."""
    return qmul(qmul(q, pure(v)), qconj(q))[1:]


def qrot_vjp(q, v, g):
    """g_v = (q* g q)[1:], g_q = -2 g (x) q (x) v (warp_common.cuh qrot_vjp).  Returns (gq, gv)."""
    gp = pure(g)
    gv = qmul(qmul(qconj(q), gp), q)[1:]
    gq = tuple(x.scale(-2.0) for x in qmul(qmul(gp, q), pure(v)))
    return gq, gv


def _col(a, *idx):
    """Leaf _E of column(s) of an fp32 array: a[..., i] for each i."""
    return tuple(_E.leaf(a[..., i]) for i in idx)


def _bones(tab_oq, tab_ot, ig):
    """The per-bone tables as (1,B) leaves broadcasting against (n,1) point values."""
    return (_col(tab_oq[None], 0, 1, 2, 3), _col(tab_ot[None], 0, 1, 2), _col(ig[None], 0, 1, 2))


def _knife_close(e):
    """0 < |v| <= K u B: a decision or a '> 0' count within its bound."""
    return (np.abs(e.v) > 0) & (np.abs(e.v) <= K * U * e.b)


def _ill(e):
    """u B > 1/64 of |v|: a normalisation or division whose first-order bound means nothing."""
    return U * e.b > KNIFE_REL * np.abs(e.v)


# ------------------------------------------------------------------------------------------------ the shared chain
def skin(x, bones, drow):
    """skin_weights: x a point (3 (n,) values), bones (oq, ot, ig) (1,B) leaves, drow (n,B) leaf or None.
    Returns dict(w (n,B), anchor (n,), ent (n,), xb (3 (n,B) bone coordinates before inv_gauss), knife (n,))."""
    oq, ot, ig = bones
    xr = qrot(oq, [_bcast(c) for c in x])
    xb = tuple(a + t for a, t in zip(xr, ot))
    s = [a * i for a, i in zip(xb, ig)]
    l = -((s[0] * s[0] + s[1] * s[1]) + s[2] * s[2])
    if drow is not None:
        l = l - drow
    B = l.v.shape[-1]
    cols = [l[:, b] for b in range(B)]
    mx, anchor = _max(cols)
    srt = np.sort(l.v, -1)
    second = srt[:, -2] if B > 1 else np.full(len(anchor), -np.inf)
    sec_b = np.take_along_axis(l.b, np.argsort(l.v, -1)[:, -2:-1], -1)[:, 0] if B > 1 else 0.0
    gap = mx.v - second
    knife = (gap > 0) & (gap <= K * U * (mx.b + sec_b))
    d = l - _E(mx.v[:, None], mx.b[:, None], mx.f[:, None])
    onehot = np.arange(B)[None] == anchor[:, None]
    d = _E(np.where(onehot, 0.0, d.v), np.where(onehot, 0.0, d.b), np.where(onehot, np.float32(0), d.f))
    e = d.exp()
    Z = _seqsum(e)
    inv = _c(1.0) / Z
    w = e * _E(inv.v[:, None], inv.b[:, None], inv.f[:, None])
    return dict(w=w, anchor=anchor, onehot=onehot, ent=Z.log(), xb=xb, knife=knife, l=l)


def _bcast(e):
    return _E(e.v[:, None], e.b[:, None], None if e.f is None else e.f[:, None])


def blend(sk, sr_m, sd_m):
    """blend of one frame: sr_m, sd_m (B,4) fp32.  Returns (QR, QD, sign (n,B), ws (n,B), knife (n,))."""
    r = _col(sr_m[None], 0, 1, 2, 3)
    dq = _col(sd_m[None], 0, 1, 2, 3)
    qa = tuple(_E.leaf(sr_m[sk["anchor"], c][:, None]) for c in range(4))
    dot = qdot(qa, r)
    sign = np.where(dot.v > 0, 1.0, -1.0)
    knife = (_knife_close(dot) & (sk["w"].f != 0)).any(-1)
    ws = sk["w"].scale(sign)
    QR = tuple(_seqsum(c * ws) for c in r)
    QD = tuple(_seqsum(c * ws) for c in dq)
    return QR, QD, sign, ws, knife, r, dq


def rigid(QR, QD, x):
    """The rsqrtf normalisation and x' = q x q* + t.  Returns dict(q, qd, inv, xt, knife)."""
    nn = qdot(QR, QR)
    inv = nn.rsqrt()
    q, qd = qscale(QR, inv), qscale(QD, inv)
    t4 = qmul(qd, qconj(q))
    xr = qrot(q, x)
    xt = tuple(a + t.scale(2.0) for a, t in zip(xr, t4[1:]))
    return dict(q=q, qd=qd, inv=inv, xt=xt, knife=_ill(nn))


def normal_vjp(R, gq, gqd):
    q, qd, inv = R["q"], R["qd"], R["inv"]
    gQD = qscale(gqd, inv)
    gQR = qscale(qadd(gq, qscale(q, -(qdot(q, gq) + qdot(qd, gqd)))), inv)
    return gQR, gQD


def blend_vjp(bl, gQR, gQD, gw):
    """gw[b] += s (qdot(gQR, r_b) + qdot(gQD, d_b)); the per-point (n,B,4) contributions to dL/dse3_r and dL/dse3_d."""
    _, _, sign, ws, _, r, dq = bl
    bc = [_bcast(c) for c in gQR], [_bcast(c) for c in gQD]
    t = (qdot(bc[0], r) + qdot(bc[1], dq)).scale(sign)
    gw = t if gw is None else gw + t
    g_sr = _stack([c * ws for c in bc[0]])
    g_sd = _stack([c * ws for c in bc[1]])
    return gw, g_sr, g_sd


def _stack(es):
    f = None if any(e.f is None for e in es) else np.stack([e.f for e in es], -1)
    return _E(np.stack([e.v for e in es], -1), np.stack([e.b for e in es], -1), f)


def skin_vjp(sk, bones, x, gw, ge, drow, g_d2):
    """The softmax (+ entropy) and Gaussian-logit VJP (skin_vjp, and bob_warp_bwd's inline copy): ge None for no entropy
    term, g_d2 None for no delta^2 term.  Returns (g_delta (n,B) or None, (n,B,3) bone terms of dL/dx, table terms
    g_oq (n,B,4), g_ot (n,B,3), g_ig (n,B,3))."""
    w = sk["w"]
    dotwg = _seqsum(w * gw)
    gl = w * (gw - _bcast(dotwg))
    if ge is not None:
        gl = gl + _bcast(ge) * _where(sk["onehot"], w - _c(1.0), w)
    g_delta = -gl if g_d2 is None else (_bcast(g_d2) * drow - gl)
    oq, ot, ig = bones
    xb = sk["xb"]
    gs = [(b.scale(-2.0) * i) * gl for b, i in zip(xb, ig)]
    gb = [g * i for g, i in zip(gs, ig)]
    gqb, ax = qrot_vjp(oq, [_bcast(c) for c in x], gb)
    return g_delta, _stack(list(ax)), _stack(list(gqb)), _stack(gb), _stack([g * b for g, b in zip(gs, xb)])


# ------------------------------------------------------------------------------------------------ reductions
class Red:
    """One table slot group's cross-thread sum: per-thread terms in blocks of `bs` threads; G passes per thread."""

    def __init__(self, bs):
        self.bs, self.v, self.b, self.a, self.nb, self.adds, self.f = bs, 0.0, 0.0, 0.0, 0, 0, []

    def add(self, t):
        """t: _E (G, n, *slot) of one run of whole blocks (n a multiple of bs; dead lanes are zeros)."""
        G, n = t.v.shape[:2]
        assert n % self.bs == 0
        nw, nbc = self.bs // 32, n // self.bs
        self.v = self.v + t.v.sum((0, 1))
        self.b = self.b + t.b.sum((0, 1))
        self.a = self.a + np.abs(t.v).sum((0, 1))
        self.nb += nbc
        self.adds = G * nw
        if t.f is not None and self.f is not None:
            f = t.f.reshape((G, nbc, nw, 32) + t.f.shape[2:])
            while f.shape[3] > 1:
                h = f.shape[3] // 2
                f = f[:, :, :, :h] + f[:, :, :, h:]
            f = np.moveaxis(f[:, :, :, 0], 0, 1).reshape((nbc, G * nw) + t.f.shape[2:])
            self.f.append(np.add.accumulate(f, 1)[:, -1])
        else:
            self.f = None

    def result(self, L=None):
        """The sum; L overrides the level count where the passes of one thread and the blocks do not follow from add()."""
        L = 5 + self.adds + self.nb if L is None else L
        f = np.add.accumulate(np.concatenate(self.f, 0), 0)[-1] if self.f else None
        return _E(self.v, self.b + L * self.a, f)


def _pad(t, n, axis=1):
    """Zero terms for the dead lanes up to n along `axis`."""
    k = n - t.v.shape[axis]
    if k == 0:
        return t
    pw = [(0, 0)] * t.v.ndim
    pw[axis] = (0, k)
    return _E(np.pad(t.v, pw), np.pad(t.b, pw), None if t.f is None else np.pad(t.f, pw))


def _rup(n, b):
    return (n + b - 1) // b * b


def _pts(a):
    """(n,3|4) fp32 rows as a tuple of (n,) leaves."""
    return tuple(_E.leaf(a[:, i]) for i in range(a.shape[1]))


def _flat(e):
    return _E(e.v[:, 0], e.b[:, 0], None if e.f is None else e.f[:, 0])


def _cat(parts, axis=0):
    f = None if any(p.f is None for p in parts) else np.concatenate([p.f for p in parts], axis)
    return _E(np.concatenate([p.v for p in parts], axis), np.concatenate([p.b for p in parts], axis), f)


# ------------------------------------------------------------------------------------------------ bob_warp
def warp_chunk(xyz, rot, tab, delta, gx, gr, ge):
    """bob_warp_fwd_kernel and bob_warp_bwd_kernel on n points (n a multiple of 128; rows past the live ones must carry
    zero upstream).  xyz (n,3), rot (n,4), delta (n,B) or None, gx (M,n,3), gr (M,n,4), ge (n,) or None (fp32).
    Returns dict of _E: xyz_cam (M,n,3), rot_cam (M,n,4), entropy (n,), g_xyz (n,3), g_rot (n,4), g_delta (n,B); table
    terms g_oq (1,n,B,4) ... g_sr (1,n,M,B,4) for Red; knife (n,)."""
    M = tab["sr"].shape[0]
    x, r = _pts(xyz), _pts(rot)
    bones = _bones(tab["oq"], tab["ot"], tab["ig"])
    drow = None if delta is None else _E.leaf(delta)
    sk = skin(x, bones, drow)
    knife = sk["knife"].copy()
    gxx = [ZERO, ZERO, ZERO]
    grot = (ZERO,) * 4
    gw = None
    out = {k: [] for k in ("xyz_cam", "rot_cam", "g_sr", "g_sd", "g_cq", "g_ct")}
    for m in range(M):
        bl = blend(sk, tab["sr"][m], tab["sd"][m])
        R = rigid(bl[0], bl[1], x)
        knife |= bl[4] | R["knife"]
        rt = qmul(R["q"], r)
        qc = tuple(_E.leaf(np.float32(c)) for c in tab["cq"][m])
        ct = tuple(_E.leaf(np.float32(c)) for c in tab["ct"][m])
        cr = qrot(qc, R["xt"])
        out["xyz_cam"].append(_stack([a + t for a, t in zip(cr, ct)]))
        out["rot_cam"].append(_stack(list(qmul(qc, rt))))
        gc = _pts(gx[m])
        grc = _pts(gr[m])
        gqc, gt = qrot_vjp(qc, R["xt"], gc)
        gqc = qadd(gqc, qmul(grc, qconj(rt)))
        grt = qmul(qconj(qc), grc)
        out["g_cq"].append(_stack(list(gqc)))
        out["g_ct"].append(_stack(list(gc)))
        gq, ax = qrot_vjp(R["q"], x, gt)
        gxx = [a + b for a, b in zip(gxx, ax)]
        gq = qadd(gq, qmul(grt, qconj(r)))
        grot = qadd(grot, qmul(qconj(R["q"]), grt))
        gct = pure(tuple(g.scale(2.0) for g in gt))
        gqd = qmul(gct, R["q"])
        gq = qadd(gq, qconj(qmul(qconj(R["qd"]), gct)))
        gQR, gQD = normal_vjp(R, gq, gqd)
        gw, g_sr, g_sd = blend_vjp(bl, gQR, gQD, gw)
        out["g_sr"].append(g_sr)
        out["g_sd"].append(g_sd)
    gev = None if ge is None else _E.leaf(ge)
    g_delta, axb, g_oq, g_ot, g_ig = skin_vjp(sk, bones, x, gw, gev, None, None)
    g_xyz = [_seqsum(axb[:, :, k], init=gxx[k]) for k in range(3)]
    st = lambda es, ax_: _stack(es) if ax_ == -1 else _E(np.stack([e.v for e in es], ax_), np.stack([e.b for e in es], ax_),  # noqa: E731
                                                         np.stack([e.f for e in es], ax_))
    return dict(xyz_cam=st(out["xyz_cam"], 0), rot_cam=st(out["rot_cam"], 0), entropy=sk["ent"],
                g_xyz=_stack(g_xyz), g_rot=_stack(list(grot)), g_delta=g_delta, g_oq=g_oq[None], g_ot=g_ot[None], g_ig=g_ig[None],
                g_sr=st(out["g_sr"], 1)[None], g_sd=st(out["g_sd"], 1)[None],
                g_cq=st(out["g_cq"], 1)[None], g_ct=st(out["g_ct"], 1)[None], knife=knife)


WARP_TABLES = ("oq", "ot", "ig", "sr", "sd", "cq", "ct")
TABLE_GRADS = tuple("g_" + k for k in WARP_TABLES)


def warp_model(xyz, rot, tab, delta, gx, gr, ge, chunk=2048):
    """The whole bob_warp (forward and backward) in chunks of points.  The upstream of knife points is zeroed (the GPU
    side must zero the same): a chunk that holds one is evaluated again for its backward.  Returns dict of _E (full
    tensors) plus knife (P,)."""
    P = xyz.shape[0]
    chunk = _rup(chunk, 128)
    reds = {k: Red(128) for k in WARP_TABLES}
    parts = {k: [] for k in ("xyz_cam", "rot_cam", "entropy", "g_xyz", "g_rot", "g_delta")}
    knives = []
    for a in range(0, P, chunk):
        e = min(P, a + chunk)
        n = _rup(e - a, 128)
        pad = lambda arr, ax=0: None if arr is None else np.concatenate(  # noqa: E731
            [np.take(arr, np.arange(a, e), ax), np.zeros(arr.shape[:ax] + (n - (e - a),) + arr.shape[ax + 1:], arr.dtype)], ax)
        args = [pad(xyz), pad(rot), tab, pad(delta), pad(gx, 1), pad(gr, 1), pad(ge)]
        if e - a < n:               # dead lanes read point 0 of the whole array (p clamped to 0), with zero upstream
            for i, arr in ((0, xyz), (1, rot), (3, delta)):
                if arr is not None:
                    args[i][e - a:] = arr[0]
        res = warp_chunk(*args)
        kn = res["knife"][:e - a]
        if kn.any():
            for i in (4, 5):
                args[i][:, :e - a][:, kn] = 0.0
            if args[6] is not None:
                args[6][:e - a][kn] = 0.0
            res2 = warp_chunk(*args)
            for k in list(res):
                if k.startswith("g_"):
                    res[k] = res2[k]
        knives.append(kn)
        for k in parts:
            t = res[k]
            parts[k].append(t[:, :e - a] if k in ("xyz_cam", "rot_cam") else t[:e - a])
        for k in WARP_TABLES:
            t = res["g_" + k]
            reds[k].add(t)
    out = {k: _cat(v, 1 if k in ("xyz_cam", "rot_cam") else 0) for k, v in parts.items()}
    for k in WARP_TABLES:
        out["g_" + k] = reds[k].result()
    out["knife"] = np.concatenate(knives)
    return out


def _rows(arr, a, e, n, fill=None):
    """Rows a..e of arr padded to n rows: the dead lanes' rows, copies of row `fill` (a dead lane's clamped index) or
    zeros."""
    if arr is None:
        return None
    out = np.zeros((n,) + arr.shape[1:], arr.dtype)
    out[:e - a] = arr[a:e]
    if fill is not None and e - a < n:
        out[e - a:] = arr[fill]
    return out


def _scal(x):
    return _E.leaf(np.float32(x))


def _scal_e(e, i=None):
    """One element of an _E as a scalar _E."""
    return _E(e.v if i is None else e.v[i], e.b if i is None else e.b[i], e.f if i is None else e.f[i])


def _block_sum(t, bs):
    """A per-thread value summed as a forward kernel sums it: t (n,) with n a multiple of bs."""
    r = Red(bs)
    r.add(t[None])
    return r


# ------------------------------------------------------------------------------------------------ reproj (match.cu)
def reproj_chunk(m, xyz, delta, tab, Km, hxy, mask, det, gls=None):
    """reproj_point and the loss ending of frame m on n pixels (rows past the live ones: mask 0).  xyz (n,3), delta (n,B)
    or None, Km (3,3), hxy (n,2), mask (n,), det the frame's is_detected (fp32).  gls: g_loss * scale as an _E scalar for
    the backward, or None.  Returns dict of _E: xy (n,2), val (n,), knife (n,); with gls also g_xyz (n,3), g_delta (n,B),
    table terms g_oq (1,n,B,4), g_ot, g_ig, g_sr (1,n,B,4), g_sd, g_cq (1,n,4), g_ct (1,n,3)."""
    x = _pts(xyz)
    bones = _bones(tab["oq"], tab["ot"], tab["ig"])
    drow = None if delta is None else _E.leaf(delta)
    sk = skin(x, bones, drow)
    bl = blend(sk, tab["sr"][m], tab["sd"][m])
    R = rigid(bl[0], bl[1], x)
    qc = tuple(_scal(c) for c in tab["cq"][m])
    ct = tuple(_scal(c) for c in tab["ct"][m])
    xc = [a + t for a, t in zip(qrot(qc, R["xt"]), ct)]
    Kq = [_scal(k) for k in np.asarray(Km, np.float32).reshape(9)]
    h = [(Kq[3 * i] * xc[0] + Kq[3 * i + 1] * xc[1]) + Kq[3 * i + 2] * xc[2] for i in range(3)]
    den = h[2] + _scal(1e-6)
    u, v = h[0] / den, h[1] / den
    dx, dy = u - _E.leaf(hxy[:, 0]), v - _E.leaf(hxy[:, 1])
    nrm = (dx * dx + dy * dy).sqrt()
    mk, dt = _E.leaf(mask), _scal(det)
    val = (nrm * mk) * dt
    knife = sk["knife"] | bl[4] | R["knife"] | _ill(den) | _ill(nrm)
    out = dict(xy=_stack([u, v]), val=val, knife=knife)
    if gls is None:
        return out
    wpx = mk * dt
    on = (nrm.v * wpx.v) > 0
    gl = _where(on, (gls * wpx) / _where(on, nrm, 1.0), 0.0)
    gu, gv = gl * dx, gl * dy
    dh = [gu / den, gv / den, -(gu * u + gv * v) / den]
    gc = [(Kq[j] * dh[0] + Kq[3 + j] * dh[1]) + Kq[6 + j] * dh[2] for j in range(3)]
    gqc, gt = qrot_vjp(qc, R["xt"], gc)
    gq, gx = qrot_vjp(R["q"], x, gt)
    gct = pure(tuple(g.scale(2.0) for g in gt))
    gqd = qmul(gct, R["q"])
    gq = qadd(gq, qconj(qmul(qconj(R["qd"]), gct)))
    gQR, gQD = normal_vjp(R, gq, gqd)
    gw, g_sr, g_sd = blend_vjp(bl, gQR, gQD, None)
    g_delta, axb, g_oq, g_ot, g_ig = skin_vjp(sk, bones, x, gw, None, None, None)
    out.update(g_xyz=_stack([_seqsum(axb[:, :, k], init=gx[k]) for k in range(3)]), g_delta=g_delta, g_oq=g_oq[None],
               g_ot=g_ot[None], g_ig=g_ig[None], g_sr=g_sr[None], g_sd=g_sd[None], g_cq=_stack(list(gqc))[None],
               g_ct=_stack(gc)[None])
    return out


def reproj_model(xyz_m, delta, tab, Kmat, hxy, mask, det, weight, train_res, g_loss, chunk=2048):
    """reproj_fwd_kernel, reproj_scale_kernel and reproj_bwd_kernel.  xyz_m (M,HW,3), delta (M,HW,B) or None, Kmat (M,3,3),
    hxy (M,HW,>=2), mask (M,HW), det (M,), weight, train_res, g_loss (fp32).  The mask of knife pixels must already be 0
    (reproj_knife).  Returns dict: xy (M,HW,2), terms (M,), loss, scale as _E, counts (M,), g_xyz (M,HW,3), g_delta
    (M,HW,B) and the table gradients (g_oq ... in sr_bob_warp_table_floats' shapes) as _E."""
    M, HW = xyz_m.shape[:2]
    chunk = _rup(chunk, 128)
    spans = [(a, min(HW, a + chunk)) for a in range(0, HW, chunk)]

    def args(m, a, e):
        n = _rup(e - a, 128)
        return (m, _rows(xyz_m[m], a, e, n, 0), _rows(None if delta is None else delta[m], a, e, n, 0), tab, Kmat[m],
                _rows(hxy[m][:, :2], a, e, n, 0), _rows(mask[m], a, e, n), det[m])

    xy, terms, counts = [], [], []
    for m in range(M):
        red, parts, cnt = Red(128), [], 0
        for a, e in spans:
            r = reproj_chunk(*args(m, a, e))
            assert not (r["knife"][:e - a] & (mask[m][a:e] != 0)).any(), "knife pixels must be masked"
            parts.append(r["xy"][:e - a])
            on = r["val"].v > 0
            red.add(_where(on, r["val"], 0.0)[None])
            cnt += int(on.sum())
        xy.append(_cat(parts))
        terms.append(red.result())
        counts.append(cnt)
    c = sum(counts)
    s = (_scal(weight) / (_c(float(c)) * _scal(train_res))) if c else _E(0.0, None, np.float32(0))
    terms = [t * s for t in terms]
    loss = ZERO
    for t in terms:
        loss = loss + t
    gls = _scal(g_loss) * s
    tabs = ("oq", "ot", "ig", "sr", "sd", "cq", "ct")
    shared = {k: Red(128) for k in ("oq", "ot", "ig")}
    per = {k: [Red(128) for _ in range(M)] for k in ("sr", "sd", "cq", "ct")}
    gx, gd = [], []
    for m in range(M):
        px, pd = [], []
        for a, e in spans:
            r = reproj_chunk(*args(m, a, e), gls=gls)
            px.append(r["g_xyz"][:e - a])
            pd.append(r["g_delta"][:e - a])
            for k in tabs:
                (shared[k] if k in shared else per[k][m]).add(r["g_" + k])
        gx.append(_cat(px))
        gd.append(_cat(pd))
    st = lambda es: _E(np.stack([e.v for e in es]), np.stack([e.b for e in es]), np.stack([e.f for e in es]))  # noqa: E731
    out = dict(xy=st(xy), terms=st(terms), loss=loss, scale=s, counts=np.array(counts), g_xyz=st(gx),
               g_delta=None if delta is None else st(gd))
    for k in tabs:
        out["g_" + k] = shared[k].result() if k in shared else st([r.result() for r in per[k]])
    return out


def reproj_knife(xyz_m, delta, tab, Kmat, hxy, chunk=2048):
    """(M,HW) knife pixels of reproj (the decisions and conditioning of reproj_chunk, which do not depend on the mask)."""
    M, HW = xyz_m.shape[:2]
    out = np.zeros((M, HW), bool)
    for m in range(M):
        for a in range(0, HW, chunk):
            e = min(HW, a + chunk)
            r = reproj_chunk(m, xyz_m[m][a:e], None if delta is None else delta[m][a:e], tab, Kmat[m], hxy[m][a:e, :2],
                             np.ones(e - a, np.float32), 1.0)
            out[m, a:e] = r["knife"]
    return out


# ------------------------------------------------------------------------------------------------ cycle (cycle.cu)
CYCLE_TABLES = ("oq", "ot", "ig", "sr", "sd", "cq", "ct")


def cycle_chunk(m, xyz, xcam, delta, tab, sc=None):
    """cycle_point and the three values of frame m on n surfels (rows past the live ones are dead lanes: pass live).
    tab: oq (M,B,4), ot (M,B,3), ig (B,3), sr, sd (M,B,4), cq (M,4), ct (M,3).  sc: (s_cyc, s_dsk, s_ent) = g_loss * scale
    as _E scalars for the backward, or None.  Returns dict of _E: cyc, dsk, ent (n,), knife (n,); with sc also go (n,3)
    (dL/dx_cycled), g_xyz_cam (n,3), g_delta (n,B), table terms g_oq (1,n,B,4), g_ot, g_ig, g_sr, g_sd, g_cq, g_ct."""
    B = tab["ig"].shape[0]
    x = _pts(xyz)
    xc = _pts(xcam)
    qi = qconj(tuple(_scal(c) for c in tab["cq"][m]))
    nct = tuple(_scal(-c) for c in tab["ct"][m])
    xt = [a + b for a, b in zip(qrot(qi, xc), qrot(qi, nct))]
    bones = _bones(tab["oq"][m], tab["ot"][m], tab["ig"])
    drow = None if delta is None else _E.leaf(delta)
    sk = skin(xt, bones, drow)
    bl = blend(sk, tab["sr"][m], tab["sd"][m])
    R = rigid(bl[0], bl[1], xt)
    d = [a - b for a, b in zip(R["xt"], x)]
    cyc = ((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]).sqrt()
    dsk = ZERO if drow is None else _seqsum(drow * drow) / _scal(float(B))
    ent = sk["ent"]
    knife = sk["knife"] | bl[4] | R["knife"] | _ill(cyc) | _knife_close(cyc) | _knife_close(ent)
    if drow is not None:
        knife |= _knife_close(dsk)
    out = dict(cyc=cyc, dsk=dsk, ent=ent, knife=knife)
    if sc is None:
        return out
    on = cyc.v > 0
    gc = _where(on, sc[0] / _where(on, cyc, 1.0), 0.0)
    go = [gc * di for di in d]
    ge = _where(ent.v > 0, sc[2], 0.0)
    g_d2 = None
    if drow is not None:
        g_d2 = _where(dsk.v > 0, sc[1].scale(2.0) / _scal(float(B)), 0.0)
    gq, gt = qrot_vjp(R["q"], xt, go)
    gct = pure(tuple(g.scale(2.0) for g in go))
    gqd = qmul(gct, R["q"])
    gq = qadd(gq, qconj(qmul(qconj(R["qd"]), gct)))
    gQR, gQD = normal_vjp(R, gq, gqd)
    gw, g_sr, g_sd = blend_vjp(bl, gQR, gQD, None)
    g_delta, axb, g_oq, g_ot, g_ig = skin_vjp(sk, bones, xt, gw, ge, drow, g_d2)
    gt = [_seqsum(axb[:, :, k], init=gt[k]) for k in range(3)]
    gqi, gxc = qrot_vjp(qi, xc, gt)
    gqn, gn = qrot_vjp(qi, nct, gt)
    out.update(go=_stack(go), g_xyz_cam=_stack(list(gxc)), g_delta=g_delta, g_oq=g_oq[None], g_ot=g_ot[None],
               g_ig=g_ig[None], g_sr=g_sr[None], g_sd=g_sd[None], g_cq=_stack(list(qconj(qadd(gqi, gqn))))[None],
               g_ct=_stack([-g for g in gn])[None])
    return out


def cycle_model(xyz, xyz_cam, tab, delta, weights, g_loss, chunk=2048):
    """cycle_fwd_kernel, cycle_scale_kernel and cycle_bwd_kernel.  xyz (P,3), xyz_cam (M,P,3), delta (M,P,B) or None,
    weights (3,), g_loss (fp32).  Returns dict: terms (M,3), loss, scale (3,) as _E, counts (M,3), knife (P,) (a knife in
    any frame), g_xyz (P,3), g_xyz_cam (M,P,3), g_delta (M,P,B) and the table gradients as _E."""
    P, M = xyz.shape[0], xyz_cam.shape[0]
    chunk = _rup(chunk, 256)
    spans = [(a, min(P, a + chunk)) for a in range(0, P, chunk)]

    def args(m, a, e):
        n = _rup(e - a, 256)
        return (m, _rows(xyz, a, e, n, 0), _rows(xyz_cam[m], a, e, n, 0), _rows(None if delta is None else delta[m], a, e, n, 0),
                tab)

    live = lambda a, e: np.arange(_rup(e - a, 256)) < e - a  # noqa: E731
    reds = [[Red(256) for _ in range(3)] for _ in range(M)]
    counts = np.zeros((M, 3), np.int64)
    knife = np.zeros(P, bool)
    for m in range(M):
        for a, e in spans:
            r = cycle_chunk(*args(m, a, e))
            lv = live(a, e)
            knife[a:e] |= r["knife"][:e - a]
            for k, key in enumerate(("cyc", "dsk", "ent")):
                t = r[key] if r[key].v.ndim else _E(np.zeros(len(lv)), None, np.zeros(len(lv), np.float32))
                on = lv & (t.v > 0)
                reds[m][k].add(_where(on, t, 0.0)[None])
                counts[m, k] += int(on.sum())
    tot = counts.sum(0)
    s = [(_scal(weights[k]) / _c(float(tot[k]))) if tot[k] else _E(0.0, None, np.float32(0)) for k in range(3)]
    terms = [[reds[m][k].result() * s[k] for k in range(3)] for m in range(M)]
    loss = ZERO
    for m in range(M):
        for k in range(3):
            loss = loss + terms[m][k]
    sc = [_scal(g_loss) * s[k] for k in range(3)]
    per = {k: [Red(128) for _ in range(M)] for k in ("oq", "ot", "sr", "sd", "cq", "ct")}
    ig = Red(128)
    gx, gxc, gd = [], [[] for _ in range(M)], [[] for _ in range(M)]
    for a, e in spans:
        lv = live(a, e)
        acc = None
        for m in range(M):
            r = cycle_chunk(*args(m, a, e), sc=sc)
            neg = -r["go"]
            acc = neg if acc is None else acc + neg          # g_xyz -= dL/dx_cycled, frame after frame
            gxc[m].append(r["g_xyz_cam"][:e - a])
            if delta is not None:
                gd[m].append(r["g_delta"][:e - a])
            for k in per:
                per[k][m].add(_dead(r["g_" + k], lv))
            ig.add(_dead(r["g_ig"], lv))
        gx.append(acc[:e - a])
    nb = sum(_rup(e - a, 256) for a, e in spans) // 128
    st = lambda es: _E(np.stack([e.v for e in es]), np.stack([e.b for e in es]), np.stack([e.f for e in es]))  # noqa: E731
    out = dict(terms=st([st(t) for t in terms]), loss=loss, scale=st(s), counts=counts, knife=knife, g_xyz=_cat(gx),
               g_xyz_cam=st([_cat(p) for p in gxc]), g_delta=None if delta is None else st([_cat(p) for p in gd]))
    for k in per:
        out["g_" + k] = st([r.result() for r in per[k]])
    out["g_ig"] = ig.result(L=5 + 4 * M + nb)
    return out


def _dead(t, lv):
    """Table terms of dead lanes are 0 (the kernel multiplies them by lv = 0 or gates them on `live`)."""
    shape = (1, len(lv)) + (1,) * (t.v.ndim - 2)
    keep = lv.reshape(shape)
    return _E(np.where(keep, t.v, 0.0), np.where(keep, t.b, 0.0), None if t.f is None else np.where(keep, t.f, np.float32(0)))


# ------------------------------------------------------------------------------------------------ scenes
def _tables(inp, cycle=False):
    import torch

    from vidu4d_b200.warp import cycle_tables, warp_tables

    from .reproj_model import q2dq
    with torch.no_grad():
        fn = cycle_tables if cycle else warp_tables
        oq, ot, ig, sr, sd = fn(q2dq(inp["rest_q"], inp["rest_t"]), q2dq(inp["art_q"], inp["art_t"]), inp["log_gauss"])
    return {k: np.ascontiguousarray(v.numpy(), np.float32) for k, v in
            dict(oq=oq, ot=ot, ig=ig, sr=sr, sd=sd, cq=inp["cam_q"], ct=inp["cam_t"]).items()}


def _inputs(seed, P, B, M, with_delta, wide):
    """The warp fixtures' articulations (make_warp_golden.make_inputs: narrow 0.03 bones), or with wide=True
    make_cycle_golden.make_case's 0.2 scales (a median surfel blends several bones)."""
    from tests.golden.make_cycle_golden import make_case
    from tests.golden.make_warp_golden import make_inputs
    return (make_case if wide else make_inputs)(seed, P, B, M, with_delta)


def warp_scene(seed, P, B, M, delta="small", wide=False):
    """bob_warp's inputs as the kernel sees them: fp32 tables from vidu4d_b200.warp.warp_tables, the surfels, delta
    (None, the fixtures' "small" one or 400 times it, "large", which decides many arg-maxes) and upstream gradients."""
    inp = _inputs(seed, P, B, M, delta is not None, wide)
    rng = np.random.default_rng(seed + 1)
    d = None if delta is None else (inp["delta"].numpy() * (1.0 if delta == "small" else 400.0)).astype(np.float32)
    up = dict(gx=rng.normal(size=(M, P, 3)).astype(np.float32), gr=rng.normal(size=(M, P, 4)).astype(np.float32),
              ge=rng.normal(size=P).astype(np.float32))
    return dict(xyz=inp["xyz"].numpy(), rot=inp["rot"].numpy(), tab=_tables(inp), delta=d, **up)


def reproj_scene(seed, M, HW, B, delta=True, wide=True, hs=3):
    """reproj_loss's inputs: the warp tables, constructed matched points (canonical surfels, no top-K), 100-pixel
    intrinsics that differ per frame, targets hxy scattered over the image, a mask of 0 and values in [0.5, 2] (pixel 0
    of every frame live: a dead lane of a ragged last block reads it), is_detected 1."""
    inp = _inputs(seed, M * HW, B, M, False, wide)
    rng = np.random.default_rng(seed + 2)
    f = np.array([[100.0, 0, 50.0], [0, 100.0, 40.0], [0, 0, 1]], np.float32)
    Kmat = np.stack([f + np.array([[0, 0, 0.5 * m], [0, 0, -0.3 * m], [0, 0, 0]], np.float32) for m in range(M)])
    hxy = np.concatenate([rng.uniform(0, 100, (M, HW, 2)), np.ones((M, HW, hs - 2))], -1).astype(np.float32)
    mask = ((rng.random((M, HW)) < 0.7) * rng.uniform(0.5, 2.0, (M, HW))).astype(np.float32)
    mask[:, 0] = 1.0
    d = (np.maximum(rng.normal(size=(M, HW, B)), 0.0) * 0.1).astype(np.float32) if delta else None
    return dict(xyz_m=inp["xyz"].numpy().reshape(M, HW, 3), delta=d, tab=_tables(inp), Kmat=Kmat, hxy=hxy, mask=mask,
                det=np.ones(M, np.float32), weight=np.float32(5e-2), train_res=256.0, g_loss=np.float32(0.75))


def cycle_scene(seed, P, B, M, delta=True):
    """cycle_loss's inputs: make_cycle_golden.make_case's wide bones, its tables from vidu4d_b200.warp.cycle_tables, and
    xyz_cam the float64 forward warp (oracle/warp_oracle.py) of the surfels, offset and rounded to fp32."""
    import torch

    from oracle import warp_oracle as wo

    from .reproj_model import q2dq
    inp = _inputs(seed, P, B, M, delta, True)
    t = {k: v.double() for k, v in inp.items() if v is not None}
    rest, art = q2dq(t["rest_q"], t["rest_t"]), q2dq(t["art_q"], t["art_t"])
    rest_m = (rest[0][None].expand(M, -1, -1), rest[1][None].expand(M, -1, -1))
    with torch.no_grad():
        xc, _, _ = wo.bob_warp(t["xyz"], t["rot"], rest, torch.exp(-t["log_gauss"]), wo.dq_mul(art, wo.dq_inverse(rest_m)),
                               (t["cam_q"], t["cam_t"]), t.get("delta"))
    # a camera-space offset of ~1e-2 keeps every cycle distance far above rounding, even where one bone dominates
    xc = xc.numpy() + 1e-2 * np.random.default_rng(seed + 3).normal(size=xc.shape)
    return dict(xyz=inp["xyz"].numpy(), xyz_cam=xc.astype(np.float32), tab=_tables(inp, cycle=True),
                delta=None if not delta else inp["cdelta"].numpy(), weights=np.array([0.01, 5e-3, 5e-4], np.float32),
                g_loss=np.float32(0.75))
