"""TEST INFRASTRUCTURE -- the global match (csrc/match.cu match_fwd, match_bwd, match_scatter) restated operation for
operation, with its rounding-error bound.

Every value is a running-error value (tests/error_bound.py): its float64 value, its bound B (units of u = 2^-24) and an
fp32 shadow.  The tests hold the GPU (and, on the CPU, the shadow) to |x - value| <= K u B + FLOOR, with K = 2.

  * score: f0 a0, then 15 FMAs in channel order, each charged two roundings (a contracted a*b + c rounds once).
  * top-K, as data: the float64 order is larger score first, the lower candidate position first on exact ties (two
    copies of one surfel score bit-identically on both sides).  A pixel is a knife pixel when two neighbours of that
    order among its first K + 1 (the K-th / (K+1)-th, or two adjacent members: the order is an output) differ by more
    than 0 and at most K u (B_i + B_j).  Outside knife pixels the kernel's list must be the float64 list, in order; at
    knife pixels it must be a valid top-K in order within the bound.  Invalid positions (< 0 or >= M P) are never
    chosen; slots beyond the valid count are -1, with prob 0 and score 0.
  * the rest of the forward and the whole backward are evaluated on the kernel's own list, so knife pixels need no
    masking of values: tau = expf(logsigma), mx = v0 tau, e_j = expf(v_j tau - mx), Z in order, iz = 1 / Z (0 when no
    candidate is valid, so Z = 0), p = e iz, the xyz sums in order; gp_k, dot in order, ds = p (gp - dot), gs = ds tau,
    gs f_c, p g, and glog = ds tau v.
    The backward takes p and the score as inputs (the GPU's own buffers on the GPU, the forward's values on the CPU).
  * reductions beyond one thread add m u sum|t| for m adds in any order: a (candidate, channel) row of g_cand its
    choosing pixels plus one global add per CTA that flushes it (the same form covers the kernel that adds straight to
    g_cand); g_logsigma K adds per strided pass, 5 shuffle levels, 32 warps, then one atomic per CTA; match_scatter the
    candidate positions sharing a surfel.  CTA counts are bounded by the host's grid, min(ceil(N / 1024), 2 SMs).
"""
import numpy as np

from .error_bound import _E, _where

U = 2.0 ** -24
K = 2.0
FLOOR = float(np.finfo(np.float32).tiny)
FEAT = 16
ROW = FEAT + 3
BWD_THREADS = 1024


def _leaf(a):
    return _E.leaf(np.asarray(a, np.float32))


def _gather(e, idx):
    """Per row n, e[n, idx[n, k]] of an (N, C) value: (N, K)."""
    t = lambda a: np.take_along_axis(a, idx, 1)  # noqa: E731
    return _E(t(e.v), t(e.b), None if e.f is None else t(e.f))


def valid_positions(cand, MP):
    return (cand >= 0) & (cand < MP)


def scores(feat, rf, cand, MP):
    """The (N, C) score chain of every pixel against every candidate row; invalid positions read row 0 (masked later)."""
    P = rf.shape[0]
    ok = valid_positions(cand, MP)
    rows = rf[np.where(ok, cand, 0).astype(np.int64) % P]
    s = _leaf(feat[:, None, 0]) * _leaf(rows[None, :, 0])
    for c in range(1, FEAT):
        s = _leaf(feat[:, None, c]) * _leaf(rows[None, :, c]) + s
    return s


def topk(s, cand, MP, Kn):
    """The float64 top-K lists (N, Kn) (-1 beyond the valid count), the knife mask (N,) and the number of valid
    candidates."""
    ok = valid_positions(cand, MP)
    N, C = s.v.shape
    nv = int(ok.sum())
    key = np.where(ok[None], s.v, -np.inf)
    pos = np.broadcast_to(np.arange(C), key.shape)
    order = np.lexsort((pos, -key), axis=-1)
    kv = min(Kn, nv)
    want = np.full((N, Kn), -1, np.int64)
    want[:, :kv] = order[:, :kv]
    L = min(Kn + 1, nv)
    sv, sb = np.take_along_axis(s.v, order[:, :L], 1), np.take_along_axis(s.b, order[:, :L], 1)
    gap = sv[:, :-1] - sv[:, 1:]
    knife = ((gap > 0) & (gap <= K * U * (sb[:, :-1] + sb[:, 1:]))).any(1) if L > 1 else np.zeros(N, bool)
    return want, knife, nv


def check_topk(s, cand, MP, Kn, idx):
    """Asserts the kernel's lists idx (N, Kn) against the float64 choice.  Returns (knife mask, float64 lists)."""
    want, knife, nv = topk(s, cand, MP, Kn)
    N, C = s.v.shape
    kv = min(Kn, nv)
    assert ((idx >= -1) & (idx < C)).all()
    assert (idx[:, kv:] == -1).all(), "slots beyond the valid count must be -1"
    if kv == 0:                                      # no valid candidate: every slot is empty
        return np.zeros(N, bool), want
    ch = idx[:, :kv]
    assert (ch >= 0).all(), "a valid slot holds no candidate"
    ok = valid_positions(cand, MP)
    assert ok[ch].all(), "an invalid candidate position was chosen"
    assert (np.diff(np.sort(ch, 1), axis=1) != 0).all(), "a candidate was chosen twice"
    bad = ~knife & (idx != want).any(1)
    assert not bad.any(), ("top-K differs from the float64 order at non-knife pixel", int(np.argmax(bad)),
                           idx[np.argmax(bad)], want[np.argmax(bad)])
    # valid within the bound: no unchosen candidate beats a chosen one by more than K u (B_i + B_j), and the list is in
    # order within the same bound
    lo = s.v - K * U * s.b
    hi = s.v + K * U * s.b
    chosen = np.zeros((N, C), bool)
    np.put_along_axis(chosen, ch, True, 1)
    rest = np.where(ok[None] & ~chosen, lo, -np.inf).max(1)
    assert (rest <= np.take_along_axis(hi, ch, 1).min(1)).all(), "not a top-K within the bound"
    cv, cb = np.take_along_axis(s.v, ch, 1), np.take_along_axis(s.b, ch, 1)
    assert (np.diff(cv, axis=1) <= K * U * (cb[:, 1:] + cb[:, :-1])).all(), "top-K out of order beyond the bound"
    return knife, want


def forward(s, idx, cand, xyz, logsigma):
    """match_fwd's arithmetic on the lists idx (N, Kn).  Returns dict(score, prob, xyz_matched (3 (N,) values), tau)."""
    P = xyz.shape[0]
    ok = idx >= 0
    pos = np.where(ok, idx, 0)
    sc = _gather(s, pos)
    sc = _where(ok, sc, 0.0)
    tau = _leaf(np.reshape(logsigma, ())).exp()
    mx = sc[:, 0] * tau
    arg = sc * tau - _E(mx.v[:, None], mx.b[:, None], None if mx.f is None else mx.f[:, None])
    e = _where(ok, arg.exp(), 0.0)
    Z = e[:, 0]
    for j in range(1, idx.shape[1]):
        Z = Z + e[:, j]
    iz = _where(Z.v > 0, _E(1.0, None, np.float32(1.0)) / Z, 0.0)     # Z = 0 only without a valid candidate
    p = e * _E(iz.v[:, None], iz.b[:, None], None if iz.f is None else iz.f[:, None])
    sidx = np.where(ok, cand[pos].astype(np.int64) % P, 0)
    out = []
    for a in range(3):
        x = _where(ok, _leaf(xyz[sidx, a]), 0.0)
        o = p[:, 0] * x[:, 0]
        for j in range(1, idx.shape[1]):
            o = p[:, j] * x[:, j] + o
        out.append(o)
    return dict(score=sc, prob=p, xyz_matched=out, tau=tau)


def grid_max(N, sms):
    """The largest grid the host launches for match_bwd: ceil(N / 1024) CTAs, at most 2 per SM."""
    return max(1, min(-(-N // BWD_THREADS), 2 * sms))


def _keyed_sum(t, keys, n, m_of_count):
    """Sum of terms t (T, W) into n rows by keys (T,), in any order: value, bound sum t.b + m u sum|t| with m given per
    row by m_of_count(count), and a float32 shadow (one sequential order)."""
    W = t.v.shape[1]
    v = np.zeros((n, W))
    b = np.zeros((n, W))
    a = np.zeros((n, W))
    np.add.at(v, keys, t.v)
    np.add.at(b, keys, t.b)
    np.add.at(a, keys, np.abs(t.v))
    cnt = np.bincount(keys, minlength=n).astype(np.float64)
    f = None
    if t.f is not None:
        f = np.zeros((n, W), np.float32)
        np.add.at(f, keys, t.f)
    return _E(v, b + m_of_count(cnt)[:, None] * a, f), cnt


def backward(feat, idx, p, sc, g, cand, xyz, logsigma, C, sms):
    """match_bwd's arithmetic on the lists idx (N, Kn), with p and sc (N, Kn) values (the GPU's fp32 buffers as leaves,
    or the forward's values).  Returns dict(g_cand (C, 19), g_logsigma (), live (N,) pixels with nonzero upstream,
    users (C,) the live (pixel, slot) pairs that chose each position)."""
    N, Kn = idx.shape
    P = xyz.shape[0]
    live = (g != 0).any(1)
    ok = (idx >= 0) & live[:, None]
    pos = np.where(ok, idx, 0)
    sidx = np.where(ok, cand[pos].astype(np.int64) % P, 0)
    tau = _leaf(np.reshape(logsigma, ())).exp()
    gx, gy, gz = (_leaf(g[:, None, a]) for a in range(3))
    X = [_leaf(xyz[sidx, a]) for a in range(3)]
    gp = _where(ok, (gx * X[0] + gy * X[1]) + gz * X[2], 0.0)
    p = _where(ok, p, 0.0)
    sc = _where(ok, sc, 0.0)
    dot = p[:, 0] * gp[:, 0]
    for k in range(1, Kn):
        dot = p[:, k] * gp[:, k] + dot
    ds = p * (gp - _E(dot.v[:, None], dot.b[:, None], None if dot.f is None else dot.f[:, None]))
    gs = ds * tau
    tl = gs * sc
    G = grid_max(N, sms)
    # g_logsigma: per thread K adds per strided pass, 5 shuffle levels, 32 warps, one atomic per CTA
    passes = -(-N // BWD_THREADS)
    m = Kn * passes + 5 + BWD_THREADS // 32 + G
    tlv = np.where(ok, tl.v, 0.0)
    glog = _E(tlv.sum(), np.where(ok, tl.b, 0.0).sum() + m * np.abs(tlv).sum(),
              None if tl.f is None else np.float32(np.where(ok, tl.f, 0).astype(np.float32).sum(dtype=np.float32)))
    # g_cand: one term per live (pixel, slot) and channel
    cols = [gs * _leaf(feat[:, None, c]) for c in range(FEAT)] + [p * gx, p * gy, p * gz]
    sel = ok.reshape(-1)
    stack = lambda get: np.stack([get(c).reshape(-1)[sel] for c in cols], 1)  # noqa: E731
    has_f = all(c.f is not None for c in cols)
    terms = _E(stack(lambda c: c.v), stack(lambda c: c.b), stack(lambda c: c.f) if has_f else None)
    gc, users = _keyed_sum(terms, pos.reshape(-1)[sel], C, lambda n: n + np.minimum(n, G))
    return dict(g_cand=gc, g_logsigma=glog, live=live, users=users)


def scatter(gc, cand, MP, P):
    """match_scatter: rows of g_cand (C, 19) values (the GPU's buffer as leaves on the GPU) added at cand mod P.
    Returns (g_regist_feat (P, 16), g_xyz (P, 3))."""
    ok = valid_positions(cand, MP)
    keys = cand[ok].astype(np.int64) % P
    t = gc[ok]
    out, _ = _keyed_sum(t, keys, P, lambda n: n)
    return out[:, :FEAT], out[:, FEAT:]


# ------------------------------------------------------------------------------------------------ scenes
def scene(seed, M, H, W, P, C, Kn, scale=1.0, logsigma=np.log(2.0), invalid=(), dup=0, hot=(), masked=0.3, weight=1.0):
    """Inputs of one case.  invalid: candidate positions holding an index outside [0, M P) (alternating -1 and M P);
    dup: number of surfels drawn twice (idx and idx + P); hot: positions whose surfel gets a large feature, so that
    many pixels choose it; masked: the fraction of pixels with zero upstream gradient."""
    rng = np.random.default_rng(seed)
    N = M * H * W
    feat = (rng.normal(size=(N, FEAT)) * scale).astype(np.float32)
    rf = (rng.normal(size=(P, FEAT)) * scale).astype(np.float32)
    xyz = rng.normal(size=(P, 3)).astype(np.float32)
    cand = rng.permutation(M * P)[:C].astype(np.int64)
    if dup:
        assert M >= 2
        base = rng.choice(P, size=dup, replace=False)
        at = rng.choice(C, size=2 * dup, replace=False)
        cand[at[:dup]], cand[at[dup:]] = base, base + P
        rest = np.setdiff1d(np.arange(C), at)
        pool = np.setdiff1d(np.arange(M * P), np.concatenate([base, base + P]))
        cand[rest] = rng.choice(pool, size=len(rest), replace=False)
    for i, c in enumerate(invalid):
        cand[c] = -1 if i % 2 else M * P + 7 * i
    for c in hot:
        rf[cand[c] % P] = (rng.normal(size=FEAT) * 4.0 * scale).astype(np.float32)
    if dup:
        rf[cand[at[0]] % P] = (rng.normal(size=FEAT) * 4.0 * scale).astype(np.float32)
    g = (rng.normal(size=(N, 3)) * weight).astype(np.float32)
    g[rng.random(N) < masked] = 0.0
    return dict(M=M, H=H, W=W, P=P, C=C, K=Kn, feat=feat, rf=rf, xyz=xyz, cand=cand.astype(np.int32),
                logsigma=np.array([logsigma], np.float32), g=g, dup_at=(at[0], at[dup]) if dup else None)


def model(s, sms, idx=None, prob=None, score=None):
    """The bound model of one scene.  idx / prob / score: the kernel's lists and buffers (N, K); without them the float64
    lists and the forward's own values are used.  Returns dict with the score matrix, knife mask, forward and backward."""
    MP = s["M"] * s["P"]
    sc = scores(s["feat"], s["rf"], s["cand"], MP)
    if idx is None:
        want, knife, _ = topk(sc, s["cand"], MP, s["K"])
        idx = want
    else:
        knife, want = check_topk(sc, s["cand"], MP, s["K"], idx)
    fw = forward(sc, idx, s["cand"], s["xyz"], s["logsigma"])
    p = fw["prob"] if prob is None else _leaf(prob)
    v = fw["score"] if score is None else _leaf(score)
    bw = backward(s["feat"], idx, p, v, s["g"], s["cand"], s["xyz"], s["logsigma"], s["C"], sms)
    return dict(scores=sc, idx=idx, want=want, knife=knife, fwd=fw, bwd=bw)
