"""TEST INFRASTRUCTURE -- Stage 3's per-surfel feature rows (csrc/feature_rows.cu: frows_absmax, frows_fwd, frows_bwd_sum,
frows_bwd) restated operation for operation, with their rounding-error bound.

Every value is a running-error value (tests/error_bound.py): its float64 value, its bound B (units of u = 2^-24) and an
fp32 shadow, evaluated in the kernels' order on their fp32 inputs.  The tests hold the GPU (and, on the CPU, the shadow)
to |x - value| <= K u B + FLOOR, with K = 2.

Exact values.  The projection, the flow, the density's r2 and the flow channels use __fmul_rn / __fadd_rn / __fsub_rn /
__fdiv_rn only: every result is correctly rounded and nothing is contracted, so the float32 NumPy shadow of project(),
of the flow, of max|flow| (an integer max on the bit pattern), of s = sm + 1e-6f, of the counts hi and lo of the flow
values equal to +sm and -sm, and of the flow channels f / s is the GPU's result bit for bit.  The shadow's tie set is
then data for the backward's routing of dL/ds, as the match model takes the kernel's own top-K lists.

Charges.
  * normal: two qrot calls, which nvcc may contract: two roundings per FMA (every product and sum is charged).
  * density: r2 from _rn ops; expf its 2 ulp, plus an absolute 2^-148 wherever the score is subnormal (the build has no
    -ftz, so subnormal scores survive and a relative charge understates their error); one rounding for the product with
    beta.  The constants 1e-4f (0.01^2) and 1e-6f are the float64 constants of tests/feature_rows_model.py with their
    fp32 rounding charged (error_bound._E.const).
  * backward: gflow = __fdiv_rn(g, s) plus the tie shares; G = g_s - acc / rn(s s), g_hi and g_lo with the halving,
    sgn_min and the division by the counts; project_vjp with plain / and FMAs; normal_vjp as two qrot_vjp; g_regist and
    dL/d(density) as in-thread sums over the frames; g_xyz the g_r2 chain at the first arg-max bone.
  * reductions beyond one thread add m u sum|t| for m adds in any order, with m from the kernels' constants (256-thread
    CTAs, 8 warps): frows_bwd_sum an in-thread sum over frame pairs, a 5-level xor tree, 8 sequential warp adds, one
    global atomic per CTA; acc_q / acc_table (g_cam_q, g_beta) a 5-level xor tree, shared-memory atomics from 8 warps,
    one global atomic per CTA; g_centres one shared-memory atomic per live thread (the largest count of one CTA's
    threads on one bone, in any order), then one global atomic per CTA.

Knife rules.
  * density arg-max: the top two float64 scores differ by more than 0 and at most K u (B1 + B2), and the top score is
    not itself within its bound of 0 (a score that has underflowed decides nothing the bound can see).  Such a surfel's
    density and g_xyz are not compared; its score is charged B1 + 2 B2 (the GPU may hold the runner-up's score) and
    |term| of both candidate bones is added to those bones' g_centres bounds: the term is not dropped.  An exact float64
    tie is not a knife: both sides take the first index.
  * projection: a surfel-frame with u B(v2) > 1/64 |v2|.  Its pair's flow and g_xyz_cam are not compared; if it holds
    the max |flow|, nothing that depends on s is.
"""
import numpy as np

from .error_bound import _E, _c, _seqsum, _where
from .skin_bounds import FLOOR, K, U, Red, _ill, _knife_close, _pad, _rup, _stack, qrot, qrot_vjp

THREADS = 256
R2 = 1e-4                                  # 0.01^2 (the kernel's FR_R2 = 1e-4f)
EPS = 1e-6                                 # the flow scale's epsilon (FR_EPS = 1e-6f)
TINY = float(np.finfo(np.float32).tiny)
SUB = 2.0 ** -148 / U                      # expf's absolute error on a subnormal result, in units of u
ZERO = _E(0.0, None, np.float32(0.0))


def _leaf(a):
    return _E.leaf(np.asarray(a, np.float32))


def _ap(e, fn):
    """fn applied to value, bound and shadow alike (a reshape or a gather)."""
    return _E(fn(e.v), fn(e.b), None if e.f is None else fn(e.f))


def partner(M):
    """The flow partner of every frame: m xor 1, or the frame itself when M = 1."""
    return np.arange(M) ^ 1 if M > 1 else np.zeros(1, np.int64)


def project_f32(Kmat, xyz_cam):
    """pi(K, x) in plain float32 NumPy, each operation rounded once, as project() computes it: (M,P) u0, u1."""
    Kf, x = np.asarray(Kmat, np.float32), np.asarray(xyz_cam, np.float32)
    row = [(Kf[:, i, 0, None] * x[..., 0] + Kf[:, i, 1, None] * x[..., 1]) + Kf[:, i, 2, None] * x[..., 2] for i in range(3)]
    return row[0] / row[2], row[1] / row[2]


def flow_f32(Kmat, xyz_cam):
    """The kernels' flow (M,P,2) in plain float32 NumPy: b.u - a.u for the pair's first frame, its negation for the
    second."""
    pm = partner(Kmat.shape[0])
    f = np.stack([u[pm] - u for u in project_f32(Kmat, xyz_cam)], -1)
    odd = (np.arange(Kmat.shape[0]) % 2 == 1)[:, None, None]
    return np.where(odd, -f[pm], f)


def project(Kmat, xyz_cam):
    x = [_leaf(xyz_cam[..., j]) for j in range(3)]
    k = lambda i, j: _leaf(Kmat[:, i, j][:, None])  # noqa: E731
    v = [(k(i, 0) * x[0] + k(i, 1) * x[1]) + k(i, 2) * x[2] for i in range(3)]
    return v, (v[0] / v[2], v[1] / v[2])


def _reduce(t, P):
    """A per-thread term (P, *slot) through acc_table / acc_q or frows_bwd_sum's block sum: 5 xor levels, 8 warp adds,
    one global atomic per CTA (dead lanes add zeros)."""
    r = Red(THREADS)
    r.add(_pad(_ap(t, lambda a: a[None]), _rup(P, THREADS)))
    return r.result()


def _centre_sum(gd, arg, B, P):
    """g_centres: -gd (3 (P,) values) added at bone arg[p]: one shared-memory atomic per thread, then one global atomic
    per CTA.  Returns an _E (B,3)."""
    cta = np.arange(P) // THREADS
    nb = int(cta.max()) + 1 if P else 0
    cnt = np.zeros((max(nb, 1), B))
    np.add.at(cnt, (cta, arg), 1.0)
    L = cnt.max(0) + nb
    v, b, a = np.zeros((B, 3)), np.zeros((B, 3)), np.zeros((B, 3))
    f = np.zeros((B, 3), np.float32)
    for k in range(3):
        t = -gd[k]
        np.add.at(v[:, k], arg, t.v)
        np.add.at(b[:, k], arg, t.b)
        np.add.at(a[:, k], arg, np.abs(t.v))
        np.add.at(f[:, k], arg, t.f)
    return _E(v, b + L[:, None] * a, f)


def model(s):
    """The bound model of one scene (see scene()).  Returns a dict of _E values, the exact fp32 data (sm, hi, lo, the tie
    masks) and the knife masks."""
    P, M, B, Cf = s["P"], s["M"], s["B"], s["Cf"]
    pm = partner(M)
    out = dict(P=P, M=M, B=B, Cf=Cf)
    # ---- frows_absmax / frows_fwd: the flow and its scale (exact: the shadow is the GPU's bits)
    v, (u0, u1) = project(s["Kmat"], s["xyz_cam"])
    # a pair with bit-identical K and xyz_cam (M = 1, the static pair) projects to the same bits: its flow is exactly 0
    same = (s["Kmat"][pm] == s["Kmat"]).all((1, 2))[:, None] & (s["xyz_cam"][pm] == s["xyz_cam"]).all(-1)
    fl = [_where(same, ZERO, u[pm] - u) for u in (u0, u1)]              # (M,P): pi(K_m1, x_m1) - pi(K_m, x_m) ...
    odd = (np.arange(M) % 2 == 1)[:, None]
    fl = [_where(odd, -f[pm], f) for f in fl]                            # ... and frame m1's is minus frame m's (-0 too)
    F = _stack(fl)                                                       # (M,P,2)
    smf = np.float32(np.abs(F.f).max()) if P else np.float32(0.0)
    sm = _E(np.abs(F.v).max() if P else 0.0, F.b.max() if P else 0.0, smf)
    sE = sm + _E.const(EPS)
    hi_m, lo_m = F.f == smf, F.f == -smf
    hi, lo = int(hi_m.sum()), int(lo_m.sum())
    assert max(hi, lo) < 2 ** 24, "the counts are converted to float exactly only below 2^24"
    out.update(flow=F, sm=smf, s=sE, hi=hi, lo=lo, hi_m=hi_m, lo_m=lo_m, flow_ch=F / sE)
    # projection knife: an ill-conditioned v2 taints its pair's flow; if it holds the max, everything that depends on s
    pk = _ill(v[2])
    pkp = pk | pk[pm]
    tied = (hi_m | lo_m).any(-1)
    out["pknife"] = pkp
    out["s_bad"] = bool((pkp & tied).any())
    # ---- the normal: cam_q[m] applied to rot_cam[m,p] applied to e_x or e_y
    ay = s["scaling"][:, 1] < s["scaling"][:, 0]
    axis = (_c(np.where(ay, 0.0, 1.0).astype(np.float32)[None]), _c(ay.astype(np.float32)[None]), ZERO)
    r = tuple(_leaf(s["rot_cam"][..., i]) for i in range(4))
    cq = tuple(_leaf(s["cam_q"][:, i, None]) for i in range(4))
    rv = qrot(r, axis)
    out["normal"] = _stack(list(qrot(cq, rv)))                          # (M,P,3)
    out["axis_y"] = ay
    # ---- the density: max_b exp(-0.5 r2 / R2) at the first arg-max, times beta
    xyz, cen = s["xyz"], s["centres"]
    d = [_leaf(xyz[:, None, k]) - _leaf(cen[None, :, k]) for k in range(3)]          # (P,B)
    r2 = (d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]
    sc = (r2 / _E.const(R2)).scale(-0.5).exp()
    sc = _E(sc.v, sc.b + np.where(sc.v < 2 * TINY, SUB, 0.0), sc.f)
    arg = np.argmax(sc.v, 1) if P else np.zeros(0, np.int64)
    take = lambda e, i: _ap(e, lambda a: np.take_along_axis(a, i[:, None], 1)[:, 0])  # noqa: E731
    best = take(sc, arg)
    dknife = np.zeros(P, bool)
    second = arg
    if B > 1 and P:
        o = np.argsort(-sc.v, 1, kind="stable")
        second = o[:, 1]
        sec = take(sc, second)
        dknife = _knife_close(_E(best.v - sec.v, best.b + sec.b)) & (best.v > K * U * best.b)
        best = _E(best.v, np.where(dknife, best.b + 2.0 * sec.b, best.b), best.f)
    beta = _leaf(np.reshape(s["beta"], ()))
    out.update(score=best, arg=arg, second=second, dknife=dknife, density=best * beta, subnormal=best.v < TINY)
    if P == 0:
        return out
    # ---- frows_bwd_sum: acc = sum of g_row_flow * flow
    gr = s["g_rows"]
    gq = [_leaf(gr[..., Cf + c]) for c in range(2)]
    acc_t = None
    for m in range(0, M, 2):
        m1 = pm[m]
        t = gq[0][m] * fl[0][m] + gq[1][m] * fl[1][m]
        acc_t = t if acc_t is None else acc_t + t
        if m1 != m:
            acc_t = acc_t - (gq[0][m1] * fl[0][m] + gq[1][m1] * fl[1][m])
    acc = _reduce(acc_t, P)
    out["acc"] = acc
    # ---- frows_bwd: dL/ds routed over the tied elements as torch's autograd routes it
    q = -(acc / (sE * sE))
    G = q if s["g_s"] is None else _leaf(s["g_s"]) + q
    half = G.scale(0.5)
    g_hi = ((half if lo else G) / _c(float(hi))) if hi else ZERO
    g_lo = ((half if hi else G).scale(-1.0 if smf > 0 else 0.0) / _c(float(lo))) if lo else ZERO
    gf = []
    for c in range(2):
        x = gq[c] / sE
        x = _where(hi_m[..., c], x + g_hi, x)
        x = _where(lo_m[..., c], x + g_lo, x)
        gf.append(x[pm] - x)                                              # dL/dpi_m = g_flow[m1] - g_flow[m]
    gv = [gf[0] / v[2], gf[1] / v[2], -(gf[0] * u0 + gf[1] * u1) / v[2]]
    k = lambda i, j: _leaf(s["Kmat"][:, i, j][:, None])  # noqa: E731
    out["g_xyz_cam"] = _stack([(k(0, j) * gv[0] + k(1, j) * gv[1]) + k(2, j) * gv[2] for j in range(3)])
    # a tainted flow (projection knife) reaches acc, hence G and every tied element's share
    mask = pkp.copy()
    if pkp.any():
        mask |= tied | tied[pm]
    if out["s_bad"]:
        mask[:] = True
    out["g_xyz_cam_mask"] = mask
    # normal_vjp
    gn = tuple(_leaf(gr[..., Cf + 2 + i]) for i in range(3))
    gcq, gvn = qrot_vjp(cq, rv, gn)
    grc, _ = qrot_vjp(r, axis, gvn)
    out["g_rot_cam"] = _stack(list(grc))
    out["g_cam_q"] = _reduce(_ap(_stack(list(gcq)), lambda a: np.moveaxis(a, 0, 1)), P)           # (M,4)
    # regist and dL/d(density): in-thread sums over the frames, in frame order
    out["g_regist"] = _seqsum(_leaf(np.moveaxis(gr[..., :Cf], 0, -1)), axis=-1)
    g_dens = _seqsum(_leaf(gr[..., Cf + 5].T), axis=-1, init=None if s["g_density"] is None else _leaf(s["g_density"]))
    out["g_beta"] = _reduce(g_dens * best, P)
    g_r2 = (((g_dens * beta) * best).scale(-0.5) / _E.const(R2)).scale(2.0)
    gd = [take(d[j], arg) * g_r2 for j in range(3)]
    out["g_xyz"] = _stack(gd)
    gc = _centre_sum(gd, arg, B, P)
    if dknife.any():                          # the GPU may route a knife surfel's term to either bone: charge both
        ext = np.zeros((B, 3))
        for j in range(3):
            for bone in (arg, second):
                t = take(d[j], bone) * g_r2
                np.add.at(ext[:, j], bone[dknife], (np.abs(t.v) + K * U * t.b)[dknife])
        gc = _E(gc.v, gc.b + ext / (K * U), gc.f)
    out["g_centres"] = gc
    return out


# ------------------------------------------------------------------------------------------------ scenes
def _unit(rng, shape):
    q = rng.normal(size=shape + (4,))
    return q / np.linalg.norm(q, axis=-1, keepdims=True)


def scene(seed, P, M, B, Cf, *, shift=0.05, dup=False, single_max=False, static=False, far=0.0, sub=0.0, eq_scale=0.0,
          bone_dup=False, bone_knife=False, g_s=True, g_density=True):
    """The kernels' fp32 inputs and upstream gradients, from seeded NumPy.

    Bones sit on a jittered grid of spacing 0.5; three quarters of the surfels (the rest of those not placed by the
    options) lie within ~0.01 of a bone.  Frame m1 = m xor 1 sees each surfel at its frame-m position plus `shift`-sized
    noise, so flows are a few pixels.  Options: dup, the surfel holding max |flow| copied onto another (ties at both
    extremes); single_max, one surfel's partner frame moved by 5 so that it alone holds the max and every other
    flow / s is small; static, paired frames with equal K and xyz_cam (sm = 0); far, the fraction of surfels 0.6 away
    from every bone (the score underflows to 0); sub, the fraction at 0.133-0.142 from one bone (a subnormal score);
    eq_scale, the fraction with equal tangent scales; bone_dup, bone 1 a copy of bone 0; bone_knife, bones 0 and 1
    mirrored about a plane that a quarter of the surfels lie on or within ~1e-10 of; g_s, g_density: whether those
    upstream gradients are given (None: a NULL pointer)."""
    rng = np.random.default_rng(seed)
    g = np.stack(np.meshgrid(*[np.arange(4)] * 3, indexing="ij"), -1).reshape(-1, 3)[rng.permutation(64)[:B]]
    cen = (g * 0.5 - 0.75 + 0.02 * rng.normal(size=(B, 3)))
    if bone_dup and B > 1:
        cen[1] = cen[0]
    if bone_knife and B > 1:                  # mirrored about x = 0, where offsets of 1e-10 are representable
        cen[0] = (-2.0 ** -8, 0.5, -0.25)
        cen[1] = (2.0 ** -8, 0.5, -0.25)
    cen = cen.astype(np.float32)
    b = rng.integers(0, B, P)
    xyz = cen[b] + 0.008 * rng.normal(size=(P, 3))
    kind = rng.random(P)
    if far:                                   # outside the grid: >= 1 from every bone
        xyz[kind < far] = (2.0, 2.0, 2.0) + 0.1 * rng.normal(size=(int((kind < far).sum()), 3))
    if sub:
        sel = (kind >= far) & (kind < far + sub)
        dirn = rng.normal(size=(int(sel.sum()), 3))
        dirn /= np.linalg.norm(dirn, axis=1, keepdims=True)
        xyz[sel] = cen[b[sel]] + dirn * rng.uniform(0.133, 0.142, (int(sel.sum()), 1))
    if bone_knife and B > 1:
        sel = kind > 0.75
        n = int(sel.sum())
        xyz[sel] = np.stack([np.where(rng.random(n) < 0.5, 0.0, 3e-10 * rng.uniform(-1, 1, n)),
                             0.5 + 0.004 * rng.normal(size=n), -0.25 + 0.004 * rng.normal(size=n)], 1)
    xyz = xyz.astype(np.float32)
    sc = np.exp(-4.0 + 0.5 * rng.normal(size=(P, 2)))
    if eq_scale:
        e = rng.random(P) < eq_scale
        sc[e, 1] = sc[e, 0]
    Kf = np.zeros((M, 3, 3))
    Kf[:, 0, 0] = 280 + 40 * rng.random(M)
    Kf[:, 1, 1] = 280 + 40 * rng.random(M)
    Kf[:, 0, 2] = 128 + 4 * rng.normal(size=M)
    Kf[:, 1, 2] = 128 + 4 * rng.normal(size=M)
    Kf[:, 2, 2] = 1.0
    xc = np.empty((M, P, 3))
    xc[0::2] = rng.normal(size=((M + 1) // 2, P, 3)) * 0.4 + (0.0, 0.0, 2.5)
    if M > 1:
        xc[1::2] = xc[0::2] + shift * rng.normal(size=(M // 2, P, 3))
    if single_max and M > 1:
        xc[1, P // 2] += (4.0, -3.0, 0.0)
    if static and M > 1:
        xc[1::2] = xc[0::2]
        Kf[1::2] = Kf[0::2]
    Kmat = Kf.astype(np.float32)
    xyz_cam = xc.astype(np.float32)
    if static:
        xyz_cam[1::2] = xyz_cam[0::2]
    rot_cam = (_unit(rng, (M, P)) * (1.0 + 0.05 * rng.normal(size=(M, P, 1)))).astype(np.float32)
    cam_q = (_unit(rng, (M,)) * (1.0 + 0.05 * rng.normal(size=(M, 1)))).astype(np.float32)
    regist = rng.normal(size=(P, Cf)).astype(np.float32)
    beta = np.array([np.exp(4.6 + 0.1 * rng.normal())], np.float32)
    W = Cf + 6
    g_rows = rng.normal(size=(M, P, W)).astype(np.float32)
    g_rows[..., Cf:Cf + 2] *= 0.01
    s = dict(P=P, M=M, B=B, Cf=Cf, regist=regist, xyz=xyz, scaling=sc.astype(np.float32), xyz_cam=xyz_cam, rot_cam=rot_cam,
             Kmat=Kmat, cam_q=cam_q, centres=cen, beta=beta, g_rows=g_rows,
             g_density=rng.normal(size=P).astype(np.float32) if g_density else None,
             g_s=np.array(rng.normal() * 3.0, np.float32) if g_s else None)
    if dup and P > 1:
        u0, u1 = project_f32(Kmat, xyz_cam)
        pm = partner(M)
        fa = np.maximum(np.abs(u0[pm] - u0), np.abs(u1[pm] - u1)).max(0)
        p = int(np.argmax(fa))
        q = (p + P // 2) % P
        for key in ("regist", "xyz", "scaling"):
            s[key][q] = s[key][p]
        for key in ("xyz_cam", "rot_cam"):
            s[key][:, q] = s[key][:, p]
        s["dup_pair"] = (p, q)
    return s
