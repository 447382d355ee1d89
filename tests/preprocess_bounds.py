"""TEST INFRASTRUCTURE -- the forward preprocess (csrc/preprocess.cu preprocess_fwd_kernel) restated for one frame in
float64, with a first-order rounding-error bound per output (tests/error_bound.py's _E) and an fp32 shadow.

The restatement follows the kernel's operation tree: the fp32 intrinsics (api.cu make_cam for scalar tangents,
common.cuh cam_of_frame for a per-frame table row), rot_matrix with rsqrtf charged its 2 ulp, w_mul, the view-space
position, M0, M1, the normal and cosv with its flip, T[0..8], computeAABB (d, 1/d, the centre, nq, the extents), the
radius (max, the 0.7071 floor and ceil(3e) in double), get_rect, the tile area, sh_to_rgb for every degree and the
clamp.  Every written multiply and add is charged one rounding, so the bound holds for whichever products nvcc contracts
into FMAs (sh_to_rgb is left to the compiler's contraction); sqrtf and / are correctly rounded (no --use_fast_math).
An operation on exact operands whose result is an fp32 value is not charged, so a scene built on exact values (a
view matrix of 0 and +-1, quaternions (w, 0, 0, 0)) reaches a decision such as cosv == 0 or d == 0 exactly.

model() returns, per surfel,
  * float fields with bounds (value v, bound b in units of u = 2^-24, fp32 shadow f): T (9), the centre (2), the
    normal after the flip (3), rgb (3) and the depth;
  * exact fields: visible, radius, the tile rectangle, tiles_touched, the clamp bits and the opacity (a copy);
  * a knife mask: surfels where a decision lies within its own bound of its threshold -- depth vs 0.2, cosv vs 0,
    d vs 0 (within 16 times its bound: closer, 1/d's first-order bound stops holding), 3e vs the next integer (with the
    0.7071 floor), px - r and px + r + 15 vs a multiple of 16 (get_rect truncates toward zero and clamps to the grid);
    and, per channel, v vs 0 for the clamp bit (it masks that bit only: max(v, 0) keeps v's bound).

check_records holds a decoded forward (vidu4d_b200.debug.decode's fields, or the same fields of the CPU oracle or of
the reference's records) to the model outside the knife mask: the visible set, radii, tiles_touched and the clamp
bits exactly, the opacity (and rgb of precomputed colours) bit for bit, every float field within K u B + FLOOR.
"""
import numpy as np

from .error_bound import _c, _E

U = 2.0 ** -24
K = 2.0
FLOOR = float(np.finfo(np.float32).tiny)
F32 = np.float32
NEAR = F32(0.2)
RADIUS_FLOOR = 0.7071067811865476
D_KNIFE = 16.0                   # d is knifed within D_KNIFE times its bound of 0
INT_MAX = 2147483647

SH_C0 = F32(0.28209479177387814)
SH_C1 = F32(0.4886025119029199)
SH_C2 = np.array([1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792,
                  0.5462742152960396], F32)
SH_C3 = np.array([-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154,
                  -0.4570457994644658, 1.445305721320277, -0.5900435899266435], F32)
MUTANTS = ("noflip", "cxcy_swap", "sh_sign", "sh_neighbour")


# ------------------------------------------------------------------------------------------------ the camera
def intrinsics(W, H, tan, off=None):
    """(focal_x, focal_y, cx, cy) in fp32 as the kernel forms them: make_cam's scalar path (off None), or
    cam_of_frame's table row (tan_x, tan_y, off_x, off_y), each operation rounded on its own."""
    tx, ty = F32(tan[0]), F32(tan[1])
    fy = F32(H) / (F32(2.0) * ty)
    fx = F32(W) / (F32(2.0) * tx)
    if off is None:
        return fx, fy, F32(F32(W) / 2.0), F32(F32(H) / 2.0)
    return fx, fy, F32(W) * F32(0.5) + F32(off[0]), F32(H) * F32(0.5) + F32(off[1])


def camera(vm, campos, W, H, tan, off=None):
    """One frame's camera: view matrix (16, the column-major glm layout the kernels read), campos (3), image size,
    tangents and, for the per-frame table path, the principal-point offsets."""
    return dict(vm=np.asarray(vm, F32).reshape(16), campos=np.asarray(campos, F32).reshape(3), W=int(W), H=int(H),
                tan=(float(tan[0]), float(tan[1])), off=None if off is None else (float(off[0]), float(off[1])))


def _leaf(x):
    return _E.leaf(np.asarray(x, F32))


def _fma(a, b, c):
    """a * b + c, charged two roundings (a contracted FMA rounds once: the bound still holds)."""
    return a * b + c


def _w_mul(m, v):
    """glm mat3(W) * v as w_mul contracts it: fma(v.z, m[8 + r], fma(v.x, m[r], v.y * m[4 + r]))."""
    return [_fma(v[2], m[8 + r], _fma(v[0], m[r], v[1] * m[4 + r])) for r in range(3)]


def _sqrt0(x):
    """sqrtf(fmaxf(0, x)): sqrt's first-order bound, capped by sqrt(|dx|), which also covers x's sign near 0."""
    v = np.sqrt(np.fmax(0.0, x.v))
    with np.errstate(divide="ignore", invalid="ignore"):
        b = np.where(x.b > 0, np.fmin(np.where(v > 0, x.b / (2.0 * v), np.inf), np.sqrt(x.b / U)), 0.0)
    exact = (x.b == 0) & (v.astype(F32).astype(np.float64) == v)
    f = None if x.f is None else np.sqrt(np.fmax(F32(0), x.f))
    return _E(v, b + np.where(exact, 0.0, v), f)


def _add(a, b):
    """a + b where adding an exact 0 (a term whose coefficient is 0) is exact."""
    r = a + b
    z = ((a.v == 0) & (a.b == 0)) | ((b.v == 0) & (b.b == 0))
    return _E(r.v, np.where(z, a.b + b.b, r.b), r.f)


def _near(x, thr, scale=1.0):
    """A decision x vs thr that x's bound does not settle (an exact x settles it, whatever its value)."""
    return (x.b > 0) & (np.abs(x.v - thr) <= scale * K * U * x.b)


# ------------------------------------------------------------------------------------------------ the kernel
def _rot(q):
    """rot_matrix: R (row-major, 9 _E) of the fp32 quaternion q (w, x, y, z) -- glm's .x is w."""
    qx, qy, qz, qw = (_leaf(q[:, i]) for i in range(4))
    n2 = _fma(qz, qz, _fma(qy, qy, _fma(qw, qw, qx * qx)))
    s = n2.rsqrt()
    w, x, y, z = qx * s, qy * s, qz * s, qw * s
    wz, wy, wx, yy, zz = w * z, w * y, w * x, y * y, z * z
    one = _c(1.0)
    R = [None] * 9
    R[0] = one - (yy + zz).scale(2.0)
    R[1] = _fma(x, y, wz).scale(2.0)
    R[2] = _fma(x, z, -wy).scale(2.0)
    R[3] = _fma(x, y, -wz).scale(2.0)
    R[4] = one - _fma(x, x, zz).scale(2.0)
    R[5] = _fma(y, z, wx).scale(2.0)
    R[6] = _fma(x, z, wy).scale(2.0)
    R[7] = _fma(y, z, -wx).scale(2.0)
    R[8] = one - _fma(x, x, yy).scale(2.0)
    return R


def _rect(px, py, r, gx, gy):
    """get_rect on float64 centres and fp32 radii: (x0, y0, x1, y1) clamped to [0, grid], truncation toward zero; the
    float-to-int conversions saturate as the GPU's do."""
    def t(v):
        return np.trunc(np.clip(np.nan_to_num(v, nan=0.0), -2.0 ** 31, 2.0 ** 31 - 1))
    x0, y0 = t((px - r) / 16.0), t((py - r) / 16.0)
    x1, y1 = t((px + r + 15.0) / 16.0), t((py + r + 15.0) / 16.0)
    c = lambda v, g: np.minimum(g, np.maximum(0.0, v)).astype(np.int64)   # noqa: E731
    return np.stack([c(x0, gx), c(y0, gy), c(x1, gx), c(y1, gy)], 1)


def _radius(e):
    """(int)(float)ceil(3 max(e, 0.7071)) in double, saturating."""
    rad = np.ceil(3.0 * np.fmax(e, RADIUS_FLOOR)).astype(F32).astype(np.float64)
    return np.clip(np.nan_to_num(rad, nan=0.0), -2.0 ** 31, INT_MAX).astype(np.int64)


def _sh(deg, sh, d, mutant=None):
    """sh_to_rgb's value per channel before the +0.5 and the clamp: sh (P, M, 3) fp32, d = (x, y, z) the unit
    direction (_E).  Operation order as written in the kernel."""
    x, y, z = d
    C1 = -SH_C1 if mutant == "sh_sign" else SH_C1
    out = []
    for ch in range(3):
        s = lambda k: _leaf(sh[:, k, ch])                                                     # noqa: E731
        v = _leaf(SH_C0) * s(0)
        if deg > 0:
            c1 = _leaf(C1)
            v = _add(_add(_add(v, -(c1 * y * s(1))), c1 * z * s(2)), -(c1 * x * s(3)))
            if deg > 1:
                xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
                c2 = [_leaf(c) for c in SH_C2]
                for t in (c2[0] * xy * s(4), c2[1] * yz * s(5), c2[2] * (zz.scale(2.0) - xx - yy) * s(6),
                          c2[3] * xz * s(7), c2[4] * (xx - yy) * s(8)):
                    v = _add(v, t)
                if deg > 2:
                    c3 = [_leaf(c) for c in SH_C3]
                    three, four = _leaf(3.0), zz.scale(4.0)
                    for t in (c3[0] * y * (three * xx - yy) * s(9), c3[1] * xy * z * s(10),
                              c3[2] * y * (four - xx - yy) * s(11),
                              c3[3] * z * (zz.scale(2.0) - three * xx - three * yy) * s(12),
                              c3[4] * x * (four - xx - yy) * s(13), c3[5] * z * (xx - yy) * s(14),
                              c3[6] * x * (xx - three * yy) * s(15)):
                        v = _add(v, t)
        out.append(v + 0.5)
    return out


def model(inputs, cam, mutant=None):
    """One frame of preprocess_fwd_kernel.  inputs: means3D (P,3), rotations (P,4), scales (P,2), opacities (P,) or
    (P,1), and either shs (P,M,3) with deg, or colors_precomp (P,3); cam: camera().  mutant (MUTANTS, for the tests
    that show the bound is not vacuous) changes the shadow's arithmetic.  Returns a dict of the fields listed in the
    module docstring ("T", "centre", "normal", "rgb", "depth": lists of _E)."""
    mu = np.asarray(inputs["means3D"], F32).reshape(-1, 3)
    P = mu.shape[0]
    q = np.asarray(inputs["rotations"], F32).reshape(P, 4)
    sc = np.asarray(inputs["scales"], F32).reshape(P, 2)
    opac = np.asarray(inputs["opacities"], F32).reshape(P)
    W, H = cam["W"], cam["H"]
    gx, gy = (W + 15) // 16, (H + 15) // 16
    fx, fy, cx, cy = (_leaf(v) for v in intrinsics(W, H, cam["tan"], cam["off"]))
    if mutant == "cxcy_swap":
        cx, cy = cy, cx
    m = [_leaf(v) for v in cam["vm"]]
    p = [_leaf(mu[:, i]) for i in range(3)]
    with np.errstate(all="ignore"):
        pv0 = _w_mul(m, p)
        pv = [pv0[i] + m[12 + i] for i in range(3)]
        depth = pv[2]
        R = _rot(q)
        sx, sy = _leaf(sc[:, 0]), _leaf(sc[:, 1])
        M0 = _w_mul(m, [R[0] * sx, R[1] * sx, R[2] * sx])
        M1 = _w_mul(m, [R[3] * sy, R[4] * sy, R[5] * sy])
        tn = _w_mul(m, [R[6], R[7], R[8]])
        cosv = _fma(-pv[2], tn[2], _fma(pv[1], -tn[1], -(pv[0] * tn[0])))
        mult = np.where(cosv.v > 0, 1.0, -1.0)
        if mutant != "noflip":
            tn = [_E(t.v * mult, t.b, None if t.f is None else t.f * mult.astype(F32)) for t in tn]
        T = [_fma(M0[2], cx, fx * M0[0]), _fma(M1[2], cx, fx * M1[0]), _fma(pv[2], cx, fx * pv[0]),
             _fma(M0[2], cy, fy * M0[1]), _fma(M1[2], cy, fy * M1[1]), _fma(pv[2], cy, fy * pv[1]),
             M0[2], M1[2], pv[2]]
        d = _fma(-T[8], T[8], _fma(T[6], T[6], T[7] * T[7]))
        r = _c(1.0) / d
        cxp = _fma(T[2] * T[8], -r, _fma(T[1] * T[7], r, T[0] * T[6] * r))
        cyp = _fma(T[5] * T[8], -r, _fma(T[4] * T[7], r, T[3] * T[6] * r))
        nqx = _fma(T[2] * T[2], r, -_fma(T[1] * T[1], r, T[0] * T[0] * r))
        nqy = _fma(T[5] * T[5], r, -_fma(T[4] * T[4], r, T[3] * T[3] * r))
        ex, ey = _sqrt0(_fma(cxp, cxp, nqx)), _sqrt0(_fma(cyp, cyp, nqy))
        # the radius: ceil(3 max(e, floor)) of e anywhere within its bound
        e = np.fmax(ex.v, ey.v)
        de = K * U * np.fmax(ex.b, ey.b) + 4 * U * e
        radius, r_lo, r_hi = _radius(e), _radius(e - de), _radius(e + de)
        k_rad = (r_lo != r_hi) | ~np.isfinite(de)
        # get_rect at the extremes of the centre (its two float adds round too: 3 u of the largest operand) and of the
        # radius; every field is monotone in both
        f = lambda r: r.astype(F32).astype(np.float64)                                        # noqa: E731
        rect = _rect(cxp.v, cyp.v, f(radius), gx, gy)
        dx = K * U * cxp.b + 3 * U * (np.abs(cxp.v) + f(r_hi) + 16.0)
        dy = K * U * cyp.b + 3 * U * (np.abs(cyp.v) + f(r_hi) + 16.0)
        lo = _rect(cxp.v - dx, cyp.v - dy, f(r_lo), gx, gy)
        hi = _rect(cxp.v + dx, cyp.v + dy, f(r_hi), gx, gy)
        lo2 = _rect(cxp.v - dx, cyp.v - dy, f(r_hi), gx, gy)
        hi2 = _rect(cxp.v + dx, cyp.v + dy, f(r_lo), gx, gy)
        ext = [np.minimum(lo2[:, :2], rect[:, :2]), np.maximum(hi2[:, :2], rect[:, :2]),
               np.minimum(lo[:, 2:], rect[:, 2:]), np.maximum(hi[:, 2:], rect[:, 2:])]
        empty = lambda a0, a1: ((a1[:, 0] - a0[:, 0]) * (a1[:, 1] - a0[:, 1])) <= 0            # noqa: E731
        # a surfel whose widest rectangle is empty is invisible whatever the rounding; else every extreme must agree
        never = empty(ext[1], ext[2])
        k_rect = ~never & (((ext[0] != ext[1]).any(1) | (ext[2] != ext[3]).any(1)) | ~np.isfinite(dx + dy))
        k_rad = k_rad & ~never
        area = (rect[:, 2] - rect[:, 0]) * (rect[:, 3] - rect[:, 1])
        front = depth.v > float(NEAR)
        faced = cosv.v != 0
        dnz = d.v != 0
        visible = front & faced & dnz & (area != 0)
        k_depth = _near(depth, float(NEAR))
        k_cos = front & _near(cosv, 0.0)
        k_d = front & faced & _near(d, 0.0, D_KNIFE)
        k_geo = front & faced & dnz & k_rect
        knife = k_depth | k_cos | k_d | k_geo
        # the colour
        if inputs.get("colors_precomp") is not None:
            col = np.asarray(inputs["colors_precomp"], F32).reshape(P, 3)
            rgb = [_leaf(col[:, c]) for c in range(3)]
            clamp = np.zeros((P, 3), bool)
            k_clamp = np.zeros((P, 3), bool)
        else:
            sh = np.asarray(inputs["shs"], F32).reshape(P, -1, 3)
            if mutant == "sh_neighbour":
                sh = np.roll(sh, 1, axis=0)
            cp = [_leaf(cam["campos"][i]) for i in range(3)]
            dv = [p[i] - cp[i] for i in range(3)]
            ln = _sqrt0(dv[0] * dv[0] + dv[1] * dv[1] + dv[2] * dv[2])
            v = _sh(int(inputs["deg"]), sh, [dv[i] / ln for i in range(3)], mutant)
            clamp = np.stack([c.v < 0 for c in v], 1)
            k_clamp = np.stack([_near(c, 0.0) for c in v], 1)
            rgb = [_E(np.fmax(c.v, 0.0), c.b, None if c.f is None else np.fmax(c.f, F32(0))) for c in v]
    radius = np.where(visible, radius, 0)
    return dict(T=T, centre=[cxp, cyp], normal=tn, rgb=rgb, depth=[depth], visible=visible, radius=radius,
                rect=rect, tiles_touched=np.where(visible, area, 0), clamp=clamp, opacity=opac, knife=knife,
                knife_clamp=k_clamp, knife_radius=front & faced & dnz & k_rad,
                knife_parts=dict(depth=k_depth, cosv=k_cos, d=k_d, rect=k_geo),
                cosv=cosv, d=d)


# ------------------------------------------------------------------------------------------------ records
def _np(x):
    return x.detach().cpu().numpy() if hasattr(x, "detach") else np.asarray(x)


def records(dec):
    """The per-surfel fields of a decoded forward (vidu4d_b200.debug.decode plus "radii") as NumPy: T (P,9), centre
    (P,2), opacity, normal (P,3), rgb (P,3), depth, radii, tiles_touched, clamp bits (P,3) bool."""
    rec = _np(dec["surfel_rec"]).astype(F32)
    P = _np(dec["radii"]).size
    rec = rec.reshape(P, 20)
    cl = _np(dec["clamped"]).astype(np.uint8).reshape(P)
    return dict(T=rec[:, 0:9], centre=rec[:, 9:11], opacity=rec[:, 11], normal=rec[:, 12:15], rgb=rec[:, 15:18],
                depth=_np(dec["depths"]).astype(F32).reshape(P), radii=_np(dec["radii"]).astype(np.int64).reshape(P),
                tiles_touched=_np(dec["tiles_touched"]).astype(np.int64).reshape(P),
                clamp=((cl[:, None] >> np.arange(3)) & 1).astype(bool))


def oracle_records(st):
    """records() of the CPU oracle's forward state (oracle.surfel_oracle.forward)."""
    return dict(T=st.transMat, centre=st.means2D, opacity=st.normal_opacity[:, 3], normal=st.normal_opacity[:, :3],
                rgb=st.rgb, depth=st.depths, radii=st.radii.astype(np.int64), tiles_touched=st.tiles_touched.astype(np.int64),
                clamp=st.clamped.astype(bool))


def golden_records(g):
    """records() of the reference's own buffers stored in a golden fixture."""
    no = g["ref_geom_normal_opacity"]
    return dict(T=g["ref_geom_transMat"], centre=g["ref_geom_means2D"], opacity=no[:, 3], normal=no[:, :3],
                rgb=g["ref_geom_rgb"], depth=g["ref_geom_depths"], radii=g["ref_radii"].astype(np.int64),
                tiles_touched=g["ref_geom_tiles_touched"].astype(np.int64), clamp=g["ref_geom_clamped"].astype(bool))


def golden_inputs(g):
    """model() inputs and camera() of a golden fixture."""
    P, W, H, deg, pre = [int(v) for v in g["in_meta"]]
    inp = dict(means3D=g["in_means3D"], rotations=g["in_rotations"], scales=g["in_scales"], opacities=g["in_opacities"],
               shs=None if pre else g["in_shs"], colors_precomp=g["in_colors_precomp"] if pre else None, deg=deg)
    return inp, camera(g["in_viewmatrix"], g["in_campos"], W, H, g["in_tanfov"])


def check_records(dec, inputs, cam, colour_source, name="", m=None):
    """Asserts a frame's per-surfel records against model() outside its knife mask.  dec: a decoded forward (or
    records() of one); colour_source: "sh" (rgb and clamp bits against sh_to_rgb), "precomp" (rgb a bit-for-bit copy,
    no clamp bit) or None (geometry only: rgb and clamp bits not checked).  Returns {field: largest err / bound,
    "knife": knifed surfels, "visible": visible surfels}."""
    r = dec if "T" in dec else records(dec)
    m = model(inputs, cam) if m is None else m
    ok = ~m["knife"]
    vis = r["radii"] > 0
    bad = np.nonzero((vis != m["visible"]) & ok)[0]
    assert bad.size == 0, (name, "visible set differs from the model at", bad[:8].tolist(),
                           [(bool(vis[i]), {k: bool(v[i]) for k, v in m["knife_parts"].items()}, float(m["depth"][0].v[i]),
                             float(m["cosv"].v[i]), float(m["d"].v[i])) for i in bad[:3]])
    for k, want, mask in (("radii", m["radius"], ok & ~m["knife_radius"]), ("tiles_touched", m["tiles_touched"], ok)):
        bad = np.nonzero((r[k] != want) & mask)[0]
        assert bad.size == 0, (name, k, "differs at", bad[:8].tolist(), r[k][bad[:4]].tolist(), want[bad[:4]].tolist())
    v = ok & m["visible"]
    o = np.asarray(r["opacity"], F32)
    assert np.array_equal(o[v].view(np.uint32), m["opacity"][v].view(np.uint32)), (name, "opacity is not a copy")
    fields = [("T", 9), ("centre", 2), ("normal", 3), ("depth", 1)]
    if colour_source == "precomp":
        rgb = np.asarray(r["rgb"], F32)[v]
        want = np.stack([c.v for c in m["rgb"]], 1).astype(F32)[v]
        assert np.array_equal(rgb.view(np.uint32), want.view(np.uint32)), (name, "rgb is not a copy of colors_precomp")
        assert not r["clamp"][v].any(), (name, "clamp bit set with precomputed colours")
    elif colour_source == "sh":
        fields.append(("rgb", 3))
        cv = v[:, None] & ~m["knife_clamp"]
        bad = np.argwhere((r["clamp"] != m["clamp"]) & cv)
        assert bad.size == 0, (name, "clamp bits differ at (surfel, channel)", bad[:8].tolist())
    report = {}
    for k, n in fields:
        g = np.asarray(r[k], np.float64).reshape(-1, n)[v]
        for i in range(n):
            e = m[k][i]
            err = np.abs(g[:, i] - e.v[v])
            tol = K * U * e.b[v] + FLOOR
            ratio = err / tol
            if ratio.size:
                j = int(np.argmax(np.nan_to_num(ratio, nan=np.inf)))
                sid = np.nonzero(v)[0][j]
                assert ratio[j] <= 1.0, (name, f"{k}[{i}]", "surfel", int(sid), "gpu", float(g[j, i]), "model",
                                         float(e.v[sid]), "tolerance", float(tol[j]))
                report[k] = max(report.get(k, 0.0), float(ratio[j]))
    report["knife"] = int(m["knife"].sum())
    report["knife_clamp"] = int((m["knife_clamp"] & m["visible"][:, None]).sum())
    report["visible"] = int(m["visible"].sum())
    return report


def shadow_records(m):
    """records() of a model's own fp32 shadow (the float fields) and exact fields."""
    st = lambda xs: np.stack([x.f for x in xs], 1)   # noqa: E731
    return dict(T=st(m["T"]), centre=st(m["centre"]), opacity=m["opacity"], normal=st(m["normal"]), rgb=st(m["rgb"]),
                depth=m["depth"][0].f, radii=m["radius"], tiles_touched=m["tiles_touched"], clamp=m["clamp"])


def exceed_share(rec, m):
    """The share of the model's visible, unknifed surfels where some float field of rec lies outside the bound."""
    v = m["visible"] & ~m["knife"]
    out = np.zeros(v.shape, bool)
    for k in ("T", "centre", "normal", "rgb", "depth"):
        g = np.asarray(rec[k], np.float64).reshape(v.size, -1)
        for i, e in enumerate(m[k]):
            out |= np.abs(g[:, i] - e.v) > K * U * e.b + FLOOR
    return float((out & v).sum()) / max(1, int(v.sum()))


def print_report(name, rep):
    print(f"\n[{name}] visible {rep['visible']}, knife {rep['knife']} surfels + {rep['knife_clamp']} clamp bits; err/bound "
          + ", ".join(f"{k} {v:.3g}" for k, v in rep.items() if k not in ("knife", "knife_clamp", "visible")))


# ------------------------------------------------------------------------------------------------ scenes
# The turned camera: view x = world z, view y = world y, view z = -world x + TURN_Z (entries 0 and +-1, exact in fp32).
# A surfel with quaternion (w, 0, 0, 0) -- R = I exactly, whatever rsqrtf returns -- has the view-space normal (1, 0, 0)
# exactly, so cosv = -(view x) exactly: its sign and zero are set by the position alone; and T[6] = -s_x, T[7] = 0,
# T[8] = depth, so d = s_x^2 - depth^2 is 0 exactly where s_x = depth (both with short mantissas).
TURN = np.array([[0.0, 0.0, 1.0], [0.0, 1.0, 0.0], [-1.0, 0.0, 0.0]])
TURN_Z = 0.0


def turned_view():
    """The turned camera's view matrix in the kernels' layout (W2C transposed) and its campos (world)."""
    w2c = np.eye(4)
    w2c[:3, :3] = TURN
    w2c[2, 3] = TURN_Z
    return w2c.T.astype(F32), (-TURN.T @ np.array([0.0, 0.0, TURN_Z])).astype(F32)


def _to_world(pv, Rv):
    """View-space positions and rotation matrices to world ones under the turned camera (exact for the positions)."""
    from .cull_model import _quat
    pw = np.stack([-(pv[:, 2] - TURN_Z), pv[:, 1], pv[:, 0]], 1)
    Rw = np.einsum("ji,njk->nik", TURN, Rv)
    return pw, _quat(Rw)


def _pixel_to_view(u, v, z, W, H, tan):
    fx, fy = W / (2 * tan), H / (2 * tan)
    return np.stack([(u - W / 2) * z / fx, (v - H / 2) * z / fy, z], 1)


def special_surfels(rng, n, W, H, tan=0.5):
    """The preprocess's own edge classes for the turned camera, as {class: dict(means, scales, rotations, opacities)}
    in world space (fp32):
      near        view z at 0.2 and its fp32 neighbours (a few ulps either side);
      edge_on     quaternions (w, 0, 0, 0) with view x = 0 (cosv exactly 0) or small either side (the flip both ways);
      d_zero      quaternions (w, 0, 0, 0) with s_x = depth exactly (d = 0) and one ulp either side;
      floor       face-on sub-pixel surfels (3e below the 0.7071 floor: radius 3);
      huge        face-on surfels far larger than the image (the rectangle clamped to the grid);
      far_off     small surfels centred far outside the image (area 0, radius 0);
      rect_edge   face-on sub-pixel surfels whose px - 3 or px + 18 lies within 0.3 px of a multiple of 16, or px - 3
                  just below 0;
      quat_norm   random quaternions scaled to |q| from 1e-3 to 1e3."""
    from .cull_model import _frame_with_normal, _logu, _unit
    out = {}

    def face_q(k):                                  # (w, 0, 0, 0), w from 1e-3 to 1e3: R = I, normal world z = view x
        return np.stack([_logu(rng, 1e-3, 1e3, k), np.zeros(k), np.zeros(k), np.zeros(k)], 1)

    def pack(pv, sc, q_world=None, Rv=None, op=None):
        k = pv.shape[0]
        if q_world is None:
            pw, q_world = _to_world(pv, Rv)
        else:
            pw = np.stack([-(pv[:, 2] - TURN_Z), pv[:, 1], pv[:, 0]], 1)
        op = rng.uniform(0.05, 1.0, k) if op is None else op
        return dict(means=pw.astype(F32), scales=np.asarray(sc, F32), rotations=np.asarray(q_world, F32),
                    opacities=np.asarray(op, F32))

    # near: view z = -world x + TURN_Z, exact for these values; ulps of 0.2f either side
    ul = rng.integers(-6, 7, n)
    z = np.array([np.float32(NEAR)], F32)
    zs = np.array([z[0]] * n, F32)
    for i in range(n):
        for _ in range(abs(int(ul[i]))):
            zs[i] = np.nextafter(zs[i], F32(np.inf) if ul[i] > 0 else F32(-np.inf))
    pv = _pixel_to_view(rng.uniform(0, W, n), rng.uniform(0, H, n), zs.astype(np.float64), W, H, tan)
    pv[:, 2] = zs
    Rv = _frame_with_normal(rng, _unit(rng.normal(size=(n, 3)) + np.array([0, 0, -2.0])))
    out["near"] = pack(pv, rng.uniform(0.002, 0.02, (n, 2)), Rv=Rv)
    # edge_on: view x = world z in {0, +-small}; (w, 0, 0, 0) gives view normal (1, 0, 0)
    z = rng.uniform(0.5, 4.0, n).astype(F32)
    xv = np.where(rng.random(n) < 0.3, 0.0, rng.choice([-1.0, 1.0], n) * _logu(rng, 1e-6, 0.3, n)).astype(F32)
    pv = np.stack([xv, (rng.uniform(0, H, n) - H / 2) * z / (H / (2 * tan)), z], 1)
    out["edge_on"] = pack(pv, np.stack([_logu(rng, 1e-3, 0.1, n), _logu(rng, 1e-3, 0.1, n)], 1), q_world=face_q(n))
    # d_zero: short-mantissa depths, s_x = depth (or one ulp off), view x nonzero so that cosv != 0
    z = (rng.integers(4, 64, n) / 8.0).astype(F32)                       # 0.5 .. 7.875, at most 6 bits
    sx = z.copy()
    k = rng.integers(-1, 2, n)
    sx[k > 0] = np.nextafter(sx[k > 0], F32(np.inf))
    sx[k < 0] = np.nextafter(sx[k < 0], F32(0))
    xv = (rng.choice([-1.0, 1.0], n) * rng.integers(1, 64, n) / 64.0 * z).astype(F32)
    pv = np.stack([xv, ((rng.uniform(0, H, n) - H / 2) * z / (H / (2 * tan))).astype(F32), z], 1)
    out["d_zero"] = pack(pv, np.stack([sx, _logu(rng, 1e-3, 0.1, n)], 1), q_world=face_q(n))
    # face-on surfels for the turned camera: view normal (0, 0, -1) = world x
    def face_on(k):
        Rv = np.repeat(np.array([[[1.0, 0, 0], [0, -1.0, 0], [0, 0, -1.0]]]), k, 0)
        return Rv
    # floor: sub-pixel
    z = rng.uniform(0.5, 8.0, n)
    pv = _pixel_to_view(rng.uniform(0, W, n), rng.uniform(0, H, n), z, W, H, tan)
    out["floor"] = pack(pv, _logu(rng, 1e-7, 1e-3, (n, 2)) * z[:, None], Rv=face_on(n))
    # huge: face-on (the plane stays in front of the camera), 1.5 to 50 image widths across
    z = rng.uniform(1.0, 4.0, n)
    pv = _pixel_to_view(rng.uniform(0, W, n), rng.uniform(0, H, n), z, W, H, tan)
    out["huge"] = pack(pv, _logu(rng, 1.5, 50.0, (n, 2)) * z[:, None], Rv=face_on(n))
    # far off the image
    side = rng.integers(0, 4, n)
    u = np.where(side == 0, -rng.uniform(60, 2000, n), np.where(side == 1, W + rng.uniform(60, 2000, n), rng.uniform(0, W, n)))
    v = np.where(side == 2, -rng.uniform(60, 2000, n), np.where(side == 3, H + rng.uniform(60, 2000, n), rng.uniform(0, H, n)))
    z = rng.uniform(1.0, 4.0, n)
    pv = _pixel_to_view(u, v, z, W, H, tan)
    out["far_off"] = pack(pv, rng.uniform(0.1, 1.0, (n, 2)) * z[:, None] / W, Rv=face_on(n))
    # rect edges: radius 3 (sub-pixel), px - 3 or px + 18 at a multiple of 16 +- up to 0.3, or px - 3 in (-1, 0)
    kind = rng.integers(0, 3, n)
    m16 = 16.0 * rng.integers(1, max(2, W // 16), n)
    off = rng.choice([-1.0, 1.0], n) * _logu(rng, 1e-4, 0.3, n)
    px = np.where(kind == 0, m16 + 3 + off, np.where(kind == 1, m16 - 18 + off, 3.0 - rng.uniform(0.01, 0.99, n)))
    py = rng.uniform(4, H - 4, n)
    z = rng.choice([0.5, 1.0, 2.0, 4.0], n)
    pv = _pixel_to_view(px, py, z, W, H, tan)
    out["rect_edge"] = pack(pv, np.full((n, 2), 1e-6) * z[:, None], Rv=face_on(n))
    # unnormalised quaternions
    z = rng.uniform(1.0, 4.0, n)
    pv = _pixel_to_view(rng.uniform(0, W, n), rng.uniform(0, H, n), z, W, H, tan)
    qn = _unit(rng.normal(size=(n, 4))) * _logu(rng, 1e-3, 1e3, n)[:, None]
    d = pack(pv, rng.uniform(1, 12, (n, 2)) * z[:, None] / W, Rv=np.eye(3)[None].repeat(n, 0))
    d["rotations"] = qn.astype(F32)
    out["quat_norm"] = d
    return out


def cull_classes(rng, n, W, H, tan=0.5):
    """tests/cull_model.py's identity-camera classes (grazing, near-parabolic, sub-pixel, off-image, threshold) moved
    into the turned camera's world frame."""
    from . import cull_model as cm
    from .cull_model import rot_columns
    out = {}
    for cls in cm.CLASSES:
        a = cm.adversarial(rng, cls, n, W, H)
        pw, q = _to_world(a["means"].astype(np.float64), rot_columns(a["rotations"]))
        out[cls] = dict(means=pw.astype(F32), scales=a["scales"], rotations=q.astype(F32), opacities=a["opacities"])
    return out


def sh_near_zero(rng, n, M=16):
    """SH rows whose channel values v = C0 sh0 + 0.5 (the other coefficients 0) lie a few ulps of sh0 from 0, one
    channel at a time or all three."""
    sh = np.zeros((n, M, 3), F32)
    base = F32(-0.5) / SH_C0
    for c in range(3):
        sh[:, 0, c] = rng.uniform(-1.5, 1.5, n)
        k = rng.integers(-12, 13, n)
        pick = rng.random(n) < 0.6
        for i in np.nonzero(pick)[0]:
            x = base
            for _ in range(abs(int(k[i]))):
                x = np.nextafter(x, F32(np.inf) if k[i] > 0 else F32(-np.inf))
            sh[i, 0, c] = x
    return sh


def adversarial_scene(seed, W, H, n, tan=0.5):
    """Every class of special_surfels and cull_classes (n each) plus n ordinary random surfels, shuffled, for the
    turned camera; SH degree 3 (random rows, sh_near_zero's for a third of the surfels).  Returns (inputs, camera,
    labels (P,) class names)."""
    rng = np.random.default_rng(seed)
    parts = dict(special_surfels(rng, n, W, H, tan), **cull_classes(rng, n, W, H, tan))
    z = rng.uniform(0.5, 6.0, n)
    pv = _pixel_to_view(rng.uniform(-W / 4, 1.25 * W, n), rng.uniform(-H / 4, 1.25 * H, n), z, W, H, tan)
    Rv = np.stack([np.linalg.qr(rng.normal(size=(3, 3)))[0] for _ in range(n)])
    Rv *= np.sign(np.linalg.det(Rv))[:, None, None]
    pw, q = _to_world(pv, Rv)
    parts["cloud"] = dict(means=pw.astype(F32), scales=(rng.uniform(0.5, 20, (n, 2)) * z[:, None] / W).astype(F32),
                          rotations=q.astype(F32), opacities=rng.uniform(0.05, 1.0, n).astype(F32))
    names = list(parts)
    label = np.concatenate([np.full(len(parts[k]["opacities"]), k) for k in names])
    perm = rng.permutation(label.size)
    cat = {k: np.concatenate([parts[c][k] for c in names])[perm] for k in ("means", "scales", "rotations", "opacities")}
    P = label.size
    sh = rng.normal(0, 0.4, (P, 16, 3)).astype(F32)
    near0 = rng.random(P) < 1 / 3
    sh[near0] = sh_near_zero(rng, int(near0.sum()))
    vm, cp = turned_view()
    inp = dict(means3D=cat["means"], rotations=cat["rotations"], scales=cat["scales"],
               opacities=cat["opacities"].reshape(P, 1), shs=sh, colors_precomp=None, deg=3)
    return inp, camera(vm, cp, W, H, (tan, tan)), label[perm]
