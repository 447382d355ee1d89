"""Every element of Stage 3's per-surfel feature rows (csrc/feature_rows.cu: sr_feature_rows_forward and
sr_feature_rows_backward) against the float64 restatement of its kernels (tests/feature_rows_bounds.py, pinned to
tests/feature_rows_model.py by tests/test_feature_rows_bounds_cpu.py).

The entry points are driven through _capi.call, so aux and the raw g_tables (g_cam_q | g_centres | g_beta | the sum of
g_row_flow * flow in slot ntab) are compared before any torch op.  Every output buffer starts as NaN, so an element the
kernels fail to write fails the comparison.  Bit for bit: aux[0] (max |flow|), aux[1:3] (the counts of flow values at
+max and -max), s, the flow channels and the regist channels.  Every other element: |gpu - value| <= K u B + FLOOR,
K = 2.  Each case asserts its own edge from the GPU's buffers and prints its knife counts and the largest err / tol per
tensor.

Cases: the row paths (Cf = 0, 1, 15, 16, 26; even Cf with regist, rows, g_rows and g_regist at a 4-byte-aligned offset,
which takes the scalar path; an odd-P FlatSurfelModel view, 8-byte aligned, which takes the float2 path); P = 1, 255,
256, 257 and 70001 (274 CTAs: the global atomics interleave), and P = 0; M = 1, 2, 8 and 1024; B = 1 and 64; the flow
scale's edges (duplicated surfels tied at both extremes, a single holder of the max, the static pair with sm = 0,
g_flow_scale NULL, g_density NULL); the density's (duplicated bone centres, two bones within rounding of each other,
scores that underflow to 0, subnormal scores); equal tangent scales.  One last test runs vidu4d_b200.warp.feature_rows
through autograd at Cf = 15, M = 8.
"""
import numpy as np
import pytest
import torch

from . import feature_rows_bounds as fb

pytestmark = pytest.mark.gpu

BASE = dict(P=3000, M=2, B=25, Cf=16)
CASES = {
    **{f"cf_{c}": dict(Cf=c) for c in (0, 1, 15, 16, 26)},
    "cf16_offset4": dict(layout="offset4"),
    "cf16_flat_p5003": dict(P=5003, layout="flat"),
    **{f"p_{p}": dict(P=p) for p in (1, 255, 256, 257, 70001)},
    "m_1": dict(M=1),
    "m_8": dict(M=8, P=2000, Cf=15),
    "m_1024": dict(M=1024, P=300, B=7, Cf=2),
    "b_1": dict(B=1),
    "b_64": dict(B=64, far=0.1),
    "dup": dict(M=4, dup=True),
    "single_max": dict(M=4, single_max=True),
    "static": dict(M=4, static=True, Cf=3),
    "g_s_null": dict(g_s=False),
    "g_density_null": dict(g_density=False, Cf=1),
    "bone_dup": dict(B=7, bone_dup=True),
    "bone_knife": dict(B=7, bone_knife=True),
    "far": dict(B=7, far=0.4),
    "subnormal": dict(B=7, sub=0.4),
    "eq_scale": dict(eq_scale=0.5, Cf=15),
}


@pytest.fixture(scope="module")
def dev(built):
    from vidu4d_b200 import _capi
    _capi.load()
    return torch.device("cuda:0")


def make(name):
    c = dict(BASE, **CASES[name])
    layout = c.pop("layout", "plain")
    return fb.scene(1000 + sum(map(ord, name)), c.pop("P"), c.pop("M"), c.pop("B"), c.pop("Cf"), **c), layout


def gpu(s, dev, layout="plain"):
    """sr_feature_rows_forward, then sr_feature_rows_backward on its own s and aux.  Returns numpy buffers and the row
    pointers."""
    from vidu4d_b200 import _capi
    P, M, B, Cf = (s[k] for k in ("P", "M", "B", "Cf"))
    W, ntab = Cf + 6, M * 4 + B * 3 + 1
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    nan = lambda *sh: torch.full(sh, float("nan"), device=dev)  # noqa: E731
    keep = []

    def row_buf(shape, data=None):
        """A row-major buffer at the layout's alignment (offset4: one float past a 256-byte-aligned allocation)."""
        n = int(np.prod(shape))
        if layout == "offset4":
            b = nan(n + 1)
            keep.append(b)
            t = b[1:].view(shape)
        else:
            t = nan(*shape)
        if data is not None:
            t.copy_(T(data))
        return t
    g_regist = None
    if layout == "flat":
        from vidu4d_b200.surfel_store import FlatSurfelModel
        z = lambda *sh: torch.zeros(sh, device=dev)  # noqa: E731
        fm = FlatSurfelModel(z(P, 3), z(P, 1, 3), z(P, 15, 3), z(P, 1), z(P, 2), z(P, 4), regist_feat=T(s["regist"]))
        keep.append(fm)
        regist = fm._regist_feat.detach()
        g_regist = fm._regist_feat.grad
        g_regist.fill_(float("nan"))
    else:
        regist = row_buf((P, Cf), s["regist"]) if Cf and P else None
    rows = row_buf((M, P, W))
    g_rows = row_buf((M, P, W), s["g_rows"])
    if g_regist is None and Cf and P:
        g_regist = row_buf((P, Cf))
    ptrs = {k: v.data_ptr() for k, v in (("regist", regist), ("rows", rows), ("g_rows", g_rows), ("g_regist", g_regist))
            if v is not None}
    per = lambda k: T(s[k]) if P else None  # noqa: E731
    xyz, scaling, xyz_cam, rot_cam = per("xyz"), per("scaling"), per("xyz_cam"), per("rot_cam")
    Kmat, cam_q, cen, beta = T(s["Kmat"]), T(s["cam_q"]), T(s["centres"]), T(s["beta"])
    density, sv = nan(P), nan(1)
    aux = torch.full((3,), -7, dtype=torch.int32, device=dev)
    _capi.call("sr_feature_rows_forward", dev, P, M, B, Cf, regist, xyz, scaling, xyz_cam, rot_cam, Kmat, cam_q, cen, beta,
               rows if P else None, density if P else None, sv, aux)
    g_xyz, g_xyz_cam, g_rot_cam, g_tab = nan(P, 3), nan(M, P, 3), nan(M, P, 4), nan(ntab + 1)
    gd = T(s["g_density"]) if s["g_density"] is not None and P else None
    gs = T(np.reshape(s["g_s"], (1,))) if s["g_s"] is not None else None
    _capi.call("sr_feature_rows_backward", dev, P, M, B, Cf, xyz, scaling, xyz_cam, rot_cam, Kmat, cam_q, cen, beta, sv, aux,
               g_rows if P else None, gd, gs, g_regist, g_xyz if P else None, g_xyz_cam if P else None,
               g_rot_cam if P else None, g_tab)
    torch.cuda.synchronize(dev)
    n = lambda t: None if t is None else t.detach().cpu().numpy()  # noqa: E731
    out = dict(rows=n(rows), density=n(density), s=n(sv)[0], aux=n(aux).view(np.uint32), g_regist=n(g_regist), g_xyz=n(g_xyz),
               g_xyz_cam=n(g_xyz_cam), g_rot_cam=n(g_rot_cam), g_tables=n(g_tab), ptrs=ptrs)
    del keep
    return out


def _cmp(name, what, mine, e, report, skip=None):
    mine = np.asarray(mine, np.float64)
    tol = fb.K * fb.U * e.b + fb.FLOOR
    ratio = np.abs(mine - e.v) / tol
    ratio = np.where(np.isnan(mine), np.inf, ratio)
    if skip is not None:
        ratio = np.where(skip, 0.0, ratio)
    if not ratio.size:
        return
    i = int(np.argmax(ratio))
    report[what] = max(report.get(what, 0.0), float(ratio.flat[i]))
    assert ratio.flat[i] <= 1.0, (name, what, "element", np.unravel_index(i, np.shape(mine)), "gpu", mine.flat[i],
                                  "value", e.v.flat[i], "bound", tol.flat[i])


def _bits(name, what, a, b):
    a, b = np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32)
    assert a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32)), (
        name, what, "not bit-identical", int((a.view(np.uint32) != b.view(np.uint32)).sum()))


def run(name, s, g):
    m = fb.model(s)
    P, M, B, Cf = (s[k] for k in ("P", "M", "B", "Cf"))
    ntab = M * 4 + B * 3 + 1
    report = {}
    # exact: the flow scale, its tie counts, the flow and regist channels
    assert g["aux"][0] == np.float32(m["sm"]).view(np.uint32), (name, "aux[0]: max |flow|")
    assert (int(g["aux"][1]), int(g["aux"][2])) == (m["hi"], m["lo"]), (name, "aux[1:3]: tie counts", g["aux"][1:], m["hi"], m["lo"])
    _bits(name, "s", g["s"], m["s"].f)
    _bits(name, "regist channels", g["rows"][..., :Cf], np.broadcast_to(s["regist"], (M, P, Cf)))
    assert not m["pknife"].any() and not m["s_bad"], (name, "projection knife", int(m["pknife"].sum()))
    _bits(name, "flow channels", g["rows"][..., Cf:Cf + 2], m["flow_ch"].f)
    # within the bound
    dk = m["dknife"]
    _cmp(name, "normal", g["rows"][..., Cf + 2:Cf + 5], m["normal"], report)
    _cmp(name, "density", g["density"], m["density"], report, dk)
    _cmp(name, "density_ch", g["rows"][..., Cf + 5], m["density"], report, dk[None])
    tab = g["g_tables"]
    _cmp(name, "acc", tab[ntab], m["acc"], report)
    _cmp(name, "g_cam_q", tab[:4 * M].reshape(M, 4), m["g_cam_q"], report)
    _cmp(name, "g_centres", tab[4 * M:4 * M + 3 * B].reshape(B, 3), m["g_centres"], report)
    _cmp(name, "g_beta", tab[4 * M + 3 * B], m["g_beta"], report)
    if Cf:
        _cmp(name, "g_regist", g["g_regist"], m["g_regist"], report)
    _cmp(name, "g_xyz", g["g_xyz"], m["g_xyz"], report, dk[:, None])
    _cmp(name, "g_xyz_cam", g["g_xyz_cam"], m["g_xyz_cam"], report, m["g_xyz_cam_mask"][..., None])
    _cmp(name, "g_rot_cam", g["g_rot_cam"], m["g_rot_cam"], report)
    print(f"\n[{name}] P={P} M={M} B={B} Cf={Cf}: knife proj {int(m['pknife'].sum())} density {int(dk.sum())}; ties "
          f"{m['hi']}/{m['lo']}; " + ", ".join(f"{k} {v:.3g}" for k, v in report.items()))
    return m


@pytest.mark.parametrize("name", list(CASES))
def test_feature_rows_every_element_within_bound(name, dev):
    s, layout = make(name)
    g = gpu(s, dev, layout)
    m = run(name, s, g)
    P, M, B, Cf = (s[k] for k in ("P", "M", "B", "Cf"))
    dk = m["dknife"]
    dens = g["density"]
    tab = g["g_tables"]
    gcen = tab[4 * M:4 * M + 3 * B].reshape(B, 3)
    if name == "bone_knife":
        assert dk.sum() > 0, "no surfel on the density knife"
    else:                               # elsewhere only scores a few subnormal ulps apart are knives
        assert (m["score"].v[dk] < fb.TINY).all()
    if layout == "offset4":
        assert all(p % 8 == 4 for p in g["ptrs"].values()) and len(g["ptrs"]) == 4, g["ptrs"]
    if layout == "flat":
        assert g["ptrs"]["regist"] % 8 == 0 and g["ptrs"]["regist"] % 16 != 0
        assert g["ptrs"]["g_regist"] % 8 == 0 and g["ptrs"]["g_regist"] % 16 != 0
    if name == "cf_0":
        assert g["rows"].shape[-1] == 6
    if name == "p_70001":
        assert -(-P // fb.THREADS) == 274
    if name == "m_1":
        assert g["aux"][0] == 0 and g["s"] == np.float32(1e-6) and (g["g_xyz_cam"] == 0).all()
    if name == "m_1024":
        gq = tab[:4 * M].reshape(M, 4)
        assert (gq != 0).all(), "a frame's g_cam_q slot is 0"
    if name == "dup":
        assert g["aux"][1] == g["aux"][2] == 2
        p, q = s["dup_pair"]
        assert np.array_equal(g["rows"][:, p], g["rows"][:, q])
    if name == "single_max":
        ch = np.abs(g["rows"][..., Cf:Cf + 2])
        assert g["aux"][1] == g["aux"][2] == 1 and ch[:, P // 2].max() == 1 and np.delete(ch, P // 2, 1).max() < 0.2
    if name == "static":
        assert g["aux"][0] == 0 and g["aux"][1] == g["aux"][2] == 2 * M * P and g["s"] == np.float32(1e-6)
        assert (g["rows"][..., Cf:Cf + 2] == 0).all() and np.abs(g["g_xyz_cam"]).max() > 0
    if name == "bone_dup":
        assert (gcen[1] == 0).all() and (gcen[0] != 0).all()
    if name == "far":
        assert (dens == 0).sum() > 0.3 * P and (g["g_xyz"][dens == 0] == 0).all()
    if name == "subnormal":
        sub = (dens > 0) & (dens < fb.TINY * float(s["beta"][0]))
        assert sub.sum() > 0.3 * P, "no subnormal score"
    if name == "eq_scale":
        assert (s["scaling"][:, 0] == s["scaling"][:, 1]).sum() > 0.4 * P
    if name == "b_1":
        assert (m["arg"] == 0).all() and (gcen != 0).all()


def test_empty_surfel_set_writes_only_s_and_zero_tables(dev):
    """P = 0 through the C entry points, with NULL per-surfel pointers: s = 1e-6f, aux zeroed, g_tables all 0."""
    s = fb.scene(5, 0, 2, 5, 16)
    g = gpu(s, dev)
    assert g["s"] == np.float32(1e-6) and (g["aux"] == 0).all()
    assert g["g_tables"].shape == (2 * 4 + 5 * 3 + 2,) and (g["g_tables"] == 0).all()
    assert np.signbit(g["g_tables"]).sum() == 0


def test_autograd_odd_cf_matches_bound_model(dev):
    """vidu4d_b200.warp.feature_rows -> weighted sum -> backward at Cf = 15 (the scalar row path both ways) and M = 8,
    every element against the bound model.  The rest bones are identity rotations, so the wrapper's centres are the
    translations exactly; beta is the wrapper's exp(logibeta), read back."""
    from vidu4d_b200.warp import feature_rows
    from .test_feature_rows_cpu import q2dq
    s = fb.scene(77, 2000, 8, 25, 15)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    leaf = lambda a: T(a).requires_grad_(True)  # noqa: E731
    regist, xyz, xc, rc, cq = (leaf(s[k]) for k in ("regist", "xyz", "xyz_cam", "rot_cam", "cam_q"))
    logibeta = torch.tensor([4.6], device=dev)
    rest = q2dq(T(np.tile(np.float32([1, 0, 0, 0]), (25, 1))), T(s["centres"]))
    out = feature_rows(regist, xyz, T(s["scaling"]), xc, rc, T(s["Kmat"]), (cq, torch.zeros((8, 3), device=dev)), rest, logibeta)
    s["beta"] = torch.exp(logibeta).cpu().numpy()
    loss = (out["rows"] * T(s["g_rows"])).sum() + out["flow_scale"] * float(s["g_s"]) + \
        (out["gauss_density"][:, 0] * T(s["g_density"])).sum()
    loss.backward()
    m = fb.model(s)
    n = lambda t: t.detach().cpu().numpy()  # noqa: E731
    report = {}
    rows = n(out["rows"])
    _bits("autograd", "flow channels", rows[..., 15:17], m["flow_ch"].f)
    _bits("autograd", "regist channels", rows[..., :15], np.broadcast_to(s["regist"], (8, 2000, 15)))
    _cmp("autograd", "normal", rows[..., 17:20], m["normal"], report)
    _cmp("autograd", "density", n(out["gauss_density"])[:, 0], m["density"], report, m["dknife"])
    for k, t in (("g_regist", regist), ("g_xyz_cam", xc), ("g_rot_cam", rc), ("g_cam_q", cq)):
        _cmp("autograd", k, n(t.grad), m[k], report)
    _cmp("autograd", "g_xyz", n(xyz.grad), m["g_xyz"], report, m["dknife"][:, None])
    assert float(np.abs(n(regist.grad)).max()) > 0
    print("\n[autograd Cf=15 M=8] " + ", ".join(f"{k} {v:.3g}" for k, v in report.items()))
