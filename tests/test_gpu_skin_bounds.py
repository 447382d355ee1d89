"""Every output and gradient element of the fused bob warp (csrc/warp.cu, sr_bob_warp_forward / sr_bob_warp_backward)
against the float64 restatement of its skinning chain (tests/skin_bounds.py, pinned to oracle/warp_oracle.py by
tests/test_skin_bounds_cpu.py), under the a-priori rounding-error bound |gpu - value| <= K u B + FLOOR, with K = 2.

The kernels are driven through vidu4d_b200.warp.bob_warp_tables with the fp32 tables as leaves, so the comparison holds
the kernels alone.  Knife points (a decision within its bound, or an ill-conditioned |QR|^2; see skin_bounds.py) get zero
upstream on both sides: their gradient rows must then come out exactly +-0, and their forward rows are not compared.
Each case prints its knife count and the largest err / tol per tensor, and keeps its knife count within a few times the
count measured on an H100 (KNIFE_MEASURED).

Cases, each asserting its edge: every B in BONES (both templates, every residue of B mod 3 and B mod 4, B = 1 and
B = 64); wide bones (median surfel >= 4 bones above 1e-3) and the warp fixtures' narrow bones (fp32 weights underflow to
0 where float64 ones do not); M = 1, 2 and the largest M whose backward tables fit at B = 64, the upstream scaled per
frame over 1 .. 1e-6 with one frame exactly 0 (its se3 and camera gradients exactly 0); P at the 128-thread backward and
256-thread forward block edges and ~20 K points; no delta, a small delta and a delta that decides the arg-max; two
bit-identical bones (the lower index is the anchor) and an exactly orthogonal rotation (sign -1).

The reprojection loss (csrc/match.cu reproj_fwd / reproj_bwd, on constructed matched points, no top-K) and the cycle
loss (csrc/cycle.cu) are held to the same bound through their C entry points: every B in BONES, M up to the largest
their tables allow at B = 64 (48 and 26), HW and P at the block edges.  Reproj knife pixels are masked out (mask 0);
cycle knife surfels are dropped from the inputs.  Counts must match exactly.
"""
import numpy as np
import pytest
import torch

from . import skin_bounds as sb
from .skin_bounds import warp_scene as scene

pytestmark = pytest.mark.gpu

BONES = (1, 2, 3, 4, 5, 31, 32, 33, 34, 63, 64)
# knife points per case, measured on an H100 80GB HBM3: none of these scenes puts a decision within its bound
KNIFE_MEASURED = {**{f"bones_{B}": 0 for B in BONES}, "wide": 0, "narrow": 0, "frames_1": 0, "frames_2": 0, "frames_48": 0,
                  **{f"ragged_{P}": 0 for P in (1, 127, 128, 129, 255, 257, 20011)}, "delta_None": 0, "delta_small": 0,
                  "delta_large": 0, "exact_edges": 0}


@pytest.fixture(scope="module")
def dev(built):
    from vidu4d_b200 import _capi
    _capi.load()
    return torch.device("cuda:0")


def max_frames(B):
    """The largest M whose tables and their gradients fit the backward's shared memory (sr_bob_warp_table_floats)."""
    from vidu4d_b200 import _capi
    from vidu4d_b200.warp import TABLE_SMEM_MAX
    lib = _capi.load()
    M = 1
    while 2 * 4 * lib.sr_bob_warp_table_floats(B, M + 1) <= TABLE_SMEM_MAX:
        M += 1
    return M


def _gpu(s, dev):
    from vidu4d_b200.warp import bob_warp_tables
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    tab = {k: T(v).requires_grad_(True) for k, v in s["tab"].items()}
    xyz, rot = T(s["xyz"]).requires_grad_(True), T(s["rot"]).requires_grad_(True)
    delta = None if s["delta"] is None else T(s["delta"]).requires_grad_(True)
    xc, rc, ent = bob_warp_tables(xyz, rot, tab["oq"], tab["ot"], tab["ig"], (tab["sr"], tab["sd"]), (tab["cq"], tab["ct"]),
                                  delta)
    torch.autograd.backward((xc, rc, ent), (T(s["gx"]), T(s["gr"]), T(s["ge"])))
    n = lambda t: t.detach().cpu().numpy().astype(np.float64)  # noqa: E731
    out = dict(xyz_cam=n(xc), rot_cam=n(rc), entropy=n(ent), g_xyz=n(xyz.grad), g_rot=n(rot.grad),
               **{"g_" + k: n(v.grad) for k, v in tab.items()})
    if delta is not None:
        out["g_delta"] = n(delta.grad)
    return out


def _cmp(name, what, mine, e, report, skip=None):
    tol = sb.K * sb.U * e.b + sb.FLOOR
    err = np.abs(mine - e.v)
    ratio = err / tol
    ratio = np.where(np.isnan(mine), np.inf, ratio)
    if skip is not None:
        ratio = np.where(skip, 0.0, ratio)
    i = int(np.argmax(ratio))
    report[what] = max(report.get(what, 0.0), float(ratio.flat[i]))
    assert ratio.flat[i] <= 1.0, (name, what, "element", np.unravel_index(i, mine.shape), "gpu", mine.flat[i], "value",
                                  e.v.flat[i], "bound", tol.flat[i])


def run(name, s, dev):
    """The model (zeroing the knife points' upstream in s), the GPU, and every element compared.  Returns (model, gpu)."""
    m = sb.warp_model(s["xyz"], s["rot"], s["tab"], s["delta"], s["gx"], s["gr"], s["ge"])
    kn = m["knife"]
    s["gx"][:, kn] = 0.0
    s["gr"][:, kn] = 0.0
    s["ge"][kn] = 0.0
    g = _gpu(s, dev)
    report = {}
    for k in ("xyz_cam", "rot_cam"):
        _cmp(name, k, g[k], m[k], report, skip=np.broadcast_to(kn[None, :, None], g[k].shape))
    _cmp(name, "entropy", g["entropy"], m["entropy"], report, skip=kn)
    for k in ("g_xyz", "g_rot", "g_delta"):
        if k in g:
            _cmp(name, k, g[k], m[k], report, skip=np.broadcast_to(kn[:, None], g[k].shape))
            assert (g[k][kn] == 0).all(), (name, k, "knife rows must be exactly 0")
    for k in sb.TABLE_GRADS:
        _cmp(name, k, g[k], m[k], report)
    nk = int(kn.sum())
    print(f"\n[{name}] P={s['xyz'].shape[0]} B={s['tab']['oq'].shape[0]} M={s['tab']['sr'].shape[0]}: knife {nk}; "
          + ", ".join(f"{k} {v:.3g}" for k, v in report.items()))
    assert nk <= 4 * KNIFE_MEASURED[name] + 8, (name, "knife points", nk)
    return m, g


@pytest.mark.parametrize("B", BONES)
def test_bone_grid(B, dev):
    """Both templates (B <= 32 and B > 32) and every residue of B mod 4 (blend_vjp's 4-bone passes) and B mod 3 (the
    3-bone passes of the skinning VJP), wide and narrow bones alternating, M = 2, 257 points."""
    s = scene(seed=200 + B, P=257, B=B, M=2, delta="small", wide=B % 2 == 1)
    run(f"bones_{B}", s, dev)


def test_bone_grid_reaches_its_edges():
    assert {B % 4 for B in BONES if B > 4} == {0, 1, 2, 3} and {B % 3 for B in BONES if B > 3} == {0, 1, 2}
    assert min(BONES) == 1 and max(BONES) == 64 and any(B <= 32 for B in BONES) and any(B > 32 for B in BONES)


def test_wide_bones(dev):
    s = scene(seed=11, P=2000, B=25, M=3, delta="small", wide=True)
    m, _ = run("wide", s, dev)
    w = sb.skin(sb._pts(s["xyz"]), sb._bones(s["tab"]["oq"], s["tab"]["ot"], s["tab"]["ig"]), sb._E.leaf(s["delta"]))["w"].v
    assert np.median((w > 1e-3).sum(-1)) >= 4


def test_narrow_bones(dev):
    s = scene(seed=12, P=2000, B=25, M=2, delta="small", wide=False)
    run("narrow", s, dev)
    sk = sb.skin(sb._pts(s["xyz"]), sb._bones(s["tab"]["oq"], s["tab"]["ot"], s["tab"]["ig"]), sb._E.leaf(s["delta"]))
    underflow = (sk["w"].f == 0) & (sk["w"].v > 0)
    assert underflow.sum() >= 0.05 * underflow.size, int(underflow.sum())


@pytest.mark.parametrize("M", [1, 2, "max"])
def test_frames(M, dev):
    """The upstream of frame m scaled by 10^(-6 m / (M-1)); the last frame's exactly 0 when M > 1."""
    B = 64
    M = max_frames(B) if M == "max" else M
    assert M in (1, 2, 48)
    s = scene(seed=300 + M, P=300, B=B, M=M, delta="small", wide=True)
    sc = (10.0 ** (-6.0 * np.arange(M) / max(M - 1, 1))).astype(np.float32)
    s["gx"] *= sc[:, None, None]
    s["gr"] *= sc[:, None, None]
    if M > 1:
        s["gx"][-1] = 0.0
        s["gr"][-1] = 0.0
    _, g = run(f"frames_{M}", s, dev)
    if M > 1:
        assert (g["g_sr"][-1] == 0).all() and (g["g_sd"][-1] == 0).all()
        assert (g["g_cq"][-1] == 0).all() and (g["g_ct"][-1] == 0).all()


@pytest.mark.parametrize("P", [1, 127, 128, 129, 255, 257, 20011])
def test_ragged_points(P, dev):
    s = scene(seed=400 + P % 97, P=P, B=25, M=2, delta="small", wide=True)
    run(f"ragged_{P}", s, dev)


@pytest.mark.parametrize("delta", [None, "small", "large"])
def test_delta(delta, dev):
    s = scene(seed=500, P=1000, B=25, M=2, delta=delta, wide=True)
    run(f"delta_{delta}", s, dev)
    if delta == "large":
        bones = sb._bones(s["tab"]["oq"], s["tab"]["ot"], s["tab"]["ig"])
        a0 = sb.skin(sb._pts(s["xyz"]), bones, None)["anchor"]
        a1 = sb.skin(sb._pts(s["xyz"]), bones, sb._E.leaf(s["delta"]))["anchor"]
        assert (a0 != a1).mean() > 0.3


def test_exact_tie_and_orthogonal_rotation(dev):
    """Bones 1 and 2 share their skinning tables bit for bit (an exact logit tie) but not their rotations: taking bone 2
    as the anchor would flip every sign and so rot_cam.  Bone 3's rotation is exactly orthogonal to bone 0's: sign -1."""
    s = scene(seed=600, P=1000, B=4, M=2, delta=None, wide=True)
    tab = s["tab"]
    for k in ("oq", "ot", "ig"):
        tab[k][2] = tab[k][1]
    tab["sr"][:, 2] = -tab["sr"][:, 1]
    tab["sd"][:, 2] = -tab["sd"][:, 1]
    tab["sr"][:, 0] = (1.0, 0.0, 0.0, 0.0)
    tab["sr"][:, 3] = (0.0, 1.0, 0.0, 0.0)
    m, g = run("exact_edges", s, dev)
    sk = sb.skin(sb._pts(s["xyz"]), sb._bones(tab["oq"], tab["ot"], tab["ig"]), None)
    assert (sk["anchor"] == 1).sum() > 10 and not (sk["anchor"] == 2).any()
    a0 = sk["anchor"] == 0
    assert a0.sum() > 10 and (sk["w"].f[a0, 3] > 0).all()
    # flipping bone 3's sign moves QR by 2 w3 |r3|: that must exceed the rot_cam tolerance by far, or the case is vacuous
    assert sk["w"].v[a0, 3].max() > 100 * sb.K * sb.U * m["rot_cam"].b[:, a0].max()


# ------------------------------------------------------------------------------------------------ reproj and cycle
def _t(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def _reproj_gpu(s, dev):
    from vidu4d_b200 import _capi
    M, HW = s["xyz_m"].shape[:2]
    B = s["tab"]["oq"].shape[0]
    T = {k: _t(v, dev) for k, v in s["tab"].items()}
    x, Km, hxy, mask, det = (_t(s[k], dev) for k in ("xyz_m", "Kmat", "hxy", "mask", "det"))
    d = None if s["delta"] is None else _t(s["delta"], dev)
    w, gl = _t(np.array([s["weight"]], np.float32), dev), _t(np.array([s["g_loss"]], np.float32), dev)
    xy = torch.empty((M, HW, 2), device=dev)
    terms, counts = torch.empty(M, device=dev), torch.empty(M, dtype=torch.int32, device=dev)
    scale, loss = torch.empty(1, device=dev), torch.empty((), device=dev)
    hs = hxy.shape[-1]
    tabs = (T["oq"], T["ot"], T["ig"], d, T["sr"], T["sd"], T["cq"], T["ct"])
    _capi.call("sr_reproj_loss_forward", dev, M, HW, 1, B, hs, float(s["train_res"]), x, *tabs, Km, hxy, mask, det, w, xy,
               terms, counts, scale, loss)
    gx = torch.empty((M, HW, 3), device=dev)
    gd = None if d is None else torch.empty((M, HW, B), device=dev)
    gtab = torch.empty(int(_capi.load().sr_bob_warp_table_floats(B, M)), device=dev)
    _capi.call("sr_reproj_loss_backward", dev, M, HW, 1, B, hs, x, *tabs, Km, hxy, mask, det, scale, gl, gx, gd, gtab)
    n = lambda t: t.cpu().numpy().astype(np.float64)  # noqa: E731
    from vidu4d_b200.warp import split_table_grads
    out = dict(xy=n(xy), terms=n(terms), counts=counts.cpu().numpy(), scale=n(scale)[0], loss=n(loss), g_xyz=n(gx),
               **{"g_" + k: n(v) for k, v in zip(sb.WARP_TABLES, split_table_grads(gtab, B, M))})
    if gd is not None:
        out["g_delta"] = n(gd)
    return out


def run_reproj(name, s, dev):
    kn = sb.reproj_knife(s["xyz_m"], s["delta"], s["tab"], s["Kmat"], s["hxy"])
    s["mask"][kn] = 0.0
    m = sb.reproj_model(s["xyz_m"], s["delta"], s["tab"], s["Kmat"], s["hxy"], s["mask"], s["det"], s["weight"],
                        s["train_res"], s["g_loss"])
    g = _reproj_gpu(s, dev)
    assert np.array_equal(g["counts"], m["counts"]), (name, g["counts"], m["counts"])
    report = {}
    _cmp(name, "xy_reproj", g["xy"], m["xy"], report, skip=np.broadcast_to(kn[..., None], g["xy"].shape))
    for k in ("terms", "loss", "scale", "g_xyz", "g_delta") + sb.TABLE_GRADS:
        if k in g:
            _cmp(name, k, g[k], m[k], report)
    assert (g["g_xyz"][kn] == 0).all() and ("g_delta" not in g or (g["g_delta"][kn] == 0).all()), name
    nk = int(kn.sum())
    print(f"\n[{name}] M={s['xyz_m'].shape[0]} HW={s['xyz_m'].shape[1]} B={s['tab']['oq'].shape[0]}: knife {nk}; "
          + ", ".join(f"{k} {v:.3g}" for k, v in report.items()))
    assert nk <= 8 + 1e-3 * kn.size, (name, "knife pixels", nk)
    return m, g


def _cycle_gpu(s, dev):
    from vidu4d_b200 import _capi
    from vidu4d_b200.warp import table_views
    P, M, B = s["xyz"].shape[0], s["xyz_cam"].shape[0], s["tab"]["ig"].shape[0]
    T = {k: _t(v, dev) for k, v in s["tab"].items()}
    x, xc, w = _t(s["xyz"], dev), _t(s["xyz_cam"], dev), _t(s["weights"], dev)
    d = None if s["delta"] is None else _t(s["delta"], dev)
    terms, counts = torch.empty((M, 3), device=dev), torch.empty((M, 3), dtype=torch.int32, device=dev)
    scale, loss = torch.empty(3, device=dev), torch.empty((), device=dev)
    tabs = (T["oq"], T["ot"], T["ig"], d, T["sr"], T["sd"], T["cq"], T["ct"])
    _capi.call("sr_cycle_loss_forward", dev, P, B, M, x, xc, *tabs, w, terms, counts, scale, loss)
    gxc, gx = torch.empty((M, P, 3), device=dev), torch.empty((P, 3), device=dev)
    gd = None if d is None else torch.empty((M, P, B), device=dev)
    gtab = torch.empty(int(_capi.load().sr_cycle_loss_table_floats(B, M)), device=dev)
    gl = _t(np.array([s["g_loss"]], np.float32), dev)
    _capi.call("sr_cycle_loss_backward", dev, P, B, M, x, xc, *tabs, scale, gl, gxc, gx, gd, gtab)
    n = lambda t: t.cpu().numpy().astype(np.float64)  # noqa: E731
    views = table_views(gtab, ((M, B, 4), (M, B, 3), (B, 3), (M, B, 4), (M, B, 4), (M, 4), (M, 3)))
    out = dict(terms=n(terms), counts=counts.cpu().numpy(), scale=n(scale), loss=n(loss), g_xyz=n(gx), g_xyz_cam=n(gxc),
               **{"g_" + k: n(v) for k, v in zip(sb.CYCLE_TABLES, views)})
    if gd is not None:
        out["g_delta"] = n(gd)
    return out


def run_cycle(name, s, dev):
    m = sb.cycle_model(s["xyz"], s["xyz_cam"], s["tab"], s["delta"], s["weights"], s["g_loss"])
    kn = m["knife"]
    if kn.any():                 # knife surfels leave the inputs on both sides
        s.update(xyz=s["xyz"][~kn], xyz_cam=s["xyz_cam"][:, ~kn], delta=None if s["delta"] is None else s["delta"][:, ~kn])
        m = sb.cycle_model(s["xyz"], s["xyz_cam"], s["tab"], s["delta"], s["weights"], s["g_loss"])
    g = _cycle_gpu(s, dev)
    assert np.array_equal(g["counts"], m["counts"]), (name, g["counts"], m["counts"])
    report = {}
    for k in ("terms", "loss", "scale", "g_xyz", "g_xyz_cam", "g_delta") + sb.TABLE_GRADS:
        if k in g:
            _cmp(name, k, g[k], m[k], report)
    nk = int(kn.sum())
    print(f"\n[{name}] P={len(kn)} B={s['tab']['ig'].shape[0]} M={s['xyz_cam'].shape[0]}: knife {nk}; "
          + ", ".join(f"{k} {v:.3g}" for k, v in report.items()))
    # a surfel is dropped for a knife value in any of its M frames; about 0.4% of (surfel, frame) pairs are knives on
    # these scenes when measured, mostly the anchor and '> 0' decisions
    assert nk <= 8 + 1e-2 * len(kn) * s["xyz_cam"].shape[0], (name, "knife surfels", nk)
    return m, g


@pytest.mark.parametrize("B", BONES)
def test_reproj_and_cycle_bone_grid(B, dev):
    """Both templates of reproj_fwd / reproj_bwd and cycle_fwd / cycle_bwd, every residue of B mod 4 and B mod 3."""
    run_reproj(f"reproj_bones_{B}", sb.reproj_scene(seed=700 + B, M=2, HW=257, B=B, delta=B % 2 == 0), dev)
    run_cycle(f"cycle_bones_{B}", sb.cycle_scene(seed=800 + B, P=257, B=B, M=2, delta=B % 2 == 1), dev)


def max_cycle_frames(B):
    from vidu4d_b200 import _capi
    from vidu4d_b200.warp import TABLE_SMEM_MAX
    lib = _capi.load()
    M = 1
    while 2 * 4 * lib.sr_cycle_loss_table_floats(B, M + 1) <= TABLE_SMEM_MAX:
        M += 1
    return M


@pytest.mark.parametrize("M", [1, 2, "max"])
def test_reproj_frames(M, dev):
    """reproj at B = 64 up to the largest M its tables allow; the upstream scaled per frame through mask (1 .. 1e-6) and
    the last frame undetected: its counts, se3 and camera gradients exactly 0."""
    M = max_frames(64) if M == "max" else M
    assert M in (1, 2, 48)
    s = sb.reproj_scene(seed=900 + M, M=M, HW=130, B=64)
    s["mask"] *= (10.0 ** (-6.0 * np.arange(M) / max(M - 1, 1))).astype(np.float32)[:, None]
    if M > 1:
        s["det"][-1] = 0.0
    _, g = run_reproj(f"reproj_frames_{M}", s, dev)
    if M > 1:
        assert g["counts"][-1] == 0
        for k in ("g_sr", "g_sd", "g_cq", "g_ct"):
            assert (g[k][-1] == 0).all(), k


@pytest.mark.parametrize("M", [1, 2, "max"])
def test_cycle_frames(M, dev):
    M = max_cycle_frames(64) if M == "max" else M
    assert M in (1, 2, 26)
    run_cycle(f"cycle_frames_{M}", sb.cycle_scene(seed=1000 + M, P=130, B=64, M=M), dev)


@pytest.mark.parametrize("n", [1, 127, 128, 129, 257, 20011])
def test_reproj_and_cycle_ragged(n, dev):
    """HW and P at the 128-thread (reproj, cycle backward) and 256-thread (cycle forward) block edges.  A dead lane of
    reproj's last block reads pixel 0 of its frame, whose mask is not 0."""
    run_reproj(f"reproj_ragged_{n}", sb.reproj_scene(seed=1100 + n % 97, M=2, HW=n, B=25), dev)
    run_cycle(f"cycle_ragged_{n}", sb.cycle_scene(seed=1200 + n % 97, P=n, B=25, M=2), dev)
