"""Every per-surfel record the forward preprocess writes (T, the AABB centre, opacity, normal, rgb, the clamp bits, the
depth, radii and tiles_touched) against the float64 restatement of tests/preprocess_bounds.py, under its rounding-error
bound, with the surfels whose decisions lie within their bound of a threshold masked.

The cases: the 7 golden fixtures (whose normal, opacity, rgb and clamp bits the kernel also reproduces bit for bit), the
SH coefficient-count grid (both staging paths, a degree below the stored one, partial last blocks), the adversarial
geometry of preprocess_bounds.adversarial_scene (near plane, edge-on, d == 0, the radius floor, huge, far-off and
rectangle-edge surfels, unnormalised quaternions, SH colours at v = 0, and tests/cull_model.py's classes), 8-frame
batches with each per-frame input switched on alone and all together, a per-frame intrinsics table, and the near-plane
test of sr_mark_visible.  Each case asserts from the GPU's own buffers that it reaches its edge, and prints its knife
count and the largest err / bound per field."""
import numpy as np
import pytest
import torch

from . import preprocess_bounds as pb
from .conftest import GOLDEN_CASES, load_golden

pytestmark = pytest.mark.gpu

TAN = 0.5
# Knifed surfels measured per case on an H100; a case may knife at most 4 times as many plus 8.
KNIFE_MEASURED = {"golden id_deg3_64": 5, "golden rigid_bg_96x64": 13, "golden ragged_80x48_deg1": 5,
                  "golden precomp_init_70x50": 1, "sh M=1 deg=0 P=20000": 22, "sh M=4 deg=1 P=20000": 15,
                  "sh M=9 deg=2 P=20000": 21, "sh M=16 deg=0 P=20000": 18, "sh M=16 deg=1 P=20000": 18,
                  "sh M=16 deg=3 P=20000": 18, "adversarial_104x72": 378, "adversarial_37x23": 167,
                  "batch8 means3D": 825, "batch8 rotations": 884, "batch8 scales": 841, "batch8 opacities": 952,
                  "batch8 shs": 952, "batch8 colors_precomp": 952, "batch8 camera": 908, "batch8 all": 827,
                  "batch8 intrinsics": 693}


@pytest.fixture(scope="module")
def dev(built):
    from vidu4d_b200 import _capi, rasterizer as RZ
    _capi.load()
    RZ.set_sync_mode(True)
    return torch.device("cuda:0")


def _np(x):
    return x.detach().cpu().numpy()


def _check_knife(name, rep):
    assert rep["knife"] <= 4 * KNIFE_MEASURED.get(name, 0) + 8, (name, "knifed surfels", rep["knife"])


def _single(inp, cam, dev, colour=None):
    """One frame through sr_forward (test_gpu_parity._run_ours); returns the decoded buffers with radii."""
    from .test_gpu_parity import _run_ours
    P = inp["means3D"].shape[0]
    pre = inp["shs"] is None
    e = np.zeros((0,), np.float32)
    from vidu4d_b200.synthetic import projection_matrix
    d = dict(means3D=inp["means3D"], scales=inp["scales"], rotations=inp["rotations"],
             opacities=np.asarray(inp["opacities"], np.float32).reshape(P, 1),
             shs=e if pre else inp["shs"], colors_precomp=inp["colors_precomp"] if pre else e,
             viewmatrix=cam["vm"].reshape(4, 4), projmatrix=projection_matrix(*cam["tan"]).astype(np.float32),
             campos=cam["campos"], bg=np.zeros(3, np.float32),
             meta=np.array([P, cam["W"], cam["H"], inp["deg"], int(pre)], np.int64),
             tanfov=np.array(cam["tan"], np.float32))
    r = _run_ours(d, dev, with_grads=False)
    r["radii"] = _np(r["radii"])
    return r


def _run_check(name, r, inp, cam, src):
    rep = pb.check_records(r, inp, cam, src, name)
    pb.print_report(name, rep)
    _check_knife(name, rep)
    return rep


# ------------------------------------------------------------------------------------------------ goldens
@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_golden(name, dev):
    g = load_golden(name)
    inp, cam = pb.golden_inputs(g)
    r = _single(inp, cam, dev)
    src = "precomp" if inp["shs"] is None else "sh"
    rep = _run_check(f"golden {name}", r, inp, cam, src)
    assert rep["visible"] == int((g["ref_radii"] > 0).sum()) or rep["knife"] > 0
    # the records the reference wrote, bit for bit: opacity and normal always, rgb and clamp bits with SH colours (the
    # reference leaves them unwritten with precomputed colours)
    rec = pb.records(r)
    vis = g["ref_radii"] > 0
    no = g["ref_geom_normal_opacity"][vis]
    assert np.array_equal(rec["normal"][vis].view(np.uint32), no[:, :3].view(np.uint32)), name
    assert np.array_equal(rec["opacity"][vis].view(np.uint32), no[:, 3].view(np.uint32)), name
    if src == "sh":
        assert np.array_equal(rec["rgb"][vis].view(np.uint32), g["ref_geom_rgb"][vis].view(np.uint32)), name
        assert np.array_equal(rec["clamp"][vis], g["ref_geom_clamped"][vis].astype(bool)), name
    if name == "near_cull_64":
        d = _np(r["depths"])
        assert (r["radii"] == 0).any() and (r["radii"] > 0).any() and (d[r["radii"] > 0] > pb.NEAR).all()
        m = pb.model(inp, cam)
        assert ((m["depth"][0].v <= float(pb.NEAR)) & (r["radii"] == 0)).any()


# ------------------------------------------------------------------------------------------------ SH grid
@pytest.mark.parametrize("P", [1, 255, 256, 257, 20000])
@pytest.mark.parametrize("M,deg", [(1, 0), (4, 1), (9, 2), (16, 0), (16, 1), (16, 3)])
def test_sh_grid(M, deg, P, dev):
    """3M in {3, 12, 27, 48}: the scalar (3M % 4 != 0) and float4 staging paths, with the padded row stride; the last
    block holds 1, 255 or 256 rows."""
    from tests.golden.make_golden import build_case
    c = build_case(P, 96, 80, 500 + M + P, sh_degree=deg)
    shs = np.ascontiguousarray(c["shs"].reshape(P, -1, 3)[:, :M])
    inp = dict(means3D=c["means3D"], rotations=c["rotations"], scales=c["scales"], opacities=c["opacities"], shs=shs,
               colors_precomp=None, deg=deg)
    cam = pb.camera(c["viewmatrix"], c["campos"], 96, 80, (TAN, TAN))
    r = _single(inp, cam, dev)
    rep = _run_check(f"sh M={M} deg={deg} P={P}", r, inp, cam, "sh")
    # the last block's rows reach the check: a visible surfel among them
    last = np.arange(P) >= (P - 1) // 256 * 256
    assert (r["radii"][last] > 0).any(), (M, deg, P)
    assert rep["visible"] > 0.5 * P


# ------------------------------------------------------------------------------------------------ adversarial geometry
ADV = {"adversarial_104x72": (11, 104, 72, 400), "adversarial_37x23": (12, 37, 23, 200)}


@pytest.mark.parametrize("name", list(ADV))
def test_adversarial(name, dev):
    seed, W, H, n = ADV[name]
    inp, cam, label = pb.adversarial_scene(seed, W, H, n)
    r = _single(inp, cam, dev)
    rep = _run_check(name, r, inp, cam, "sh")
    m = pb.model(inp, cam)
    rec = pb.records(r)
    vis, ok = r["radii"] > 0, ~m["knife"]
    depth = m["depth"][0].v                                     # exact for the near class (the turned camera)
    near = (label == "near") & ok
    z = float(pb.NEAR)
    assert (near & (depth <= z) & ~vis).any() and (near & (depth > z) & (depth < z + 1e-6) & vis).any()
    eo = (label == "edge_on") & ok
    x_v = inp["means3D"][:, 2]                                  # view x; the view normal (1, 0, 0) flips by -sign(x_v)
    assert (eo & vis & (rec["normal"][:, 0] < 0)).any() and (eo & vis & (rec["normal"][:, 0] > 0)).any()
    assert (eo & (x_v == 0) & ~vis).sum() > 0 and not (eo & (x_v == 0) & vis).any()
    dz = (label == "d_zero") & ok & (m["d"].v == 0)
    assert dz.any() and not vis[dz].any()
    fl = (label == "floor") & vis & ok
    assert fl.any() and (r["radii"][fl] == 3).all()
    gx, gy = (W + 15) // 16, (H + 15) // 16
    tt = pb.records(r)["tiles_touched"]
    assert (tt[(label == "huge") & vis] == gx * gy).any()
    assert not vis[label == "far_off"].any()
    # rectangle edges: a visible surfel with px - 3 or px + 18 within 0.3 px of a multiple of 16, and one with px - 3
    # in (-1, 0)
    px = rec["centre"][:, 0].astype(np.float64)
    re = (label == "rect_edge") & vis
    on16 = np.abs((px - 3) / 16 - np.round((px - 3) / 16)) * 16
    on16b = np.abs((px + 18) / 16 - np.round((px + 18) / 16)) * 16
    assert (re & (on16 < 0.3) & (px > 16)).any() and (re & (on16b < 0.3)).any() and (re & (px - 3 < 0) & (px - 3 > -1)).any()
    qn = np.linalg.norm(inp["rotations"].astype(np.float64), axis=1)
    qs = (label == "quat_norm") & vis
    assert (qn[qs] < 1e-2).any() and (qn[qs] > 1e2).any()
    cl = rec["clamp"][vis & ok]
    assert cl.any(0).all() and (~cl).any(0).all()
    for c in ("grazing", "dc_zero", "subpixel", "offimage", "threshold", "cloud"):
        assert ((label == c) & vis).any(), c


def test_near_plane_mark_visible(dev):
    """sr_mark_visible's near-plane decision equals the forward's, bit for bit, at view z = 0.2 and its fp32
    neighbours (where the forward's other decisions let a surfel through)."""
    from vidu4d_b200 import rasterizer as RZ
    from vidu4d_b200.synthetic import projection_matrix
    inp, cam, label = pb.adversarial_scene(13, 64, 64, 400)
    r = _single(inp, cam, dev)
    m = pb.model(inp, cam)
    means = torch.from_numpy(inp["means3D"]).to(dev)
    vm = torch.from_numpy(cam["vm"].reshape(4, 4)).to(dev)
    pm = torch.from_numpy(projection_matrix(TAN, TAN).astype(np.float32)).to(dev)
    mark = _np(RZ._C.mark_visible(means, vm, pm)).astype(bool)
    near = label == "near"
    front = m["depth"][0].v > float(pb.NEAR)                     # exact at these surfels: their depth has no rounding
    assert (m["depth"][0].b[near] == 0).all()
    assert np.array_equal(mark[near], front[near])
    assert mark[near].any() and (~mark[near]).any()
    assert not (r["radii"] > 0)[~mark].any()                     # the forward draws nothing mark_visible drops
    ok = near & ~m["knife"] & front
    assert (r["radii"][ok] > 0).any()


# ------------------------------------------------------------------------------------------------ batches
M8 = 8
SWITCHES = ("means3D", "rotations", "scales", "opacities", "shs", "colors_precomp", "camera", "all")


def _batch_inputs(switch, P, rng):
    from vidu4d_b200.synthetic import object_scene
    sc = object_scene(P, seed=70, center=(0.0, 0.0, 0.0))
    base = dict(means3D=sc.means3D, rotations=sc.rotations, scales=sc.scales, opacities=sc.opacities.reshape(P),
                shs=sc.shs, colors_precomp=rng.uniform(-0.2, 1.2, (P, 3)).astype(np.float32))
    names = [k for k in base if k != "colors_precomp"] if switch == "all" else [switch] if switch in base else []
    per = {}
    for k in names:
        x = base[k]
        fr = []
        for f in range(M8):
            d = 0.02 * f * rng.normal(size=x.shape)
            if k == "rotations":
                fr.append((x + d) * rng.uniform(0.1, 10.0, (P, 1)))     # unnormalised, differently per frame
            elif k == "scales":
                fr.append(x * (1 + np.abs(d)))
            elif k == "opacities":
                fr.append(np.clip(x + d, 0.0, 1.0))
            else:
                fr.append(x + d)
        per[k] = np.stack(fr).astype(np.float32)
    return base, per


def _frame_inputs(base, per, f, precomp):
    g = lambda k: per[k][f] if k in per else base[k]                        # noqa: E731
    return dict(means3D=g("means3D"), rotations=g("rotations"), scales=g("scales"), opacities=g("opacities"),
                shs=None if precomp else g("shs"), colors_precomp=g("colors_precomp") if precomp else None, deg=3)


def _batch(name, dev, base, per, cams, W, H, precomp, rows=None):
    from vidu4d_b200 import debug as dbg, rasterizer as RZ
    P = base["means3D"].shape[0]
    vms, cps = cams
    t = lambda k: torch.from_numpy(per[k] if k in per else base[k]).to(dev)   # noqa: E731
    e = torch.empty((0,), device=dev)
    opac = t("opacities")
    opac = opac.reshape(*opac.shape, 1)
    tan = (float("nan"), float("nan")) if rows is not None else (TAN, TAN)
    kw = {} if rows is None else {"intrinsics": torch.tensor(rows, device=dev)}
    vm_t, cp_t = torch.from_numpy(vms).to(dev), torch.from_numpy(cps).to(dev)
    nr, color, allmap, radii, gb, bb, ib = RZ._C.rasterize_gaussians_batch(
        torch.zeros(3, device=dev), t("means3D"), t("colors_precomp") if precomp else e, opac, t("scales"), t("rotations"),
        1.0, vm_t, vm_t, tan[0], tan[1], H, W, e if precomp else t("shs"), 3, cp_t, **kw)[:7]
    reps, recs = [], []
    for f in range(M8):
        dec = dbg.decode(gb.view(M8, -1)[f], bb.view(M8, -1)[f], ib.view(M8, -1)[f], P, W, H, nr[f])
        dec["radii"] = _np(radii[f])
        row = rows[f] if rows is not None else None
        cam = pb.camera(vms[f], cps[f], W, H, row[:2] if row else (TAN, TAN), row[2:] if row else None)
        rep = pb.check_records(dec, _frame_inputs(base, per, f, precomp), cam, "precomp" if precomp else "sh",
                               f"{name} frame {f}")
        reps.append(rep)
        recs.append(pb.records(dec))
    tot = dict(max((r for r in reps), key=lambda r: r["knife"]))
    for k in tot:
        tot[k] = sum(r[k] for r in reps) if k in ("knife", "knife_clamp", "visible") else max(r.get(k, 0.0) for r in reps)
    pb.print_report(name, tot)
    _check_knife(name, tot)
    return recs, _np(radii)


def _orbit_cams(M, same):
    from vidu4d_b200.synthetic import orbit_view
    vms, cps = [], []
    for f in range(M):
        R, tr = orbit_view(0 if same else 3 * f + 1, 64)
        w2c = np.eye(4)
        w2c[:3, :3] = R
        w2c[:3, 3] = tr
        vms.append(w2c.T.astype(np.float32))
        cps.append((-R.T @ tr).astype(np.float32))
    return np.stack(vms), np.stack(cps)


@pytest.mark.parametrize("switch", SWITCHES)
def test_batch8_per_frame_input(switch, dev):
    """8 frames; one per-frame input (or the camera, or every input) differs between frames, the rest is shared.  Every
    frame's records against the model of that frame's inputs."""
    rng = np.random.default_rng(71 + SWITCHES.index(switch))
    P, W, H = 5000, 120, 88
    base, per = _batch_inputs(switch, P, rng)
    precomp = switch == "colors_precomp"
    if precomp:
        per["colors_precomp"] = np.stack([base["colors_precomp"] + 0.05 * f for f in range(M8)]).astype(np.float32)
    cams = _orbit_cams(M8, same=switch not in ("camera", "all"))
    recs, radii = _batch(f"batch8 {switch}", dev, base, per, cams, W, H, precomp)
    # the switched input reaches the records: frames 0 and 7 differ in the fields it feeds
    field = {"means3D": "T", "rotations": "normal", "scales": "T", "opacities": "opacity", "shs": "rgb",
             "colors_precomp": "rgb", "camera": "T", "all": "T"}[switch]
    both = (radii[0] > 0) & (radii[M8 - 1] > 0)
    assert both.sum() > 0.3 * P
    assert not np.array_equal(recs[0][field][both], recs[M8 - 1][field][both]), switch
    assert switch == "camera" or per, switch


def test_batch8_intrinsics_table(dev):
    """Per-frame tangents and non-integer principal-point offsets of either sign from a device table, one frame with the
    object half off the image, per-frame positions and cameras."""
    rng = np.random.default_rng(79)
    P, W, H = 5000, 120, 88
    base, per = _batch_inputs("means3D", P, rng)
    cams = _orbit_cams(M8, same=False)
    rows = [(0.5, 0.45, 7.25, -3.5), (0.44, 0.39, -11.75, 5.125), (0.55, 0.5, 60.5, -30.0), (0.5, 0.5, 0.0, 0.0),
            (0.61, 0.37, -0.375, 0.625), (0.3, 0.33, 2.5, 19.75), (0.52, 0.48, -40.125, -12.5), (0.47, 0.58, 0.5, -0.5)]
    recs, radii = _batch("batch8 intrinsics", dev, base, per, cams, W, H, False, rows)
    # frame 2 (cx offset 60.5 = half the width): the object's right half falls off the image
    cx = recs[2]["centre"][radii[2] > 0, 0]
    assert (cx > W).any() and (cx < W).any()
    # the offsets reach T: frame 3 (zero offsets) against the scalar path is pinned by test_gpu_cameras; here frame 0's
    # T[2] carries cx = W/2 + 7.25
    assert not np.array_equal(recs[0]["T"][radii[0] > 0], recs[3]["T"][radii[0] > 0])
