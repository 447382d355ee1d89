"""The forward preprocess's float64 restatement (tests/preprocess_bounds.py) pinned without a GPU: its own fp32 shadow,
the CPU oracle's fp32 forward and the reference's own records in the golden fixtures all lie within its bound, the
table path's intrinsics equal the scalar path's, and each of five plausible kernel mistakes, applied to the shadow,
falls outside the bound on a clear share of the visible surfels."""
import numpy as np
import pytest

from . import preprocess_bounds as pb
from .conftest import GOLDEN_CASES, load_golden, oracle_forward_from_golden

MUTANT_SHARE = 0.25          # a mistake must put at least this share of the visible surfels outside the bound


def _build(P, W, H, seed, **kw):
    from tests.golden.make_golden import build_case
    c = build_case(P, W, H, seed, **kw)
    pre = int(c["meta"][4])
    inp = dict(means3D=c["means3D"], rotations=c["rotations"], scales=c["scales"], opacities=c["opacities"],
               shs=None if pre else c["shs"], colors_precomp=c["colors_precomp"] if pre else None, deg=int(c["meta"][3]))
    return inp, pb.camera(c["viewmatrix"], c["campos"], W, H, c["tanfov"]), c


BUILT = {"id_2000_96x80": dict(P=2000, W=96, H=80, seed=401),
         "rigid_3000_120x72": dict(P=3000, W=120, H=72, seed=402, rigid=True),
         "deg1_rigid_1500_64": dict(P=1500, W=64, H=64, seed=403, rigid=True, sh_degree=1),
         "precomp_1000_70x50": dict(P=1000, W=70, H=50, seed=404, colors_precomp=True),
         "near_900_64": dict(P=900, W=64, H=64, seed=405, center=(0.0, 0.0, 0.45), sh_degree=2)}


@pytest.mark.parametrize("name", list(BUILT))
def test_shadow_and_oracle_within_bound_on_built_scenes(name):
    from oracle import surfel_oracle as so
    inp, cam, c = _build(**BUILT[name])
    m = pb.model(inp, cam)
    src = "precomp" if inp["shs"] is None else "sh"
    pb.print_report(name + " shadow", pb.check_records(pb.shadow_records(m), inp, cam, src, name, m))
    P, W, H = [int(v) for v in c["meta"][:3]]
    st = so.forward(c["means3D"], c["opacities"], c["scales"], c["rotations"], shs=inp["shs"],
                    colors_precomp=inp["colors_precomp"], sh_degree=inp["deg"], W=W, H=H, tanfovx=0.5, tanfovy=0.5,
                    bg=c["bg"], viewmatrix=c["viewmatrix"], projmatrix=c["projmatrix"], campos=c["campos"])
    # the oracle leaves rgb unwritten with precomputed colours
    rep = pb.check_records(pb.oracle_records(st), inp, cam, "sh" if src == "sh" else None, name + " oracle", m)
    pb.print_report(name + " oracle", rep)
    assert rep["visible"] > 0.3 * P


@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_oracle_and_reference_records_within_bound(name):
    """The CPU oracle's forward and the reference's own records (ref_geom_*) stored in each golden fixture.  The
    reference writes no rgb or clamp bit with precomputed colours, so those are checked on the SH fixtures only."""
    g = load_golden(name)
    inp, cam = pb.golden_inputs(g)
    m = pb.model(inp, cam)
    src = None if inp["shs"] is None else "sh"
    for who, rec in (("oracle", pb.oracle_records(oracle_forward_from_golden(g))), ("reference", pb.golden_records(g))):
        rep = pb.check_records(rec, inp, cam, src, f"{name} {who}", m)
        pb.print_report(f"{name} {who}", rep)
    assert rep["visible"] > 0
    if name == "near_cull_64":
        assert (m["depth"][0].v <= float(pb.NEAR)).any() and (m["depth"][0].v > float(pb.NEAR)).any()


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_shadow_within_bound_on_adversarial_classes(seed):
    """Every class of preprocess_bounds.adversarial_scene: the model's own fp32 evaluation stays within its bound and
    the classes reach their edges in the model."""
    W, H = (104, 72) if seed != 2 else (37, 23)
    inp, cam, label = pb.adversarial_scene(seed, W, H, 200)
    m = pb.model(inp, cam)
    rep = pb.check_records(pb.shadow_records(m), inp, cam, "sh", f"adversarial seed {seed}", m)
    pb.print_report(f"adversarial seed {seed}", rep)
    ok, vis, depth, z = ~m["knife"], m["visible"], m["depth"][0].v, float(pb.NEAR)
    near = label == "near"
    assert (near & ok & (depth <= z)).any() and (near & ok & (depth > z) & vis).any()
    eo = (label == "edge_on") & ok
    assert (eo & (m["cosv"].v == 0) & (depth > z)).any() and (eo & vis & (m["cosv"].v > 0)).any() and \
        (eo & vis & (m["cosv"].v < 0)).any()
    assert ((label == "d_zero") & ok & (m["d"].v == 0) & (m["cosv"].v != 0)).any()
    assert (m["radius"][(label == "floor") & vis & ok] == 3).all()
    huge = (label == "huge") & vis & ok
    gx, gy = (W + 15) // 16, (H + 15) // 16
    assert huge.sum() > 0 and (m["tiles_touched"][huge] == gx * gy).any()
    assert not vis[label == "far_off"].any()
    assert ((m["clamp"] & ~m["knife_clamp"]).any(0)).all() and ((~m["clamp"] & ~m["knife_clamp"] & vis[:, None]).any(0)).all()


def test_table_path_forms_scalar_intrinsics():
    """cam_of_frame with (tan_x, tan_y, 0, 0) forms make_cam's fp32 intrinsics bit for bit."""
    for W, H in ((64, 64), (75, 53), (136, 88), (1, 65535)):
        for tx, ty in ((0.5, 0.5), (0.42, 0.37), (1e-3, 7.5), (0.61, 0.55)):
            a = np.array(pb.intrinsics(W, H, (tx, ty)), np.float32)
            b = np.array(pb.intrinsics(W, H, (tx, ty), (0.0, 0.0)), np.float32)
            assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), (W, H, tx, ty)
    fx, fy, cx, cy = pb.intrinsics(75, 53, (0.5, 0.5), (7.25, -3.5))
    assert (cx, cy) == (np.float32(44.75), np.float32(23.0))


@pytest.mark.parametrize("mutant", pb.MUTANTS + ("campos0",))
def test_mutants_exceed_the_bound(mutant):
    """A plausible kernel mistake -- the flip dropped, cx / cy swapped in T[2] / T[5], SH_C1's sign flipped, the
    neighbouring surfel's SH row, frame 0's campos for another frame -- applied to the shadow falls outside the bound
    on a clear share of the visible surfels."""
    inp, cam, _ = _build(P=2000, W=120, H=72, seed=406, rigid=True)
    m = pb.model(inp, cam)
    if mutant == "campos0":
        cam0 = dict(cam, campos=cam["campos"] + np.float32([0.3, -0.2, 0.1]))
        bad = pb.model(inp, cam0)
    else:
        bad = pb.model(inp, cam, mutant=mutant)
    assert pb.exceed_share(pb.shadow_records(m), m) == 0.0
    share = pb.exceed_share(pb.shadow_records(bad), m)
    print(f"\n[{mutant}] share of visible surfels outside the bound {share:.3f}")
    assert share >= MUTANT_SHARE, (mutant, share)
