"""Forward-only rendering under the float64 oracle's rounding-error bound, element by element.

A. sr_post_forward_frames (csrc/postprocess.cu) on constructed allmaps, with no rasterizer in the loop: M frames of
   test_gpu_loss_bounds._frames (smooth depth with planted degenerate pixels on block seams and borders), each with its
   own world-view transform and, on the table path, its own camera row (both tangents and both offsets differ per
   frame).  Every map is held to tests/post_bounds.py's model of the frame's own camera.  The learnable background must be
   numpy's c + (1 - a) bk with each operation rounded, bit for bit, on a colour buffer whose frame stride is padded, and
   the padding must stay untouched.  The scalar path must equal sr_post_forward frame by frame, a table of the scalar
   tangents with zero offsets the scalar path, and the table path's surf_depth the loss pass's, all bit for bit.

B. renderer.render_frames end to end: test_gpu_batch_bounds' 104 x 72 scene of 6,000 surfels over T = 5 frames, with
   per-frame positions and orientations, that file's camera rows (the last frame's object cut by the right edge), and no
   features, 7 shared or 32 per-frame feature channels over a 3+F background.  The oracle composites each frame from the
   training forward's records, point list and tile ranges (test_gpu_grad_bounds._oracle_frame, which first holds those
   records to the preprocess model of that frame's inputs and camera row; one colour oracle per group of three feature
   channels, as test_gpu_feature_bounds._oracle_fwd builds them).  The forward-only walk, driven as render_frames drives
   it, must put colour, the eight allmap planes and every feature plane within the forward bound outside the oracle's
   knife mask; it keeps no n_contrib or final_T, so those are not compared.  A walk that built other records or read
   another frame's camera leaves the bound.  render_frames' own colour, features and radii must equal that walk's bit for
   bit at 1, 2 and 5 frames per call, and its maps are held to part A's model on the walk's own allmap, so composite
   error and post-processing error stay apart.

Negative controls: on the F = 0 case's maps, the model evaluated with a camera mistake (row 0's tangents, fx and fy
swapped, cx off by half a pixel, the y offset's sign flipped, the depth ratio as 1 - r) must leave the bound on a
quarter of the covered pixels at least.

Each case prints its knife counts and per plane or map the largest err / (K u B + FLOOR).
"""
import numpy as np
import pytest
import torch

from . import post_bounds as PB
from .test_gpu_grad_bounds import FLOOR, K, U, _np, _oracle_frame
from .test_gpu_loss_bounds import NAN, OPTS, POST_CH, POST_KEYS, TANX, TANY, _frames, _loss_gpu, _wvts

pytestmark = pytest.mark.gpu

T_ = 5                   # part B's frames
RATIO = 0.37             # part B's depth ratio
FPC = (1, 2, 5)          # frames per call: one frame, chunks that do not divide T, all at once
B_CASES = {"F0": 0, "F7_shared": 7, "F32_per_frame": -32}

# Masked pixels per part-B case over its frames, measured on an H100: the composite's knife edges (a case may mask at
# most 4 n + 8) and the post stencil's.
KNIFE_MEASURED = {"F0": 0, "F7_shared": 1, "F32_per_frame": 2}
STENCIL_MEASURED = {"F0": 0, "F7_shared": 0, "F32_per_frame": 0}


@pytest.fixture(scope="module")
def dev(built):
    from vidu4d_b200 import _capi
    _capi.load()
    return torch.device("cuda:0")


def _t(x, dev):
    return None if x is None else torch.from_numpy(np.ascontiguousarray(x)).to(dev)


def _bits(a, b, what):
    a, b = torch.as_tensor(a), torch.as_tensor(b)
    assert a.shape == b.shape, (what, tuple(a.shape), tuple(b.shape))
    x, y = a.contiguous().view(torch.int32), b.contiguous().view(torch.int32)
    n = int((x != y).sum())
    assert n == 0, f"{what}: {n} of {x.numel()} elements differ"


# ------------------------------------------------------------------------------------------------ A: the post kernels
def _post_frames(M, W, H, am, wvt, table, r, bk, color, stride, dev):
    """sr_post_forward_frames into NaN-filled (M, c, H, W) maps; table None = the shared TANX / TANY."""
    from vidu4d_b200 import _capi
    maps = {k: torch.full((M, c, H, W), NAN, device=dev) for k, c in zip(POST_KEYS, POST_CH)}
    _capi.call("sr_post_forward_frames", dev, M, W, H, TANX, TANY, table, r, am, wvt, bk, color, stride,
               *[maps[k] for k in POST_KEYS])
    torch.cuda.synchronize(dev)
    return maps


@pytest.mark.parametrize("W,H,M,path,r,bk", PB.GRID, ids=[f"{w}x{h}-M{m}-{p}-r{r}-{'bk' if b else 'nobk'}"
                                                          for w, h, m, p, r, b in PB.GRID])
def test_post_frames_elementwise(W, H, M, path, r, bk, dev):
    from vidu4d_b200 import _capi
    name = f"{W}x{H} M={M} {path} r={r} bk={bk}"
    seed = W * 1000 + H * 10 + M
    am, _, _, _, _ = _frames(M, W, H, seed, False, False)
    wvt = _wvts(M, seed).contiguous().numpy()
    scalar_rows = np.tile(np.array([TANX, TANY, 0.0, 0.0], np.float32), (M, 1))
    rows = PB.frame_rows(M, W, H) if path == "table" else scalar_rows
    am_d, wvt_d = _t(am, dev), _t(wvt, dev)
    N = H * W
    stride = 3 * N + 37                         # a padded frame stride: the padding must stay untouched
    rng = np.random.default_rng(seed)
    color0 = rng.uniform(-1.0, 2.0, (M, stride)).astype(np.float32)
    col = _t(color0, dev)
    bkn = np.array([0.7, -0.25, 0.4], np.float32) if bk else None
    table = _t(rows, dev) if path == "table" else None
    maps = _post_frames(M, W, H, am_d, wvt_d, table, r, _t(bkn, dev), col, stride, dev)

    # the background: numpy float32, each operation rounded; without one the colour buffer is not touched
    want = color0.copy()
    if bk:
        c = color0[:, :3 * N].reshape(M, 3, N)
        a = am[:, 1].reshape(M, 1, N)
        want[:, :3 * N] = (c + (np.float32(1.0) - a) * bkn[None, :, None]).reshape(M, 3 * N)
    _bits(col.cpu(), torch.from_numpy(want), f"{name} colour")

    report, knife = {}, 0
    got = {k: v.cpu().numpy() for k, v in maps.items()}
    for f in range(M):
        knife += PB.check_frame(f"{name} frame {f}", PB.maps_of(got, f), am[f], wvt[f], rows[f], r, report)
    print(f"\n[{name}] stencil knife {knife} of {M * W * H} px; " + ", ".join(f"{k} {v:.3g}" for k, v in report.items()))
    assert knife <= 8 + 1e-4 * M * W * H, (name, knife)

    if path == "scalar":
        # sr_post_forward frame by frame, and a table of the scalar tangents with zero offsets
        for f in range(M):
            one = [torch.full((c, H, W), NAN, device=dev) for c in POST_CH]
            _capi.call("sr_post_forward", dev, W, H, TANX, TANY, r, am_d[f], wvt_d[f], *one)
            for k, t in zip(POST_KEYS, one):
                _bits(maps[k][f], t, f"{name} frame {f} {k} vs sr_post_forward")
        tab = _post_frames(M, W, H, am_d, wvt_d, _t(scalar_rows, dev), r, None, None, 0, dev)
        for k in POST_KEYS:
            _bits(tab[k], maps[k], f"{name} {k}: table of the scalar tangents vs scalar path")
    else:
        # the loss pass's surf_depth with the same table
        o = dict(OPTS["bench"], depth_ratio=r)
        color = torch.rand((M, 3, H, W), device=dev)
        target = torch.rand((M, 3, H, W), device=dev)
        sd = _loss_gpu(M, W, H, o, color, am_d, wvt_d, target, None, None, None, None, dev, table=table)[4]
        _bits(maps["surf_depth"][:, 0], sd, f"{name} surf_depth vs the loss pass")


# ------------------------------------------------------------------------------------------------ B: render_frames
_runs = {}


def _case(key, dev):
    """Part B's scene, the training forward, the forward-only walk and render_frames at every FPC; cached per case."""
    if key in _runs:
        return _runs[key]
    from vidu4d_b200 import rasterizer as R
    from vidu4d_b200.renderer import BatchCameras, PipelineParams, render_frames
    from . import test_gpu_batch_bounds as BB
    from .test_gpu_batch import _cams
    from .test_gpu_render import _PC
    Fs = B_CASES[key]
    F, P, W, H = abs(Fs), BB.P, BB.W, BB.H
    c = dict(M=T_, means3D="per_frame", rotations="per_frame", scales="shared", opacities="shared", colour="sh_shared",
             sh=(3, 16), features=Fs, background="3+F")
    inp = BB._inputs(c, 9000 + F)
    ti = {k: _t(inp[k], dev) for k in ("means3D", "rotations", "scales", "opacities", "sh", "features")}
    bg = _t(inp["bg"], dev)
    assert bg.numel() == 3 + F
    rows = BB._rows(T_, True)
    table = _t(rows, dev)
    # _forward takes contiguous cameras (its callers pass them through _f32c); _cams' view matrices are strided views
    vm, pm, cp = (x.contiguous() for x in _cams(T_, dev))
    e = torch.empty((0,), device=dev)
    kw = {} if not F else dict(features=ti["features"], concat=False)
    nan = float("nan")
    train = R._C.rasterize_gaussians_batch(bg, ti["means3D"], e, ti["opacities"], ti["scales"], ti["rotations"], 1.0, vm,
                                           pm, nan, nan, H, W, ti["sh"], 3, cp, intrinsics=table, **kw)
    # the forward-only walk, as render_frames drives it, into NaN-filled outputs
    ins, strides = R._batch_inputs(T_, means3D=(ti["means3D"], (3,)), sh=(ti["sh"], None), opacity=(ti["opacities"], (1,)),
                                   scales=(ti["scales"], (2,)), rotations=(ti["rotations"], (4,)),
                                   features=(ti["features"], None))
    full = lambda *s: torch.full((T_,) + s, NAN, device=dev)  # noqa: E731
    ro = R._RenderOut(full(3, H, W), full(F, H, W) if F else None, full(8, H, W),
                      torch.full((T_, P), -7, dtype=torch.int32, device=dev))
    nr = R._forward(T_, True, strides, bg, ins["means3D"], ins["sh"], None, ins["opacity"], ins["scales"],
                    ins["rotations"], ins["features"], vm, pm, cp, H, W, 3, 0.0, 0.0, 1.0, False, False, intrinsics=table,
                    render=ro)[0]
    assert list(nr) == list(train[0]) and min(nr) > 0, (key, nr, train[0])
    cams = BatchCameras(W, H, 0.0, 0.0, vm, pm, cp, table)
    pc = _PC(dict(means3D=ti["means3D"][0], rotations=ti["rotations"][0], scales=ti["scales"],
                  opacities=ti["opacities"], shs=ti["sh"]))
    outs = {n: render_frames(cams, pc, PipelineParams(depth_ratio=RATIO), bg, means3D=ti["means3D"],
                             rotations=ti["rotations"], features=ti["features"], frames_per_call=n) for n in FPC}
    bk = torch.tensor([0.7, -0.25, 0.4], device=dev)
    with_bk = render_frames(cams, pc, PipelineParams(depth_ratio=RATIO), bg, means3D=ti["means3D"],
                            rotations=ti["rotations"], features=ti["features"], learnable_bkgd=bk, frames_per_call=2)
    torch.cuda.synchronize(dev)
    run = dict(inp=inp, F=F, P=P, W=W, H=H, rows=rows, cams=(vm, pm, cp), train=train, ro=ro, outs=outs, with_bk=with_bk,
               bk=bk)
    _runs.clear()
    _runs[key] = run
    return run


def _planes(name, mine, ref, fbound, ok, report, what):
    """Each plane of mine (n, H, W) within K u fbound + FLOOR of the oracle's outside the knife mask."""
    for i in range(mine.shape[0]):
        x = np.where(ok, np.abs(mine[i].astype(np.float64) - ref[i]) / (K * U * fbound[i] + FLOOR), 0.0)
        x = np.where(np.isnan(mine[i]) & ok, np.inf, x)
        k = what if what == "features" else f"{what}[{i}]"
        report[k] = max(report.get(k, 0.0), float(x.max()))
        assert x.max() <= 1.0, (name, f"{what}[{i}]", float(x.max()), np.argwhere(x > 1.0)[:4].tolist())


@pytest.mark.parametrize("key", list(B_CASES))
def test_render_frames_against_the_oracle(key, dev):
    from vidu4d_b200 import debug as dbg
    from . import test_gpu_feature_bounds as FB
    run = _case(key, dev)
    inp, F, P, W, H, rows, ro = (run[k] for k in ("inp", "F", "P", "W", "H", "rows", "ro"))
    vms, pms, cps = (_np(x) for x in run["cams"])
    nr, _, _, radii, gb, bb, ib = run["train"][:7]
    color, allmap = _np(ro.color), _np(ro.others)
    feat = None if not F else _np(ro.features)
    report, knife = {}, 0
    for f in range(T_):
        tag = f"{key} frame {f}"
        dec = dbg.decode(gb.view(T_, -1)[f], bb.view(T_, -1)[f], ib.view(T_, -1)[f], P, W, H, nr[f])
        dec["radii"] = _np(radii[f])
        dec["num_rendered"] = nr[f]
        tan, off = (float(rows[f][0]), float(rows[f][1])), (float(rows[f][2]), float(rows[f][3]))
        means, rots = inp["means3D"][f], inp["rotations"][f]
        geo = (means, inp["opacities"], inp["scales"], rots)
        st, ext = _oracle_frame(dec, P, W, H, *geo, inp["sh"], None, 3, inp["bg"][:3], vms[f], pms[f], cps[f], tan,
                                off=off, name=tag)
        ok = ~ext["knife"]
        knife += int(ext["knife"].sum())
        _planes(tag, color[f], st.color, ext["fbound"][0:3], ok, report, "color")
        _planes(tag, allmap[f], st.allmap, ext["fbound"][3:11], ok, report, "allmap")
        if F:
            ff = inp["features"][f] if inp["features"].ndim == 3 else inp["features"]
            for g, (cols, b3, n) in enumerate(FB._groups(ff, inp["bg"][3:])):
                sg, eg = _oracle_frame(dec, P, W, H, *geo, None, cols, 0, b3, vms[f], pms[f], cps[f], tan, off=off,
                                       records=None, name=f"{tag} group {g}")
                assert np.array_equal(eg["knife"], ext["knife"]), (tag, "group", g, "knife mask differs from the colour's")
                _planes(f"{tag} group {g}", feat[f, 3 * g:3 * g + n], sg.color, eg["fbound"], ok, report, "features")
    # the last frame's object crosses the right image edge
    assert float(allmap[T_ - 1, 1, :, -1].max()) > 0.5, key

    # render_frames: its own colour, features and radii are the walk's, at every chunking
    _bits(ro.radii, radii, f"{key} walk radii vs the records'")
    for n, r in run["outs"].items():
        _bits(r["render"], ro.color, f"{key} fpc={n} render")
        if F:
            _bits(r["features"], ro.features, f"{key} fpc={n} features")
        else:
            assert "features" not in r
        _bits(r["radii"], radii, f"{key} fpc={n} radii")
        assert torch.equal(r["visibility_filter"], radii > 0), key
        for k in POST_KEYS:
            _bits(r[k], run["outs"][1][k], f"{key} fpc={n} {k}")
    # the learnable background on top, numpy float32 with each operation rounded
    a = allmap[:, 1:2]
    want = color + (np.float32(1.0) - a) * _np(run["bk"])[None, :, None, None]
    _bits(run["with_bk"]["render"].cpu(), torch.from_numpy(want), f"{key} render with learnable_bkgd")

    # the maps, on the walk's own allmap
    got = run["outs"][1]
    stencil = 0
    for f in range(T_):
        stencil += PB.check_frame(f"{key} frame {f} post", PB.maps_of(got, f), allmap[f], vms[f], rows[f], RATIO, report)
    print(f"\n[{key}] T={T_} {W}x{H}: knife composite {knife} stencil {stencil} of {T_ * W * H} px; "
          + ", ".join(f"{k} {v:.3g}" for k, v in report.items()))
    assert knife <= 4 * KNIFE_MEASURED[key] + 8, (key, "knife pixels", knife)
    assert stencil <= 4 * STENCIL_MEASURED[key] + 8, (key, "stencil knife pixels", stencil)


@pytest.mark.parametrize("control", list(PB.CONTROLS))
def test_negative_controls_leave_the_bound(control, dev):
    """Held to the model with a plausible camera mistake, the F = 0 case's maps leave the bound on many pixels."""
    run = _case("F0", dev)
    vms = _np(run["cams"][0])
    got = run["outs"][1]
    maps = [PB.maps_of(got, f) for f in range(T_)]
    bad, live = PB.control_failures(control, maps, _np(run["ro"].others), vms, run["rows"], RATIO)
    print(f"\n[control {control}] {PB.CONTROLS[control]}: {bad} of {live} covered pixels out of the bound")
    assert live > 0 and bad >= PB.CONTROL_SHARE * live, (control, bad, live)
