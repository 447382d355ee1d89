"""GPU: forward-only rendering (include/surfel_render.h, renderer.render_frames) against the training forward.

The forward-only walk composites the same contributors with the same weights in the same order as composite_fwd +
feature_fwd, so colour, the eight allmap planes, the feature planes and radii must equal _C.rasterize_gaussians_batch's
bit for bit; render_frames' maps must equal sr_post_forward's frame by frame."""
import math

import numpy as np
import pytest
import torch

from .conftest import load_golden

pytestmark = pytest.mark.gpu

FS = [0, 1, 3, 4, 8, 16, 22, 32]
SIZES = [(16, 16, 20_000), (75, 53, 20_000), (80, 48, 20_000), (512, 512, 300_000)]
TAN = 0.5
FOV = 2.0 * math.atan(TAN)
TANF = math.tan(FOV * 0.5)     # the tangent render() derives from FoV (renderer._cam_tans): both arms use it


@pytest.fixture(scope="module")
def dev(built):
    from vidu4d_b200 import _capi
    _capi.load()
    return torch.device("cuda:0")


_scenes = {}


def _scene(P, dev):
    if P not in _scenes:
        from vidu4d_b200.synthetic import object_scene
        _scenes.clear()
        _scenes[P] = object_scene(P, seed=0, opacity="trained", center=(0.0, 0.0, 0.0)).to_torch(dev)
    return _scenes[P]


class _PC:
    def __init__(self, s, degree=3):
        self.get_xyz, self.get_rotation, self.get_scaling = s["means3D"], s["rotations"], s["scales"]
        self.get_opacity, self.get_features, self.active_sh_degree = s["opacities"], s["shs"], degree


def _cams(M, W, H, dev, table=None, first=0):
    from vidu4d_b200.renderer import BatchCameras
    from vidu4d_b200.synthetic import orbit_view, projection_matrix
    vms, cps = [], []
    for f in range(M):
        R, t = orbit_view(first + 5 * f, 64)
        W2C = np.eye(4)
        W2C[:3, :3], W2C[:3, 3] = R, t
        vms.append(W2C.T.astype(np.float32))
        cps.append((-R.T @ t).astype(np.float32))
    vm = torch.from_numpy(np.stack(vms)).to(dev)
    pm = vm @ torch.from_numpy(projection_matrix(TAN, TAN)).to(dev)
    return BatchCameras(W, H, FOV, FOV, vm.contiguous(), pm.contiguous(), torch.from_numpy(np.stack(cps)).to(dev), table)


def _inputs(P, M, F, per_frame, dev, seed=1):
    """Surfels (shared or per frame, jittered) and features (shared (P,F) or per frame (M,P,F))."""
    s = _scene(P, dev)
    g = torch.Generator(device=dev).manual_seed(seed)
    means = rots = None
    if per_frame:
        means = (s["means3D"][None] + 0.003 * torch.randn((M, P, 3), device=dev, generator=g)).contiguous()
        r = s["rotations"][None] + 0.05 * torch.randn((M, P, 4), device=dev, generator=g)
        rots = (r / r.norm(dim=-1, keepdim=True)).contiguous()
    feat = None
    if F:
        shape = (M, P, F) if per_frame else (P, F)
        feat = torch.rand(shape, device=dev, generator=g) * 2 - 1
    return s, means, rots, feat


def _training(s, cams, bg, means, rots, feat, depth_ratio=0.0):
    """Today's route: the training forward under no_grad, then sr_post_forward frame by frame."""
    from vidu4d_b200 import _capi
    from vidu4d_b200.rasterizer import _C
    M, H, W = len(cams), cams.image_height, cams.image_width
    dev = s["means3D"].device
    e = torch.empty((0,), device=dev)
    kw = {} if feat is None else {"features": feat, "concat": False}
    if cams.intrinsics is not None:
        kw["intrinsics"] = cams.intrinsics
    with torch.no_grad():
        out = _C.rasterize_gaussians_batch(bg, s["means3D"] if means is None else means, e, s["opacities"], s["scales"],
                                           s["rotations"] if rots is None else rots, 1.0, cams.world_view_transform,
                                           cams.full_proj_transform, TANF, TANF, H, W, s["shs"], 3, cams.camera_center, **kw)
        maps = []
        if cams.intrinsics is None:
            for f in range(M):
                mk = lambda c: torch.empty((c, H, W), device=dev)  # noqa: E731
                m = [mk(1), mk(3), mk(1), mk(1), mk(1), mk(1), mk(3)]
                _capi.call("sr_post_forward", dev, W, H, TANF, TANF, depth_ratio, out[2][f], cams.world_view_transform[f], *m)
                maps.append(m)
    return out, maps


def _render_only(s, cams, bg, means, rots, feat):
    """sr_render_forward through _forward's forward-only mode: colour, allmap, radii, features."""
    from vidu4d_b200.rasterizer import _RenderOut, _batch_inputs, _forward
    M, H, W = len(cams), cams.image_height, cams.image_width
    dev = s["means3D"].device
    P = int(s["means3D"].shape[0])
    F = 0 if feat is None else int(feat.shape[-1])
    ins, strides = _batch_inputs(M, means3D=(s["means3D"] if means is None else means, (3,)), sh=(s["shs"], None),
                                 opacity=(s["opacities"], (1,)), scales=(s["scales"], (2,)),
                                 rotations=(s["rotations"] if rots is None else rots, (4,)), features=(feat, None))
    out = _RenderOut(torch.empty((M, 3, H, W), device=dev), torch.empty((M, F, H, W), device=dev) if F else None,
                     torch.empty((M, 8, H, W), device=dev), torch.empty((M, P), dtype=torch.int32, device=dev))
    xyz = ins["means3D"] if ins["means3D"] is not None else s["means3D"]       # P = 0: the empty tensors
    nr = _forward(M, True, strides, bg, xyz, ins["sh"], None, ins["opacity"], ins["scales"], ins["rotations"],
                  ins["features"] if ins["features"] is not None else feat, cams.world_view_transform, cams.full_proj_transform, cams.camera_center, H, W, 3, TANF, TANF,
                  1.0, False, False, intrinsics=cams.intrinsics, render=out)[0]
    return nr, out


def _bits(a, b, what):
    assert a.shape == b.shape, (what, a.shape, b.shape)
    x, y = a.contiguous().view(torch.int32), b.contiguous().view(torch.int32)
    n = int((x != y).sum())
    assert n == 0, f"{what}: {n} of {x.numel()} elements differ"


def _table(M, dev, offsets=False):
    rows = [(TANF, TANF, (3.5 - 2.25 * f) if offsets else 0.0, (-1.75 + 1.5 * f) if offsets else 0.0) for f in range(M)]
    return torch.tensor(rows, dtype=torch.float32, device=dev)


@pytest.mark.parametrize("W,H,P", SIZES, ids=[f"{w}x{h}" for w, h, _ in SIZES])
@pytest.mark.parametrize("table", [False, True], ids=["scalar", "table"])
@pytest.mark.parametrize("per_frame", [False, True], ids=["shared", "per_frame"])
@pytest.mark.parametrize("F", FS)
def test_bit_identical_to_training_forward(F, per_frame, table, W, H, P, dev):
    M = 2
    s, means, rots, feat = _inputs(P, M, F, per_frame, dev)
    cams = _cams(M, W, H, dev, _table(M, dev, offsets=True) if table else None)
    bg = torch.tensor([0.1, 0.2, 0.3] + [0.05 * k for k in range(F)] if F % 2 else [0.1, 0.2, 0.3], device=dev)
    ref, _ = _training(s, cams, bg, means, rots, feat)
    nr, out = _render_only(s, cams, bg, means, rots, feat)
    assert nr == ref[0]
    _bits(out.color, ref[1], "colour")
    for ch in range(8):
        _bits(out.others[:, ch], ref[2][:, ch], f"allmap plane {ch}")
    _bits(out.radii, ref[3], "radii")
    if F:
        _bits(out.features, ref[7], "features")


@pytest.mark.parametrize("case", ["empty", "culled"])
@pytest.mark.parametrize("F", [0, 4, 22])
def test_empty_and_culled(case, F, dev):
    """P = 0 zero-fills the planes as the training forward does; with every surfel behind the camera the planes are the
    background's, bit for bit with the training forward."""
    M, W, H = 2, 75, 53
    s = _scene(20_000, dev)
    if case == "empty":
        s = {k: v[:0] for k, v in s.items()}
    else:
        s = dict(s, means3D=(s["means3D"] * 0.01 - torch.tensor([0.0, 0.0, 5.0], device=dev)).contiguous())
    feat = torch.rand((int(s["means3D"].shape[0]), F), device=dev) if F else None
    cams = _cams(M, W, H, dev)
    cams.world_view_transform = torch.eye(4, device=dev).expand(M, 4, 4).contiguous()
    bg = torch.tensor([0.1, 0.2, 0.3] + [0.5] * F, device=dev)
    nr, out = _render_only(s, cams, bg, None, None, feat)
    r = _render_frames(s, cams, bg, feat=feat)
    assert max(nr) == 0 and not bool((r["radii"] > 0).any())
    if case == "empty":            # rasterize_points.cu:106: zero-filled planes
        ref = (None, torch.zeros_like(out.color), torch.zeros_like(out.others), None, None, None, None,
               torch.zeros_like(out.features) if F else None)
    else:
        ref, _ = _training(s, cams, bg, None, None, feat)
        assert nr == ref[0]
    _bits(out.color, ref[1], "colour")
    _bits(out.others, ref[2], "allmap")
    _bits(r["render"], ref[1], "render_frames colour")
    if F:
        _bits(out.features, ref[7], "features")
        _bits(r["features"], ref[7], "render_frames features")


def _render_frames(s, cams, bg, means=None, rots=None, feat=None, **kw):
    from vidu4d_b200.renderer import PipelineParams, render_frames
    return render_frames(cams, _PC(s), PipelineParams(depth_ratio=kw.pop("depth_ratio", 0.0)), bg, means3D=means,
                         rotations=rots, features=feat, **kw)


MAPS = ["acc", "rend_normal", "rend_dist", "render_depth_median", "render_depth_expected", "surf_depth", "surf_normal"]


@pytest.mark.parametrize("depth_ratio", [0.0, 1.0])
@pytest.mark.parametrize("F", [0, 22])
def test_render_frames_scalar_path_matches_sr_post_forward(F, depth_ratio, dev):
    M, W, H = 3, 80, 48
    s, means, rots, feat = _inputs(20_000, M, F, True, dev)
    cams = _cams(M, W, H, dev)
    bg = torch.tensor([0.1, 0.2, 0.3], device=dev)
    ref, maps = _training(s, cams, bg, means, rots, feat, depth_ratio)
    r = _render_frames(s, cams, bg, means, rots, feat, depth_ratio=depth_ratio)
    _bits(r["render"], ref[1], "render")
    _bits(r["radii"], ref[3], "radii")
    assert torch.equal(r["visibility_filter"], ref[3] > 0)
    if F:
        _bits(r["features"], ref[7], "features")
    for f in range(M):
        for k, m in zip(MAPS, maps[f]):
            got = r[k][f] if m.shape[0] == r[k].shape[1] else r[k][f, :1]
            _bits(got, m, f"{k} frame {f}")


def test_render_frames_table_of_shared_tangents_equals_scalar_path(dev):
    M, W, H = 3, 75, 53
    s, means, rots, feat = _inputs(20_000, M, 8, False, dev)
    bg = torch.tensor([0.1, 0.2, 0.3], device=dev)
    a = _render_frames(s, _cams(M, W, H, dev), bg, feat=feat)
    b = _render_frames(s, _cams(M, W, H, dev, _table(M, dev)), bg, feat=feat)
    for k in ["render", "features", "radii"] + MAPS:
        _bits(a[k], b[k], k)


def test_render_frames_offsets_match_post_oracle(dev):
    """Off-centre principal points: each frame's maps against post_oracle.post_forward with tests/camera_model.py's
    offset rays, within test_gpu_cameras' tolerance; the centred oracle disagrees."""
    from oracle import post_oracle as po
    from . import camera_model as cm
    from .test_gpu_cameras import RTOL
    M, W, H = 2, 75, 53
    s, means, rots, feat = _inputs(20_000, M, 0, False, dev)
    table = _table(M, dev, offsets=True)
    cams = _cams(M, W, H, dev, table)
    bg = torch.tensor([0.0, 0.0, 0.0], device=dev)
    r = _render_frames(s, cams, bg)
    _, out = _render_only(s, cams, bg, None, None, None)
    for f in range(M):
        tx, ty, ox, oy = (float(v) for v in table[f])
        allmap, wvt = out.others[f].cpu().numpy(), cams.world_view_transform[f].cpu().numpy()
        want = cm._with_rays(ox, oy, po.post_forward, allmap, wvt, tx, ty)
        centred = po.post_forward(allmap, wvt, tx, ty)
        for k in ("surf_normal",):
            got = r[k][f].cpu().numpy().astype(np.float64)
            scale = np.abs(want[k]).max() + 1e-12
            assert np.abs(got - want[k]).max() <= RTOL * 50 * scale, (f, k)
            assert np.abs(got - centred[k]).max() > RTOL * 500 * scale, (f, k)        # the offsets are not ignored
        for k in ("acc", "rend_dist", "render_depth_median", "render_depth_expected"):
            got = r[k][f].cpu().numpy().astype(np.float64)
            assert np.abs(got - want[k][:1]).max() <= RTOL * (np.abs(want[k]).max() + 1e-12), (f, k)


def test_learnable_background_is_torchs_expression(dev):
    M, W, H = 3, 80, 48
    s, means, rots, feat = _inputs(20_000, M, 0, False, dev)
    cams = _cams(M, W, H, dev)
    bg = torch.tensor([0.1, 0.2, 0.3], device=dev)
    bk = torch.tensor([0.7, -0.25, 0.4], device=dev)
    plain = _render_frames(s, cams, bg)
    r = _render_frames(s, cams, bg, learnable_bkgd=bk)
    want = plain["render"] + (1 - plain["acc"]) * bk[None, :, None, None]
    _bits(r["render"], want, "render with learnable_bkgd")
    _bits(r["acc"], plain["acc"], "acc")


def test_chunks_give_the_same_bits(dev):
    M, W, H = 13, 80, 48
    s, means, rots, feat = _inputs(20_000, M, 22, True, dev)
    cams = _cams(M, W, H, dev, _table(M, dev, offsets=True))
    bg = torch.tensor([0.1, 0.2, 0.3], device=dev)
    outs = [_render_frames(s, cams, bg, means, rots, feat, frames_per_call=n) for n in (1, 4, 13)]
    for o in outs[1:]:
        for k in ["render", "features", "radii"] + MAPS:
            _bits(o[k], outs[0][k], k)


def test_overflow_reruns_with_the_same_bits(dev):
    from vidu4d_b200 import rasterizer as RZ
    M, W, H = 4, 512, 512
    s, means, rots, feat = _inputs(300_000, M, 4, False, dev)
    cams = _cams(M, W, H, dev)
    bg = torch.tensor([0.1, 0.2, 0.3], device=dev)
    ref, _ = _training(s, cams, bg, None, None, feat)
    key = (dev.index, W, H)
    RZ._cap_hint[key] = 1                  # a capacity hint far too small: the first call overflows
    r = _render_frames(s, cams, bg, feat=feat, frames_per_call=2)
    assert RZ._cap_hint[key] > 4 * 4096 and min(ref[0]) > 4 * 4096      # the chunks overflowed and were re-run
    _bits(r["render"], ref[1], "render")
    _bits(r["features"], ref[7], "features")
    _bits(r["radii"], ref[3], "radii")


def test_reference_record_headline_orbit0(dev):
    """Colour and allmap of the forward-only render of bench.py's orbit camera 0 within test_gpu_headline's tolerances of
    the reference extension's record."""
    from vidu4d_b200.renderer import BatchCameras
    from .test_gpu_headline import bench_inputs
    from .test_gpu_parity import TOL, XBUILD_TOL
    rec = load_golden("ref_headline_orbit0")
    inp = bench_inputs(0)
    t = {k: torch.from_numpy(np.ascontiguousarray(v)).to(dev) for k, v in inp.items() if k != "meta"}
    s = {"means3D": t["means3D"], "rotations": t["rotations"], "scales": t["scales"], "opacities": t["opacities"],
         "shs": t["shs"]}
    cams = BatchCameras(512, 512, 0.0, 0.0, t["viewmatrix"][None].contiguous(), t["projmatrix"][None].contiguous(),
                        t["campos"][None].contiguous())
    nr, out = _render_only(s, cams, t["bg"], None, None, None)
    assert nr[0] == int(rec["num_rendered"][0])
    near = ("color",) + tuple(f"allmap{ch}" for ch in (0, 1, 2, 3, 4, 5, 7))
    mine = {"color": out.color[0].cpu().numpy()}
    for ch in range(8):
        mine[f"allmap{ch}"] = out.others[0, ch].cpu().numpy()
    for k, v in mine.items():
        idx, want, mx = rec["idx_" + k], rec["val_" + k], float(rec["max_" + k][0])
        if idx.size == 0:
            continue
        tol = (XBUILD_TOL if k in near else TOL) * max(mx, 1e-30)
        flat = v.reshape(-1)
        assert np.abs(flat[idx] - want).max() <= tol, k
        assert abs(float(np.abs(flat).max()) - mx) <= tol, k


def test_no_autograd_state_and_only_the_outputs_stay_allocated(dev):
    M, W, H = 5, 80, 48
    s, means, rots, feat = _inputs(20_000, M, 22, True, dev)
    s = {k: v.clone().requires_grad_(True) for k, v in s.items()}
    means, rots, feat = means.requires_grad_(True), rots.requires_grad_(True), feat.requires_grad_(True)
    cams = _cams(M, W, H, dev)
    bg = torch.tensor([0.1, 0.2, 0.3], device=dev)
    bk = torch.tensor([0.7, -0.25, 0.4], device=dev, requires_grad=True)
    _render_frames(s, cams, bg, means, rots, feat, learnable_bkgd=bk, frames_per_call=2)     # warm the caches
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated(dev)
    r = _render_frames(s, cams, bg, means, rots, feat, learnable_bkgd=bk, frames_per_call=2)
    torch.cuda.synchronize()
    after = torch.cuda.memory_allocated(dev)
    storages = {}
    for v in r.values():
        assert v.grad_fn is None and not v.requires_grad
        storages[v.untyped_storage().data_ptr()] = v.untyped_storage().nbytes()
    assert after - before == sum((n + 511) // 512 * 512 for n in storages.values())
