"""GPU: per-surfel contribution statistics of render_frames (sr_render_forward_contrib) and pruning by them.

No new oracle is needed.  With one-hot features -- column s mod 32 is 1 for the surfels of group g = s // 32, 0 for the
others -- and a zero feature background, plane s mod 32 of group g's render is surfel s's per-pixel weight w = T alpha
exactly: a zero column leaves the composite's accumulator unchanged, and the one non-zero pair adds ff(T, fm(alpha, 1),
0) = w.  So weight_q must be the sum of rn(plane 2^32), max_weight the plane's maximum, pixels its count of positive
values, bit for bit, and the statistics of the F = 0 and F = 22 renders must be those of the one-hot (F = 32) render."""
import ctypes as C

import numpy as np
import pytest
import torch

from .test_gpu_render import TANF, _cams, _inputs, _table

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev(built):
    from vidu4d_b200 import _capi
    _capi.load()
    return torch.device("cuda:0")


class _PC:
    def __init__(self, s):
        self.get_xyz, self.get_rotation, self.get_scaling = s["means3D"], s["rotations"], s["scales"]
        self.get_opacity, self.get_features, self.active_sh_degree = s["opacities"], s["shs"], 3


def _render(s, cams, means, rots, feat=None, fpc=8, contrib=None, bg=None, bkgd=None):
    from vidu4d_b200.renderer import PipelineParams, render_frames
    dev = s["means3D"].device
    bg = torch.zeros(3, device=dev) if bg is None else bg
    return render_frames(cams, _PC(s), PipelineParams(depth_ratio=0.37), bg, means3D=means, rotations=rots,
                         features=feat, learnable_bkgd=bkgd, frames_per_call=fpc, contributions=contrib)


OUTPUTS = ("render", "acc", "rend_normal", "rend_dist", "render_depth_median", "render_depth_expected", "surf_depth",
           "surf_normal", "radii")


def _same_outputs(a, b, what):
    for k in OUTPUTS + (("features",) if "features" in a else ()):
        x, y = a[k].contiguous().view(torch.int32), b[k].contiguous().view(torch.int32)
        n = int((x != y).sum())
        assert n == 0, f"{what}: {k} differs in {n} of {x.numel()} elements"


def _with_capacity_hint(dev, W, H, hint, fn):
    """fn() with the rasterizer's capacity hint for (W, H) set to `hint`, then the hint restored."""
    from vidu4d_b200 import rasterizer as RZ
    key = (dev.index, W, H)
    saved = RZ._cap_hint.get(key)
    try:
        RZ._cap_hint[key] = hint
        r = fn()
        grown = RZ._cap_hint[key]
    finally:
        if saved is None:
            RZ._cap_hint.pop(key, None)
        else:
            RZ._cap_hint[key] = saved
    return r, grown


def _zeros(P, dev):
    from vidu4d_b200.renderer import SurfelContributions
    return SurfelContributions.zeros(P, dev)


def _same(a, b, what):
    for name in ("weight_q", "max_weight", "pixels", "frames"):
        x, y = getattr(a, name), getattr(b, name)
        assert x.dtype == y.dtype and x.shape == y.shape, (what, name)
        n = int((x != y).sum())
        assert n == 0, f"{what}: {name} differs for {n} of {x.numel()} surfels"


def _onehot_stats(s, cams, means, rots):
    """weight_q, max_weight bits and pixels per surfel from the one-hot feature planes, in float64 / int64 numpy."""
    P = int(s["means3D"].shape[0])
    dev = s["means3D"].device
    wq, mx, px = np.zeros(P, np.int64), np.zeros(P, np.float32), np.zeros(P, np.int64)
    for g in range((P + 31) // 32):
        lo, hi = 32 * g, min(P, 32 * g + 32)
        feat = torch.zeros((P, 32), device=dev)
        feat[torch.arange(lo, hi, device=dev), torch.arange(hi - lo, device=dev)] = 1.0
        planes = _render(s, cams, means, rots, feat)["features"][:, :hi - lo].cpu().numpy()      # (T, k, H, W)
        q = np.rint(planes.astype(np.float64) * 2.0 ** 32).astype(np.int64)
        wq[lo:hi] = q.sum(axis=(0, 2, 3))
        mx[lo:hi] = planes.max(axis=(0, 2, 3))
        px[lo:hi] = (planes > 0).sum(axis=(0, 2, 3))
    return wq, mx.view(np.int32), px


SIZES = [(16, 16, 600), (75, 53, 2000), (128, 128, 3000), (512, 512, 256)]


@pytest.mark.parametrize("W,H,P", SIZES, ids=[f"{w}x{h}_P{p}" for w, h, p in SIZES])
@pytest.mark.parametrize("table", [False, True], ids=["scalar", "table"])
@pytest.mark.parametrize("per_frame", [False, True], ids=["shared", "per_frame"])
def test_statistics_equal_the_one_hot_feature_planes(per_frame, table, W, H, P, dev):
    T = 3
    s, means, rots, _ = _inputs(P, T, 0, per_frame, dev)
    cams = _cams(T, W, H, dev, _table(T, dev, offsets=True) if table else None)
    wq, mx, px = _onehot_stats(s, cams, means, rots)
    assert px.sum() > 0

    got = {}
    g = torch.Generator(device=dev).manual_seed(3)
    onehot = torch.zeros((P, 32), device=dev)
    onehot[torch.arange(min(P, 32), device=dev), torch.arange(min(P, 32), device=dev)] = 1.0
    for F, feat in ((0, None), (22, torch.rand((P, 22), device=dev, generator=g)), (32, onehot)):
        c = _zeros(P, dev)
        out = _render(s, cams, means, rots, feat, fpc=2, contrib=c)
        assert np.array_equal(c.weight_q.cpu().numpy(), wq), F
        assert np.array_equal(c.max_weight.cpu().numpy(), mx), F
        assert np.array_equal(c.pixels.cpu().numpy(), px), F
        assert torch.equal(c.frames, (out["radii"] > 0).sum(0)), F
        assert bool((c.weight.cpu() == torch.from_numpy(wq).double() / 2.0 ** 32).all())
        got[F] = c
    _same(got[0], got[22], "F = 0 vs F = 22")
    _same(got[0], got[32], "F = 0 vs F = 32")


def test_render_is_unchanged_by_the_accumulator(dev):
    T, W, H, P = 4, 128, 96, 20_000
    s, means, rots, feat = _inputs(P, T, 22, True, dev)
    cams = _cams(T, W, H, dev)
    a = _render(s, cams, means, rots, feat, fpc=3)
    b = _render(s, cams, means, rots, feat, fpc=3, contrib=_zeros(P, dev))
    _same_outputs(a, b, "with and without the accumulator")


def test_invariances(dev):
    """frames_per_call, frame order, several calls into one accumulator, overflow re-runs and repeated runs give the
    same bits."""
    from vidu4d_b200.renderer import BatchCameras
    T, W, H, P = 8, 160, 120, 20_000
    s, means, rots, _ = _inputs(P, T, 0, True, dev, seed=4)
    cams = _cams(T, W, H, dev)
    ref = _zeros(P, dev)
    _render(s, cams, means, rots, fpc=8, contrib=ref)
    assert int(ref.pixels.sum()) > 0
    for fpc in (1, 3, 8):
        c = _zeros(P, dev)
        _render(s, cams, means, rots, fpc=fpc, contrib=c)
        _same(c, ref, f"frames_per_call {fpc}")

    def sub(idx):
        i = torch.tensor(idx, device=dev)
        return BatchCameras(W, H, cams.FoVx, cams.FoVy, cams.world_view_transform[i].contiguous(),
                            cams.full_proj_transform[i].contiguous(), cams.camera_center[i].contiguous()), \
            means[i].contiguous(), rots[i].contiguous()
    perm = [5, 2, 7, 0, 3, 6, 1, 4]
    c = _zeros(P, dev)
    _render(s, *sub(perm), fpc=3, contrib=c)
    _same(c, ref, "permuted frames")

    c = _zeros(P, dev)
    _render(s, *sub([6, 7, 0]), fpc=2, contrib=c)
    _render(s, *sub([1, 2, 3, 4, 5]), fpc=4, contrib=c)
    _same(c, ref, "two calls into one accumulator")

    c = _zeros(P, dev)
    # a hint far too small: the first chunk overflows, and its frames re-run alone
    _, grown = _with_capacity_hint(dev, W, H, 1, lambda: _render(s, cams, means, rots, fpc=3, contrib=c))
    assert grown > 4096
    _same(c, ref, "overflow and re-run")

    c = _zeros(P, dev)
    _render(s, cams, means, rots, fpc=8, contrib=c)
    _same(c, ref, "second run")


@pytest.mark.parametrize("table", [False, True], ids=["scalar", "table"])
def test_overflow_rerun_keeps_every_output(table, dev):
    """With an accumulator a chunk that overflows re-runs its frames one at a time; every output of the chunk -- colour
    with the learnable background, feature planes, all maps and radii -- must still be the bits of a run that does not
    overflow, and so must the statistics.  7 frames in chunks of 3: every frame of the first chunk overflows (the last
    re-run is the chunk's third frame), then the later chunks run with the grown capacity."""
    T, W, H, P = 7, 160, 120, 20_000
    s, means, rots, feat = _inputs(P, T, 22, True, dev, seed=6)
    cams = _cams(T, W, H, dev, _table(T, dev, offsets=True) if table else None)
    bkgd = torch.tensor([0.25, -0.5, 0.75], device=dev)
    ref_c = _zeros(P, dev)
    plain = _render(s, cams, means, rots, feat, fpc=3, bkgd=bkgd)
    ref = _render(s, cams, means, rots, feat, fpc=3, contrib=ref_c, bkgd=bkgd)
    _same_outputs(ref, plain, "no overflow, with and without the accumulator")
    c = _zeros(P, dev)
    got, grown = _with_capacity_hint(dev, W, H, 1,
                                     lambda: _render(s, cams, means, rots, feat, fpc=3, contrib=c, bkgd=bkgd))
    assert grown > 4096
    _same_outputs(got, plain, "overflow and per-frame re-runs")
    _same(c, ref_c, "overflow and per-frame re-runs")


def test_overflowed_frame_adds_nothing_at_the_abi(dev):
    """A frame that overflows is not composited and adds nothing; a frame that fits adds its share."""
    from vidu4d_b200 import rasterizer as RZ
    from vidu4d_b200.rasterizer import _RenderOut, _batch_inputs, _forward
    from vidu4d_b200 import _capi
    T, W, H, P = 1, 96, 96, 20_000
    s, _, _, _ = _inputs(P, T, 0, False, dev)
    cams = _cams(T, W, H, dev)
    ins, strides = _batch_inputs(T, means3D=(s["means3D"], (3,)), sh=(s["shs"], None), opacity=(s["opacities"], (1,)),
                                 scales=(s["scales"], (2,)), rotations=(s["rotations"], (4,)))
    c = _zeros(P, dev)
    out = _RenderOut(torch.empty((T, 3, H, W), device=dev), None, torch.empty((T, 8, H, W), device=dev),
                     torch.empty((T, P), dtype=torch.int32, device=dev),
                     contrib=_capi.SrContrib(c.weight_q.data_ptr(), c.max_weight.data_ptr(), c.pixels.data_ptr()))
    lib = _capi.load()
    arena = torch.empty((int(lib.sr_render_bytes(P, 4096, W, H)),), dtype=torch.uint8, device=dev)
    nr = torch.zeros((T, 2), dtype=torch.int32, device=dev)
    host = torch.zeros((T, 2), dtype=torch.int32, pin_memory=True)
    fr, frp = RZ._frame(P, 3, 16, W, H, TANF, TANF, 1.0, False, False, None)
    bt = _capi.SrBatch(T, 0, 0, 0, 0, 0, 0, 0)
    _capi.call("sr_render_forward_contrib", dev, frp, C.byref(bt), torch.zeros(3, device=dev), 3, ins["means3D"], ins["sh"], None,
               ins["opacity"], ins["scales"], ins["rotations"], None, 0, 0, cams.world_view_transform,
               cams.full_proj_transform, cams.camera_center, out.color, 0, None, 0, out.others, out.radii, arena, 4096,
               nr, host, C.byref(out.contrib))
    torch.cuda.synchronize()
    assert int(host[0, 1]) & _capi.SR_STATUS_OVERFLOW and int(host[0, 0]) > 4096
    assert int(c.weight_q.abs().sum()) == 0 and int(c.pixels.sum()) == 0 and int(c.max_weight.abs().sum()) == 0
    _forward(T, True, strides, torch.zeros(3, device=dev), ins["means3D"], ins["sh"], None, ins["opacity"], ins["scales"],
             ins["rotations"], None, cams.world_view_transform, cams.full_proj_transform, cams.camera_center, H, W, 3,
             TANF, TANF, 1.0, False, False, render=out)
    ref = _zeros(P, dev)
    _render(s, cams, None, None, contrib=ref)
    assert torch.equal(c.weight_q, ref.weight_q) and torch.equal(c.pixels, ref.pixels)
    assert torch.equal(c.max_weight, ref.max_weight)


@pytest.mark.parametrize("case", ["empty", "culled"])
def test_empty_and_culled(case, dev):
    T, W, H = 3, 64, 48
    P = 0 if case == "empty" else 5000
    s, _, _, _ = _inputs(max(P, 1), T, 0, False, dev)
    if P == 0:
        s = {k: v[:0] for k, v in s.items()}
    means = None
    if case == "culled":
        cams = _cams(T, W, H, dev)
        # every surfel behind every camera: the view-space z of each frame's centre reflected through the camera
        wvt = cams.world_view_transform
        x = s["means3D"]
        cam_pos = cams.camera_center
        means = (2 * cam_pos[:, None, :] - x[None]).contiguous()            # point reflection through the camera
        z = torch.einsum("tpk,tk->tp", torch.nn.functional.pad(means, (0, 1), value=1.0), wvt[:, :, 2])
        assert bool((z < 0.2).all())
    else:
        cams = _cams(T, W, H, dev)
    c = _zeros(P, dev)
    out = _render(s, cams, means, None, contrib=c)
    for name in ("weight_q", "max_weight", "pixels", "frames"):
        assert int(getattr(c, name).abs().sum()) == 0, name
    assert int((out["radii"] > 0).sum()) == 0
    assert int(c.prune_mask().sum()) == P


def _occluded_model(dev):
    """A small scene in front of three large opaque discs, and one small surfel (the last) behind them."""
    from vidu4d_b200.surfel_store import FlatSurfelModel
    g = torch.Generator().manual_seed(11)
    n_front = 300
    front = torch.cat([(torch.rand((n_front, 2), generator=g) - 0.5) * 1.2, torch.full((n_front, 1), 1.5)], 1)
    discs = torch.tensor([[0.0, 0.0, 2.0], [0.05, -0.03, 2.1], [-0.04, 0.02, 2.2]])
    hidden = torch.tensor([[0.0, 0.0, 3.0]])
    xyz = torch.cat([front, discs, hidden])
    P = xyz.shape[0]
    scale = torch.cat([torch.full((n_front, 2), 0.02), torch.full((3, 2), 20.0), torch.full((1, 2), 0.05)])
    op = torch.cat([torch.full((n_front, 1), 0.8), torch.full((3, 1), 0.999), torch.full((1, 1), 0.9)])
    rot = torch.zeros((P, 4)); rot[:, 0] = 1.0
    fdc = torch.rand((P, 1, 3), generator=g) - 0.5
    frest = (torch.rand((P, 15, 3), generator=g) - 0.5) * 0.1
    t = lambda a: a.to(dev).contiguous()  # noqa: E731
    return FlatSurfelModel(t(xyz), t(fdc), t(frest), t(torch.log(op / (1 - op))), t(torch.log(scale)), t(rot),
                           sh_degree=3, regist_feat=t(torch.rand((P, 16), generator=g)))


def _front_cams(T, W, H, dev):
    from vidu4d_b200.renderer import make_camera, stack_cameras
    import math
    fov = 2 * math.atan(0.5)
    return stack_cameras([make_camera(W, H, fov, fov, T=(0.03 * f - 0.03, 0.02 * f, 0.0), device=dev) for f in range(T)])


def test_hidden_surfel_is_pruned_and_the_images_stay(dev):
    from vidu4d_b200.renderer import PipelineParams, render_frames
    T, W, H = 3, 96, 80
    m = _occluded_model(dev)
    P = m.P
    cams = _front_cams(T, W, H, dev)
    bg = torch.zeros(3, device=dev)
    c = _zeros(P, dev)
    before = render_frames(cams, m, PipelineParams(), bg, contributions=c)
    assert int(c.frames[P - 1]) == T                           # seen by the preprocess in every frame ...
    assert int(c.weight_q[P - 1]) == 0 and int(c.pixels[P - 1]) == 0 and int(c.max_weight[P - 1]) == 0   # ... never blended
    assert int(c.pixels[P - 4]) > 0                             # the nearest disc is
    mask = c.prune_mask()
    keep_feat = m._regist_feat.detach()[~mask].clone()
    n = m.prune_by_contribution(c)
    assert n == int(mask.sum()) >= 1 and m.P == P - n
    assert torch.equal(m._regist_feat.detach(), keep_feat)
    after = render_frames(cams, m, PipelineParams(), bg)
    for k in ("render", "acc", "rend_normal", "rend_dist", "surf_depth", "surf_normal"):
        assert torch.equal(before[k].contiguous().view(torch.int32), after[k].contiguous().view(torch.int32)), k
    # nothing left to prune: the buffers stay where they are
    c2 = _zeros(m.P, dev)
    render_frames(cams, m, PipelineParams(), bg, contributions=c2)
    flat = m.flat.data_ptr()
    assert m.prune_by_contribution(c2) == 0 and m.flat.data_ptr() == flat
    with pytest.raises(RuntimeError, match="contributions are for"):
        m.prune_by_contribution(_zeros(m.P + 1, dev))


def test_prune_then_graphed_step_recaptures(dev):
    """prune_by_contribution between steps of a captured Stage-3 step: the change of P re-captures, and the step runs."""
    import math
    from vidu4d_b200.graph import GraphedStep
    from vidu4d_b200.renderer import PipelineParams, make_camera, render_frames, render_loss_batch, stack_cameras
    from vidu4d_b200.synthetic import orbit_view
    from vidu4d_b200.surfel_store import FlatSurfelModel
    from vidu4d_b200.synthetic import object_scene
    sc = object_scene(20000, seed=2, center=(0.0, 0.0, 0.0))
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    op = np.clip(sc.opacities, 1e-6, 1 - 1e-6)
    m = FlatSurfelModel(t(sc.means3D), t(sc.shs[:, :1]), t(sc.shs[:, 1:]), t(np.log(op / (1 - op))), t(np.log(sc.scales)),
                        t(sc.rotations))
    M, W, H = 2, 96, 96
    fov = 2 * math.atan(0.5)
    cams = []
    for f in range(M):
        R, tt = orbit_view(7 * f + 3, 64)
        cams.append(make_camera(W, H, fov, fov, R=R.T, T=tt, device=dev))
    cams = stack_cameras(cams)
    pipe, bg = PipelineParams(), torch.zeros(3, device=dev)
    rgb = torch.rand((M, 3, H, W), device=dev, generator=torch.Generator(device=dev).manual_seed(1))
    losses = []

    def body():
        m.zero_grad_flat()
        out = render_loss_batch(cams, m, pipe, bg, rgb)
        out["loss"].backward()
        m.step()
        losses.append(out["loss"].detach())

    from vidu4d_b200 import rasterizer as RZ
    try:
        gs = GraphedStep(body, key=lambda: m.P, device=dev)
        gs()
        assert gs.captures == 1
        c = _zeros(m.P, dev)
        render_frames(cams, m, pipe, bg, contributions=c)
        P0 = m.P
        n = m.prune_by_contribution(c, min_pixels=4)
        assert n > 0 and m.P == P0 - n
        step0 = int(m.device_step)
        gs()
        assert gs.captures == 2 and int(m.device_step) > step0
        gs()
        assert gs.captures == 2
        torch.cuda.synchronize()
        assert math.isfinite(float(losses[-1]))
        assert bool(torch.isfinite(m.flat).all())
    finally:
        RZ.set_sync_mode(True)                 # GraphedStep leaves the rasterizer in no-sync mode
        RZ._pending.clear()
