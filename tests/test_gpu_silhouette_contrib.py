"""GPU: the background share of the contribution statistics (render_frames(..., masks=), sr_render_forward_contrib_masked)
and pruning by it.

The oracle is test_gpu_contrib's: with one-hot features, plane s mod 32 of group s // 32's render is surfel s's per-pixel
weight w = T alpha exactly.  So weight_bg_q must be the sum over background pixels of rn(plane 2^32) and pixels_bg the
number of background pixels where the plane is positive, bit for bit; and the three older words must stay those of the
unmasked walk."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from .test_gpu_contrib import OUTPUTS, _PC, _front_cams, _same_outputs, _with_capacity_hint
from .test_gpu_render import TANF, _cams, _inputs, _table

pytestmark = pytest.mark.gpu

WORDS = ("weight_q", "max_weight", "pixels", "frames", "weight_bg_q", "pixels_bg")


@pytest.fixture(scope="module")
def dev(built):
    from vidu4d_b200 import _capi
    _capi.load()
    return torch.device("cuda:0")


def _render(s, cams, means, rots, feat=None, fpc=8, contrib=None, masks=None, bkgd=None):
    from vidu4d_b200.renderer import PipelineParams, render_frames
    dev = s["means3D"].device
    return render_frames(cams, _PC(s), PipelineParams(depth_ratio=0.37), torch.zeros(3, device=dev), means3D=means,
                         rotations=rots, features=feat, learnable_bkgd=bkgd, frames_per_call=fpc, contributions=contrib,
                         masks=masks)


def _zeros(P, dev, silhouettes=True):
    from vidu4d_b200.renderer import SurfelContributions
    return SurfelContributions.zeros(P, dev, silhouettes=silhouettes)


def _same(a, b, what, names=WORDS):
    for name in names:
        x, y = getattr(a, name), getattr(b, name)
        assert x.dtype == y.dtype and x.shape == y.shape, (what, name)
        n = int((x != y).sum())
        assert n == 0, f"{what}: {name} differs for {n} of {x.numel()} surfels"


def _masks(kind, T, W, H, dev, seed=0):
    """(masks as passed, the (T,H,W) bool foreground they mean)."""
    y, x = torch.meshgrid(torch.arange(H, device=dev), torch.arange(W, device=dev), indexing="ij")
    g = torch.Generator(device=dev).manual_seed(seed)
    if kind == "random":                            # bool
        fg = torch.rand((T, H, W), device=dev, generator=g) < 0.5
        return fg, fg
    if kind == "float":                             # float (T,1,H,W), foreground where > 0.5
        f = torch.rand((T, 1, H, W), device=dev, generator=g)
        f[..., ::7, :] = 0.5                        # exactly 0.5 is background
        return f, (f > 0.5)[:, 0]
    # "seams": uint8 with edges on the 16x16 tile seams and the 8x4 sub-tile seams, nonzero values other than 1
    tiles = ((x // 16) + (y // 16)) % 2 == 0
    subs = ((x // 8) + (y // 4)) % 2 == 0
    fg = torch.stack([(tiles, subs, ~tiles)[t % 3] for t in range(T)])
    return fg.to(torch.uint8) * 7, fg


def _onehot(s, cams, means, rots, fg):
    """Per surfel, from the one-hot feature planes: weight_q, max_weight bits and pixels over every pixel, and
    weight_bg_q and pixels_bg over the background pixels of `fg` ((T,H,W) bool)."""
    P = int(s["means3D"].shape[0])
    dev = s["means3D"].device
    bg = (~fg).cpu().numpy()[:, None]
    wq, mx, px, wb, pb = (np.zeros(P, np.int64), np.zeros(P, np.float32), np.zeros(P, np.int64), np.zeros(P, np.int64),
                          np.zeros(P, np.int64))
    for g in range((P + 31) // 32):
        lo, hi = 32 * g, min(P, 32 * g + 32)
        feat = torch.zeros((P, 32), device=dev)
        feat[torch.arange(lo, hi, device=dev), torch.arange(hi - lo, device=dev)] = 1.0
        planes = _render(s, cams, means, rots, feat)["features"][:, :hi - lo].cpu().numpy()      # (T, k, H, W)
        q = np.rint(planes.astype(np.float64) * 2.0 ** 32).astype(np.int64)
        wq[lo:hi] = q.sum(axis=(0, 2, 3))
        mx[lo:hi] = planes.max(axis=(0, 2, 3))
        px[lo:hi] = (planes > 0).sum(axis=(0, 2, 3))
        wb[lo:hi] = (q * bg).sum(axis=(0, 2, 3))
        pb[lo:hi] = ((planes > 0) & bg).sum(axis=(0, 2, 3))
    return wq, mx.view(np.int32), px, wb, pb


SIZES = [(16, 16, 600), (75, 53, 2000), (130, 98, 3000)]


@pytest.mark.parametrize("W,H,P", SIZES, ids=[f"{w}x{h}_P{p}" for w, h, p in SIZES])
@pytest.mark.parametrize("table", [False, True], ids=["scalar", "table"])
@pytest.mark.parametrize("per_frame", [False, True], ids=["shared", "per_frame"])
def test_background_words_equal_the_one_hot_planes(per_frame, table, W, H, P, dev):
    T = 3
    s, means, rots, _ = _inputs(P, T, 0, per_frame, dev)
    cams = _cams(T, W, H, dev, _table(T, dev, offsets=True) if table else None)
    plain = _zeros(P, dev, silhouettes=False)
    _render(s, cams, means, rots, fpc=2, contrib=plain)
    assert int(plain.pixels.sum()) > 0
    for kind in ("random", "float", "seams"):
        masks, fg = _masks(kind, T, W, H, dev)
        wq, mx, px, wb, pb = _onehot(s, cams, means, rots, fg)
        assert 0 < pb.sum() < px.sum(), kind
        c = _zeros(P, dev)
        _render(s, cams, means, rots, fpc=2, contrib=c, masks=masks)
        assert np.array_equal(c.weight_bg_q.cpu().numpy(), wb), kind
        assert np.array_equal(c.pixels_bg.cpu().numpy(), pb), kind
        assert np.array_equal(c.weight_q.cpu().numpy(), wq), kind
        assert np.array_equal(c.max_weight.cpu().numpy(), mx), kind
        assert np.array_equal(c.pixels.cpu().numpy(), px), kind
        _same(c, plain, f"{kind}: the unmasked words", WORDS[:4])


@pytest.mark.parametrize("table", [False, True], ids=["scalar", "table"])
@pytest.mark.parametrize("F", [0, 1, 8, 22, 32])
def test_nothing_else_moves(F, table, dev):
    """Every output -- colour with a learnable background, allmap-derived maps, feature planes and radii -- and the four
    older words are the bits of the unmasked render; without statistics too."""
    T, W, H, P = 4, 120, 90, 20_000
    s, means, rots, feat = _inputs(P, T, F, True, dev, seed=7)
    cams = _cams(T, W, H, dev, _table(T, dev, offsets=True) if table else None)
    bkgd = torch.tensor([0.25, -0.5, 0.75], device=dev)
    masks, _ = _masks("random", T, W, H, dev, seed=F)
    none = _render(s, cams, means, rots, feat, fpc=3, bkgd=bkgd)
    c0 = _zeros(P, dev, silhouettes=False)
    plain = _render(s, cams, means, rots, feat, fpc=3, contrib=c0, bkgd=bkgd)
    c = _zeros(P, dev)
    got = _render(s, cams, means, rots, feat, fpc=3, contrib=c, masks=masks[:, None], bkgd=bkgd)      # (T,1,H,W)
    _same_outputs(plain, none, "statistics without masks")
    _same_outputs(got, none, "statistics with masks")
    _same(c, c0, "with and without masks", WORDS[:4])
    assert int(c.pixels_bg.sum()) > 0


def test_all_foreground_and_all_background(dev):
    T, W, H, P = 3, 96, 72, 10_000
    s, means, rots, _ = _inputs(P, T, 0, True, dev, seed=8)
    cams = _cams(T, W, H, dev)
    c0 = _zeros(P, dev, silhouettes=False)
    _render(s, cams, means, rots, contrib=c0)
    for name, masks in (("all foreground", torch.ones((T, H, W), dtype=torch.uint8, device=dev)),
                        ("all foreground (float)", torch.ones((T, H, W), device=dev)),
                        ("all background", torch.zeros((T, H, W), dtype=torch.bool, device=dev))):
        c = _zeros(P, dev)
        _render(s, cams, means, rots, contrib=c, masks=masks)
        _same(c, c0, name, WORDS[:4])
        if name.startswith("all foreground"):
            assert int(c.weight_bg_q.abs().sum()) == 0 and int(c.pixels_bg.abs().sum()) == 0, name
            assert int((c.background_fraction != 0).sum()) == 0
        else:
            assert torch.equal(c.weight_bg_q, c.weight_q) and torch.equal(c.pixels_bg, c.pixels)
            assert bool((c.background_fraction[c.weight_q > 0] == 1.0).all())
    assert int(c0.pixels.sum()) > 0


def test_invariances(dev):
    """frames_per_call, frame order (the masks follow their frames), several calls into one accumulator, overflow re-runs
    of single frames (each with its own mask) and repeated runs give the same bits."""
    from vidu4d_b200.renderer import BatchCameras
    T, W, H, P = 8, 150, 110, 20_000
    s, means, rots, _ = _inputs(P, T, 0, True, dev, seed=4)
    cams = _cams(T, W, H, dev)
    masks, _ = _masks("seams", T, W, H, dev)
    masks[5] = _masks("random", 1, W, H, dev, seed=5)[0][0].to(torch.uint8)
    ref = _zeros(P, dev)
    _render(s, cams, means, rots, fpc=8, contrib=ref, masks=masks)
    assert int(ref.pixels_bg.sum()) > 0
    for fpc in (1, 3, 8):
        c = _zeros(P, dev)
        _render(s, cams, means, rots, fpc=fpc, contrib=c, masks=masks)
        _same(c, ref, f"frames_per_call {fpc}")

    def sub(idx):
        i = torch.tensor(idx, device=dev)
        return BatchCameras(W, H, cams.FoVx, cams.FoVy, cams.world_view_transform[i].contiguous(),
                            cams.full_proj_transform[i].contiguous(), cams.camera_center[i].contiguous()), \
            means[i].contiguous(), rots[i].contiguous()
    perm = [5, 2, 7, 0, 3, 6, 1, 4]
    c = _zeros(P, dev)
    _render(s, *sub(perm), fpc=3, contrib=c, masks=masks[perm])
    _same(c, ref, "permuted frames")

    c = _zeros(P, dev)
    _render(s, *sub([6, 7, 0]), fpc=2, contrib=c, masks=masks[[6, 7, 0]])
    _render(s, *sub([1, 2, 3, 4, 5]), fpc=4, contrib=c, masks=masks[1:6])
    _same(c, ref, "two calls into one accumulator")

    c = _zeros(P, dev)
    # a hint far too small: the first chunk overflows, and its frames re-run alone with their own masks
    _, grown = _with_capacity_hint(dev, W, H, 1, lambda: _render(s, cams, means, rots, fpc=3, contrib=c, masks=masks))
    assert grown > 4096
    _same(c, ref, "overflow and re-run")

    c = _zeros(P, dev)
    _render(s, cams, means, rots, fpc=8, contrib=c, masks=masks)
    _same(c, ref, "second run")


def test_abi_null_mask_and_overflow(dev):
    """At the ABI: a mask struct whose mask is NULL gives sr_render_forward_contrib's words and leaves its own output
    words alone; an overflowed frame adds nothing to any word."""
    from vidu4d_b200 import _capi
    from vidu4d_b200 import rasterizer as RZ
    from vidu4d_b200.rasterizer import _batch_inputs
    T, W, H, P = 1, 96, 96, 20_000
    s, _, _, _ = _inputs(P, T, 0, False, dev)
    cams = _cams(T, W, H, dev)
    ins, _ = _batch_inputs(T, means3D=(s["means3D"], (3,)), sh=(s["shs"], None), opacity=(s["opacities"], (1,)),
                           scales=(s["scales"], (2,)), rotations=(s["rotations"], (4,)))
    lib = _capi.load()
    color, others = torch.empty((T, 3, H, W), device=dev), torch.empty((T, 8, H, W), device=dev)
    radii = torch.empty((T, P), dtype=torch.int32, device=dev)
    fr, frp = RZ._frame(P, 3, 16, W, H, TANF, TANF, 1.0, False, False, None)
    bt = _capi.SrBatch(T, 0, 0, 0, 0, 0, 0, 0)
    fg = _masks("random", T, W, H, dev)[0].to(torch.uint8)

    def call(cap, c, mask_ptr):
        arena = torch.empty((int(lib.sr_render_bytes(P, cap, W, H)),), dtype=torch.uint8, device=dev)
        nr = torch.zeros((T, 2), dtype=torch.int32, device=dev)
        host = torch.zeros((T, 2), dtype=torch.int32, pin_memory=True)
        ct = _capi.SrContrib(c.weight_q.data_ptr(), c.max_weight.data_ptr(), c.pixels.data_ptr())
        mk = _capi.SrContribMask(mask_ptr, W * H, c.weight_bg_q.data_ptr(), c.pixels_bg.data_ptr())
        _capi.call("sr_render_forward_contrib_masked", dev, frp, C.byref(bt), torch.zeros(3, device=dev), 3,
                   ins["means3D"], ins["sh"], None, ins["opacity"], ins["scales"], ins["rotations"], None, 0, 0,
                   cams.world_view_transform, cams.full_proj_transform, cams.camera_center, color, 0, None, 0, others,
                   radii, arena, cap, nr, host, C.byref(ct), C.byref(mk))
        torch.cuda.synchronize()
        return host

    c = _zeros(P, dev)
    host = call(4096, c, fg.data_ptr())
    assert int(host[0, 1]) & _capi.SR_STATUS_OVERFLOW and int(host[0, 0]) > 4096
    for name in WORDS[:3] + WORDS[4:]:
        assert int(getattr(c, name).abs().sum()) == 0, name
    cap = RZ._round_cap(int(host[0, 0]) + 4096)
    call(cap, c, fg.data_ptr())
    ref = _zeros(P, dev)
    _render(s, cams, None, None, contrib=ref, masks=fg)
    _same(c, ref, "overflow then re-run at the ABI", WORDS[:3] + WORDS[4:])

    c = _zeros(P, dev)
    c.weight_bg_q.fill_(-3)
    c.pixels_bg.fill_(5)
    call(cap, c, None)
    plain = _zeros(P, dev, silhouettes=False)
    _render(s, cams, None, None, contrib=plain)
    _same(c, plain, "NULL mask", WORDS[:3])
    assert bool((c.weight_bg_q == -3).all()) and bool((c.pixels_bg == 5).all())


def _model(xyz, scale, op, dev, seed=11):
    from vidu4d_b200.surfel_store import FlatSurfelModel
    g = torch.Generator().manual_seed(seed)
    P = xyz.shape[0]
    rot = torch.zeros((P, 4)); rot[:, 0] = 1.0
    fdc = torch.rand((P, 1, 3), generator=g) - 0.5
    frest = (torch.rand((P, 15, 3), generator=g) - 0.5) * 0.1
    t = lambda a: a.to(dev).contiguous()  # noqa: E731
    return FlatSurfelModel(t(xyz), t(fdc), t(frest), t(torch.log(op / (1 - op))), t(torch.log(scale)), t(rot),
                           sh_degree=3, regist_feat=t(torch.arange(P, dtype=torch.float32)[:, None].expand(P, 16)))


def test_floating_clump_is_pruned_and_the_object_stays(dev):
    """An object inside the silhouette and an opaque clump off to its side, which every front camera sees over
    background only: with max_background_fraction 0.5 exactly the clump goes, and every foreground pixel the clump never
    covered renders the same bits."""
    from vidu4d_b200.renderer import PipelineParams, render_frames
    T, W, H = 4, 96, 80
    g = torch.Generator().manual_seed(3)
    n_obj, n_clump = 400, 24
    obj = torch.cat([(torch.rand((n_obj, 2), generator=g) - 0.5) * 0.8, 1.5 + 0.05 * torch.rand((n_obj, 1), generator=g)], 1)
    clump = torch.tensor([0.6, 0.48, 1.4]) + 0.03 * (torch.rand((n_clump, 3), generator=g) - 0.5)
    xyz = torch.cat([obj, clump])
    scale = torch.full((n_obj + n_clump, 2), 0.02)
    op = torch.cat([torch.full((n_obj, 1), 0.8), torch.full((n_clump, 1), 0.95)])
    m = _model(xyz, scale, op, dev)
    cams = _front_cams(T, W, H, dev)
    pipe, bg = PipelineParams(), torch.zeros(3, device=dev)
    fg = render_frames(cams, _model(obj, scale[:n_obj], op[:n_obj], dev), pipe, bg)["acc"][:, 0] > 0     # silhouettes
    clump_cover = render_frames(cams, _model(clump, scale[n_obj:], op[n_obj:], dev), pipe, bg)["acc"][:, 0] > 0
    assert int(clump_cover.sum()) > 0 and not bool((fg & clump_cover).any())
    c = _zeros(m.P, dev)
    before = render_frames(cams, m, pipe, bg, contributions=c, masks=fg)
    frac = c.background_fraction
    assert bool((c.pixels > 0).all())                           # every surfel is blended somewhere
    assert bool((frac[:n_obj] == 0).all()) and bool((frac[n_obj:] == 1).all())
    assert m.prune_by_contribution(c, max_background_fraction=0.5) == n_clump and m.P == n_obj
    assert torch.equal(m._regist_feat.detach()[:, 0], torch.arange(n_obj, dtype=torch.float32, device=dev))
    after = render_frames(cams, m, pipe, bg)
    keep = (fg & ~clump_cover)[:, None]
    assert int(keep.sum()) > 0
    for k in ("render", "acc", "rend_normal", "rend_dist", "surf_depth", "surf_normal", "render_depth_median"):
        a, b = before[k].contiguous(), after[k].contiguous()
        sel = keep.expand(-1, a.shape[1], -1, -1)
        assert torch.equal(a[sel].view(torch.int32), b[sel].view(torch.int32)), k
    assert bool((after["acc"][clump_cover[:, None]] < before["acc"][clump_cover[:, None]]).any())


def test_prune_then_graphed_step_recaptures(dev):
    """prune_by_contribution(..., max_background_fraction) between steps of a captured Stage-3 step: the change of P
    re-captures, and the step runs."""
    from vidu4d_b200.graph import GraphedStep
    from vidu4d_b200.renderer import PipelineParams, make_camera, render_frames, render_loss_batch, stack_cameras
    from vidu4d_b200.surfel_store import FlatSurfelModel
    from vidu4d_b200.synthetic import object_scene, orbit_view
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
        # the left half of every frame is foreground: what lands mostly on the right half goes
        masks = torch.zeros((M, H, W), dtype=torch.bool, device=dev)
        masks[:, :, : W // 2] = True
        c = _zeros(m.P, dev)
        render_frames(cams, m, pipe, bg, contributions=c, masks=masks)
        P0 = m.P
        want = int(c.prune_mask(max_background_fraction=0.5).sum())
        n = m.prune_by_contribution(c, max_background_fraction=0.5)
        assert n == want > int(c.prune_mask().sum()) and m.P == P0 - n
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
