"""GPU: per-pixel maps lifted onto the surfels (render_frames(..., lift=, values=), sr_render_forward_lift).

The oracle is test_gpu_contrib's: with one-hot features -- plane k equal to 1 on surfel sub[k] of a chosen subset of 32
and 0 on every other surfel, over a zero feature background -- plane k of the render is surfel sub[k]'s per-pixel weight
w = T alpha exactly.  So sums[sub[k], c] must be, bit for bit, the int64 sum over the pixels where plane k is positive of
rn(fl(w v) 2^s), formed here in numpy: fl(w v) is numpy's float32 product, the scaling is exact in float64 and rint
rounds half to even.  Non-finite values give 0 and |fl(w v) 2^s| > 2^32 gives +-2^32, each counted in `saturated`."""
import ctypes as C

import numpy as np
import pytest
import torch

from .test_gpu_contrib import _PC, _front_cams, _same_outputs, _with_capacity_hint
from .test_gpu_render import TANF, _cams, _inputs, _table
from .test_gpu_silhouette_contrib import _masks, _model

pytestmark = pytest.mark.gpu

WORDS = ("weight_q", "max_weight", "pixels", "frames")


@pytest.fixture(scope="module")
def dev(built):
    from vidu4d_b200 import _capi
    _capi.load()
    return torch.device("cuda:0")


def _render(s, cams, means, rots, feat=None, fpc=8, contrib=None, masks=None, lift=None, values=None, bkgd=None):
    from vidu4d_b200.renderer import PipelineParams, render_frames
    dev = s["means3D"].device
    return render_frames(cams, _PC(s), PipelineParams(depth_ratio=0.37), torch.tensor([0.1, 0.2, 0.3], device=dev),
                         means3D=means, rotations=rots, features=feat, learnable_bkgd=bkgd, frames_per_call=fpc,
                         contributions=contrib, masks=masks, lift=lift, values=values)


def _zeros(P, dev, silhouettes=False):
    from vidu4d_b200.renderer import SurfelContributions
    return SurfelContributions.zeros(P, dev, silhouettes=silhouettes)


def _lift(P, Cn, dev, B=1.0):
    from vidu4d_b200.renderer import SurfelLift
    return SurfelLift.zeros(P, Cn, dev, value_bound=B)


def _same(a, b, what, names=WORDS):
    for name in names:
        x, y = getattr(a, name), getattr(b, name)
        assert x.dtype == y.dtype and x.shape == y.shape, (what, name)
        n = int((x != y).sum())
        assert n == 0, f"{what}: {name} differs in {n} of {x.numel()} elements"


def _same_lift(a, b, what):
    _same(a, b, what, ("sums", "saturated"))
    assert a.scale_log2 == b.scale_log2


def _subset(c, P, seed=0):
    """32 surfels: the 16 that blend the most pairs and 16 others drawn at random."""
    top = torch.argsort(c.pixels, descending=True)[:16].cpu().numpy()
    rest = np.setdiff1d(np.arange(P), top)
    rng = np.random.default_rng(seed)
    return np.concatenate([top, rng.choice(rest, 32 - len(top), replace=False)])


def _planes(s, cams, means, rots, sub):
    """(T, 32, H, W) float32: plane k is surfel sub[k]'s per-pixel weight."""
    P = int(s["means3D"].shape[0])
    dev = s["means3D"].device
    feat = torch.zeros((P, 32), device=dev)
    feat[torch.from_numpy(sub).to(dev), torch.arange(32, device=dev)] = 1.0
    return _render(s, cams, means, rots, feat)["features"].cpu().numpy()


def _oracle(planes, values, s):
    """(32, C) int64 sums and the saturated count of the 32 planes' surfels, by the contract."""
    v = values.cpu().numpy().astype(np.float32)                         # (T, C, H, W)
    out = np.zeros((planes.shape[1], v.shape[1]), np.int64)
    sat = 0
    for k in range(planes.shape[1]):
        w = planes[:, k][:, None]                                       # (T, 1, H, W)
        on = np.broadcast_to(w > 0, v.shape)
        with np.errstate(invalid="ignore", over="ignore"):
            p = (w * v).astype(np.float32)                              # one float32 rounding
            x = p.astype(np.float64) * 2.0 ** s                         # exact
        bad = on & ~np.isfinite(v)
        big = on & np.isfinite(v) & (np.abs(x) > 2.0 ** 32)
        q = np.where(on & np.isfinite(v) & ~big, np.rint(np.where(np.isfinite(x), x, 0.0)), 0.0).astype(np.int64)
        q += np.where(big, np.sign(x) * 2.0 ** 32, 0.0).astype(np.int64)
        out[k] = q.sum(axis=(0, 2, 3))
        sat += int(bad.sum() + big.sum())
    return out, sat


def _values(kind, T, Cn, W, H, dev, seed=0):
    """(values (T,C,H,W) float32, value_bound) of one kind."""
    g = torch.Generator(device=dev).manual_seed(seed)
    u = torch.rand((T, Cn, H, W), device=dev, generator=g)
    if kind == "random":                    # both signs, within B = 4
        return (u * 8 - 4), 4.0
    if kind == "negative":                  # large negative values, B = 1000
        return -(u * 1000), 1000.0
    if kind == "seams":                     # sign and magnitude change on the 16x16 tile and 8x4 sub-tile seams
        y, x = torch.meshgrid(torch.arange(H, device=dev), torch.arange(W, device=dev), indexing="ij")
        sgn = torch.where(((x // 16) + (y // 16)) % 2 == 0, 1.0, -1.0)
        mag = torch.where(((x // 8) + (y // 4)) % 2 == 0, 1.0, 0.25)
        ch = torch.arange(Cn, device=dev, dtype=torch.float32)[None, :, None, None]
        return (sgn * mag)[None, None] * (1.0 - ch / 64) * torch.ones((T, 1, 1, 1), device=dev), 1.0
    # "subres": |w v 2^s| mostly below a few units, so the rounding to integers decides (ties included)
    v = (torch.floor(u * 8) - 4) * 2.0 ** -33
    return v, 1.0


SIZES = [(75, 53, 2000), (130, 98, 3000)]


@pytest.mark.parametrize("W,H,P", SIZES, ids=[f"{w}x{h}_P{p}" for w, h, p in SIZES])
@pytest.mark.parametrize("table", [False, True], ids=["scalar", "table"])
@pytest.mark.parametrize("per_frame", [False, True], ids=["shared", "per_frame"])
@pytest.mark.parametrize("Cn", [1, 7, 16, 32])
def test_sums_equal_the_one_hot_oracle(Cn, per_frame, table, W, H, P, dev):
    T = 3
    s, means, rots, _ = _inputs(P, T, 0, per_frame, dev)
    cams = _cams(T, W, H, dev, _table(T, dev, offsets=True) if table else None)
    plain = _zeros(P, dev)
    _render(s, cams, means, rots, fpc=2, contrib=plain)
    sub = _subset(plain, P)
    planes = _planes(s, cams, means, rots, sub)
    assert (planes > 0).sum() > 0
    for kind in ("random", "negative", "seams", "subres"):
        values, B = _values(kind, T, Cn, W, H, dev, seed=Cn)
        c, lf = _zeros(P, dev), _lift(P, Cn, dev, B)
        _render(s, cams, means, rots, fpc=2, contrib=c, lift=lf, values=values)
        want, sat = _oracle(planes, values, lf.scale_log2)
        assert sat == 0 and int(lf.saturated) == 0, kind
        got = lf.sums.cpu().numpy()[sub]
        n = int((got != want).sum())
        assert n == 0, f"{kind}: {n} of {want.size} sums differ"
        assert np.abs(want).sum() > 0, kind
        _same(c, plain, f"{kind}: the statistics")


def test_ones_give_weight_q(dev):
    """v = 1 with value bound 1: every channel's sums are weight_q, bit for bit."""
    T, W, H, P = 4, 120, 90, 20_000
    s, means, rots, _ = _inputs(P, T, 0, True, dev, seed=2)
    cams = _cams(T, W, H, dev)
    c, lf = _zeros(P, dev), _lift(P, 3, dev)
    assert lf.scale_log2 == 32
    _render(s, cams, means, rots, fpc=3, contrib=c, lift=lf, values=torch.ones((T, 3, H, W), device=dev))
    assert int(c.pixels.sum()) > 0 and int(lf.saturated) == 0
    for k in range(3):
        assert torch.equal(lf.sums[:, k], c.weight_q), k
    m = lf.mean(c)
    assert bool((m[c.weight_q > 0] == 1.0).all()) and bool((m[c.weight_q == 0] == 0.0).all())


def test_background_indicator_gives_weight_bg_q(dev):
    """Lifting the indicator of the background pixels gives the masked call's weight_bg_q."""
    T, W, H, P = 4, 150, 110, 20_000
    s, means, rots, _ = _inputs(P, T, 0, True, dev, seed=3)
    cams = _cams(T, W, H, dev, _table(T, dev, offsets=True))
    for kind in ("random", "seams"):
        masks, fg = _masks(kind, T, W, H, dev)
        cm = _zeros(P, dev, silhouettes=True)
        _render(s, cams, means, rots, fpc=3, contrib=cm, masks=masks)
        c, lf = _zeros(P, dev), _lift(P, 2, dev)
        ind = torch.stack([(~fg).float(), fg.float()], 1).contiguous()
        _render(s, cams, means, rots, fpc=3, contrib=c, lift=lf, values=ind)
        assert int(cm.weight_bg_q.sum()) > 0
        assert torch.equal(lf.sums[:, 0], cm.weight_bg_q), kind
        assert torch.equal(lf.sums[:, 0] + lf.sums[:, 1], c.weight_q), kind
        _same(c, cm, kind)


@pytest.mark.parametrize("table", [False, True], ids=["scalar", "table"])
def test_nothing_else_moves(table, dev):
    """Every output -- colour with a learnable background, allmap-derived maps and radii -- and the statistics are the
    bits of the render without a lift, at every channel width."""
    T, W, H, P = 4, 120, 90, 20_000
    s, means, rots, _ = _inputs(P, T, 0, True, dev, seed=7)
    cams = _cams(T, W, H, dev, _table(T, dev, offsets=True) if table else None)
    bkgd = torch.tensor([0.25, -0.5, 0.75], device=dev)
    none = _render(s, cams, means, rots, fpc=3, bkgd=bkgd)
    c0 = _zeros(P, dev)
    plain = _render(s, cams, means, rots, fpc=3, contrib=c0, bkgd=bkgd)
    _same_outputs(plain, none, "statistics without a lift")
    for Cn in (1, 8, 9, 24, 32):
        values, B = _values("random", T, Cn, W, H, dev, seed=Cn)
        c = _zeros(P, dev)
        got = _render(s, cams, means, rots, fpc=3, contrib=c, lift=_lift(P, Cn, dev, B), values=values, bkgd=bkgd)
        _same_outputs(got, none, f"lift of {Cn} channels")
        _same(c, c0, f"lift of {Cn} channels")


def test_invariances(dev):
    """frames_per_call, frame order (the values follow their frames), several calls into one accumulator, overflow
    re-runs of single frames and repeated runs give the same bits."""
    from vidu4d_b200.renderer import BatchCameras
    T, W, H, P, Cn = 8, 150, 110, 20_000, 5
    s, means, rots, _ = _inputs(P, T, 0, True, dev, seed=4)
    cams = _cams(T, W, H, dev)
    values, B = _values("random", T, Cn, W, H, dev, seed=9)

    def run(fn):
        c, lf = _zeros(P, dev), _lift(P, Cn, dev, B)
        fn(c, lf)
        return c, lf
    rc, ref = run(lambda c, lf: _render(s, cams, means, rots, fpc=8, contrib=c, lift=lf, values=values))
    assert int(ref.sums.abs().sum()) > 0
    for fpc in (1, 3, 8):
        c, lf = run(lambda c, lf: _render(s, cams, means, rots, fpc=fpc, contrib=c, lift=lf, values=values))
        _same_lift(lf, ref, f"frames_per_call {fpc}")
        _same(c, rc, f"frames_per_call {fpc}")

    def sub(idx):
        i = torch.tensor(idx, device=dev)
        return BatchCameras(W, H, cams.FoVx, cams.FoVy, cams.world_view_transform[i].contiguous(),
                            cams.full_proj_transform[i].contiguous(), cams.camera_center[i].contiguous()), \
            means[i].contiguous(), rots[i].contiguous()
    perm = [5, 2, 7, 0, 3, 6, 1, 4]
    _, lf = run(lambda c, lf: _render(s, *sub(perm), fpc=3, contrib=c, lift=lf, values=values[perm].contiguous()))
    _same_lift(lf, ref, "permuted frames")

    def two(c, lf):
        _render(s, *sub([6, 7, 0]), fpc=2, contrib=c, lift=lf, values=values[[6, 7, 0]].contiguous())
        _render(s, *sub([1, 2, 3, 4, 5]), fpc=4, contrib=c, lift=lf, values=values[1:6].contiguous())
    _, lf = run(two)
    _same_lift(lf, ref, "two calls into one accumulator")

    # a hint far too small: the first chunk overflows, and its frames re-run alone with their own values
    holder = {}

    def overflow(c, lf):
        holder["grown"] = _with_capacity_hint(
            dev, W, H, 1, lambda: _render(s, cams, means, rots, fpc=3, contrib=c, lift=lf, values=values))[1]
    c, lf = run(overflow)
    assert holder["grown"] > 4096
    _same_lift(lf, ref, "overflow and re-run")
    _same(c, rc, "overflow and re-run")

    _, lf = run(lambda c, lf: _render(s, cams, means, rots, fpc=8, contrib=c, lift=lf, values=values))
    _same_lift(lf, ref, "second run")


def test_abi_overflowed_frame_adds_nothing(dev):
    """At the ABI an overflowed frame adds nothing to any word; re-run with room it adds what render_frames adds."""
    from vidu4d_b200 import _capi
    from vidu4d_b200 import rasterizer as RZ
    from vidu4d_b200.rasterizer import _batch_inputs
    T, W, H, P, Cn = 1, 96, 96, 20_000, 3
    s, _, _, _ = _inputs(P, T, 0, False, dev)
    cams = _cams(T, W, H, dev)
    ins, _ = _batch_inputs(T, means3D=(s["means3D"], (3,)), sh=(s["shs"], None), opacity=(s["opacities"], (1,)),
                           scales=(s["scales"], (2,)), rotations=(s["rotations"], (4,)))
    lib = _capi.load()
    color, others = torch.empty((T, 3, H, W), device=dev), torch.empty((T, 8, H, W), device=dev)
    radii = torch.empty((T, P), dtype=torch.int32, device=dev)
    fr, frp = RZ._frame(P, 3, 16, W, H, TANF, TANF, 1.0, False, False, None)
    bt = _capi.SrBatch(T, 0, 0, 0, 0, 0, 0, 0)
    values, B = _values("random", T, Cn, W, H, dev)
    values[0, 0, 40:56, 40:56] = float("nan")           # the centre, where the scene is

    def call(cap, c, lf):
        arena = torch.empty((int(lib.sr_render_bytes(P, cap, W, H)),), dtype=torch.uint8, device=dev)
        nr = torch.zeros((T, 2), dtype=torch.int32, device=dev)
        host = torch.zeros((T, 2), dtype=torch.int32, pin_memory=True)
        ct = _capi.SrContrib(c.weight_q.data_ptr(), c.max_weight.data_ptr(), c.pixels.data_ptr())
        sl = _capi.SrLift(values.data_ptr(), Cn, Cn * W * H, lf.scale_log2, lf.sums.data_ptr(), lf.saturated.data_ptr())
        _capi.call("sr_render_forward_lift", dev, frp, C.byref(bt), torch.tensor([0.1, 0.2, 0.3], device=dev), 3,
                   ins["means3D"], ins["sh"], None, ins["opacity"], ins["scales"], ins["rotations"], None, 0, 0,
                   cams.world_view_transform, cams.full_proj_transform, cams.camera_center, color, 0, None, 0, others,
                   radii, arena, cap, nr, host, C.byref(ct), C.byref(sl))
        torch.cuda.synchronize()
        return host

    c, lf = _zeros(P, dev), _lift(P, Cn, dev, B)
    host = call(4096, c, lf)
    assert int(host[0, 1]) & _capi.SR_STATUS_OVERFLOW and int(host[0, 0]) > 4096
    for name in WORDS[:3]:
        assert int(getattr(c, name).abs().sum()) == 0, name
    assert int(lf.sums.abs().sum()) == 0 and int(lf.saturated) == 0
    call(RZ._round_cap(int(host[0, 0]) + 4096), c, lf)
    rc, ref = _zeros(P, dev), _lift(P, Cn, dev, B)
    _render(s, cams, None, None, contrib=rc, lift=ref, values=values)
    _same(c, rc, "overflow then re-run at the ABI", WORDS[:3])
    _same_lift(lf, ref, "overflow then re-run at the ABI")
    assert int(ref.saturated) > 0


def test_saturation_is_counted_and_clamped(dev):
    """Non-finite values contribute 0 and values beyond the bound are clamped to +-2^32, each (pair, channel) term
    counted once in `saturated`; the oracle follows the same rule, so every sum of the subset is still exact, and so is
    every sum of a surfel that never lands on the bad pixels."""
    T, W, H, P, Cn = 2, 130, 98, 3000, 6
    s, means, rots, _ = _inputs(P, T, 0, True, dev, seed=5)
    cams = _cams(T, W, H, dev)
    values, B = _values("random", T, Cn, W, H, dev, seed=1)          # within B = 4
    bad = torch.zeros((H, W), dtype=torch.bool, device=dev)
    bad[:, : W // 2] = True                                            # the left half of every frame
    y = torch.arange(H, device=dev)[:, None].expand(H, W)
    vals = values.clone()
    vals[:, 0][:, bad] = float("nan")
    vals[:, 1][:, bad] = torch.where(y[bad] % 2 == 0, float("inf"), float("-inf"))
    vals[:, 2][:, bad] = 1e30
    vals[:, 3][:, bad] = -1e30
    vals[:, 4][:, bad] = 4.0                                            # exactly B: never clamped
    cm = _zeros(P, dev, silhouettes=True)
    _render(s, cams, means, rots, contrib=cm, masks=~bad.expand(T, H, W))
    c, lf = _zeros(P, dev), _lift(P, Cn, dev, B)
    _render(s, cams, means, rots, contrib=c, lift=lf, values=vals)
    _same(c, cm, "statistics")
    # channels 0..3 saturate on every pair of a left-half pixel, channels 4 and 5 never
    left_pairs = int(cm.pixels_bg.sum())
    assert left_pairs > 0 and int(lf.saturated) == 4 * left_pairs
    sub = _subset(c, P)
    planes = _planes(s, cams, means, rots, sub)
    want, want_sat = _oracle(planes, vals, lf.scale_log2)
    got = lf.sums.cpu().numpy()[sub]
    assert int((got != want).sum()) == 0 and want_sat == 4 * int(cm.pixels_bg[torch.from_numpy(sub).to(dev)].sum())
    # channel 2 is clamped to +2^32 on every left pair: the surfels that land only there sum pixels_bg 2^32
    only_left = (cm.pixels_bg == cm.pixels) & (cm.pixels > 0)
    assert int(only_left.sum()) > 0
    assert torch.equal(lf.sums[only_left, 2], cm.pixels_bg[only_left] * 2 ** 32)
    assert torch.equal(lf.sums[only_left, 3], cm.pixels_bg[only_left] * -(2 ** 32))
    assert bool((lf.sums[only_left, 0] == 0).all()) and bool((lf.sums[only_left, 1] == 0).all())
    # a surfel that never lands on the left half has the sums of the clean values
    c2, clean = _zeros(P, dev), _lift(P, Cn, dev, B)
    _render(s, cams, means, rots, contrib=c2, lift=clean, values=values)
    right = cm.pixels_bg == 0
    assert int((right & (cm.pixels > 0)).sum()) > 0
    assert torch.equal(lf.sums[right], clean.sums[right])
    assert int(clean.saturated) == 0


@pytest.mark.parametrize("case", ["empty", "culled"])
def test_empty_and_culled(case, dev):
    T, W, H, Cn = 3, 64, 48, 4
    P = 0 if case == "empty" else 5000
    s, _, _, _ = _inputs(max(P, 1), T, 0, False, dev)
    if P == 0:
        s = {k: v[:0] for k, v in s.items()}
    cams = _cams(T, W, H, dev)
    means = None
    if case == "culled":
        means = (2 * cams.camera_center[:, None, :] - s["means3D"][None]).contiguous()   # behind every camera
    c, lf = _zeros(P, dev), _lift(P, Cn, dev)
    out = _render(s, cams, means, None, contrib=c, lift=lf, values=torch.ones((T, Cn, H, W), device=dev))
    assert int((out["radii"] > 0).sum()) == 0
    assert lf.sums.shape == (P, Cn) and int(lf.sums.abs().sum()) == 0 and int(lf.saturated) == 0
    for name in WORDS:
        assert int(getattr(c, name).abs().sum()) == 0, name
    assert lf.mean(c).shape == (P, Cn) and int((lf.mean(c) != 0).sum()) == 0


def test_label_maps_give_each_surfel_its_side(dev):
    """A two-part object, left and right of a gap, seen by front cameras; per-pixel label maps (one-hot, from which part
    covers the pixel, 0 where neither does) lifted onto the surfels: mean() gives every blended surfel its own part's
    label."""
    from vidu4d_b200.renderer import PipelineParams, SurfelLift, render_frames
    T, W, H = 4, 96, 80
    g = torch.Generator().manual_seed(5)
    n = 300
    xy = (torch.rand((2 * n, 2), generator=g) - 0.5) * torch.tensor([0.3, 0.8])
    xy[:n, 0] -= 0.25                                                   # left part: x in [-0.4, -0.1]
    xy[n:, 0] += 0.25                                                   # right part: x in [0.1, 0.4]
    xyz = torch.cat([xy, 1.5 + 0.05 * torch.rand((2 * n, 1), generator=g)], 1)
    scale = torch.full((2 * n, 2), 0.015)
    op = torch.full((2 * n, 1), 0.8)
    cams = _front_cams(T, W, H, dev)
    pipe, bg = PipelineParams(), torch.zeros(3, device=dev)
    cover = [render_frames(cams, _model(xyz[k * n:(k + 1) * n], scale[:n], op[:n], dev), pipe, bg)["acc"][:, 0] > 0
             for k in (0, 1)]
    assert not bool((cover[0] & cover[1]).any()) and int(cover[0].sum()) > 0 and int(cover[1].sum()) > 0
    labels = torch.stack([cover[0], cover[1]], 1).float().contiguous()  # (T, 2, H, W)
    m = _model(xyz, scale, op, dev)
    c, lf = _zeros(m.P, dev), SurfelLift.zeros(m.P, 2, dev)
    render_frames(cams, m, pipe, bg, contributions=c, lift=lf, values=labels)
    mean = lf.mean(c)
    seen = c.pixels > 0
    assert int(seen.sum()) > 1.9 * n
    side = torch.cat([torch.zeros(n, dtype=torch.long), torch.ones(n, dtype=torch.long)]).to(dev)
    assert torch.equal(mean.argmax(1)[seen], side[seen])
    assert bool((mean[seen].gather(1, side[seen][:, None]) > 0.5).all())
    assert bool((mean[seen].gather(1, 1 - side[seen][:, None]) == 0).all())
    assert int(lf.saturated) == 0
