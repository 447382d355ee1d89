"""GPU: pixel anchors (render_frames(..., anchors=K), sr_render_forward_anchors) and tracking on them (track_pixels).

The anchors' oracle is test_gpu_lift's: with one-hot features, plane k of the render is surfel k's per-pixel weight
w = T alpha exactly, so a pixel's slots must hold, bit for bit, the K largest of its planes' positive values.  Tracking is
held to tests/track_model.py's float64 model under its rounding-error bound."""
import math

import numpy as np
import pytest
import torch

from .test_gpu_contrib import _PC, _same_outputs
from .test_gpu_render import _cams, _inputs, _table
from .track_model import track, within

pytestmark = pytest.mark.gpu

ANCHOR_KEYS = ("anchor_ids", "anchor_weights", "anchor_uv")


@pytest.fixture(scope="module")
def dev(built):
    from vidu4d_b200 import _capi
    _capi.load()
    return torch.device("cuda:0")


def _render(s, cams, means, rots, anchors=None, feat=None, fpc=8, bkgd=None, contrib=None):
    from vidu4d_b200.renderer import PipelineParams, render_frames
    d = s["means3D"].device
    return render_frames(cams, _PC(s), PipelineParams(depth_ratio=0.37), torch.tensor([0.1, 0.2, 0.3], device=d),
                         means3D=means, rotations=rots, features=feat, learnable_bkgd=bkgd, frames_per_call=fpc,
                         anchors=anchors, contributions=contrib)


def _bits(a, b, what):
    x, y = a.contiguous().view(torch.int32), b.contiguous().view(torch.int32)
    n = int((x != y).sum())
    assert n == 0, f"{what}: differs in {n} of {x.numel()} elements"


def _planes(s, cams, means, rots):
    """(T, P, H, W) float32: plane i is surfel i's per-pixel weight, from one-hot features 32 surfels at a time."""
    P = int(s["means3D"].shape[0])
    d = s["means3D"].device
    out = []
    for lo in range(0, P, 32):
        hi = min(P, lo + 32)
        feat = torch.zeros((P, 32), device=d)
        feat[torch.arange(lo, hi, device=d), torch.arange(hi - lo, device=d)] = 1.0
        out.append(_render(s, cams, means, rots, feat=feat)["features"][:, :hi - lo])
    return torch.cat(out, 1).cpu().numpy()


def _sparse_scene(dev, seed=0):
    """Small discs on two jittered grid layers in front of the orbit camera of frame 0: no pixel has more than a few
    contributors, so K = 8 captures every one of them."""
    from vidu4d_b200.synthetic import orbit_view
    rng = np.random.default_rng(seed)
    R, t = orbit_view(0, 64)
    pts = []
    for z, off in ((1.0, 0.0), (1.1, 0.03)):
        g = np.arange(-0.28, 0.29, 0.06)
        x, y = np.meshgrid(g + off, g + off)
        pc = np.stack([x.ravel(), y.ravel(), np.full(x.size, z)], 1) + rng.normal(0, 0.004, (x.size, 3))
        pts.append(pc)
    pc = np.concatenate(pts)
    P = len(pc)
    world = (pc - t[None]) @ R                                          # R^T (x_c - t)
    from scipy.spatial.transform import Rotation
    q = Rotation.from_matrix(R.T).as_quat()                             # (x, y, z, w): the disc faces the camera
    quat = np.tile(np.array([q[3], q[0], q[1], q[2]]), (P, 1)) + rng.normal(0, 0.05, (P, 4))
    quat /= np.linalg.norm(quat, axis=1, keepdims=True)
    f = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(dev)   # noqa: E731
    shs = np.zeros((P, 16, 3), np.float32)
    shs[:, 0] = rng.uniform(-1, 1, (P, 3))
    return {"means3D": f(world), "rotations": f(quat), "scales": f(rng.uniform(0.008, 0.014, (P, 2))),
            "opacities": f(rng.uniform(0.3, 0.8, (P, 1))), "shs": f(shs)}


@pytest.mark.parametrize("table", [False, True], ids=["scalar", "table"])
@pytest.mark.parametrize("per_frame", [False, True], ids=["shared", "per_frame"])
def test_outputs_unchanged_and_anchors_independent_of_chunking(per_frame, table, dev):
    """Colour (with a learnable background), the allmap maps and radii have the bits of the render without anchors, for
    K = 1, 2, 4, 8 and frames_per_call 1, 3, 8; the anchors have the same bits for every frames_per_call."""
    T, W, H, P = 8, 75, 53, 3000
    s, means, rots, _ = _inputs(P, T, 0, per_frame, dev, seed=3)
    cams = _cams(T, W, H, dev, _table(T, dev, offsets=True) if table else None)
    bkgd = torch.tensor([0.25, -0.5, 0.75], device=dev)
    none = _render(s, cams, means, rots, bkgd=bkgd)
    for K in (1, 2, 4, 8):
        first = None
        for fpc in (1, 3, 8):
            got = _render(s, cams, means, rots, anchors=K, fpc=fpc, bkgd=bkgd)
            _same_outputs(got, none, f"K = {K}, frames_per_call = {fpc}")
            assert got["anchor_ids"].shape == (T, K, H, W) and got["anchor_ids"].dtype == torch.int32
            assert got["anchor_weights"].shape == (T, K, H, W) and got["anchor_uv"].shape == (T, K, 2, H, W)
            if first is None:
                first = got
                assert int((got["anchor_ids"][:, 0] >= 0).sum()) > 0
            for k in ANCHOR_KEYS:
                _bits(got[k], first[k], f"{k}, K = {K}, frames_per_call = {fpc}")


@pytest.mark.parametrize("per_frame", [False, True], ids=["shared", "per_frame"])
def test_slots_hold_the_heaviest_one_hot_weights(per_frame, dev):
    """Over every P of a small scene: each filled slot's weight is its surfel's feature plane at the pixel, bit for bit;
    the slots hold the K largest weights in descending order; a pixel with n contributors fills min(n, K) slots and the
    rest are empty (id -1, w 0, uv (0, 0)); the surfels of a pixel's slots are distinct."""
    T, W, H, P = 2, 48, 40, 96
    s, means, rots, _ = _inputs(P, T, 0, per_frame, dev, seed=5)
    cams = _cams(T, W, H, dev)
    planes = _planes(s, cams, means, rots)                               # (T, P, H, W)
    n = (planes > 0).sum(1)                                              # (T, H, W)
    assert n.max() >= 3
    top = -np.sort(-planes, axis=1)                                      # descending, per pixel
    for K in (1, 2, 4, 8):
        a = _render(s, cams, means, rots, anchors=K)
        ids, w, uv = (a[k].cpu().numpy() for k in ANCHOR_KEYS)
        filled = ids >= 0
        assert np.array_equal(filled.sum(1), np.minimum(n, K))
        assert np.array_equal(w.view(np.int32), top[:, :K].view(np.int32)), f"K = {K}: slot weights"
        g = np.take_along_axis(planes, np.where(filled, ids, 0), axis=1)
        assert np.array_equal(np.where(filled, g, 0).view(np.int32), w.view(np.int32)), f"K = {K}: surfel planes"
        assert np.all(uv[:, :, 0][~filled] == 0) and np.all(uv[:, :, 1][~filled] == 0)
        srt = np.sort(np.where(filled, ids, -1 - np.arange(K)[None, :, None, None]), axis=1)
        assert np.all(np.diff(srt, axis=1) != 0), f"K = {K}: a surfel fills two slots"


def test_slot_sums_are_the_contribution_statistics(dev):
    """Where no pixel has more than K - 1 contributors (K = 8: the last slot is empty everywhere), summing
    rn(w 2^32), the count and the max over the slots, per surfel, gives SurfelContributions' weight_q, pixels and
    max_weight bit for bit."""
    from vidu4d_b200.renderer import SurfelContributions
    s = _sparse_scene(dev)
    P = int(s["means3D"].shape[0])
    T, W, H = 3, 96, 80
    cams = _cams(T, W, H, dev, first=0)
    a = _render(s, cams, None, None, anchors=8)
    ids, w = a["anchor_ids"], a["anchor_weights"]
    assert int((ids[:, 7] >= 0).sum()) == 0, "a pixel fills every slot: the scene is not sparse enough"
    assert int((ids[:, 1] >= 0).sum()) > 0
    c = SurfelContributions.zeros(P, dev)
    _render(s, cams, None, None, contrib=c)
    on = ids >= 0
    idl = ids[on].long().cpu().numpy()
    wl = w[on].cpu().numpy()
    q = np.rint(wl.astype(np.float64) * 2.0 ** 32).astype(np.int64)
    wq = np.zeros(P, np.int64)
    np.add.at(wq, idl, q)
    px = np.bincount(idl, minlength=P)
    mx = np.zeros(P, np.float32)
    np.maximum.at(mx, idl, wl)
    assert np.array_equal(c.weight_q.cpu().numpy().astype(np.int64), wq)
    assert np.array_equal(c.pixels.cpu().numpy().astype(np.int64), px)
    assert np.array_equal(c.max_weight.cpu().numpy().view(np.int32), mx.view(np.int32))


def _world_points(s, ids, uv, means=None, rots=None, frame=0):
    """float64 (.., 3) surface points mean + u s_u t_u + v s_v t_v of the slots, with the surfels of `frame`."""
    from scipy.spatial.transform import Rotation
    mu = (s["means3D"] if means is None else means[frame]).double().cpu().numpy()
    q = (s["rotations"] if rots is None else rots[frame]).double().cpu().numpy()
    Rm = Rotation.from_quat(q[:, [1, 2, 3, 0]]).as_matrix()            # columns: t_u, t_v, normal
    sc = s["scales"].double().cpu().numpy()
    i = np.where(ids >= 0, ids, 0)
    u, v = uv[..., 0, :, :], uv[..., 1, :, :]
    return (mu[i] + (u * sc[i][..., 0])[..., None] * Rm[i][..., :, 0] + (v * sc[i][..., 1])[..., None] * Rm[i][..., :, 1])


def _project(X, cam, t, W, H):
    """float64 pixel coordinates and depth of world points X (.., 3) through frame t of a scalar-tangent BatchCamera."""
    vm = cam.world_view_transform[t].double().cpu().numpy()             # W2C transposed
    Xc = X @ vm[:3, :3] + vm[3, :3]
    f = W / (2.0 * math.tan(cam.FoVx * 0.5)), H / (2.0 * math.tan(cam.FoVy * 0.5))
    return f[0] * Xc[..., 0] / Xc[..., 2] + W / 2.0, f[1] * Xc[..., 1] / Xc[..., 2] + H / 2.0, Xc[..., 2]


def test_hit_points_lie_on_the_pixel_and_blend_to_the_depth_plane(dev):
    """Each disc-branch hit point projects back onto its pixel's centre, and where every contributor is captured the
    slots' weighted depth, divided by their weight, is render_depth_expected."""
    s = _sparse_scene(dev, seed=1)
    T, W, H = 2, 96, 80
    cams = _cams(T, W, H, dev)
    a = _render(s, cams, None, None, anchors=8)
    ids, w, uv = (a[k].cpu().numpy() for k in ANCHOR_KEYS)
    X = _world_points(s, ids, uv.astype(np.float64))
    for t in range(T):
        x, y, z = _project(X[t], cams, t, W, H)
        disc = (ids[t] >= 0) & ((uv[t, :, 0] != 0) | (uv[t, :, 1] != 0))
        yy, xx = np.meshgrid(np.arange(H) + 0.5, np.arange(W) + 0.5, indexing="ij")
        assert disc.sum() > 100
        err = np.maximum(np.abs(x - xx[None]), np.abs(y - yy[None]))[disc]
        assert err.max() < 2e-3, err.max()
        cov = (w[t] * (ids[t] >= 0)).sum(0)
        zd = (w[t] * np.where(ids[t] >= 0, z, 0)).sum(0)
        ex = a["render_depth_expected"][t, 0].cpu().numpy()
        on = cov > 0
        assert np.all(np.abs(zd[on] / cov[on] - ex[on]) <= 1e-4 * np.abs(ex[on]) + 1e-6)


def _queries(a, s_frame=0):
    ids = a["anchor_ids"]
    T, K, H, W = ids.shape
    yy, xx = torch.meshgrid(torch.arange(H, device=ids.device), torch.arange(W, device=ids.device), indexing="ij")
    return torch.stack([torch.full_like(xx, s_frame), xx, yy], -1).reshape(-1, 3).int().contiguous()


def _track(a, q, cams, s, means=None, rots=None, depth=None, tol=0.05):
    from vidu4d_b200.tracking import track_pixels
    return track_pixels(tuple(a[k] for k in ANCHOR_KEYS), q, cams, _PC(s), means3D=means, rotations=rots, depth=depth,
                        depth_tolerance=tol)


@pytest.mark.parametrize("table", [False, True], ids=["scalar", "table"])
@pytest.mark.parametrize("K", [1, 4, 8])
def test_tracking_matches_the_float64_model(K, table, dev):
    T, W, H, P = 3, 64, 48, 4000
    s, means, rots, _ = _inputs(P, T, 0, True, dev, seed=11)
    tab = _table(T, dev, offsets=True) if table else None
    cams = _cams(T, W, H, dev, tab)
    a = _render(s, cams, means, rots, anchors=K)
    q = torch.cat([_queries(a, 0), _queries(a, 2)[::7]]).contiguous()
    got = _track(a, q, cams, s, means, rots)
    npy = lambda t: t.cpu().numpy()                                      # noqa: E731
    from vidu4d_b200.renderer import _cam_tans
    m = track(npy(a["anchor_ids"]), npy(a["anchor_weights"]), npy(a["anchor_uv"]), npy(q), npy(means), npy(rots),
              npy(s["scales"]), npy(cams.world_view_transform).reshape(T, 16), W, H,
              tans=None if table else _cam_tans(cams), table=None if tab is None else npy(tab))
    valid = m["valid"]
    assert valid.sum() > 500
    cov = npy(got["coverage"])
    assert np.all(cov[~valid] == 0) and np.all(within(cov[valid], m["coverage"][valid]))
    xy, z = npy(got["xy"]), npy(got["z"])
    assert np.all(np.isnan(xy[~valid])) and np.all(np.isnan(z[~valid])) and not npy(got["visible"])[~valid].any()
    for name, g in (("x", xy[..., 0]), ("y", xy[..., 1]), ("z", z)):
        ok = within(g[valid], m[name][valid])
        assert ok.all(), f"{name}: {int((~ok).sum())} of {ok.size} outside the bound"
    vis = npy(got["visible"])[valid]
    inside = (m["z"].v[valid] >= 0.2) & (m["x"].v[valid] >= 0) & (m["x"].v[valid] < W) & (m["y"].v[valid] >= 0) \
        & (m["y"].v[valid] < H)
    knife = (np.abs(m["x"].v[valid]) < 1e-3) | (np.abs(m["x"].v[valid] - W) < 1e-3) | (np.abs(m["y"].v[valid]) < 1e-3) \
        | (np.abs(m["y"].v[valid] - H) < 1e-3)
    assert np.array_equal(vis[~knife], inside[~knife])


def test_tracking_into_the_source_frame_returns_pixel_centres(dev):
    """A query followed into its own frame with its own surfels lands on its pixel's centre: every hit point lies on the
    pixel's ray, and so does their weighted mean.  Queries with a slot on the screen-space filter branch (which stores
    the centre) are left out."""
    T, W, H, P = 2, 64, 48, 4000
    s, means, rots, _ = _inputs(P, T, 0, True, dev, seed=13)
    cams = _cams(T, W, H, dev)
    a = _render(s, cams, means, rots, anchors=4)
    for sf in range(T):
        q = _queries(a, sf)
        got = _track(a, q, cams, s, means, rots)
        ids, uv = a["anchor_ids"][sf], a["anchor_uv"][sf]
        disc = ((ids < 0) | (uv[:, 0] != 0) | (uv[:, 1] != 0)).all(0).reshape(-1) & (got["coverage"] > 0)
        assert int(disc.sum()) > 500
        c = q[:, 1:].float() + 0.5
        err = (got["xy"][:, sf] - c).abs().amax(-1)[disc]
        assert float(err.max()) < 2e-3, float(err.max())
        assert bool(got["visible"][:, sf][disc].all())


def _quat_mul(a, b):
    w1, x1, y1, z1 = a.unbind(-1)
    w2, x2, y2, z2 = b.unbind(-1)
    return torch.stack([w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2, w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2,
                        w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2, w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2], -1)


def test_rigid_motion_moves_the_tracks_analytically(dev):
    """Every surfel of frame t is frame 0's, rotated by R_t about the object's centre and shifted by c_t; one camera
    sees all frames.  A frame-0 pixel's track into frame t is the projection of R_t X_0 + c_t."""
    T, W, H, P = 4, 64, 48, 4000
    s, _, _, _ = _inputs(P, T, 0, False, dev, seed=17)
    cam1 = _cams(1, W, H, dev)
    cams = type(cam1)(W, H, cam1.FoVx, cam1.FoVy, cam1.world_view_transform.expand(T, 4, 4).contiguous(),
                      cam1.full_proj_transform.expand(T, 4, 4).contiguous(), cam1.camera_center.expand(T, 3).contiguous(),
                      None)
    mus, qs, Rs, cs = [], [], [], []
    for t in range(T):
        ang = 0.05 * t
        Rt = torch.tensor([[math.cos(ang), 0, math.sin(ang)], [0, 1, 0], [-math.sin(ang), 0, math.cos(ang)]],
                          dtype=torch.float64, device=dev)
        ct = torch.tensor([0.01 * t, -0.005 * t, 0.0], dtype=torch.float64, device=dev)
        qt = torch.tensor([math.cos(ang / 2), 0.0, math.sin(ang / 2), 0.0], dtype=torch.float64, device=dev)
        mus.append((s["means3D"].double() @ Rt.T + ct).float())
        qs.append(_quat_mul(qt.expand(P, 4), s["rotations"].double()).float())
        Rs.append(Rt.cpu().numpy()), cs.append(ct.cpu().numpy())
    means, rots = torch.stack(mus).contiguous(), torch.stack(qs).contiguous()
    a = _render(s, cams, means, rots, anchors=4)
    q = _queries(a, 0)
    got = _track(a, q, cams, s, means, rots)
    on = (got["coverage"] > 0).cpu().numpy()
    assert on.sum() > 500
    ids, uv = a["anchor_ids"][0].cpu().numpy(), a["anchor_uv"][0].cpu().numpy().astype(np.float64)
    w = a["anchor_weights"][0].cpu().numpy().astype(np.float64) * (ids >= 0)
    X0 = _world_points(s, ids, uv, means, rots, 0)                      # (K, H, W, 3)
    X0 = (w[..., None] * X0).sum(0) / np.maximum(w.sum(0), 1e-30)[..., None]
    X0 = X0.reshape(-1, 3)[on]
    xy = got["xy"].cpu().numpy()[on]
    for t in range(T):
        x, y, _ = _project(X0 @ Rs[t].T + cs[t], cams, t, W, H)
        err = np.maximum(np.abs(xy[:, t, 0] - x), np.abs(xy[:, t, 1] - y))
        assert err.max() < 2e-3, (t, err.max())


def test_an_occluding_wall_hides_the_tracks_behind_it(dev):
    """Frame 1 puts an opaque wall in front of the left half of the object; frame 0 keeps it behind the camera.  With
    frame 1's surf_depth, the frame-0 pixels whose tracks land behind the wall are not visible, though they are without
    the depth test; right of the wall, visibility is what it is when the wall stays behind the camera in both frames."""
    from scipy.spatial.transform import Rotation
    from vidu4d_b200.synthetic import orbit_view
    T, W, H, P = 2, 64, 48, 4000
    s, _, _, _ = _inputs(P, T, 0, False, dev, seed=19)
    cams = _cams(1, W, H, dev)
    cams = type(cams)(W, H, cams.FoVx, cams.FoVy, cams.world_view_transform.expand(T, 4, 4).contiguous(),
                      cams.full_proj_transform.expand(T, 4, 4).contiguous(), cams.camera_center.expand(T, 3).contiguous(),
                      None)
    R, t = orbit_view(0, 64)
    g = np.arange(-0.4, 0.0, 0.01)
    x, y = np.meshgrid(g, np.arange(-0.4, 0.41, 0.01))
    wc = np.stack([x.ravel(), y.ravel(), np.full(x.size, 0.5)], 1)
    Pw = len(wc)
    q = Rotation.from_matrix(R.T).as_quat()
    wall = {"means3D": (wc - t[None]) @ R, "behind": (wc * [1, 1, -1] - t[None]) @ R,
            "rot": np.tile([q[3], q[0], q[1], q[2]], (Pw, 1))}
    f = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(dev)   # noqa: E731
    s2 = {"means3D": torch.cat([s["means3D"], f(wall["means3D"])]),
          "rotations": torch.cat([s["rotations"], f(wall["rot"])]),
          "scales": torch.cat([s["scales"], torch.full((Pw, 2), 0.012, device=dev)]),
          "opacities": torch.cat([s["opacities"], torch.full((Pw, 1), 0.99, device=dev)]),
          "shs": torch.cat([s["shs"], torch.zeros((Pw,) + tuple(s["shs"].shape[1:]), device=dev)])}
    means = torch.stack([torch.cat([s["means3D"], f(wall["behind"])]), s2["means3D"]]).contiguous()
    a = _render(s2, cams, means, None, anchors=4)
    depth = a["surf_depth"][:, 0].contiguous()
    qq = _queries(a, 0)
    with_d = _track(a, qq, cams, s2, means, None, depth=depth)
    no_d = _track(a, qq, cams, s2, means, None)
    on = with_d["coverage"] > 0
    xs = with_d["xy"][:, 1, 0]
    left, right = on & (xs < W / 2 - 3), on & (xs > W / 2 + 3)
    assert int(left.sum()) > 100 and int(right.sum()) > 100
    assert not bool(with_d["visible"][:, 1][left].any())
    assert bool(no_d["visible"][:, 1][left].all())
    m0 = torch.stack([means[0], means[0]]).contiguous()
    a0 = _render(s2, cams, m0, None, anchors=4)
    ref = _track(a0, qq, cams, s2, m0, None, depth=a0["surf_depth"][:, 0].contiguous())
    right = right & (xs > W / 2 + 8)
    assert int(right.sum()) > 50 and float(ref["visible"][:, 1][on].float().mean()) > 0.5
    assert float((with_d["visible"][:, 1][right] == ref["visible"][:, 1][right]).float().mean()) > 0.95


def test_guarded_queries(dev):
    """Background pixels, frames and pixels out of range and ids >= P give coverage 0, NaN and not visible; P = 0
    renders empty slots."""
    T, W, H, P = 2, 64, 48, 2000
    s, means, rots, _ = _inputs(P, T, 0, True, dev, seed=23)
    cams = _cams(T, W, H, dev)
    a = _render(s, cams, means, rots, anchors=2)
    bg = (a["anchor_ids"][0, 0] < 0).nonzero()
    assert bg.shape[0] > 0
    fg = (a["anchor_ids"][0, 0] >= 0).nonzero()[:3]
    q = torch.cat([torch.stack([torch.zeros_like(bg[:, 0]), bg[:, 1], bg[:, 0]], 1),
                   torch.tensor([[2, 1, 1], [-1, 1, 1], [0, W, 0], [0, 0, H], [0, -1, 0]], device=dev),
                   torch.stack([torch.zeros_like(fg[:, 0]), fg[:, 1], fg[:, 0]], 1)]).int().contiguous()
    got = _track(a, q, cams, s, means, rots)
    n = q.shape[0] - fg.shape[0]
    assert bool((got["coverage"][:n] == 0).all()) and bool(torch.isnan(got["xy"][:n]).all())
    assert bool(torch.isnan(got["z"][:n]).all()) and not bool(got["visible"][:n].any())
    assert bool((got["coverage"][n:] > 0).all())
    bad = {k: a[k].clone() for k in ANCHOR_KEYS}
    bad["anchor_ids"][0, 1] = torch.where(bad["anchor_ids"][0, 1] >= 0, P, -1)
    got = _track(bad, q[n:], cams, s, means, rots)
    two = (a["anchor_ids"][0, 1][fg[:, 0], fg[:, 1]] >= 0)
    assert bool((got["coverage"][two] == 0).all()) and bool(torch.isnan(got["xy"][two]).all())
    e = {k: torch.empty((0,) + tuple(v.shape[1:]), device=dev, dtype=v.dtype) for k, v in s.items()}
    z = _render(e, cams, means[:, :0].contiguous(), rots[:, :0].contiguous(), anchors=4)
    assert bool((z["anchor_ids"] == -1).all()) and bool((z["anchor_weights"] == 0).all())
    assert bool((z["anchor_uv"] == 0).all())
    got = _track(z, q[n:], cams, e, means[:, :0].contiguous(), rots[:, :0].contiguous())
    assert bool((got["coverage"] == 0).all()) and bool(torch.isnan(got["xy"]).all())


def test_overflowed_chunk_reruns_with_the_same_anchors(dev):
    """A chunk that overflows the instance buffer re-runs whole with a larger one; its anchors and outputs are those of
    a render that never overflowed."""
    from .test_gpu_contrib import _with_capacity_hint
    T, W, H, P = 4, 75, 53, 3000
    s, means, rots, _ = _inputs(P, T, 0, True, dev, seed=29)
    cams = _cams(T, W, H, dev)
    ref = _render(s, cams, means, rots, anchors=4, fpc=4)
    got, grown = _with_capacity_hint(dev, W, H, 64, lambda: _render(s, cams, means, rots, anchors=4, fpc=4))
    assert grown > 64
    _same_outputs(got, ref, "after an overflow")
    for k in ANCHOR_KEYS:
        _bits(got[k], ref[k], f"{k} after an overflow")
