"""GPU tests of the frame-looped forward preprocess: one thread runs one surfel through every frame of a batch, reading
the inputs the frames share once.  Each frame of a batched call must equal a single-frame call on the same inputs bit
for bit -- radii, the surfel record / depth / tiles_touched / clamped bits the preprocess writes, the number of
instances, the sorted keys and surfel list, and the colour -- for shared and per-frame inputs, precomputed colours,
every SH degree, block-edge surfel counts, a frame that sees no surfel, and the `prefiltered` status bit."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

W, H = 96, 64
DEGREE_OF = {1: 0, 4: 1, 9: 2, 16: 3}


@pytest.fixture(scope="module")
def dev(built):
    from vidu4d_b200 import _capi
    _capi.load()
    return torch.device("cuda:0")


def _cams(M, dev, empty=()):
    """Orbiting cameras; a frame in `empty` is moved so that every surfel lies behind it."""
    from vidu4d_b200.synthetic import orbit_view, projection_matrix
    Pm = projection_matrix(0.5, 0.5).astype(np.float64)
    vms, pms, cps = [], [], []
    for f in range(M):
        R, t = orbit_view(5 * f + 2, 64)
        if f in empty:
            t = t - np.array([0.0, 0.0, 6.0])
        W2C = np.eye(4); W2C[:3, :3] = R; W2C[:3, 3] = t
        vms.append(W2C.T.astype(np.float32)); pms.append((W2C.T @ Pm).astype(np.float32)); cps.append((-R.T @ t).astype(np.float32))
    return tuple(torch.from_numpy(np.stack(a)).to(dev) for a in (vms, pms, cps))


def _inputs(P, K, M, dev, per_frame=(), seed=3):
    """Surfels of a sphere about the origin with K SH coefficients; each name in `per_frame` gets its own copy per frame."""
    from vidu4d_b200.synthetic import object_scene
    t = object_scene(P, seed=seed, center=(0.0, 0.0, 0.0)).to_torch(dev)
    ins = {"means3D": t["means3D"], "opacities": t["opacities"], "scales": t["scales"], "rotations": t["rotations"],
           "shs": t["shs"][:, :K].contiguous(), "colors": torch.rand((P, 3), device=dev, generator=torch.Generator(device=dev).manual_seed(seed))}
    g = torch.Generator(device=dev).manual_seed(seed + 1)
    ins["per_frame"] = set(per_frame)
    for n in per_frame:
        x = ins[n]
        noise = [0.02 * f * torch.randn(x.shape, device=dev, generator=g) for f in range(M)]
        if n == "rotations":
            ins[n] = torch.stack([torch.nn.functional.normalize(x + d) for d in noise])
        elif n == "opacities":
            ins[n] = torch.stack([(x + d).clamp(0.0, 1.0) for d in noise])
        elif n == "scales":
            ins[n] = torch.stack([x * (1.0 + d).abs() for d in noise])
        else:
            ins[n] = torch.stack([x + d for d in noise])
    return ins


def _frame(ins, name, f):
    return ins[name][f] if name in ins["per_frame"] else ins[name]


def _run(ins, K, vms, pms, cps, precomp, prefiltered=False):
    from vidu4d_b200 import rasterizer as RZ
    dev = vms.device
    e = torch.empty((0,), device=dev)
    bg = torch.tensor([0.2, 0.1, 0.4], device=dev)
    colors, shs = (ins["colors"], e) if precomp else (e, ins["shs"])
    C = RZ._C
    batch = C.rasterize_gaussians_batch(bg, ins["means3D"], colors, ins["opacities"], ins["scales"], ins["rotations"], 1.0, vms, pms,
                                        0.5, 0.5, H, W, shs, DEGREE_OF[K], cps, prefiltered=prefiltered)
    singles = []
    for f in range(vms.shape[0]):
        singles.append(C.rasterize_gaussians(bg, _frame(ins, "means3D", f), _frame(ins, "colors", f) if precomp else e,
                                             _frame(ins, "opacities", f), _frame(ins, "scales", f), _frame(ins, "rotations", f), 1.0, e,
                                             vms[f], pms[f], 0.5, 0.5, H, W, e if precomp else _frame(ins, "shs", f), DEGREE_OF[K],
                                             cps[f], prefiltered, False))
    return batch, singles


def _check(batch, singles, P):
    from vidu4d_b200.debug import decode
    nr, color, allmap, radii, gb, bb, ib = batch
    M = len(singles)
    assert len(nr) == M and radii.shape == (M, P)
    for f, o in enumerate(singles):
        assert o[0] == nr[f], f
        assert torch.equal(o[3], radii[f]), f
        assert torch.equal(o[1], color[f]) and torch.equal(o[2], allmap[f]), f
        d1 = decode(o[4], o[5], o[6], P, W, H, o[0])
        db = decode(gb.view(M, -1)[f], bb.view(M, -1)[f], ib.view(M, -1)[f], P, W, H, nr[f])
        vis = o[3] > 0                                   # the record, depth and clamped bits are written for these only
        assert torch.equal(d1["tiles_touched"], db["tiles_touched"]), f
        assert torch.equal(d1["surfel_rec"][vis], db["surfel_rec"][vis]), f
        assert torch.equal(d1["depths"][vis], db["depths"][vis]), f
        assert torch.equal(d1["clamped"][vis], db["clamped"][vis]), f
        assert torch.equal(d1["keys"], db["keys"]) and torch.equal(d1["point_list"], db["point_list"]), f


@pytest.mark.parametrize("P", [1, 255, 257, 300_000])
@pytest.mark.parametrize("M", [1, 2, 5, 8])
def test_shared_inputs(M, P, dev):
    ins = _inputs(P, 16, M, dev)
    vms, pms, cps = _cams(M, dev)
    batch, singles = _run(ins, 16, vms, pms, cps, precomp=False)
    _check(batch, singles, P)
    if P > 1:
        assert all(n > 0 for n in batch[0])


@pytest.mark.parametrize("P", [257, 300_000])
@pytest.mark.parametrize("per_frame", [("means3D", "rotations"), ("means3D", "rotations", "opacities", "scales", "shs")],
                         ids=["geometry", "everything"])
def test_per_frame_inputs(per_frame, P, dev):
    M = 5
    ins = _inputs(P, 16, M, dev, per_frame=per_frame)
    vms, pms, cps = _cams(M, dev)
    batch, singles = _run(ins, 16, vms, pms, cps, precomp=False)
    _check(batch, singles, P)


@pytest.mark.parametrize("per_frame", [(), ("colors", "means3D")], ids=["shared", "per_frame"])
def test_colors_precomp(per_frame, dev):
    M, P = 5, 257
    ins = _inputs(P, 16, M, dev, per_frame=per_frame)
    vms, pms, cps = _cams(M, dev)
    batch, singles = _run(ins, 16, vms, pms, cps, precomp=True)
    _check(batch, singles, P)


@pytest.mark.parametrize("K", [1, 4, 9, 16])
@pytest.mark.parametrize("M", [2, 5])
def test_sh_degrees(M, K, dev):
    P = 255
    ins = _inputs(P, K, M, dev)
    vms, pms, cps = _cams(M, dev)
    batch, singles = _run(ins, K, vms, pms, cps, precomp=False)
    _check(batch, singles, P)


def test_frame_without_visible_surfels(dev):
    M, P = 5, 257
    ins = _inputs(P, 16, M, dev)
    vms, pms, cps = _cams(M, dev, empty=(2,))
    batch, singles = _run(ins, 16, vms, pms, cps, precomp=False)
    _check(batch, singles, P)
    assert batch[0][2] == 0 and int(batch[3][2].abs().sum()) == 0
    assert all(batch[0][f] > 0 for f in (0, 1, 3, 4))


def test_prefiltered_status(dev):
    from vidu4d_b200 import rasterizer as RZ
    M, P = 3, 257
    ins = _inputs(P, 16, M, dev)
    vms, pms, cps = _cams(M, dev)
    plain, _ = _run(ins, 16, vms, pms, cps, precomp=False)
    pre, singles = _run(ins, 16, vms, pms, cps, precomp=False, prefiltered=True)   # every surfel in front: no status bit
    _check(pre, singles, P)
    for a, b in zip(plain[:4], pre[:4]):
        assert a == b if isinstance(a, list) else torch.equal(a, b)
    # a surfel behind one camera of the batch raises the status bit of that frame; the others stay clean
    vms, pms, cps = _cams(M, dev, empty=(1,))
    e = torch.empty((0,), device=dev)
    bg = torch.zeros(3, device=dev)
    C = RZ._C
    with pytest.raises(RuntimeError, match="prefiltered"):
        C.rasterize_gaussians_batch(bg, ins["means3D"], e, ins["opacities"], ins["scales"], ins["rotations"], 1.0, vms, pms, 0.5, 0.5,
                                    H, W, ins["shs"], 3, cps, prefiltered=True)
        RZ.check_overflow()
    for f in (0, 2):
        C.rasterize_gaussians(bg, ins["means3D"], e, ins["opacities"], ins["scales"], ins["rotations"], 1.0, e, vms[f], pms[f], 0.5,
                              0.5, H, W, ins["shs"], 3, cps[f], True, False)
        RZ.check_overflow()
