"""The kernel variants that only an environment switch selects, against the default path.

  * tile          SURFEL_COMPOSITE_FWD=tile   composite_tile_fwd_kernel (one CTA per tile, shared chunk ring) instead of
                                              composite_fwd_kernel (one warp per sub-tile);
  * sort_blocked  SURFEL_SORT_INTERLEAVE=0    the onesweep passes map blocks to (frame, slot) frame by frame instead of
                                              interleaving the frames.

Each switch is read once per process, so each variant runs the case list in a spawned child process and saves its
results; the parent runs the same cases on the default path and compares.  The tile forward promises the same per-pair
arithmetic, contribution masks and outputs as the default one, and the sort grid only changes which block sorts what, so
every forward buffer must match bit for bit; gradients may differ only in the order of the atomic sums.  Each case also
asserts, from the default path's buffers, that it reaches the tile-list edge it exists for (chunk and ring boundaries,
early stops, sub-tiles outside the image, pair-buffer overflow of the composite backward), and the hand-built scenes are
checked against the CPU oracle."""
import hashlib
import os
import re
import sys
import time

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from .conftest import GOLDEN_CASES, ROOT, load_golden

VARIANTS = {"tile": {"SURFEL_COMPOSITE_FWD": "tile"}, "sort_blocked": {"SURFEL_SORT_INTERLEAVE": "0"}}
SWITCHES = ("SURFEL_COMPOSITE_FWD", "SURFEL_COMPOSITE", "SURFEL_SORT_INTERLEAVE")
TAN = 0.5
CH = 256                 # instances per chunk of the tile forward and of the composite backward
BWD_CAP = 4608           # pair-buffer slots of the composite backward (composite_tile.cu BWD_CAP)
GRAD_TOL = 2e-5          # of each tensor's max: the inputs of the backward are bit-identical, only atomic order differs
TOL = 1e-4               # CPU oracle (test_gpu_parity's bar)
SORT_TILE = 3072         # SR_SORT_TILE: keys per onesweep block
DIGEST_ABOVE = 1 << 20   # exact tensors with more elements travel as a SHA-256 of their bytes
FEATURE_COUNTS = (1, 16, 22)


# ------------------------------------------------------------------------------------------------ scenes
def _facing_case(W, H, px, py, z, sigma, opac, seed, bg=(0.1, 0.2, 0.3)):
    """Surfels facing an identity camera (rotation (1,0,0,0), tan(fov/2) = 0.5), centred on pixel (px, py) at depth z with a
    footprint of about sigma pixels, colours precomputed; in build_case's format."""
    rng = np.random.default_rng(seed)
    px, py, z, sigma, opac = (np.asarray(v, np.float64) for v in (px, py, z, sigma, opac))
    P = px.size
    means = np.stack([z * TAN * ((2 * px + 1) / W - 1), z * TAN * ((2 * py + 1) / H - 1), z], 1).astype(np.float32)
    s = (sigma * z / W).astype(np.float32)                   # focal length in x = W / (2 tan) = W pixels
    from vidu4d_b200.synthetic import projection_matrix
    return dict(
        means3D=means, scales=np.stack([s, s], 1), rotations=np.tile(np.array([1, 0, 0, 0], np.float32), (P, 1)),
        opacities=opac.astype(np.float32).reshape(P, 1), shs=np.zeros((0,), np.float32),
        colors_precomp=rng.uniform(0, 1, size=(P, 3)).astype(np.float32),
        viewmatrix=np.eye(4, dtype=np.float32), projmatrix=projection_matrix(TAN, TAN).astype(np.float32),
        campos=np.zeros(3, np.float32), bg=np.asarray(bg, np.float32),
        dL_dcolor=rng.normal(size=(3, H, W)).astype(np.float32), dL_dallmap=rng.normal(size=(8, H, W)).astype(np.float32),
        meta=np.array([P, W, H, 0, 1], np.int64), tanfov=np.array([TAN, TAN], np.float32))


def _cat(*parts):
    return [np.concatenate([p[i] for p in parts]) for i in range(5)]


def _tile_blob(rng, n, tx, ty, z0, z1, sigma, o0, o1, spread=0.75):
    """n small surfels about the centre of tile (tx, ty), each inside that tile alone (radius 3 sigma <= 5 px)."""
    return (16 * tx + 8 + rng.uniform(-spread, spread, n), 16 * ty + 8 + rng.uniform(-spread, spread, n),
            rng.uniform(z0, z1, n), np.full(n, sigma), rng.uniform(o0, o1, n))


EXACT_LENGTHS = (1, 31, 32, 33, 255, 256, 257, 511, 512, 513, 769)


def scene_exact_lengths():
    """c: tile k of a 4 x 3 tile image holds exactly EXACT_LENGTHS[k] instances (the last tile none): lengths on the
    32-instance stage, 256-instance chunk and 2-slot ring boundaries.  Low opacity: nothing saturates."""
    rng = np.random.default_rng(101)
    parts = [_tile_blob(rng, n, k % 4, k // 4, 0.5, 5.0, 1.5, 0.006, 0.01) for k, n in enumerate(EXACT_LENGTHS)]
    return _facing_case(64, 48, *_cat(*parts), seed=102)


def scene_cta_stop():
    """d: eight opaque surfels over the whole image (alpha >= 0.89 everywhere) in front of 1,200 instances in tile 0: every
    pixel saturates within the first stage, so the tile forward stops requesting chunks long before the end of tile 0's
    list."""
    rng = np.random.default_rng(103)
    n = 8
    front = (np.full(n, 32.0), np.full(n, 32.0), 0.40 + 0.01 * np.arange(n), np.full(n, 96.0), np.ones(n))
    back = _tile_blob(rng, 1200, 0, 0, 1.0, 5.0, 1.5, 0.3, 0.6)
    return _facing_case(64, 64, *_cat(front, back), seed=104)


def scene_warp_stop():
    """e: sixteen opaque surfels saturate the top-left 8 x 4 sub-tile of tile (1, 1) but barely touch its bottom-right one;
    1,500 faint surfels lie behind them over the whole tile."""
    rng = np.random.default_rng(105)
    n, m = 16, 1500
    front = (np.full(n, 20.0), np.full(n, 18.0), 0.40 + 0.002 * np.arange(n), np.full(n, 4.0), np.ones(n))
    back = (rng.uniform(16, 32, m), rng.uniform(16, 32, m), rng.uniform(1.0, 5.0, m), np.full(m, 2.0), rng.uniform(0.01, 0.03, m))
    return _facing_case(64, 64, *_cat(front, back), seed=106)


DENSE_N = CH + 16


def scene_dense():
    """f: 272 large faint surfels over a 32 x 32 image: every instance contributes to every pixel, so chunk 0 of each tile
    has 256 x 256 pairs (beyond the backward's pair buffer) and chunk 1 has 16 x 256 (inside it)."""
    rng = np.random.default_rng(107)
    n = DENSE_N
    return _facing_case(32, 32, 16 + rng.uniform(-2, 2, n), 16 + rng.uniform(-2, 2, n), rng.uniform(0.5, 5.0, n),
                        np.full(n, 48.0), rng.uniform(0.008, 0.012, n), seed=108)


CONSTRUCTED = {"exact_lengths": scene_exact_lengths, "cta_stop": scene_cta_stop, "warp_stop": scene_warp_stop,
               "dense": scene_dense}


# ------------------------------------------------------------------------------------------------ running a case
def _np(x):
    return x.detach().cpu().numpy()


def _live_stages(ranges, sub_last):
    """(tile * 8 + sub-tile, stage) of every contribution-mask row the backward and the feature kernels read: stage s of
    sub-tile w of tile t for s < ceil(min(sub_last, len) / 32) (debug.contributing_pairs' rows).  Other rows are undefined."""
    rg = ranges.to(torch.int64)
    sl = sub_last.to(torch.int64)
    nb = ((torch.minimum(sl, (rg[:, 1] - rg[:, 0])[:, None]) + 31) >> 5).reshape(-1)
    ids = torch.repeat_interleave(torch.arange(nb.numel(), device=nb.device), nb)
    return ids, torch.arange(ids.numel(), device=nb.device) - (torch.cumsum(nb, 0) - nb)[ids]


def _frame(dec, nr, color, allmap, radii):
    from vidu4d_b200 import debug as dbg
    ids, s = _live_stages(dec["ranges"], dec["sub_last"])
    t = ids // 8
    masks = dec["contrib_masks"][(dec["ranges"][:, 0].to(torch.int64) >> 5)[t] + t + s, ids % 8]
    assert dbg.contributing_pairs(dec) == int(_popcount(masks).sum())
    return dict(num_rendered=torch.tensor([int(nr)]), radii=radii, keys=dec["keys"], point_list=dec["point_list"],
                ranges=dec["ranges"], color=color, allmap=allmap, final_T=dec["final_T"], n_contrib=dec["n_contrib"],
                sub_last=dec["sub_last"], masks=masks)


_POP8 = torch.tensor([bin(i).count("1") for i in range(256)], dtype=torch.int64)


def _popcount(words):
    """Set bits per row of an int32 (rows, 32) tensor."""
    b = words.contiguous().view(torch.uint8).to(torch.int64)
    return _POP8.to(b.device)[b].reshape(words.shape[0], 4 * words.shape[1]).sum(1)


def _pack(exact, grad, extra=None):
    """Move a case's results to the CPU; big exact tensors as digests."""
    out = {"exact": {}, "grad": {}, "extra": extra or {}}
    for k, v in exact.items():
        v = v.detach().contiguous().cpu()
        if v.numel() > DIGEST_ABOVE:
            v = ("sha256", tuple(v.shape), str(v.dtype), hashlib.sha256(v.view(torch.uint8).numpy().tobytes()).hexdigest())
        out["exact"][k] = v
    for k, v in grad.items():
        if v is not None:
            out["grad"][k] = v.detach().cpu()
    return out


def _single(inp, dev, F=0, seed=0):
    """One frame through rasterize_gaussians (or rasterize_gaussians_features with F random channels) and its backward."""
    from vidu4d_b200 import debug as dbg, rasterizer as R
    from .test_gpu_parity import GRADS, _run_ours
    if F == 0:
        r = _run_ours(inp, dev)
        frame = _frame(r, r["num_rendered"], r["color"], r["allmap"], r["radii"])
        return frame, r["grads"], r
    P, W, H, deg, pre = [int(v) for v in inp["meta"]]
    t = {k: torch.from_numpy(np.ascontiguousarray(v)).to(dev) for k, v in inp.items() if k != "meta"}
    g = torch.Generator(device=dev).manual_seed(seed)
    feat = torch.randn((P, F), device=dev, generator=g)
    dLc = torch.cat([t["dL_dcolor"], torch.randn((F, H, W), device=dev, generator=g)])
    e = torch.empty((0,), device=dev)
    shs, col = (e, t["colors_precomp"]) if pre else (t["shs"], e)
    nr, color, allmap, radii, gb, bb, ib = R._C.rasterize_gaussians_features(
        t["bg"], t["means3D"], col, t["opacities"], t["scales"], t["rotations"], 1.0, e, t["viewmatrix"], t["projmatrix"],
        TAN, TAN, H, W, shs, deg, t["campos"], False, False, feat)
    grads = R._C.rasterize_gaussians_features_backward(
        t["bg"], t["means3D"], radii, col, t["scales"], t["rotations"], 1.0, e, t["viewmatrix"], t["projmatrix"], TAN, TAN,
        dLc, t["dL_dallmap"], shs, deg, t["campos"], gb, nr, bb, ib, False, feat)
    dec = dbg.decode(gb, bb, ib, P, W, H, nr)
    return _frame(dec, nr, color, allmap, radii), dict(zip(GRADS + ("dL_dfeatures",), grads)), dec


def _batch(dev, M, W, H, scene, means, cams, seed, F=0, shs=None, deg=3):
    """M frames through rasterize_gaussians_batch and rasterize_gaussians_backward_batch (sum_shared off and on)."""
    from vidu4d_b200 import debug as dbg, rasterizer as R
    from .test_gpu_parity import GRADS
    C = R._C
    t = scene.to_torch(dev)
    shs = t["shs"] if shs is None else shs
    P = int(t["opacities"].shape[0])
    vms, pms, cps = cams
    g = torch.Generator(device=dev).manual_seed(seed)
    feat = torch.randn((P, F), device=dev, generator=g) if F else None
    dLc = torch.randn((M, 3 + F, H, W), device=dev, generator=g)
    dLo = 0.1 * torch.randn((M, 8, H, W), device=dev, generator=g)
    e = torch.empty((0,), device=dev)
    bg = torch.tensor([0.2, 0.1, 0.4], device=dev)
    out = C.rasterize_gaussians_batch(bg, means, e, t["opacities"], t["scales"], t["rotations"], 1.0, vms, pms, TAN, TAN, H, W,
                                      shs, deg, cps, features=feat)
    nr, color, allmap, radii, gb, bb, ib = out[:7]
    names = GRADS + (("dL_dfeatures",) if F else ())
    exact, grad, decs = {}, {}, []
    for f in range(M):
        dec = dbg.decode(gb.view(M, -1)[f], bb.view(M, -1)[f], ib.view(M, -1)[f], P, W, H, nr[f])
        decs.append(dec)
        for k, v in _frame(dec, nr[f], color[f], allmap[f], radii[f]).items():
            exact[f"f{f}.{k}"] = v
    for sum_shared in (False, True):
        gr = C.rasterize_gaussians_backward_batch(bg, means, radii, e, t["scales"], t["rotations"], 1.0, vms, pms, TAN, TAN,
                                                  dLc, dLo, shs, deg, cps, gb, bb, ib, sum_shared=sum_shared, features=feat)
        for k, v in zip(names, gr):
            grad[f"sum_shared={sum_shared}.{k}"] = v
    return exact, grad, decs


def _orbit_cams(M, dev):
    from .test_gpu_batch import _cams
    return _cams(M, dev)


def case_golden(name, dev):
    g = load_golden(name)
    frame, grads, _ = _single({k[3:]: v for k, v in g.items() if k.startswith("in_")}, dev)
    return frame, grads, {}


def case_build(kw, dev):
    from tests.golden.make_golden import build_case
    frame, grads, _ = _single(build_case(**kw), dev)
    return frame, grads, {}


def case_constructed(name, dev):
    frame, grads, _ = _single(CONSTRUCTED[name](), dev)
    return frame, grads, {}


def case_cull(name, dev):
    """A scene of tests/test_gpu_cull_bounds.py: the tile forward reads the same cull words."""
    from .test_gpu_cull_bounds import SINGLE, scene_single
    frame, grads, _ = _single(scene_single(**SINGLE[name])[0], dev)
    return frame, grads, {}


def case_features_single(F, dev):
    from tests.golden.make_golden import build_case
    frame, grads, _ = _single(build_case(6000, 96, 80, 90 + F, bg=(0.2, 0.1, 0.3)), dev, F=F, seed=F)
    return frame, grads, {}


def case_features_batch(F, dev):
    from vidu4d_b200.synthetic import object_scene
    sc = object_scene(6000, seed=40 + F, center=(0.0, 0.0, 0.0))
    means = torch.from_numpy(sc.means3D).to(dev)
    exact, grad, _ = _batch(dev, 3, 104, 72, sc, means, _orbit_cams(3, dev), seed=F, F=F)
    return exact, grad, {}


def _hidden_means(sc, cps, dev):
    """Per-frame positions for 5 frames: frame 0 sees nothing, frame 1 one surfel, frame 2 fewer instances than one sort
    block, frames 3 and 4 the whole object.  Hidden surfels sit 1 behind the camera (it orbits the origin at distance 1)."""
    base = torch.from_numpy(sc.means3D).to(dev)
    means = base[None].repeat(5, 1, 1)
    cam = cps.to(dev)
    single = int(torch.argmax(base @ cam[1] / cam[1].norm()))     # the surfel nearest to frame 1's camera, on its axis
    means[0] = 2 * cam[0]
    means[1] = 2 * cam[1]
    means[1, single] = base[single]
    means[2, 150:] = 2 * cam[2]
    return means.contiguous(), single


def case_batch5(dev):
    from vidu4d_b200.synthetic import object_scene
    sc = object_scene(20000, seed=5, center=(0.0, 0.0, 0.0))
    cams = _orbit_cams(5, dev)
    means, single = _hidden_means(sc, cams[2], dev)
    exact, grad, _ = _batch(dev, 5, 120, 88, sc, means, cams, seed=55)
    return exact, grad, {"single": single}


def case_batch8(dev):
    """The benchmark's shape: 300 K surfels, 512^2, 8 orbit cameras, per-frame positions (SH degree 0 keeps the
    (M,P,.) gradients small enough to ship between processes)."""
    from vidu4d_b200.synthetic import object_scene
    sc = object_scene(300_000, seed=0, center=(0.0, 0.0, 0.0))
    g = torch.Generator(device=dev).manual_seed(88)
    base = torch.from_numpy(sc.means3D).to(dev)
    means = torch.stack([base + 0.002 * f * torch.randn(base.shape, device=dev, generator=g) for f in range(8)])
    shs = torch.from_numpy(np.ascontiguousarray(sc.shs[:, :1])).to(dev)
    exact, grad, _ = _batch(dev, 8, 512, 512, sc, means, _orbit_cams(8, dev), seed=8, shs=shs, deg=0)
    return exact, grad, {}


def case_graphed(dev):
    """render_loss_batch forward + backward captured as one CUDA graph, replayed with two RGB targets."""
    from vidu4d_b200 import rasterizer as RZ
    from vidu4d_b200.graph import GraphedStep
    from vidu4d_b200.renderer import PipelineParams, render_loss_batch
    from .test_gpu_feature_loss import _model, _scene
    M, P, W, H = 2, 20000, 96, 96
    bc, _, _ = _scene(P, W, H, M, dev, seed=51)
    gen = torch.Generator(device=dev).manual_seed(6)
    rgbs = [torch.rand((M, 3, H, W), device=dev, generator=gen) for _ in range(2)]
    mask = (torch.rand((M, H, W), device=dev, generator=gen) > 0.4).float()
    ftgt = torch.randn((M, 16, H, W), device=dev, generator=gen) * 0.1
    rest = torch.rand((P, 6), device=dev, generator=gen)
    det = torch.tensor([1.0, 1.0], device=dev)
    w = torch.tensor([1e-2, 1e-2], device=dev)
    pipe, bg = PipelineParams(), torch.zeros(3, device=dev)
    m = _model(P, dev, seed=7)
    rgb = rgbs[0].clone()
    loss = torch.zeros((), device=dev)

    def body():
        m.zero_grad_flat()
        out = render_loss_batch(bc, m, pipe, bg, rgb, mask_gt=mask, w_mask=0.1, features=torch.cat([m._regist_feat, rest], 1),
                                feature_target=ftgt, is_detected=det, gauss_mask_channel=21, feature_loss_weights=w)
        out["loss"].backward()
        loss.copy_(out["loss"].detach())

    grad = {}
    if _graph_mode():
        step = GraphedStep(body, device=dev)
        try:
            for i, target in enumerate(rgbs):
                rgb.copy_(target)
                step()
                grad[f"replay{i}.loss"] = loss.clone()
                grad[f"replay{i}.grad_flat"] = m.grad_flat.clone()
            assert step.captures == 1
        finally:
            RZ.set_sync_mode(True)
            RZ._pending.clear()
    else:
        for i, target in enumerate(rgbs):
            rgb.copy_(target)
            body()
            grad[f"replay{i}.loss"] = loss.clone()
            grad[f"replay{i}.grad_flat"] = m.grad_flat.clone()
    return {}, grad, {}


def _graph_mode():
    """The variants capture the step; the default path runs it eagerly (the reference the replays are compared with)."""
    return any(os.environ.get(k) for k in SWITCHES)


CASES = {}
for _n in GOLDEN_CASES:
    CASES[f"golden_{_n}"] = (case_golden, _n)
CASES["ragged_72x52"] = (case_build, dict(P=6000, W=72, H=52, seed=81))
# the object moved towards the bottom-right corner so that it reaches the last tile row and column
CASES["ragged_200x116"] = (case_build, dict(P=12000, W=200, H=116, seed=82, center=(0.25, 0.2, 0.8)))
for _n in CONSTRUCTED:
    CASES[_n] = (case_constructed, _n)
CASES["long_lists"] = (case_build, dict(P=50000, W=32, H=32, seed=72))
for _n in ("cull_mix_72x52", "cull_mix_37x23"):
    CASES[_n] = (case_cull, _n)
CASES["batch8_512"] = (case_batch8, None)
CASES["batch5_edges"] = (case_batch5, None)
for _f in FEATURE_COUNTS:
    CASES[f"features{_f}_single"] = (case_features_single, _f)
    CASES[f"features{_f}_batch"] = (case_features_batch, _f)
CASES["graphed_step"] = (case_graphed, None)


def run_case(name, dev):
    fn, arg = CASES[name]
    exact, grad, extra = fn(dev) if arg is None else fn(arg, dev)
    torch.cuda.synchronize(dev)
    return _pack(exact, grad, extra)


def composite_kernels(dev):
    """Names of the CUDA kernels one forward of the first golden case launches."""
    from torch.profiler import ProfilerActivity, profile
    g = load_golden(GOLDEN_CASES[0])
    inp = {k[3:]: v for k, v in g.items() if k.startswith("in_")}
    from .test_gpu_parity import _run_ours
    _run_ours(inp, dev, with_grads=False)                          # warm: library loaded, buffers sized
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        _run_ours(inp, dev, with_grads=False)
        torch.cuda.synchronize(dev)
    return sorted({e.key for e in prof.key_averages()})


# ------------------------------------------------------------------------------------------------ variant workers
def _worker(rank, variant, out):
    sys.path.insert(0, ROOT)
    for k in SWITCHES:
        os.environ.pop(k, None)
    os.environ.update(VARIANTS[variant])                          # before the library's first call reads the switches
    from vidu4d_b200 import _capi
    _capi.load()
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    results = {"kernels": composite_kernels(dev), "cases": {}}
    for name in CASES:
        results["cases"][name] = run_case(name, dev)
    torch.save(results, out)


def _spawn(variant, out, timeout_s=1500):
    ctx = mp.start_processes(_worker, args=(variant, out), nprocs=1, join=False, start_method="spawn")
    deadline = time.monotonic() + timeout_s
    while not ctx.join(timeout=5):
        if time.monotonic() > deadline:
            for p in ctx.processes:
                p.kill()
                p.join()
            pytest.fail(f"the {variant} worker did not finish in {timeout_s} s")


@pytest.fixture(scope="module")
def dev(built):
    from vidu4d_b200 import _capi
    _capi.load()
    for k in SWITCHES:
        assert not os.environ.get(k), f"{k} is set: the parent must run the default path"
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def default_results(dev):
    return {"kernels": composite_kernels(dev), "cases": {name: run_case(name, dev) for name in CASES}}


@pytest.fixture(scope="module", params=list(VARIANTS))
def variant(request, dev, tmp_path_factory):
    out = str(tmp_path_factory.mktemp("variant_" + request.param) / "results.pt")
    _spawn(request.param, out)
    return request.param, torch.load(out, weights_only=False)


# ------------------------------------------------------------------------------------------------ comparisons
def _assert_exact(a, b, what):
    if isinstance(a, tuple) or isinstance(b, tuple):
        assert a == b, f"{what} differs (digest)"
        return
    assert a.shape == b.shape and a.dtype == b.dtype, what
    if a.dtype.is_floating_point:
        a, b = a.contiguous().view(torch.int32), b.contiguous().view(torch.int32)
    bad = a != b
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} of {bad.numel()} elements differ"


def _assert_grad(mine, ref, what):
    assert mine.shape == ref.shape, what
    err = float((mine.double() - ref.double()).abs().max()) if ref.numel() else 0.0
    assert err <= GRAD_TOL * float(ref.abs().max() if ref.numel() else 0.0) + 1e-30, (what, err)


@pytest.mark.gpu
@pytest.mark.timeout(1800)
def test_variant_switch_selects_its_kernels(variant, default_results):
    name, res = variant
    assert any("composite_fwd_kernel" in k for k in default_results["kernels"])
    assert not any("composite_tile_fwd_kernel" in k for k in default_results["kernels"])
    tile = any("composite_tile_fwd_kernel" in k for k in res["kernels"])
    warp = any("composite_fwd_kernel" in k for k in res["kernels"])
    assert (tile, warp) == ((True, False) if name == "tile" else (False, True)), res["kernels"]


@pytest.mark.gpu
@pytest.mark.timeout(1800)
@pytest.mark.parametrize("case", list(CASES))
def test_variant_matches_default(variant, default_results, case):
    name, res = variant
    mine, ref = res["cases"][case], default_results["cases"][case]
    assert mine["extra"] == ref["extra"]
    assert sorted(mine["exact"]) == sorted(ref["exact"]) and sorted(mine["grad"]) == sorted(ref["grad"])
    for k in ref["exact"]:
        _assert_exact(mine["exact"][k], ref["exact"][k], f"{name}/{case}: {k}")
    for k in ref["grad"]:
        if k.endswith(".loss"):
            assert abs(float(mine["grad"][k]) - float(ref["grad"][k])) <= 1e-5 * abs(float(ref["grad"][k])), (name, case, k)
        else:
            _assert_grad(mine["grad"][k], ref["grad"][k], f"{name}/{case}: {k}")
    if case.startswith("golden_") and name == "tile":
        g = load_golden(case[len("golden_"):])
        assert np.array_equal(mine["exact"]["color"].numpy(), g["ref_color"]), "tile forward colour vs the reference"


# ------------------------------------------------------------------------------------------------ edges reached
def _lengths(res, prefix=""):
    rg = res["exact"][prefix + "ranges"].to(torch.int64)
    return rg[:, 1] - rg[:, 0]


def _chunk_pairs(res, prefix=""):
    """{(tile, chunk): contributing pairs} from the live contribution masks."""
    ex = res["exact"]
    ids, s = _live_stages(ex[prefix + "ranges"], ex[prefix + "sub_last"])     # the row order of the stored masks
    out = {}
    for t, c, n in zip((ids // 8).tolist(), (s // (CH // 32)).tolist(), _popcount(ex[prefix + "masks"]).tolist()):
        out[(t, c)] = out.get((t, c), 0) + n
    return out


def _outside_subtiles(W, H):
    """(tile, sub-tile) pairs whose 8 x 4 pixels all lie outside the image."""
    tx, ty = (W + 15) // 16, (H + 15) // 16
    out = []
    for t in range(tx * ty):
        for w in range(8):
            x0, y0 = (t % tx) * 16 + (w & 1) * 8, (t // tx) * 16 + (w >> 1) * 4
            if x0 >= W or y0 >= H:
                out.append((t, w))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["ragged_72x52", "ragged_200x116"])
def test_edge_ragged_images_have_subtiles_outside(default_results, case):
    W, H = CASES[case][1]["W"], CASES[case][1]["H"]
    assert W % 16 == 8 and H % 16 == 4
    ln = _lengths(default_results["cases"][case])
    busy = [(t, w) for t, w in _outside_subtiles(W, H) if int(ln[t]) > 0]
    assert busy, "no tile with instances has a sub-tile wholly outside the image"


@pytest.mark.gpu
def test_edge_exact_tile_list_lengths(default_results):
    ln = _lengths(default_results["cases"]["exact_lengths"]).tolist()
    assert ln == list(EXACT_LENGTHS) + [0]


@pytest.mark.gpu
def test_edge_whole_cta_stop_leaves_chunks_unrequested(default_results):
    res = default_results["cases"]["cta_stop"]
    ln = _lengths(res)
    sl = res["exact"]["sub_last"].to(torch.int64).max(1).values
    # the tile forward requests chunks 0 and 1 up front, and chunk c + 2 once chunk c is released unless every warp is
    # done; here every pixel saturates in the chunk of the tile's deepest contributor
    unrequested = (ln + CH - 1) // CH - (torch.div(sl - 1, CH, rounding_mode="floor") + 2)
    assert int(ln[0]) == 1208 and int(unrequested[0]) == 3 and bool((sl + 2 * CH < ln).any()), (ln.tolist(), sl.tolist())


@pytest.mark.gpu
def test_edge_one_warp_stops_while_another_goes_deep(default_results):
    res = default_results["cases"]["warp_stop"]
    ln = _lengths(res)
    sl = res["exact"]["sub_last"].to(torch.int64)
    T = res["exact"]["final_T"][0]
    found = False
    for t in range(sl.shape[0]):
        early = [w for w in range(8) if 0 < int(sl[t, w]) <= CH]
        deep = [w for w in range(8) if int(sl[t, w]) > 2 * CH]
        for w in early:
            x0, y0 = (t % 4) * 16 + (w & 1) * 8, (t // 4) * 16 + (w >> 1) * 4
            saturated = bool((T[y0:y0 + 4, x0:x0 + 8] < 0.02).all())
            found = found or (saturated and bool(deep) and int(ln[t]) > 3 * CH)
    assert found, (ln.tolist(), sl.tolist())


@pytest.mark.gpu
def test_edge_dense_chunks_straddle_the_pair_buffer(default_results):
    pairs = _chunk_pairs(default_results["cases"]["dense"])
    counts = sorted(pairs.values())
    assert max(counts) == CH * CH and any(c > BWD_CAP for c in counts) and any(0 < c < BWD_CAP for c in counts), counts


@pytest.mark.gpu
def test_edge_long_lists_span_many_chunks(default_results):
    assert int(_lengths(default_results["cases"]["long_lists"]).max()) > 32 * CH


@pytest.mark.gpu
def test_edge_batch_frames(default_results):
    res = default_results["cases"]["batch5_edges"]
    nr = [int(res["exact"][f"f{f}.num_rendered"][0]) for f in range(5)]
    radii1 = res["exact"]["f1.radii"]
    assert nr[0] == 0 and nr[1] >= 1 and 0 < nr[2] < SORT_TILE and min(nr[3:]) > SORT_TILE, nr
    assert (radii1 > 0).nonzero().flatten().tolist() == [res["extra"]["single"]]
    res8 = default_results["cases"]["batch8_512"]
    nr8 = [int(res8["exact"][f"f{f}.num_rendered"][0]) for f in range(8)]
    assert min(nr8) > 100 * SORT_TILE and len(set(nr8)) > 1, nr8


# ------------------------------------------------------------------------------------------------ CPU oracle
@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CONSTRUCTED))
def test_constructed_scene_against_cpu_oracle(case, dev):
    from oracle import surfel_oracle as so
    from .test_gpu_parity import GRADS, _assert_close_robust
    inp = CONSTRUCTED[case]()
    P, W, H = [int(v) for v in inp["meta"][:3]]
    _, grads, r = _single(inp, dev)
    st = so.forward(inp["means3D"], inp["opacities"], inp["scales"], inp["rotations"], colors_precomp=inp["colors_precomp"],
                    sh_degree=0, W=W, H=H, tanfovx=TAN, tanfovy=TAN, bg=inp["bg"], viewmatrix=inp["viewmatrix"],
                    projmatrix=inp["projmatrix"], campos=inp["campos"])
    og = so.backward(st, inp["dL_dcolor"], inp["dL_dallmap"])
    assert r["num_rendered"] == st.num_rendered
    np.testing.assert_array_equal(_np(r["point_list"]).astype(np.uint32), st.point_list)
    np.testing.assert_array_equal(_np(r["ranges"]).astype(np.uint32), st.ranges)
    _assert_close_robust(_np(r["color"]), st.color, TOL, "color")
    for i in range(8):
        _assert_close_robust(_np(r["allmap"][i]), st.allmap[i], TOL, f"allmap[{i}]")
    for k in GRADS:
        if og[k].size == 0:                          # dL_dsh with precomputed colours
            assert grads[k].numel() == 0, k
            continue
        _assert_close_robust(_np(grads[k]), og[k], TOL, k)


# ------------------------------------------------------------------------------------------------ switch names (CPU)
def test_switch_names_match_the_workers():
    """The workers select their variant by environment; a renamed switch would turn every comparison above into the
    default path against itself."""
    src = os.path.join(ROOT, "vidu4d_b200", "csrc")
    with open(os.path.join(src, "composite_tile.cu")) as fh:
        tile = fh.read()
    with open(os.path.join(src, "sort.cu")) as fh:
        sort = fh.read()
    assert re.search(r'getenv\("SURFEL_COMPOSITE_FWD"\)', tile)
    m = re.search(r"return e && e\[0\] == '(.)';", tile)
    assert m and VARIANTS["tile"]["SURFEL_COMPOSITE_FWD"][0] == m.group(1)
    assert re.search(r'const char\* e = getenv\("SURFEL_SORT_INTERLEAVE"\); return e && atoi\(e\) == 0 \? 0 : 1;', sort)
    assert int(VARIANTS["sort_blocked"]["SURFEL_SORT_INTERLEAVE"]) == 0
    # the sort's switch reaches the onesweep pass as its `interleave` argument
    assert re.search(r"a\.bl\.sort_tiles, inter\);", sort)
