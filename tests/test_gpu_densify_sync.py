"""GPU: the batched densification statistics (sr_densify_stats) against M calls of the one-frame torch update, and a
multi-rank Stage-3 run -- render -> backward -> all-reduce -> statistics -> clip -> step, densify and prune at step 2,
reset opacity at step 3, radius outliers at step 4 -- whose ranks stay bit-identical and make the decisions one process
rendering every frame makes.

Rounding: the kernel reproduces torch's float32 3-norm (fl(fl(fl(x^2) + fl(z^2)) + fl(y^2)), correctly rounded sqrt)
and the per-frame adds, so its statistics equal the torch path's bit for bit.  A multi-rank run and a one-process run
sum the frames' gradients in another order, and the rasterizer backward sums with atomics, so the two agree within a
margin, not in every bit: EPS below, relative.  The test checks that the runs' differences stay inside EPS / 2 and that
no decision input lies within four times the measured difference of its threshold, so a knife edge fails loudly instead
of flipping a decision."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from .conftest import ROOT

pytestmark = pytest.mark.gpu

NF, P, W, H = 8, 40000, 256, 192
STEPS, DENSIFY_AT, RESET_AT, OUTLIER_AT = 5, 2, 3, 4
THRESHOLD, MIN_OPACITY, EXTENT = 6e-5, 0.25, 0.55
NB_POINTS, RADIUS = 1, 0.03
MAX_NORM = 1.0
LRS = {"xyz": 1e-6, "f_dc": 1e-5, "f_rest": 1e-5, "opacity": 1e-5, "scaling": 1e-5, "rotation": 1e-5}
EPS = 1e-3
SEED = 77


@pytest.fixture(scope="module")
def dev(built):
    from vidu4d_b200 import _capi
    _capi.load()
    return torch.device("cuda:0")


def _model(P, dev, seed=0, isolated=0):
    """object_scene's sphere of radius 0.35; with `isolated`, its last surfels (at most 6) moved to 0.15 along +-x, +-y,
    +-z: far from each other and from the shell next to RADIUS, so they are the outliers, and clearly so."""
    from vidu4d_b200.surfel_store import FlatSurfelModel
    from vidu4d_b200.synthetic import object_scene
    sc = object_scene(P, seed=seed, center=(0.0, 0.0, 0.0))
    xyz = sc.means3D.copy()
    if isolated:
        xyz[P - isolated:] = 0.15 * np.concatenate([np.eye(3), -np.eye(3)])[:isolated]
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    op = np.clip(sc.opacities, 1e-6, 1 - 1e-6)
    return FlatSurfelModel(t(xyz), t(sc.shs[:, :1]), t(sc.shs[:, 1:]), t(np.log(op / (1 - op))), t(np.log(sc.scales)),
                           t(sc.rotations), lrs=dict(LRS))


# ---- the kernel against the one-frame path ----------------------------------------------------------------------------
def _inputs(M, P, dev, seed, blank_frames=()):
    g = torch.Generator(device=dev).manual_seed(seed)
    grad = torch.randn((M, P, 3), device=dev, generator=g)
    # magnitudes over many binades, exact zeros, and rows whose squares sum across a rounding boundary
    grad *= torch.pow(10.0, torch.randint(-12, 4, (M, P, 1), device=dev, generator=g).float())
    grad[:, ::7] = 0.0
    grad[:, 3::11, 1] = grad[:, 3::11, 0]
    radii = torch.randint(0, 40, (M, P), device=dev, generator=g, dtype=torch.int32)
    radii[:, ::5] = 0
    for f in blank_frames:
        radii[f] = 0
    return grad, radii


@pytest.mark.parametrize("M,P,grad_scale,blank", [(1, 5003, 1.0, ()), (2, 40000, 0.125, ()), (8, 20001, 0.3, (0, 5)),
                                                  (8, 1023, 1.0, tuple(range(8))), (3, 0, 1.0, ()), (2, 4, 7.0, ())])
def test_kernel_equals_per_frame_torch_path(M, P, grad_scale, blank, dev):
    grad, radii = _inputs(M, P, dev, seed=M * 1000 + P, blank_frames=blank)
    ker, ref = _model(max(P, 1), dev), _model(max(P, 1), dev)
    if P == 0:
        ker.prune_points(torch.ones(1, dtype=torch.bool, device=dev))
        ref.prune_points(torch.ones(1, dtype=torch.bool, device=dev))
    # statistics already under way: the kernel adds to what is there, in the same order
    g0, r0 = _inputs(1, P, dev, seed=5)
    for m in (ker, ref):
        m.add_densification_stats(g0[0], r0[0] > 0, r0[0])
    ker.add_densification_stats(grad, radii > 0, radii, grad_scale=grad_scale)
    for f in range(M):
        ref.add_densification_stats(grad[f] * grad_scale, radii[f] > 0, radii[f])
    assert torch.equal(ker.denom, ref.denom)
    assert torch.equal(ker.max_radii2D, ref.max_radii2D)
    assert torch.equal(ker.xyz_gradient_accum, ref.xyz_gradient_accum)
    # run to run: the same bits
    again = _model(max(P, 1), dev)
    if P == 0:
        again.prune_points(torch.ones(1, dtype=torch.bool, device=dev))
    again.add_densification_stats(g0[0], r0[0] > 0, r0[0])
    again.add_densification_stats(grad, None, radii, grad_scale=grad_scale)
    assert torch.equal(again.densify_stats, ker.densify_stats) and torch.equal(again.max_radii2D, ker.max_radii2D)


def test_kernel_rejects_a_foreign_device_tensor(dev):
    m = _model(100, dev)
    grad, radii = _inputs(2, 100, dev, seed=1)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        m.add_densification_stats(grad, None, radii.cpu())


def test_prune_points_keeps_the_statistics_packed(dev):
    m = _model(1000, dev)
    grad, radii = _inputs(2, 1000, dev, seed=2)
    m.add_densification_stats(grad, None, radii)
    want = m.densify_stats[:, 10:].clone()
    m.prune_points(torch.arange(1000, device=dev) < 10)
    assert torch.equal(m.densify_stats, want) and m.xyz_gradient_accum.data_ptr() == m.densify_stats.data_ptr()


# ---- a multi-rank run against one process rendering every frame ---------------------------------------------------
def _scene(dev):
    from vidu4d_b200.renderer import make_camera
    from vidu4d_b200.synthetic import orbit_view
    cams = []
    for f in range(NF):
        R, t = orbit_view(7 * f + 1, 64)
        cams.append(make_camera(W, H, 2 * np.arctan(0.5), 2 * np.arctan(0.375), R=R.T, T=t, device=dev))
    target = torch.rand((NF, 3, H, W), generator=torch.Generator().manual_seed(11)).to(dev)
    return cams, target


def _train(frames, dev, check=None):
    """STEPS Stage-3 steps over `frames` (this rank's share of NF).  check(): distributed.check_replicas, or None on one
    process.  Returns the arrays the comparisons need."""
    from vidu4d_b200 import distributed as D
    from vidu4d_b200.renderer import PipelineParams, render_loss_batch, stack_cameras
    cams, target = _scene(dev)
    model = _model(P, dev, seed=3, isolated=6)
    cams = stack_cameras([cams[f] for f in frames])
    bg = torch.zeros(3, device=dev)
    rec = {}
    for step in range(STEPS):
        model.zero_grad_flat()
        out = render_loss_batch(cams, model, PipelineParams(), bg, target[frames], w_rgb=1.0, lambda_normal=0.05,
                                lambda_dist=0.01)
        out["loss"].backward()
        model.allreduce_grads_()
        model.add_densification_stats(out["viewspace_points"].grad, out["visibility_filter"], out["radii"], grad_scale=1.0 / NF)
        model.clip_grad_norm_(MAX_NORM, grad_scale=1.0 / NF)
        model.step(grad_scale=1.0 / NF)
        if step == DENSIFY_AT:
            model.sync_densification_stats()
            if check:
                check(model.replica_state())
            ratio = model.xyz_gradient_accum[:, 0] / model.denom[:, 0]
            rec["ratio"] = torch.nan_to_num(ratio, nan=0.0).cpu().numpy()
            rec["max_scale"] = model.get_scaling.detach().max(dim=1).values.cpu().numpy()
            rec["sigma"] = model.get_opacity.detach()[:, 0].cpu().numpy()
            info = model.densify_and_prune(THRESHOLD, MIN_OPACITY, EXTENT, None, generator=D.shared_generator(dev, SEED))
            rec.update({f"info_{k}": np.int64(v) for k, v in info.items()})
        if step == RESET_AT:
            model.reset_opacity()
        if step == OUTLIER_AT:
            rec["xyz_before_outliers"] = model._xyz.detach().cpu().numpy().copy()
            rec["outliers"] = np.int64(model.remove_radius_outliers(NB_POINTS, RADIUS))
        if check:
            state = model.replica_state()
            if step != DENSIFY_AT:          # each rank's own statistics until the next sync
                del state["densify_stats"], state["max_radii2D"]
            check(state)
    torch.cuda.synchronize()
    rec["P"] = np.int64(model.P)
    rec["flat"] = model.flat.cpu().numpy()
    return rec, model


def _worker(rank, world, port, out, backend):
    sys.path.insert(0, ROOT)
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    from vidu4d_b200 import _capi
    from vidu4d_b200 import distributed as D
    dev = torch.device("cuda", rank if backend == "nccl" else 0)
    torch.cuda.set_device(dev)
    _capi.load()
    D.init_distributed(backend, dev if backend == "nccl" else None)
    rec, model = _train(D.shard_frames(NF, rank, world), dev, check=D.check_replicas)
    # one element set differently on one rank, from the host: check_replicas must see it on every rank
    if rank == 1:
        model.flat[12345] = float(model.flat[12345]) + 1.0
    try:
        D.check_replicas(model.replica_state())
        rec["detect"] = ""
    except RuntimeError as e:
        rec["detect"] = str(e)
    np.savez(out + f".{rank}.npz", **rec)
    dist.destroy_process_group()


def _spawn(tmp_path, backend, port):
    out = str(tmp_path / "rank")
    ctx = mp.start_processes(_worker, args=(2, port, out, backend), nprocs=2, join=False, start_method="spawn")
    import time
    deadline = time.time() + 900
    while not ctx.join(timeout=5):
        if time.time() > deadline:
            for p in ctx.processes:
                p.kill()
            raise TimeoutError("the two ranks did not finish in 900 s")
    return [dict(np.load(out + f".{r}.npz")) for r in range(2)]


def _compare(ranks, dev):
    from vidu4d_b200.knn import radius_outlier_mask
    one, model = _train(list(range(NF)), dev)
    big = model.percent_dense * EXTENT
    print(f"one process: accum/denom quantiles (0.5, 0.9, 0.99) {np.quantile(one['ratio'], [0.5, 0.9, 0.99])}, "
          f"max scale {np.quantile(one['max_scale'], [0.5, 0.9, 0.99])}, opacity {np.quantile(one['sigma'], [0.01, 0.1, 0.5])}, "
          f"decisions {[int(one[k]) for k in ('info_cloned', 'info_split', 'info_pruned', 'outliers', 'P')]}, "
          f"max |accum/denom diff| {float(np.abs(ranks[0]['ratio'] - one['ratio']).max()):.3g}, "
          f"max |param diff| {float(np.abs(ranks[0]['flat'] - one['flat']).max()) if ranks[0]['flat'].shape == one['flat'].shape else -1:.3g}")
    for r in ranks:
        assert "'flat'" in str(r["detect"]) and "[1]" in str(r["detect"]), str(r["detect"])
    two = ranks[0]
    # the runs differ by summation order only: inside EPS / 2 ...
    for k, thr, what in (("ratio", THRESHOLD, "accum / denom"), ("max_scale", big, "scale"), ("sigma", MIN_OPACITY, "opacity")):
        d = np.abs(two[k].astype(np.float64) - one[k])
        assert np.all(d <= EPS / 2 * np.maximum(np.abs(one[k]), thr)), (k, float(d.max()))
        # ... and no decision input within (four times) that difference of its threshold
        band = max(4 * float(d.max()), 1e-9 * thr)
        assert not np.any(np.abs(one[k] - thr) <= band), f"a surfel's {what} is on the knife edge of {thr}"
    # positions differ by at most dx per coordinate, so a distance by at most 2 sqrt(3) dx: no neighbour count may change
    # between RADIUS -/+ twice that (many pairs lie within EPS * RADIUS of RADIUS, so the band is the measured one)
    dx = float(np.abs(two["xyz_before_outliers"].astype(np.float64) - one["xyz_before_outliers"]).max())
    assert dx <= EPS / 2 * RADIUS, dx
    band = max(4 * np.sqrt(3) * dx, 1e-7)
    xyz = torch.from_numpy(one["xyz_before_outliers"]).to(dev)
    assert torch.equal(radius_outlier_mask(xyz, NB_POINTS, RADIUS - band), radius_outlier_mask(xyz, NB_POINTS, RADIUS + band)), \
        ("a neighbour distance is on the knife edge of the outlier radius", dx)
    # so the decisions are the same
    for k in ("info_cloned", "info_split", "info_pruned", "info_P", "outliers", "P"):
        assert int(two[k]) == int(one[k]), (k, int(two[k]), int(one[k]))
    assert int(one["info_cloned"]) > 0 and int(one["info_split"]) > 0 and int(one["info_pruned"]) > 0 and int(one["outliers"]) > 0
    # and the parameters agree within what STEPS Adam steps of differently rounded gradients can move them
    from vidu4d_b200.surfel_store import GROUPS
    bounds = np.concatenate([np.full(int(one["P"]) * k, 4 * STEPS * LRS[n]) for n, k in GROUPS])
    d = np.abs(two["flat"].astype(np.float64) - one["flat"])
    assert np.all(d <= bounds + 1e-6 * np.abs(one["flat"])), float((d - bounds).max())


@pytest.mark.timeout(1200)
def test_two_ranks_on_one_gpu_over_gloo_stay_identical_and_match_one_process(dev, tmp_path):
    ranks = _spawn(tmp_path, "gloo", 29400 + (os.getpid() % 200))
    _compare(ranks, dev)


@pytest.mark.timeout(1200)
def test_two_gpus_over_nccl_stay_identical_and_match_one_process(dev, tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    ranks = _spawn(tmp_path, "nccl", 29800 + (os.getpid() % 100))
    _compare(ranks, dev)
