"""GPU: FlatSurfelModel checkpoints in a training run.

  * exact resume: a captured Stage-3 step (render_loss_batch -> backward -> densification statistics -> clip -> step())
    with the deterministic rasterizer backward and one densify_and_prune; a store built afresh at another P that loads
    the checkpoint of step 6 reaches step 18 with the uninterrupted run's bits -- parameters, both moments, step count,
    statistics -- and so does the live store, its graph still captured, after an in-place load of step 16's checkpoint;
    every step's loss agrees to a few ulp (below);
  * a store built from torch.optim.Adam's state continues as torch's Adam does, within tests/optim_model.py's bound;
  * after the reference's load_checkpoint sequence (trainer.py:386-396) the store still trains;
  * two ranks over gloo on one GPU: rank 0 saves, both load, and the replicas agree.

Losses are recorded by device_step inside the step itself (index_copy_ at the step count), so eager bodies and replays
write them alike; a GraphedStep capture runs its body five times (one sync pass, two warm-ups, one side-stream pass,
then the replay).  The loss scalar itself is not bit-reproducible: the loss pass sums each frame's terms with float
atomics (loss.cu), which the deterministic mode (a backward-only switch) leaves as they are.  Its gradients are, and
they are what the resumed state is made of."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from . import optim_model as om
from .conftest import ROOT

pytestmark = pytest.mark.gpu

M, W, H = 2, 96, 96
MAX_NORM = 0.5
LRS = {"xyz": 1e-4, "f_dc": 2.5e-3, "f_rest": 1.25e-4, "opacity": 5e-2, "scaling": 5e-3, "rotation": 1e-3}


@pytest.fixture(scope="module")
def dev(built):
    from vidu4d_b200 import _capi
    _capi.load()
    return torch.device("cuda:0")


def _model(P, dev, seed=0):
    from vidu4d_b200.surfel_store import FlatSurfelModel
    from vidu4d_b200.synthetic import object_scene
    sc = object_scene(P, seed=seed, center=(0.0, 0.0, 0.0))
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    op = np.clip(sc.opacities, 1e-6, 1 - 1e-6)
    return FlatSurfelModel(t(sc.means3D), t(sc.shs[:, :1]), t(sc.shs[:, 1:]), t(np.log(op / (1 - op))), t(np.log(sc.scales)),
                           t(sc.rotations), lrs=dict(LRS))


def _data(dev, seed=5):
    from vidu4d_b200.renderer import PipelineParams, make_camera, stack_cameras
    from vidu4d_b200.synthetic import orbit_view
    cams = []
    for f in range(M):
        R, t = orbit_view(7 * f + 3, 64)
        cams.append(make_camera(W, H, 2 * np.arctan(0.5), 2 * np.arctan(0.5), R=R.T, T=t, device=dev))
    g = torch.Generator(device=dev).manual_seed(seed)
    return dict(cams=stack_cameras(cams), pipe=PipelineParams(), bg=torch.zeros(3, device=dev),
                rgb=torch.rand((M, 3, H, W), device=dev, generator=g),
                mask=(torch.rand((M, H, W), device=dev, generator=g) > 0.4).float())


def _loss(m, d):
    from vidu4d_b200.renderer import render_loss_batch
    out = render_loss_batch(d["cams"], m, d["pipe"], d["bg"], d["rgb"], mask_gt=d["mask"], w_mask=0.1)
    out["loss"].backward()
    return out


def _body(m, d, losses):
    m.zero_grad_flat()
    out = _loss(m, d)
    m.add_densification_stats(out["viewspace_points"].grad, out["visibility_filter"], out["radii"])
    m.clip_grad_norm_(MAX_NORM)
    losses.index_copy_(0, m.device_step.view(1), out["loss"].detach().float().view(1))
    m.step()


def _graphed(m, d, losses, dev):
    from vidu4d_b200.graph import GraphedStep
    return GraphedStep(lambda: _body(m, d, losses), key=lambda: (m.P, m.active_sh_degree), device=dev)


def _call(gs, m, want_step, want_captures):
    gs()
    assert int(m.device_step) == want_step and gs.captures == want_captures, (int(m.device_step), gs.captures)


def _densify(m, dev):
    ratio = torch.nan_to_num(m.xyz_gradient_accum[:, 0] / m.denom[:, 0], nan=0.0)
    thr = float(torch.quantile(ratio[m.denom[:, 0] > 0], 0.7))
    P0 = m.P
    m.densify_and_prune(thr, 0.005, 0.55, None, generator=torch.Generator(device=dev).manual_seed(9))
    assert m.P != P0


def _snapshot(m):
    return {k: v.detach().clone() for k, v in m.state_dict().items()}


def _same(got, want, what):
    assert got.keys() == want.keys()
    for k in want:
        a, b = got[k], want[k]
        assert a.shape == b.shape and a.dtype == b.dtype, (what, k, a.shape, b.shape)
        n = int((a.reshape(-1).view(torch.uint8) != b.reshape(-1).view(torch.uint8)).sum())
        assert n == 0, f"{what}: {k} differs in {n} bytes of {a.numel() * a.element_size()}"


def _close_losses(got, want, what):
    """Within 8 ulp: the order of the loss pass's float atomic sums is the only difference."""
    err = (got.double() - want.double()).abs()
    assert bool((err <= 8 * 2.0 ** -23 * want.double().abs()).all()), (what, err.max().item())


def test_exact_resume_from_a_checkpoint(dev, tmp_path):
    from vidu4d_b200 import rasterizer as RZ
    d = _data(dev)
    RZ.set_deterministic(True)
    try:
        # the uninterrupted run: capture (steps 1-5), replays, densify at 11, re-capture (12-16), replays to 18
        m = _model(20000, dev, seed=1)
        losses = torch.zeros(32, device=dev)
        gs = _graphed(m, d, losses, dev)
        _call(gs, m, 5, 1)
        _call(gs, m, 6, 1)
        torch.save(m.state_dict(), tmp_path / "ck6.pt")
        for s in range(7, 12):
            _call(gs, m, s, 1)
        _densify(m, dev)
        _call(gs, m, 16, 2)
        ck16 = _snapshot(m)
        _call(gs, m, 17, 2)
        _call(gs, m, 18, 2)
        ck18, loss18 = _snapshot(m), losses.clone()
        assert bool((loss18[:18] > 0).all())

        # a fresh store of another size resumes at step 6 and meets the same densification at step 11
        r = _model(12345, dev, seed=2)
        r.load_state_dict(torch.load(tmp_path / "ck6.pt", map_location=dev, weights_only=True))
        assert r.P == 20000 and int(r.device_step) == 6
        rl = torch.zeros(32, device=dev)
        gr = _graphed(r, d, rl, dev)
        _call(gr, r, 11, 1)
        _densify(r, dev)
        _call(gr, r, 16, 2)
        _call(gr, r, 17, 2)
        _call(gr, r, 18, 2)
        _same(_snapshot(r), ck18, "resumed run")
        _close_losses(rl[6:18], loss18[6:18], "resumed run")

        # the live store rewinds to step 16 in place: same P, same addresses, the captured graph replays on
        ptrs = [t.data_ptr() for t in (m.flat, m.grad_flat, m.exp_avg, m.exp_avg_sq, m.device_step, m.densify_stats)]
        m.load_state_dict(ck16)
        assert ptrs == [t.data_ptr() for t in (m.flat, m.grad_flat, m.exp_avg, m.exp_avg_sq, m.device_step, m.densify_stats)]
        _call(gs, m, 17, 2)
        _call(gs, m, 18, 2)
        _same(_snapshot(m), ck18, "in-place load into the captured store")
        _close_losses(losses[16:18], loss18[16:18], "in-place load into the captured store")
    finally:
        RZ.set_deterministic(False)
        RZ.set_sync_mode(True)
        RZ._pending.clear()


class _GaussianModel(torch.nn.Module):
    """The reference's parameter attributes (gaussian_model.py), from a store's values."""

    def __init__(self, m):
        super().__init__()
        for a, p in zip(("_xyz", "_features_dc", "_features_rest", "_opacity", "_scaling", "_rotation"), m.flat_params()):
            setattr(self, a, torch.nn.Parameter(p.detach().clone()))
        self.active_sh_degree, self.percent_dense = m.active_sh_degree, m.percent_dense


@pytest.mark.parametrize("rates", ["stage3", "fp32"])
def test_continuing_from_torch_adam(rates, dev):
    """Three torch Adam steps on a reference-layout model, then from_gaussian_model(gm, optimizer) and five more steps
    on both, on the same gradients: the moments stay torch's bit for bit, and each parameter update is inside the rate's
    rounding of torch's (both start each step from torch's parameters); with fp32 rates the parameters stay torch's bit
    for bit on their own."""
    from vidu4d_b200.surfel_store import FlatSurfelModel
    lrs = {n: (float(np.float32(v)) if rates == "fp32" else v) for n, v in LRS.items()}
    gm = _GaussianModel(_model(5003, dev, seed=3))
    names = list(LRS)
    params = [getattr(gm, a) for a in ("_xyz", "_features_dc", "_features_rest", "_opacity", "_scaling", "_rotation")]
    opt = torch.optim.Adam([{"params": [p], "lr": lrs[n], "name": n} for p, n in zip(params, names)], lr=0.0, eps=1e-15,
                           foreach=True)
    gen = torch.Generator(device=dev).manual_seed(4)
    grads = lambda: [torch.randn(p.shape, device=dev, generator=gen) * 1e-2 for p in params]  # noqa: E731
    for _ in range(3):
        for p, g in zip(params, grads()):
            p.grad = g
        opt.step()
    m = FlatSurfelModel.from_gaussian_model(gm, opt)
    assert int(m.device_step) == 3 and m.lrs == lrs
    for step in range(4, 9):
        gs = grads()
        for p, g, q in zip(params, gs, m.flat_params()):
            p.grad = g
            q.grad.copy_(g)
        before = torch.cat([p.detach().flatten() for p in params])
        if rates != "fp32":
            with torch.no_grad():
                m.flat.copy_(before)
        m.step()
        opt.step()
        assert int(m.device_step) == step
        for key, buf in (("exp_avg", m.exp_avg), ("exp_avg_sq", m.exp_avg_sq)):
            want = torch.cat([opt.state[p][key].flatten() for p in params])
            assert torch.equal(buf, want), (step, key, int((buf != want).sum()))
        pk, pt = m.flat, torch.cat([p.detach().flatten() for p in params])
        if rates == "fp32":
            assert torch.equal(pk, pt), (step, int((pk != pt).sum()))
        else:
            assert om.rate_rounding_ok(pk.cpu().numpy(), pt.cpu().numpy(), before.cpu().numpy()).all(), step


def test_reference_load_sequence_keeps_training(dev):
    """trainer.py:386-396 on a live store (at another P, then load_state_dict): a backward lands in grad_flat, and
    step() changes what the next render reads."""
    src = _model(9000, dev, seed=6)
    src.logscale = torch.nn.Parameter(torch.tensor([0.3], device=dev))
    states = {"fields.field_params.fg." + k: v for k, v in src.state_dict().items()}
    m = _model(15000, dev, seed=7)
    model = torch.nn.Module()
    model.fields = torch.nn.Module()
    model.fields.field_params = torch.nn.ModuleDict({"fg": m})
    scale = torch.tensor([1])  # scale of the field
    model.fields.field_params.fg.logscale = torch.nn.Parameter(scale.log())
    num_pts = states["fields.field_params.fg._xyz"].shape[0]
    new_xyz = model.fields.field_params.fg._xyz[:num_pts].clone().detach()
    model.fields.field_params.fg._xyz = torch.nn.Parameter(new_xyz)
    model.fields.field_params.fg._xyz = torch.nn.Parameter(model.fields.field_params.fg._xyz[:num_pts].clone().detach())
    model.fields.field_params.fg._features_dc = torch.nn.Parameter(model.fields.field_params.fg._features_dc[:num_pts].clone().detach())
    model.fields.field_params.fg._features_rest = torch.nn.Parameter(model.fields.field_params.fg._features_rest[:num_pts].clone().detach())
    model.fields.field_params.fg._opacity = torch.nn.Parameter(model.fields.field_params.fg._opacity[:num_pts].clone().detach())
    model.fields.field_params.fg._scaling = torch.nn.Parameter(model.fields.field_params.fg._scaling[:num_pts].clone().detach())
    model.fields.field_params.fg._rotation = torch.nn.Parameter(model.fields.field_params.fg._rotation[:num_pts].clone().detach())
    model.load_state_dict(states, strict=False)
    assert m.P == 9000 and torch.equal(m.flat, src.flat) and float(m.logscale.detach()) == np.float32(0.3)
    d = _data(dev)
    m.zero_grad_flat()
    out = _loss(m, d)
    assert float(m.grad_flat.abs().max()) > 0 and all(p.grad.data_ptr() >= m.grad_flat.data_ptr() for p in m.flat_params())
    loss0 = float(out["loss"].detach())
    m.step()
    m.zero_grad_flat()
    loss1 = float(_loss(m, d)["loss"].detach())
    assert loss1 != loss0 and not torch.equal(m.flat, src.flat)


# ---- two ranks on one GPU ---------------------------------------------------------------------------------------------------
def _worker(rank, world, port, path):
    sys.path.insert(0, ROOT)
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    from vidu4d_b200 import _capi
    from vidu4d_b200 import distributed as D
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    _capi.load()
    D.init_distributed("gloo")
    m = _model(8000 + 1000 * rank, dev, seed=10 + rank)         # the ranks start apart: only the checkpoint joins them
    if rank == 0:
        src = _model(6000, dev, seed=20)
        src.exp_avg.normal_()
        src.device_step.fill_(42)
        src.densify_and_prune(1e9, 0.005, 0.55, None)           # statistics reset, as right after a densification
        torch.save(src.state_dict(), path)
    dist.barrier()
    m.load_state_dict(torch.load(path, map_location=dev, weights_only=True))
    D.check_replicas(m.replica_state())
    assert m.P == 6000 and int(m.device_step) == 42
    dist.destroy_process_group()


@pytest.mark.timeout(600)
def test_two_ranks_load_rank_zeros_checkpoint(dev, tmp_path):
    port = 29300 + (os.getpid() % 100)
    ctx = mp.start_processes(_worker, args=(2, port, str(tmp_path / "ck.pt")), nprocs=2, join=False, start_method="spawn")
    import time
    deadline = time.time() + 500
    while not ctx.join(timeout=5):
        if time.time() > deadline:
            for p in ctx.processes:
                p.kill()
            raise TimeoutError("the two ranks did not finish in 500 s")
