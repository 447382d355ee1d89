"""2-GPU NCCL test of SURVEY.md section 8(e)'s parity check with the CUDA path: frames sharded over two ranks, each rank
renders its frames with ONE batched launch set (render_loss_batch), gradients land in the flat buffer, one NCCL
all-reduce -- the summed FlatGrads must equal one GPU looping over the same frames, to 1e-5 relative (fp32 summation
order).  Skipped on machines with fewer than 2 GPUs."""
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


def _setup(dev):
    from vidu4d_b200.renderer import PipelineParams, make_camera, stack_cameras
    from vidu4d_b200.synthetic import SurfelCloud, object_scene, orbit_view
    cloud = SurfelCloud(object_scene(P, seed=3, center=(0.0, 0.0, 0.0)), dev)
    cams = []
    for f in range(NF):
        R, t = orbit_view(7 * f + 1, 64)
        cams.append(make_camera(W, H, 2 * np.arctan(0.5), 2 * np.arctan(0.375), R=R.T, T=t, device=dev))
    g = torch.Generator().manual_seed(11)
    target = torch.rand((NF, 3, H, W), generator=g).to(dev)
    return cloud, cams, target, PipelineParams(), stack_cameras


def _grads_of_frames(frames, dev):
    from vidu4d_b200 import distributed as D
    from vidu4d_b200.renderer import render_loss_batch
    cloud, cams, target, pipe, stack = _setup(dev)
    fg = D.FlatGrads(cloud.flat_params())
    out = render_loss_batch(stack([cams[f] for f in frames]), cloud, pipe, torch.zeros(3, device=dev), target[frames],
                            w_rgb=1.0, lambda_normal=0.05, lambda_dist=0.01)
    out["loss"].backward()
    return fg


def _worker(rank, world, port, out):
    sys.path.insert(0, ROOT)
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    from vidu4d_b200 import distributed as D
    dev = torch.device("cuda", rank)
    torch.cuda.set_device(dev)
    D.init_distributed("nccl", dev)
    fg = _grads_of_frames(D.shard_frames(NF, rank, world), dev)
    flat = fg.allreduce_(average_over=NF)
    torch.cuda.synchronize()
    if rank == 0:
        np.save(out, flat.cpu().numpy())
    dist.destroy_process_group()


@pytest.mark.timeout(600)
def test_two_gpu_nccl_allreduce_equals_one_gpu_loop(built, tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    out = str(tmp_path / "flat.npy")
    port = 29700 + (os.getpid() % 200)
    mp.start_processes(_worker, args=(2, port, out), nprocs=2, join=True, start_method="spawn")
    got = np.load(out)
    dev = torch.device("cuda:0")
    # one GPU, the same 8 frames in two sequential batches of 4 (another summation order on purpose)
    a = _grads_of_frames([0, 1, 2, 3], dev).flat.double()
    b = _grads_of_frames([4, 5, 6, 7], dev).flat.double()
    want = ((a + b) / NF).cpu().numpy()
    scale = np.abs(want).max()
    assert scale > 0 and np.abs(got - want).max() <= 1e-5 * scale
