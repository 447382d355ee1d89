"""Cost of per-frame intrinsics (include/surfel_camera.h): a Stage-3 training step -- render_loss_batch, forward +
backward, one CUDA graph, L2 flushed between steps -- with every frame's intrinsics read from a device table
(BatchCameras.intrinsics) against the same step on the scalar path (one shared field of view passed as host floats),
alternating in one process.  The table holds the scalar path's tangents and zero offsets, so both steps compute the same
images.  Workloads: Stage-3 training (300 K surfels, 256x256, 2 frames, F = 22 feature channels) and the headline
(300 K surfels, 512x512, 8 frames).  Prints one JSON line per workload: median step times both ways, the per-launch
CUDA-event times (sr_set_profiling) of the three kernels that read the table (preprocess_fwd, surfel_bwd, loss_grad;
loss_depth for reference), and the GPU's name and power limit.

    python tools/bench_cameras.py [--steps 30 --warmup 5]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

KERNELS = ("preprocess_fwd", "surfel_bwd", "loss_depth", "loss_grad")


def _gpu_name():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True).stdout.strip().splitlines()[0]
    except Exception:
        return torch.cuda.get_device_name(0)


def _kernel_ms(body, reps=5):
    """Per-launch CUDA-event time of each kernel that reads intrinsics, over `reps` eager runs of body."""
    from vidu4d_b200 import _capi
    body()
    torch.cuda.synchronize()
    _capi.get_profile()
    _capi.set_profiling(True)
    for _ in range(reps):
        body()
    prof = _capi.get_profile()
    _capi.set_profiling(False)
    return {k: round(v["ms"] / max(v["count"], 1), 4) for k, v in prof.items() if k in KERNELS}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--surfels", type=int, default=300_000)
    args = ap.parse_args()
    from vidu4d_b200 import _capi, rasterizer as RZ
    from vidu4d_b200.graph import GraphedStep
    from vidu4d_b200.renderer import PipelineParams, make_camera, render_loss_batch, stack_cameras
    from vidu4d_b200.synthetic import SurfelCloud, object_scene, orbit_view
    assert torch.cuda.is_available(), "this measurement needs a GPU"
    dev = torch.device("cuda:0")
    _capi.load()
    gpu = _gpu_name()
    P, TAN = args.surfels, 0.5
    scene = object_scene(P, seed=0, opacity="trained", center=(0.0, 0.0, 0.0))
    flush = torch.empty((256 << 20,), dtype=torch.uint8, device=dev)
    for RES, M, F in ((256, 2, 22), (512, 8, 0)):
        cams = []
        for f in range(M):
            R, t = orbit_view(f, 64)
            cams.append(make_camera(RES, RES, 2 * np.arctan(TAN), 2 * np.arctan(TAN), R=R.T, T=t, device=dev))
        g = torch.Generator(device=dev).manual_seed(99)
        rgb = torch.rand((M, 3, RES, RES), device=dev, generator=g)
        mask = (torch.rand((M, RES, RES), device=dev, generator=g) > 0.5).float()
        pipe, bg = PipelineParams(), torch.zeros(3, device=dev)
        cloud = SurfelCloud(scene, dev)
        feat = (torch.randn((P, F), device=dev, generator=g) * 0.3).requires_grad_(True) if F else None
        scalar = stack_cameras(cams)
        table = stack_cameras(cams)
        table.intrinsics = torch.tensor([[TAN, TAN, 0.0, 0.0]] * M, device=dev)
        outs = {}

        def make_body(bc, name):
            def body():
                out = render_loss_batch(bc, cloud, pipe, bg, rgb, mask_gt=mask, w_mask=0.1, lambda_normal=0.05,
                                        lambda_dist=10.0, features=feat)
                (out["loss"] + (out["features"].square().mean() if F else 0.0)).backward()
                outs[name] = out["render"]
            return body
        bodies = {"table": make_body(table, "table"), "scalar": make_body(scalar, "scalar")}
        steps = {k: GraphedStep(b, device=dev) for k, b in bodies.items()}
        for s in steps.values():
            s()
        same = bool(torch.equal(outs["table"], outs["scalar"]))
        for s in steps.values():
            for _ in range(args.warmup):
                s(check=False)
        torch.cuda.synchronize()
        ms = {k: [] for k in steps}
        for i in range(args.steps):
            for k, s in steps.items():
                flush.fill_(i & 255)
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(); s.graph.replay(); b.record()
                b.synchronize()
                ms[k].append(a.elapsed_time(b))
        for s in steps.values():
            s.arm(); RZ.check_overflow(keep=True)
        RZ._pending.clear()
        RZ.set_sync_mode(True)
        kern = {k: _kernel_ms(b) for k, b in bodies.items()}
        med = {k: float(np.median(v)) for k, v in ms.items()}
        spread = {k: [round(float(np.percentile(v, 25)), 4), round(float(np.percentile(v, 75)), 4)] for k, v in ms.items()}
        print(json.dumps({"workload": "render_loss_batch step, per-frame camera table vs shared scalar FoV", "surfels": P,
                          "resolution": RES, "frames": M, "F": F, "ms_per_step_table": round(med["table"], 4),
                          "ms_per_step_scalar": round(med["scalar"], 4), "ms_iqr": spread,
                          "kernel_ms_per_launch": kern, "same_images": same, "steps": args.steps,
                          "statistic": "median step time", "gpu": gpu}), flush=True)
        del steps
    RZ.set_sync_mode(True)
    RZ._pending.clear()


if __name__ == "__main__":
    main()
