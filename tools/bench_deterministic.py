"""Cost of the deterministic rasterizer backward (include/surfel_deterministic.h, DESIGN.md 3.4b) against the default one.

Two workloads, each with F = 0 and F = 22 feature channels, at 512x512 x 8 frames and 256x256 x 2 frames, 300 K surfels
on orbiting cameras:
  * value: bench.py's value-arm step -- batched forward + backward with sums into the shared gradients;
  * loss:  a Stage-3 training step -- render_loss_batch (RGB, mask, normal and distortion terms; with F = 22 the fused
           feature and Gaussian-mask losses too), loss.backward().
Each step is captured in one CUDA graph per mode (the mode is read when the backward is recorded); the default and the
deterministic graph are replayed alternately in one process, the L2 flushed before each replay, and the median of the
CUDA-event times is reported.  Then the backward's kernels are timed per launch in each mode (sr_set_profiling, eager
calls).  One JSON line per (workload, size, F), with the GPU's name, power limit and maximum SM clock.

Usage: python tools/bench_deterministic.py [--steps 30] [--warmup 5] [--surfels 300000]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

KERNELS = ("composite_bwd", "feature_bwd", "surfel_bwd", "det_zero", "composite_bwd_det", "feature_bwd_det", "det_gather")


def _gpu():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True).stdout.strip().splitlines()[0]
    except Exception:
        return torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--surfels", type=int, default=300_000)
    args = ap.parse_args()
    from vidu4d_b200 import _capi, rasterizer as RZ
    from vidu4d_b200.graph import GraphedStep
    from vidu4d_b200.renderer import PipelineParams, make_camera, render_loss_batch, stack_cameras
    from vidu4d_b200.synthetic import SurfelCloud, object_scene, orbit_view, projection_matrix
    assert torch.cuda.is_available(), "this measurement needs a GPU"
    dev = torch.device("cuda:0")
    _capi.load()
    gpu = _gpu()
    P, TAN = args.surfels, 0.5
    scene = object_scene(P, seed=0, opacity="trained", center=(0.0, 0.0, 0.0))
    t = scene.to_torch(dev)
    flush = torch.empty((256 << 20,), dtype=torch.uint8, device=dev)
    e = torch.empty((0,), device=dev)
    C = RZ._C

    def timed(steps):
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
        return {k: float(np.median(v)) for k, v in ms.items()}

    def kernels(body):
        out = {}
        for mode in (False, True):
            RZ.set_deterministic(mode)
            body()
            torch.cuda.synchronize()
            _capi.get_profile()
            _capi.set_profiling(True)
            for _ in range(5):
                body()
            prof = _capi.get_profile()
            _capi.set_profiling(False)
            out["deterministic" if mode else "default"] = {k: round(v["ms"] / max(v["count"], 1), 4)
                                                          for k, v in prof.items() if k in KERNELS}
        RZ.set_deterministic(False)
        return out

    def compare(body):
        steps = {}
        for mode in (False, True):
            RZ.set_deterministic(mode)
            steps[mode] = GraphedStep(body, device=dev)
            steps[mode]()
        RZ.set_deterministic(False)
        ms = timed({"default": steps[False], "deterministic": steps[True]})
        return ms, kernels(body)

    for RES, M in ((512, 8), (256, 2)):
        Pm = projection_matrix(TAN, TAN).astype(np.float64)
        vms, pms, cps, cams = [], [], [], []
        for f in range(M):
            R, tt = orbit_view(f, 64)
            W2C = np.eye(4); W2C[:3, :3] = R; W2C[:3, 3] = tt
            vms.append(W2C.T.astype(np.float32)); pms.append((W2C.T @ Pm).astype(np.float32)); cps.append((-R.T @ tt).astype(np.float32))
            cams.append(make_camera(RES, RES, 2 * np.arctan(TAN), 2 * np.arctan(TAN), R=R.T, T=tt, device=dev))
        vms, pms, cps = (torch.from_numpy(np.stack(a)).to(dev) for a in (vms, pms, cps))
        bc = stack_cameras(cams)
        g = torch.Generator(device=dev).manual_seed(1234)
        dLc = torch.randn((M, 3, RES, RES), device=dev, generator=g)
        dLo = torch.randn((M, 8, RES, RES), device=dev, generator=g) * 0.1
        rgb = torch.rand((M, 3, RES, RES), device=dev, generator=g)
        mask = (torch.rand((M, RES, RES), device=dev, generator=g) > 0.5).float()
        for F in (0, 22):
            feat = torch.randn((P, F), device=dev, generator=g) * 0.3 if F else None
            dLf = torch.randn((M, F, RES, RES), device=dev, generator=g) * 0.1 if F else None
            bg = torch.zeros(3 + F, device=dev)

            def value():
                kw = {} if feat is None else {"features": feat, "concat": False}
                o = C.rasterize_gaussians_batch(bg, t["means3D"], e, t["opacities"], t["scales"], t["rotations"], 1.0, vms, pms,
                                                TAN, TAN, RES, RES, t["shs"], 3, cps, **kw)
                kb = {} if feat is None else {"features": feat, "dL_dout_features": dLf}
                C.rasterize_gaussians_backward_batch(bg, t["means3D"], o[3], e, t["scales"], t["rotations"], 1.0, vms, pms, TAN,
                                                     TAN, dLc, dLo, t["shs"], 3, cps, o[4], o[5], o[6], sum_shared=True,
                                                     want_transmat=False, **kb)

            cloud = SurfelCloud(scene, dev)
            lf = feat.clone().requires_grad_(True) if F else None
            ftgt = torch.randn((M, 16, RES, RES), device=dev, generator=g) * 0.3 if F else None
            fl = dict(features=lf, feature_target=ftgt, is_detected=torch.ones(M, device=dev), gauss_mask_channel=21,
                      feature_loss_weights=torch.tensor([1e-2, 1e-2], device=dev)) if F else {}

            def loss():
                out = render_loss_batch(bc, cloud, PipelineParams(), torch.zeros(3, device=dev), rgb, mask_gt=mask, w_mask=0.1,
                                        lambda_normal=0.05, lambda_dist=10.0, **fl)
                out["loss"].backward()

            for name, body in (("value", value), ("loss", loss)):
                ms, kern = compare(body)
                print(json.dumps({"workload": name, "surfels": P, "resolution": RES, "frames": M, "F": F,
                                  "ms_per_step_default": round(ms["default"], 4),
                                  "ms_per_step_deterministic": round(ms["deterministic"], 4),
                                  "ratio": round(ms["deterministic"] / ms["default"], 3),
                                  "kernel_ms_per_launch": kern, "steps": args.steps,
                                  "statistic": "median step time, default and deterministic graphs alternating, L2 flushed",
                                  "gpu": gpu}), flush=True)


if __name__ == "__main__":
    main()
