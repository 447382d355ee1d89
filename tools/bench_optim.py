"""Cost of the Stage-3 optimizer step on the flat surfel store: gradient-norm clipping (max_norm 5, as trainer.py:547's
check_grad) followed by the surfel Adam step, two ways, alternating in one process:

  torch: torch.nn.utils.clip_grad_norm_(surfel params + extras, 5.0), then FlatSurfelModel.adam_step()
         -- the norm reads the 89 MB gradient buffer, the multiply reads and writes it, then Adam reads it again;
  fused: FlatSurfelModel.clip_grad_norm_(5.0, extras), then FlatSurfelModel.step()
         -- one read for the group sums of squares; the coefficient is applied inside the Adam pass.

Workload: 300 K surfels with the registration feature (7 groups, 74 floats per surfel, 22.2 M floats), plus an extras
set standing for the model's other trainable parameters: 8 tensors of 0.86 M floats in all, and a 3-value background.
Each timed call is eager, bracketed by CUDA events, with the gradients refilled and L2 flushed (256 MB written) before
it.  Algorithmic bytes of the surfel buffers (the extras are the same in both arms and left out):
  torch: 4 B x N x (1 + 2 + 4 + 3) = 40 B/float  -> 0.89 GB;   fused: 4 B x N x (1 + 4 + 3) = 32 B/float -> 0.71 GB,
over 3.35 TB/s (H100 SXM data sheet) for the bound.  Prints one JSON line with the median and p10 / p90 per arm, the
library kernels' CUDA-event times, the two arms' outputs compared at this size, and the GPU's name and power limit.

    python tools/bench_optim.py [--surfels 300000 --steps 50 --warmup 5]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

EXTRA_SHAPES = [(256, 1024), (128, 1024), (64, 1024), (64, 1024), (256, 512), (100, 1000), (32, 1024), (72, 1000)]


def _gpu_name():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True).stdout.strip().splitlines()[0]
    except Exception:
        return torch.cuda.get_device_name(0)


def _model(P, dev):
    from vidu4d_b200.surfel_store import FlatSurfelModel
    from vidu4d_b200.synthetic import object_scene
    sc = object_scene(P, seed=0, center=(0.0, 0.0, 0.0))
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    op = np.clip(sc.opacities, 1e-6, 1 - 1e-6)
    rf = torch.randn((P, 16), device=dev, generator=torch.Generator(device=dev).manual_seed(1)) * 0.1
    return FlatSurfelModel(t(sc.means3D), t(sc.shs[:, :1]), t(sc.shs[:, 1:]), t(np.log(op / (1 - op))), t(np.log(sc.scales)),
                           t(sc.rotations), regist_feat=rf)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--surfels", type=int, default=300000)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    from vidu4d_b200 import _capi
    assert torch.cuda.is_available(), "this measurement needs a GPU"
    dev = torch.device("cuda:0")
    _capi.load()
    gpu = _gpu_name()
    g = torch.Generator(device=dev).manual_seed(5)
    models = {"torch": _model(args.surfels, dev), "fused": _model(args.surfels, dev)}
    N = models["torch"].flat.numel()
    grads = torch.randn((N,), device=dev, generator=g) * 1e-2          # norm ~47: every step clips
    x0 = [torch.randn(s, device=dev, generator=g) for s in EXTRA_SHAPES] + [torch.rand(3, device=dev, generator=g)]
    extras = {k: [torch.nn.Parameter(x.clone()) for x in x0] for k in models}
    xgrads = [torch.randn(x.shape, device=dev, generator=g) * 1e-3 for x in x0]
    flush = torch.empty((256 << 20,), dtype=torch.uint8, device=dev)

    def refill(k):
        models[k].grad_flat.copy_(grads)
        for p, x in zip(extras[k], xgrads):
            p.grad = x.clone()

    def arm(k):
        m = models[k]
        if k == "torch":
            total = torch.nn.utils.clip_grad_norm_(m.flat_params() + extras[k], 5.0)
            m.adam_step()
        else:
            total = m.clip_grad_norm_(5.0, extras[k])
            m.step()
        return total

    # the two arms from the same state at this size
    totals = {}
    for k in models:
        refill(k)
        totals[k] = float(arm(k))
    a, b, m0 = models["fused"], models["torch"], _model(args.surfels, dev)
    du_a, du_b = a.flat - m0.flat, b.flat - m0.flat
    compare = {"total_norm_rel_diff": abs(totals["fused"] - totals["torch"]) / totals["torch"],
               "update_max_abs_diff_over_max_update": float((du_a - du_b).abs().max() / du_b.abs().max()),
               "exp_avg_max_abs_diff_over_max": float((a.exp_avg - b.exp_avg).abs().max() / b.exp_avg.abs().max()),
               "extra_grads_max_abs_diff": max(float((p.grad - q.grad).abs().max()) for p, q in zip(extras["fused"], extras["torch"]))}
    del m0, du_a, du_b

    for _ in range(args.warmup):
        for k in models:
            refill(k)
            arm(k)
    torch.cuda.synchronize()
    ms = {k: [] for k in models}
    for i in range(args.steps):
        for k in models:
            refill(k)
            flush.fill_(i & 255)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            arm(k)
            e1.record()
            e1.synchronize()
            ms[k].append(e0.elapsed_time(e1))
    _capi.get_profile()
    _capi.set_profiling(True)
    for i in range(10):
        for k in models:
            refill(k)
            flush.fill_(i & 255)
            arm(k)
    prof = _capi.get_profile()
    _capi.set_profiling(False)
    kern = {k: round(v["ms"] / max(v["count"], 1) * 1e3, 2) for k, v in prof.items()
            if k in ("grad_sumsq", "grad_norm_finish", "adam_step_count", "adam_flat_state", "adam_flat")}
    bytes_ = {"torch": 40 * N, "fused": 32 * N}
    stats = {k: {"median_us": round(float(np.median(v)) * 1e3, 1), "p10_us": round(float(np.percentile(v, 10)) * 1e3, 1),
                 "p90_us": round(float(np.percentile(v, 90)) * 1e3, 1)} for k, v in ms.items()}
    print(json.dumps({"workload": "clip_grad_norm_(5.0) + surfel Adam step", "surfels": args.surfels, "surfel_floats": N,
                      "extra_floats": sum(p.numel() for p in extras["torch"]), "extra_tensors": len(extras["torch"]),
                      "time_per_step": stats, "algorithmic_gb": {k: round(v / 1e9, 3) for k, v in bytes_.items()},
                      "hbm_bound_us_at_3.35TBps": {k: round(v / 3.35e12 * 1e6, 1) for k, v in bytes_.items()},
                      "kernel_us_per_launch": kern, "outputs": compare, "steps": args.steps,
                      "timing": "CUDA events around one eager call, gradients refilled and L2 flushed before each", "gpu": gpu}),
          flush=True)


if __name__ == "__main__":
    main()
