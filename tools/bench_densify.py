"""Cost of one step's densification statistics (trainer.py:553-560) on the flat surfel store, two ways, alternating in
one process:

  loop:  M calls of FlatSurfelModel.add_densification_stats on frame m's (P,3) gradient, (P,) filter and (P,) radii
         -- about 8 torch kernels per frame, each reading or writing the (P,) statistics again;
  fused: one add_densification_stats call on the (M,P,3) / (M,P) batch -- one sr_densify_stats kernel.

Workload: 300 K surfels, M frames of render_loss_batch-shaped inputs (60 % of the surfels visible per frame).  Each timed
call is eager, bracketed by CUDA events, with L2 flushed (256 MB written) before it.  Algorithmic bytes of the fused
kernel: the (M,P) radii, the visible frames' gradient rows and the (3,P) statistics read and written,
  4 B x P x (M + 3 M v + 6), v the visible fraction,
over 3.35 TB/s (H100 SXM data sheet) for the bound.  Prints one JSON line per M with the median and p10 / p90 per arm,
the two arms' outputs compared (they must be equal), and the GPU's name and power limit.

    python tools/bench_densify.py [--surfels 300000 --frames 2,8 --steps 100 --warmup 10]
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

VISIBLE = 0.6


def _gpu_name():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True).stdout.strip().splitlines()[0]
    except Exception:
        return torch.cuda.get_device_name(0)


def _model(P, dev):
    from vidu4d_b200.surfel_store import FlatSurfelModel
    z = lambda *s: torch.zeros(s, device=dev)  # noqa: E731
    return FlatSurfelModel(z(P, 3), z(P, 1, 3), z(P, 15, 3), z(P, 1), z(P, 2), z(P, 4))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--surfels", type=int, default=300000)
    ap.add_argument("--frames", default="2,8")
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    from vidu4d_b200 import _capi
    assert torch.cuda.is_available(), "this measurement needs a GPU"
    dev = torch.device("cuda:0")
    _capi.load()
    gpu = _gpu_name()
    flush = torch.empty((256 << 20,), dtype=torch.uint8, device=dev)
    P = args.surfels
    for M in (int(x) for x in args.frames.split(",")):
        g = torch.Generator(device=dev).manual_seed(M)
        grad = torch.randn((M, P, 3), device=dev, generator=g) * 1e-4
        radii = torch.randint(1, 60, (M, P), device=dev, generator=g, dtype=torch.int32)
        radii[torch.rand((M, P), device=dev, generator=g) >= VISIBLE] = 0
        vis = radii > 0
        scale = 1.0 / M
        models = {"loop": _model(P, dev), "fused": _model(P, dev)}

        def arm(k):
            m = models[k]
            if k == "loop":
                for f in range(M):
                    m.add_densification_stats(grad[f] * scale, vis[f], radii[f])
            else:
                m.add_densification_stats(grad, vis, radii, grad_scale=scale)

        for _ in range(args.warmup):
            for k in models:
                arm(k)
        torch.cuda.synchronize()
        same = all(torch.equal(getattr(models["loop"], a), getattr(models["fused"], a)) for a in ("densify_stats", "max_radii2D"))
        ms = {k: [] for k in models}
        for i in range(args.steps):
            for k in models:
                flush.fill_(i & 255)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                arm(k)
                e1.record()
                e1.synchronize()
                ms[k].append(e0.elapsed_time(e1))
        nbytes = 4 * P * (M + 3 * M * VISIBLE + 6)
        stats = {k: {"median_us": round(float(np.median(v)) * 1e3, 1), "p10_us": round(float(np.percentile(v, 10)) * 1e3, 1),
                     "p90_us": round(float(np.percentile(v, 90)) * 1e3, 1)} for k, v in ms.items()}
        print(json.dumps({"workload": "densification statistics of one step", "surfels": P, "frames": M, "visible": VISIBLE,
                          "time_per_step": stats, "speedup_median": round(stats["loop"]["median_us"] / stats["fused"]["median_us"], 2),
                          "fused_algorithmic_mb": round(nbytes / 1e6, 2),
                          "fused_hbm_bound_us_at_3.35TBps": round(nbytes / 3.35e12 * 1e6, 1),
                          "outputs_equal": same, "steps": args.steps,
                          "timing": "CUDA events around one eager call, L2 flushed before each", "gpu": gpu}), flush=True)


if __name__ == "__main__":
    main()
