"""Cost of Stage 3's periodic radius outlier filter (lab4d/engine/trainer.py:573-588: `remove_radius_outlier(nb_points=20,
radius=0.004)`) on the device, against the host path the reference takes.

GPU: `knn.radius_outlier_mask` (csrc/outlier.cu) on a (P,3) CUDA tensor, CUDA events around `--reps` calls after
`--warmup` calls; the median per call is reported.  Host: what the reference does -- a device-to-host copy of the
surfel centres, then a CPU KD-tree radius count.  Open3D is not available, so scipy's cKDTree
(`query_ball_point(..., return_length=True)`, all cores) stands in for Open3D's KD-tree; its time is labelled as a
stand-in.  Host times are wall-clock medians over `--host-reps` runs, the copy included.  Scenes: a Stage-3-like shell
with 1 % scattered strays (synthetic.shell_with_strays) at 200 K, 300 K and 1 M surfels.  Also reported: the scratch
the call needs (sr_radius_outlier_scratch_bytes) and the peak of torch's allocator above the input during one call,
and whether the stand-in's decision agrees with the kernel's (they can differ only on pairs at exactly the radius).
Prints one JSON line per size, each with the GPU's name, power limit and max SM clock from the same run.

Usage: python tools/bench_outliers.py [--sizes 200000 300000 1000000] [--reps 20] [--warmup 5] [--host-reps 3]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

NB, R = 20, 0.004


def _gpu_name():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True).stdout.strip().splitlines()[0]
    except Exception:
        return torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[200_000, 300_000, 1_000_000])
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--host-reps", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_outliers.py needs a CUDA device")
    from scipy.spatial import cKDTree
    from vidu4d_b200 import _capi
    from vidu4d_b200.knn import radius_outlier_mask
    from vidu4d_b200.synthetic import shell_with_strays
    lib = _capi.load()
    dev = torch.device("cuda:0")
    gpu = _gpu_name()
    for P in a.sizes:
        x = torch.from_numpy(shell_with_strays(P, seed=P)).to(dev)
        for _ in range(a.warmup):
            prune = radius_outlier_mask(x, NB, R)
        torch.cuda.synchronize(dev)
        times = []
        for _ in range(a.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            prune = radius_outlier_mask(x, NB, R)
            e1.record()
            e1.synchronize()
            times.append(e0.elapsed_time(e1))
        torch.cuda.synchronize(dev)
        torch.cuda.reset_peak_memory_stats(dev)
        base = torch.cuda.memory_allocated(dev)
        radius_outlier_mask(x, NB, R)
        torch.cuda.synchronize(dev)
        peak = torch.cuda.max_memory_allocated(dev) - base
        host = []
        for _ in range(a.host_reps):
            t0 = time.perf_counter()
            xyz = x.cpu().numpy().astype(np.float64)
            n = cKDTree(xyz).query_ball_point(xyz, R, return_length=True, workers=-1)
            host.append((time.perf_counter() - t0) * 1e3)
        host_prune = n <= NB
        gpu_prune = prune.cpu().numpy()
        print(json.dumps({
            "P": P, "nb_points": NB, "radius": R, "gpu": gpu,
            "gpu_ms_median": round(statistics.median(times), 4), "gpu_ms_min": round(min(times), 4),
            "host_kdtree_standin_ms_median": round(statistics.median(host), 1),
            "host_standin": "D2H copy + scipy cKDTree query_ball_point (stand-in for Open3D's KD-tree), all cores",
            "host_cores": os.cpu_count(),
            "pruned": int(gpu_prune.sum()), "standin_disagreements": int((host_prune != gpu_prune).sum()),
            "scratch_bytes": int(lib.sr_radius_outlier_scratch_bytes(P)), "peak_alloc_bytes": int(peak),
        }), flush=True)


if __name__ == "__main__":
    main()
