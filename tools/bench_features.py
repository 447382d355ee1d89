"""Cost of per-surfel feature channels on the headline workload: the batched step of bench.py's value arm (300 K surfels,
512x512, 8 frames on orbiting cameras, forward + backward + frame sums into shared gradients, one CUDA graph, L2 flushed
between steps) with F feature channels, and the colour-only step timed the same way in the same process, alternating.
Prints one JSON line per F: fwd+bwd frames/s both ways, and the feature / composite kernels' CUDA-event times
(sr_set_profiling), with the GPU's name and power limit.

    python tools/bench_features.py --features 4 22 32 [--steps 20 --warmup 5]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--features", type=int, nargs="+", default=[22])
    ap.add_argument("--surfels", type=int, default=300_000)
    ap.add_argument("--res", type=int, default=512)
    ap.add_argument("--frames", type=int, default=8)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    from vidu4d_b200 import _capi, rasterizer as RZ
    from vidu4d_b200.graph import GraphedStep
    from vidu4d_b200.synthetic import object_scene, orbit_view, projection_matrix
    assert torch.cuda.is_available(), "this measurement needs a GPU"
    dev = torch.device("cuda:0")
    _capi.load()
    M, RES, P, TAN = args.frames, args.res, args.surfels, 0.5
    t = object_scene(P, seed=0, opacity="trained", center=(0.0, 0.0, 0.0)).to_torch(dev)
    Pm = projection_matrix(TAN, TAN).astype(np.float64)
    vms, pms, cps = [], [], []
    for f in range(M):
        R, tt = orbit_view(f, 64)
        W2C = np.eye(4); W2C[:3, :3] = R; W2C[:3, 3] = tt
        vms.append(W2C.T.astype(np.float32)); pms.append((W2C.T @ Pm).astype(np.float32)); cps.append((-R.T @ tt).astype(np.float32))
    vms, pms, cps = (torch.from_numpy(np.stack(a)).to(dev) for a in (vms, pms, cps))
    e = torch.empty((0,), device=dev)
    gen = torch.Generator(device=dev).manual_seed(1234)
    dLc = torch.randn((M, 3, RES, RES), device=dev, generator=gen)
    dLo = torch.randn((M, 8, RES, RES), device=dev, generator=gen) * 0.1
    flush = torch.empty((256 << 20,), dtype=torch.uint8, device=dev)
    C = RZ._C
    try:
        gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True).stdout.strip().splitlines()[0]
    except Exception:
        gpu = torch.cuda.get_device_name(dev)

    def make_body(feat, dLf):
        bg = torch.zeros(3 + (0 if feat is None else feat.shape[1]), device=dev)

        def body():
            kw = {} if feat is None else {"features": feat, "concat": False}
            o = C.rasterize_gaussians_batch(bg, t["means3D"], e, t["opacities"], t["scales"], t["rotations"], 1.0, vms, pms,
                                            TAN, TAN, RES, RES, t["shs"], 3, cps, **kw)
            kb = {} if feat is None else {"features": feat, "dL_dout_features": dLf}
            C.rasterize_gaussians_backward_batch(bg, t["means3D"], o[3], e, t["scales"], t["rotations"], 1.0, vms, pms, TAN,
                                                 TAN, dLc, dLo, t["shs"], 3, cps, o[4], o[5], o[6], sum_shared=True,
                                                 want_transmat=False, **kb)
        return body

    def timed(steps):
        """steps: {name: GraphedStep}; replays them alternately, L2 flushed before each; returns ms per step."""
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
        return {k: float(np.median(v)) for k, v in ms.items()}

    base = GraphedStep(make_body(None, None), device=dev)
    base()
    for F in args.features:
        g = torch.Generator(device=dev).manual_seed(4321)
        feat = torch.randn((P, F), device=dev, generator=g)
        dLf = torch.randn((M, F, RES, RES), device=dev, generator=g) * 0.1
        body = make_body(feat, dLf)
        step = GraphedStep(body, device=dev)
        step()
        ms = timed({"features": step, "colour": base})
        RZ._pending.clear()
        RZ.set_sync_mode(True)
        body()
        torch.cuda.synchronize()
        _capi.get_profile()
        _capi.set_profiling(True)
        for _ in range(3):
            body()
        prof = _capi.get_profile()
        _capi.set_profiling(False)
        kern = {k: round(v["ms"] / max(v["count"], 1), 4) for k, v in prof.items()
                if k in ("feature_fwd", "feature_bwd", "composite_fwd", "composite_bwd")}
        print(json.dumps({"F": F, "fps": round(M / (ms["features"] * 1e-3), 1),
                          "fps_colour_only": round(M / (ms["colour"] * 1e-3), 1),
                          "ms_per_step": round(ms["features"], 4), "ms_per_step_colour_only": round(ms["colour"], 4),
                          "launches_per_step": step.launches, "launches_per_step_colour_only": base.launches,
                          "kernel_ms_per_launch": kern, "frames_per_launch": M, "surfels": P, "resolution": RES,
                          "steps": args.steps, "statistic": "median step time", "gpu": gpu}), flush=True)
    RZ.set_sync_mode(True)
    RZ._pending.clear()


if __name__ == "__main__":
    main()
