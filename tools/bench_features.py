"""Cost of per-surfel feature channels on the headline workload: the batched step of bench.py's value arm (300 K surfels,
512x512, 8 frames on orbiting cameras, forward + backward + frame sums into shared gradients, one CUDA graph, L2 flushed
between steps) with F feature channels, and the colour-only step timed the same way in the same process, alternating.
Prints one JSON line per F: fwd+bwd frames/s both ways, and the feature / composite kernels' CUDA-event times
(sr_set_profiling), with the GPU's name and power limit.

--losses times instead a Stage-3 training step -- render_loss_batch over 300 K surfels with F = 22 channels, forward +
backward, one CUDA graph -- with the feature and Gaussian-mask losses fused (csrc/loss.cu) against the same losses
written in torch on out["features"], alternating in one process, at 256x256 x 2 frames (Stage-3 training) and
512x512 x 8 frames (headline).  The torch version uses the sync-free form of the reference's positive mean
(sum(v * (v > 0)) / max(count, 1), equal to it for v >= 0), so that it can be captured too.

    python tools/bench_features.py --features 4 22 32 [--steps 20 --warmup 5]
    python tools/bench_features.py --losses [--steps 20 --warmup 5]
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
    ap.add_argument("--losses", action="store_true")
    args = ap.parse_args()
    if args.losses:
        return bench_losses(args)
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
    gpu = _gpu_name()

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


def _gpu_name():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True).stdout.strip().splitlines()[0]
    except Exception:
        return torch.cuda.get_device_name(0)


def _torch_feature_terms(planes, alpha, target, mask, det, gm, w):
    """lab4d/engine/model.py:663-667,742-745,952-967,1000-1012 in torch, without the host sync of v[v > 0]."""
    def positive_mean(v):
        on = (v > 0).to(v.dtype)
        return (v * on).sum() / on.sum().clamp(min=1.0)
    v = (planes[:, :target.shape[1]] - target).norm(2, 1) * mask * det[:, None, None]
    return w[0] * positive_mean(v) + w[1] * positive_mean((planes[:, gm] - alpha.detach()).pow(2))


def bench_losses(args):
    from vidu4d_b200 import _capi, rasterizer as RZ
    from vidu4d_b200.graph import GraphedStep
    from vidu4d_b200.renderer import PipelineParams, make_camera, render_loss_batch, stack_cameras
    from vidu4d_b200.synthetic import SurfelCloud, object_scene, orbit_view
    assert torch.cuda.is_available(), "this measurement needs a GPU"
    dev = torch.device("cuda:0")
    _capi.load()
    gpu = _gpu_name()
    P, F, Cf, GM = args.surfels, 22, 16, 21
    scene = object_scene(P, seed=0, opacity="trained", center=(0.0, 0.0, 0.0))
    flush = torch.empty((256 << 20,), dtype=torch.uint8, device=dev)
    for RES, M in ((256, 2), (512, 8)):
        cams = []
        for f in range(M):
            R, t = orbit_view(f, 64)
            cams.append(make_camera(RES, RES, 2 * np.arctan(0.5), 2 * np.arctan(0.5), R=R.T, T=t, device=dev))
        bc = stack_cameras(cams)
        g = torch.Generator(device=dev).manual_seed(99)
        rgb = torch.rand((M, 3, RES, RES), device=dev, generator=g)
        ftgt = torch.randn((M, Cf, RES, RES), device=dev, generator=g) * 0.3
        mask = (torch.rand((M, RES, RES), device=dev, generator=g) > 0.5).float()
        det = torch.ones(M, device=dev)
        w = torch.tensor([1e-2, 1e-2], device=dev)
        pipe, bg = PipelineParams(), torch.zeros(3, device=dev)
        cloud = SurfelCloud(scene, dev)
        feat = (torch.randn((P, F), device=dev, generator=g) * 0.3).requires_grad_(True)

        def make_body(fused):
            def body():
                extra = dict(feature_target=ftgt, is_detected=det, gauss_mask_channel=GM, feature_loss_weights=w) if fused else {}
                out = render_loss_batch(bc, cloud, pipe, bg, rgb, mask_gt=mask, w_mask=0.1, lambda_normal=0.05,
                                        lambda_dist=10.0, features=feat, **extra)
                loss = out["loss"] if fused else out["loss"] + _torch_feature_terms(out["features"], out["allmap"][:, 1], ftgt,
                                                                                    mask, det, GM, w)
                loss.backward()
            return body
        bodies = {"fused": make_body(True), "torch": make_body(False)}
        steps = {k: GraphedStep(b, device=dev) for k, b in bodies.items()}
        for s in steps.values():
            s()
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
        bodies["fused"]()
        torch.cuda.synchronize()
        _capi.get_profile()
        _capi.set_profiling(True)
        for _ in range(5):
            bodies["fused"]()
        prof = _capi.get_profile()
        _capi.set_profiling(False)
        kern = {k: round(v["ms"] / max(v["count"], 1), 4) for k, v in prof.items()
                if k in ("feat_loss", "feat_loss_scale", "loss_grad", "feature_fwd", "feature_bwd")}
        med = {k: float(np.median(v)) for k, v in ms.items()}
        print(json.dumps({"workload": "render_loss_batch step with feature losses", "surfels": P, "resolution": RES,
                          "frames": M, "F": F, "ms_per_step_fused": round(med["fused"], 4),
                          "ms_per_step_torch": round(med["torch"], 4), "fps_fused": round(M / (med["fused"] * 1e-3), 1),
                          "fps_torch": round(M / (med["torch"] * 1e-3), 1), "launches_per_step_fused": steps["fused"].launches,
                          "kernel_ms_per_launch": kern, "steps": args.steps, "statistic": "median step time",
                          "gpu": gpu}), flush=True)
    RZ.set_sync_mode(True)
    RZ._pending.clear()


if __name__ == "__main__":
    main()
