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

--reproj times Stage 3's feature-matching reprojection loss: global_match over 2048 candidates + warp + projection +
feat_reproj loss, forward + backward, one CUDA graph, L2 flushed between steps, fused (csrc/match.cu) against the same
statements in torch (global_match's score matrix + topk, oracle/warp_oracle.py in fp32, projection, the sync-free
positive mean), alternating in one process, at 256x256 x 2 frames with 300 K surfels; and the fused path alone at
512x512 x 8 frames, where the torch path's score matrix alone is 17 GB.

--cycle times Stage 3's deformation-cycle regulariser: the fused forward warp (bob_warp) -> cycle loss -> backward at
300 K surfels, B = 25 with delta, M = 2 and M = 8, one CUDA graph, L2 flushed between steps, with the cycle loss fused
(csrc/cycle.cu) against the same statements in torch (tests/cycle_model.py cycle_values in fp32 and the sync-free
positive means), alternating in one process.

--rows times Stage 3's per-surfel feature rows alone: [regist | flow / s | normal | Gaussian-bone density] for every
frame, forward + backward with seeded upstream gradients, at 300 K surfels, B = 25, Cf = 16, M = 2 and M = 8, one CUDA
graph, L2 flushed between steps, fused (csrc/feature_rows.cu) against the reference's statements in fp32 torch
(tests/feature_rows_model.py), alternating in one process.

--ssim times the fused SSIM op (csrc/ssim.cu), forward + backward of 1 - ssim(img1, img2), one CUDA graph, L2 flushed
between steps, against an independently written torch expression of the same formula (conv2d with the 11x11 window and
groups=C), alternating in one process, at 1x3x512^2, 8x3x512^2 and 1x3x1080x1920; then a render_loss_batch step (300 K
surfels, 512x512, 8 frames) with w_ssim = 0 and 0.2.  The op's algorithmic bound, per channel-pixel: the forward reads
x and y (8 B) and writes the three gradient maps (12 B); the backward reads the maps, x and y (20 B) and writes dL/dx
(4 B), so 44 B in all; about 400 FLOP (five 11-tap passes each way, two for each of the five forward and three backward
quantities, plus the per-pixel formula).  Printed with each size: the bytes / 3.35 TB/s and FLOP / 67 TFLOP/s bounds
(H100 SXM data sheet) and the measured share of the larger.

--mask times a Stage-3 training step -- render_loss_batch over 300 K surfels, forward + backward -- with the silhouette
term as the reference weighs it (batch balance weights, vis2d and is_detected masks, positive mean over the batch): fused
(csrc/mask_loss.cu, mask_loss_weight=) with the whole step captured in one CUDA graph, against the reference's torch
statements on out["allmap"][:, 1] run eagerly (they synchronise with the host, so that step cannot be captured),
alternating in one process, at 256x256 x 2 frames (Stage-3 training) and 512x512 x 8 frames (headline).  Reports step
times from CUDA events, the three kernels' times (sr_set_profiling), peak memory above the inputs, the torch-level host
synchronisations of one eager step (torch.cuda.set_sync_debug_mode), and the two paths' loss and gradients.

    python tools/bench_features.py --features 4 22 32 [--steps 20 --warmup 5]
    python tools/bench_features.py --losses [--steps 20 --warmup 5]
    python tools/bench_features.py --reproj [--steps 20 --warmup 5]
    python tools/bench_features.py --cycle [--steps 20 --warmup 5]
    python tools/bench_features.py --rows [--steps 20 --warmup 5]
    python tools/bench_features.py --ssim [--steps 20 --warmup 5]
    python tools/bench_features.py --mask [--steps 20 --warmup 5]
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
    ap.add_argument("--reproj", action="store_true")
    ap.add_argument("--cycle", action="store_true")
    ap.add_argument("--rows", action="store_true")
    ap.add_argument("--ssim", action="store_true")
    ap.add_argument("--mask", action="store_true")
    args = ap.parse_args()
    if args.mask:
        return bench_mask(args)
    if args.ssim:
        return bench_ssim(args)
    if args.rows:
        return bench_rows(args)
    if args.cycle:
        return bench_cycle(args)
    if args.losses:
        return bench_losses(args)
    if args.reproj:
        return bench_reproj(args)
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


def _reproj_inputs(M, RES, P, B, dev, seed=0):
    from tests.golden.make_warp_golden import make_inputs
    wi = {k: v.to(dev) for k, v in make_inputs(seed, P, B, M, False).items() if v is not None}
    g = torch.Generator(device=dev).manual_seed(seed)
    d = dict(feat_px=torch.randn((M, RES, RES, 16), device=dev, generator=g),
             regist=torch.randn((P, 16), device=dev, generator=g).requires_grad_(True),
             xyz=wi["xyz"].clone().requires_grad_(True), logsigma=torch.tensor([np.log(2.0)], device=dev, dtype=torch.float32))
    d["logsigma"].requires_grad_(True)
    for k in ("rest_q", "rest_t", "log_gauss", "art_q", "art_t", "cam_q", "cam_t"):
        d[k] = wi[k].clone().requires_grad_(True)
    f = torch.tensor([[1.2 * RES, 0, RES / 2], [0, 1.2 * RES, RES / 2], [0, 0, 1]], device=dev)
    d["Kmat"] = f[None].expand(M, -1, -1).contiguous()
    ys, xs = torch.meshgrid(torch.arange(RES, device=dev), torch.arange(RES, device=dev), indexing="ij")
    d["hxy"] = torch.stack([xs, ys, torch.ones_like(xs)], -1)[None].expand(M, -1, -1, -1).float().contiguous()
    d["mask"] = (torch.rand((M, RES, RES), device=dev, generator=g) > 0.5).float()
    d["det"] = torch.ones(M, device=dev)
    d["delta"] = (torch.randn((M, RES, RES, B), device=dev, generator=g).clamp(min=0) * 0.1).requires_grad_(True)
    d["w"] = torch.tensor([5e-2], device=dev)
    d["cand"] = torch.randperm(M * P, generator=torch.Generator().manual_seed(seed))[:2048].to(dev, torch.int32)
    return d


def _q2dq(q, t):
    from oracle import warp_oracle as wo
    return q, 0.5 * wo.qmul(torch.cat((torch.zeros_like(t[..., :1]), t), -1), q)


def _reproj_fused(d):
    from vidu4d_b200.registration import global_match, reproj_loss
    xyz_m = global_match(d["feat_px"], d["regist"], d["xyz"], d["cand"], d["logsigma"], num_grad=8)
    return reproj_loss(xyz_m, d["hxy"], d["Kmat"], _q2dq(d["rest_q"], d["rest_t"]), _q2dq(d["art_q"], d["art_t"]), d["log_gauss"],
                       (d["cam_q"], d["cam_t"]), d["mask"], d["det"], weight=d["w"], train_res=256, delta=d["delta"])["loss"], xyz_m


def _reproj_torch(d):
    """Today's caller path: deformable_gaussian.py:1455-1486 statements, oracle/warp_oracle.py in fp32, pinhole
    projection, model.py's masking and the sync-free positive mean."""
    from oracle import warp_oracle as wo
    M, H, W = d["feat_px"].shape[:3]
    P = d["regist"].shape[0]
    sidx = d["cand"].long() % P
    score = d["feat_px"].reshape(-1, 16) @ d["regist"][sidx].T
    score, idx = torch.topk(score, 8, dim=1, largest=True)
    prob = torch.softmax(score * d["logsigma"].exp(), 1)
    xyz_m = (prob[..., None] * d["xyz"][sidx][idx]).sum(1).reshape(M, H, W, 3)
    rest, art = _q2dq(d["rest_q"], d["rest_t"]), _q2dq(d["art_q"], d["art_t"])
    rest_m = (rest[0][None].expand(M, -1, -1), rest[1][None].expand(M, -1, -1))
    se3 = wo.dq_mul(art, wo.dq_inverse(rest_m))
    rot = torch.zeros((H * W, 4), device=xyz_m.device)
    rot[:, 0] = 1.0
    xys = []
    for m in range(M):
        xc = wo.bob_warp(xyz_m[m].reshape(-1, 3), rot, rest, torch.exp(-d["log_gauss"]), (se3[0][m:m + 1], se3[1][m:m + 1]),
                         (d["cam_q"][m:m + 1], d["cam_t"][m:m + 1]), d["delta"][m].reshape(-1, d["delta"].shape[-1]))[0][0]
        h = xc @ d["Kmat"][m].T
        xys.append(h[:, :2] / (h[:, 2:] + 1e-6))
    v = (torch.stack(xys).reshape(M, H, W, 2) - d["hxy"][..., :2]).norm(dim=-1) * d["mask"] * d["det"][:, None, None]
    on = (v > 0).to(v.dtype)
    return d["w"][0] * (v * on).sum() / on.sum().clamp(min=1.0) / 256.0, xyz_m


def bench_reproj(args):
    from vidu4d_b200 import _capi, rasterizer as RZ
    from vidu4d_b200.graph import GraphedStep
    assert torch.cuda.is_available(), "this measurement needs a GPU"
    dev = torch.device("cuda:0")
    _capi.load()
    gpu = _gpu_name()
    P, B = args.surfels, 25
    flush = torch.empty((256 << 20,), dtype=torch.uint8, device=dev)
    leaves = ("regist", "xyz", "logsigma", "rest_q", "rest_t", "log_gauss", "art_q", "art_t", "cam_q", "cam_t", "delta")
    for RES, M, arms in ((256, 2, ("fused", "torch")), (512, 8, ("fused",))):
        d = _reproj_inputs(M, RES, P, B, dev)
        fns = {"fused": _reproj_fused, "torch": _reproj_torch}

        def make_body(fn):
            def body():
                for k in leaves:
                    d[k].grad = None
                fn(d)[0].backward()
            return body
        bodies = {k: make_body(fns[k]) for k in arms}
        peak = {}
        for k, b in bodies.items():                                  # eager peak memory above the inputs
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            b()
            torch.cuda.synchronize()
            peak[k] = round((torch.cuda.max_memory_allocated() - base) / 2**20, 1)
        compare = {}
        if "torch" in arms:                                          # the two paths' outputs on the same inputs
            with torch.no_grad():
                lf, xf = _reproj_fused(d)
                lt, xt = _reproj_torch(d)
            compare = {"loss_rel_diff": float((lf - lt).abs() / lt.abs()),
                       "xyz_matched_max_abs_diff_over_max": float((xf - xt).abs().max() / xt.abs().max())}
        steps = {k: GraphedStep(b, device=dev) for k, b in bodies.items()}
        for s_ in steps.values():
            s_()
            for _ in range(args.warmup):
                s_(check=False)
        torch.cuda.synchronize()
        ms = {k: [] for k in steps}
        for i in range(args.steps):
            for k, s_ in steps.items():
                flush.fill_(i & 255)
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(); s_.graph.replay(); b.record()
                b.synchronize()
                ms[k].append(a.elapsed_time(b))
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
                if k in ("match_fwd", "match_bwd", "match_scatter", "reproj_fwd", "reproj_scale", "reproj_bwd")}
        print(json.dumps({"workload": "feat_reproj step (match + warp + projection + loss, fwd + bwd)", "surfels": P,
                          "resolution": RES, "frames": M, "candidates": 2048, "num_grad": 8, "bones": B,
                          "ms_per_step": {k: round(float(np.median(v)), 4) for k, v in ms.items()},
                          "peak_mem_mb_above_inputs": peak, "kernel_ms_per_launch": kern,
                          "launches_per_step_fused": steps["fused"].launches, "outputs": compare, "steps": args.steps,
                          "statistic": "median step time", "gpu": gpu}), flush=True)
        del steps, bodies, d
        torch.cuda.empty_cache()
    RZ.set_sync_mode(True)
    RZ._pending.clear()


CYCLE_LEAVES = ("xyz", "rot", "rest_q", "rest_t", "log_gauss", "art_q", "art_t", "cam_q", "cam_t", "delta", "cdelta")


def _cycle_inputs(M, P, B, dev, seed=0):
    from tests.golden.make_warp_golden import make_inputs
    d = {k: v.to(dev).requires_grad_(True) for k, v in make_inputs(seed, P, B, M, True).items()}
    g = torch.Generator(device=dev).manual_seed(seed)
    d["cdelta"] = (torch.randn((M, P, B), device=dev, generator=g).clamp(min=0) * 0.1).requires_grad_(True)
    d["w"] = torch.tensor([0.01, 5e-3, 5e-4], device=dev)
    return d


def _cycle_warp(d):
    from vidu4d_b200.warp import bob_warp
    rest, art = _q2dq(d["rest_q"], d["rest_t"]), _q2dq(d["art_q"], d["art_t"])
    xc, _, _ = bob_warp(d["xyz"], d["rot"], rest, art, d["log_gauss"], (d["cam_q"], d["cam_t"]), d["delta"])
    return xc, rest, art


def _cycle_fused(d):
    from vidu4d_b200.warp import cycle_loss
    xc, rest, art = _cycle_warp(d)
    out = cycle_loss(d["xyz"], xc, rest, art, d["log_gauss"], (d["cam_q"], d["cam_t"]), d["cdelta"], weights=d["w"])
    return out["loss"], out["terms"].sum(0)


def _cycle_torch(d):
    """Today's caller path after the fused warp: deformable_gaussian.py:1517-1574 as tests/cycle_model.py's statements
    in fp32, and model.py's reduction as the sync-free positive mean."""
    from tests import cycle_model as cm
    xc, rest, art = _cycle_warp(d)
    vals = cm.cycle_values(d["xyz"], xc, rest, art, torch.exp(-d["log_gauss"]), (d["cam_q"], d["cam_t"]), d["cdelta"])
    terms = []
    for k, v in enumerate(vals):
        on = (v > 0).to(v.dtype)
        terms.append(d["w"][k] * (v * on).sum() / on.sum().clamp(min=1.0))
    terms = torch.stack(terms)
    return terms.sum(), terms


def bench_cycle(args):
    from vidu4d_b200 import _capi, rasterizer as RZ
    from vidu4d_b200.graph import GraphedStep
    assert torch.cuda.is_available(), "this measurement needs a GPU"
    dev = torch.device("cuda:0")
    _capi.load()
    gpu = _gpu_name()
    P, B = args.surfels, 25
    flush = torch.empty((256 << 20,), dtype=torch.uint8, device=dev)
    for M in (2, 8):
        d = _cycle_inputs(M, P, B, dev)
        fns = {"fused": _cycle_fused, "torch": _cycle_torch}

        def make_body(fn):
            def body():
                for k in CYCLE_LEAVES:
                    d[k].grad = None
                fn(d)[0].backward()
            return body
        bodies = {k: make_body(f) for k, f in fns.items()}
        peak = {}
        for k, b in bodies.items():                                  # eager peak memory above the inputs
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            b()
            torch.cuda.synchronize()
            peak[k] = round((torch.cuda.max_memory_allocated() - base) / 2**20, 1)
        grads = {}
        for k, b in bodies.items():                                  # the two paths on the same inputs
            b()
            grads[k] = {n: d[n].grad.clone() for n in ("xyz", "art_q", "log_gauss", "cdelta")}
        with torch.no_grad():
            lf, tf = _cycle_fused(d)
            lt, tt = _cycle_torch(d)
        compare = {"loss_rel_diff": float((lf - lt).abs() / lt.abs()),
                   "terms_rel_diff": [float(v) for v in ((tf - tt).abs() / tt.abs().clamp(min=1e-30))],
                   "grad_max_abs_diff_over_max": {n: float((grads["fused"][n] - grads["torch"][n]).abs().max()
                                                           / grads["torch"][n].abs().max()) for n in grads["fused"]}}
        steps = {k: GraphedStep(b, device=dev) for k, b in bodies.items()}
        for s_ in steps.values():
            s_()
            for _ in range(args.warmup):
                s_(check=False)
        torch.cuda.synchronize()
        ms = {k: [] for k in steps}
        for i in range(args.steps):
            for k, s_ in steps.items():
                flush.fill_(i & 255)
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(); s_.graph.replay(); b.record()
                b.synchronize()
                ms[k].append(a.elapsed_time(b))
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
                if k in ("bob_warp_fwd", "bob_warp_bwd", "cycle_fwd", "cycle_scale", "cycle_bwd")}
        print(json.dumps({"workload": "bob_warp -> cycle loss -> backward (fwd + bwd)", "surfels": P, "frames": M, "bones": B,
                          "delta": True, "ms_per_step": {k: round(float(np.median(v)), 4) for k, v in ms.items()},
                          "peak_mem_mb_above_inputs": peak, "kernel_ms_per_launch": kern,
                          "launches_per_step": {k: s_.launches for k, s_ in steps.items()}, "outputs": compare,
                          "steps": args.steps, "statistic": "median step time", "gpu": gpu}), flush=True)
        del steps, bodies, d
        torch.cuda.empty_cache()
    RZ.set_sync_mode(True)
    RZ._pending.clear()


ROWS_LEAVES = ("regist", "xyz", "xyz_cam", "rot_cam", "cam_q", "rest_q", "rest_t", "logibeta")


def _rows_inputs(M, P, B, dev, seed=0):
    """make_feature_rows_golden.make_case's inputs at full size; xyz_cam / rot_cam are the fused forward warp's."""
    from tests.golden.make_feature_rows_golden import make_case
    from vidu4d_b200.warp import bob_warp
    inp = make_case(seed, P, B, M)
    d = {k: v.to(dev) for k, v in inp.items()}
    with torch.no_grad():
        d["xyz_cam"], d["rot_cam"], _ = bob_warp(d["xyz"], d["rot"], _q2dq(d["rest_q"], d["rest_t"]), _q2dq(d["art_q"], d["art_t"]),
                                                 d["log_gauss"], (d["cam_q"], d["cam_t"]), d["delta"])
    d["Kmat"] = torch.linalg.inv(d["Kinv"])
    for k in ROWS_LEAVES:
        d[k].requires_grad_(True)
    g = torch.Generator(device=dev).manual_seed(seed)
    d["g_rows"] = torch.randn((M, P, inp["regist"].shape[1] + 6), device=dev, generator=g)
    d["g_s"] = torch.randn((), device=dev, generator=g)
    d["g_dens"] = torch.randn((P, 1), device=dev, generator=g)
    return d


def _rows_fused(d):
    from vidu4d_b200.warp import feature_rows
    o = feature_rows(d["regist"], d["xyz"], d["scaling"], d["xyz_cam"], d["rot_cam"], d["Kmat"], (d["cam_q"], d["cam_t"]),
                     _q2dq(d["rest_q"], d["rest_t"]), d["logibeta"])
    return o["rows"], o["flow_scale"], o["gauss_density"]


def _rows_torch(d):
    """deformable_gaussian.py:1106-1182 as tests/feature_rows_model.py's statements, in fp32."""
    from tests import feature_rows_model as fm
    rows, s, dens, _ = fm.feature_rows(d["regist"], d["xyz"], d["scaling"], d["xyz_cam"], d["rot_cam"], d["Kmat"],
                                       (d["cam_q"], d["cam_t"]), _q2dq(d["rest_q"], d["rest_t"]), d["logibeta"])
    return rows, s, dens


def bench_rows(args):
    from vidu4d_b200 import _capi, rasterizer as RZ
    from vidu4d_b200.graph import GraphedStep
    assert torch.cuda.is_available(), "this measurement needs a GPU"
    dev = torch.device("cuda:0")
    _capi.load()
    gpu = _gpu_name()
    P, B = args.surfels, 25
    flush = torch.empty((256 << 20,), dtype=torch.uint8, device=dev)
    for M in (2, 8):
        d = _rows_inputs(M, P, B, dev)
        fns = {"fused": _rows_fused, "torch": _rows_torch}

        def make_body(fn):
            def body():
                for k in ROWS_LEAVES:
                    d[k].grad = None
                torch.autograd.backward(fn(d), (d["g_rows"], d["g_s"], d["g_dens"]))
            return body
        bodies = {k: make_body(f) for k, f in fns.items()}
        peak = {}
        for k, b in bodies.items():                                  # eager peak memory above the inputs
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            b()
            torch.cuda.synchronize()
            peak[k] = round((torch.cuda.max_memory_allocated() - base) / 2**20, 1)
        grads = {}
        for k, b in bodies.items():                                  # the two paths on the same inputs
            b()
            grads[k] = {n: d[n].grad.clone() for n in ROWS_LEAVES}
        with torch.no_grad():
            of, ot = _rows_fused(d), _rows_torch(d)
        rel = lambda a, b: float((a - b).abs().max() / b.abs().max().clamp(min=1e-30))  # noqa: E731
        compare = {"outputs_max_abs_diff_over_max": {n: rel(a, b) for n, a, b in zip(("rows", "flow_scale", "gauss_density"), of, ot)},
                   "grad_max_abs_diff_over_max": {n: rel(grads["fused"][n], grads["torch"][n]) for n in ROWS_LEAVES}}
        launches = {}
        for k, b in bodies.items():                                  # GPU activities (kernels, memsets, copies) of one step
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as tp:
                b()
                torch.cuda.synchronize()
            launches[k] = sum(e.count for e in tp.key_averages() if e.device_type == torch.autograd.DeviceType.CUDA)
        steps = {k: GraphedStep(b, device=dev) for k, b in bodies.items()}
        for s_ in steps.values():
            s_()
            for _ in range(args.warmup):
                s_(check=False)
        torch.cuda.synchronize()
        ms = {k: [] for k in steps}
        for i in range(args.steps):
            for k, s_ in steps.items():
                flush.fill_(i & 255)
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(); s_.graph.replay(); b.record()
                b.synchronize()
                ms[k].append(a.elapsed_time(b))
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
        kern = {k: round(v["ms"] / max(v["count"], 1), 4) for k, v in prof.items() if k.startswith("frows_")}
        print(json.dumps({"workload": "feature rows (fwd + bwd)", "surfels": P, "frames": M, "bones": B,
                          "regist_channels": int(d["regist"].shape[1]), "ms_per_step": {k: round(float(np.median(v)), 4) for k, v in ms.items()},
                          "peak_mem_mb_above_inputs": peak, "kernel_ms_per_launch": kern,
                          "gpu_activities_per_step": launches, "library_launches_per_step": steps["fused"].launches, "outputs": compare,
                          "steps": args.steps, "statistic": "median step time", "gpu": gpu}), flush=True)
        del steps, bodies, d
        torch.cuda.empty_cache()
    RZ.set_sync_mode(True)
    RZ._pending.clear()


SSIM_BYTES_PER_PX, SSIM_FLOP_PER_PX = 44, 400


def _torch_window(C, dev):
    """The 11x11 Gaussian window (sigma 1.5) of a depthwise conv2d over C channels."""
    import math
    g = torch.tensor([math.exp(-(i - 5) ** 2 / (2 * 1.5 ** 2)) for i in range(11)], dtype=torch.float32)
    g = g / g.sum()
    return (g[:, None] @ g[None, :]).expand(C, 1, 11, 11).contiguous().to(dev)


def _torch_ssim(img1, img2, win):
    """1 - SSIM in plain torch, written from the formula: depthwise conv2d with the window, groups = C."""
    C = img1.shape[1]
    f = lambda t: torch.nn.functional.conv2d(t, win, padding=5, groups=C)  # noqa: E731
    mu1, mu2 = f(img1), f(img2)
    s11, s22, s12 = f(img1 * img1) - mu1 * mu1, f(img2 * img2) - mu2 * mu2, f(img1 * img2) - mu1 * mu2
    m = ((2 * mu1 * mu2 + 0.01 ** 2) * (2 * s12 + 0.03 ** 2)) / ((mu1 * mu1 + mu2 * mu2 + 0.01 ** 2) * (s11 + s22 + 0.03 ** 2) + 1e-10)
    return 1.0 - m.mean()


def _alternate(bodies, args, flush):
    """Captures each body in a CUDA graph and replays them alternately, L2 flushed before each; median ms per body."""
    from vidu4d_b200.graph import GraphedStep
    steps = {k: GraphedStep(b, device=flush.device) for k, b in bodies.items()}
    for s_ in steps.values():
        s_()
        for _ in range(args.warmup):
            s_(check=False)
    torch.cuda.synchronize()
    ms = {k: [] for k in steps}
    for i in range(args.steps):
        for k, s_ in steps.items():
            flush.fill_(i & 255)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(); s_.graph.replay(); b.record()
            b.synchronize()
            ms[k].append(a.elapsed_time(b))
    return {k: float(np.median(v)) for k, v in ms.items()}, steps


def bench_ssim(args):
    from vidu4d_b200 import _capi, rasterizer as RZ
    from vidu4d_b200.renderer import PipelineParams, make_camera, render_loss_batch, stack_cameras
    from vidu4d_b200.ssim import ssim
    from vidu4d_b200.synthetic import SurfelCloud, object_scene, orbit_view
    assert torch.cuda.is_available(), "this measurement needs a GPU"
    dev = torch.device("cuda:0")
    _capi.load()
    gpu = _gpu_name()
    flush = torch.empty((256 << 20,), dtype=torch.uint8, device=dev)
    for shape in ((1, 3, 512, 512), (8, 3, 512, 512), (1, 3, 1080, 1920)):
        g = torch.Generator(device=dev).manual_seed(1)
        x = torch.rand(shape, device=dev, generator=g).requires_grad_(True)
        y = (x.detach() + 0.1 * torch.randn(shape, device=dev, generator=g)).clamp(0, 1)
        win = _torch_window(shape[1], dev)
        fns = {"fused": lambda: 1.0 - ssim(x, y), "torch": lambda: _torch_ssim(x, y, win)}

        def make_body(fn):
            def body():
                x.grad = None
                fn().backward()
            return body
        bodies = {k: make_body(f) for k, f in fns.items()}
        peak, vals, grads = {}, {}, {}
        for k, b in bodies.items():
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            b()
            torch.cuda.synchronize()
            peak[k] = round((torch.cuda.max_memory_allocated() - base) / 2**20, 1)
            grads[k] = x.grad.clone()
            with torch.no_grad():
                vals[k] = float(fns[k]())
        med, _ = _alternate(bodies, args, flush)
        RZ.set_sync_mode(True)
        RZ._pending.clear()
        torch.cuda.synchronize()
        _capi.get_profile()
        _capi.set_profiling(True)
        for _ in range(5):
            bodies["fused"]()
        prof = _capi.get_profile()
        _capi.set_profiling(False)
        kern = {k: round(v["ms"] / max(v["count"], 1), 4) for k, v in prof.items() if k.startswith("ssim")}
        px = int(np.prod(shape))
        t_bytes, t_flop = px * SSIM_BYTES_PER_PX / 3.35e12 * 1e3, px * SSIM_FLOP_PER_PX / 67e12 * 1e3
        kms = sum(kern.values())
        print(json.dumps({"workload": "1 - ssim, fwd + bwd", "shape": list(shape), "ms_per_step": {k: round(v, 4) for k, v in med.items()},
                          "peak_mem_mb_above_inputs": peak, "kernel_ms_per_launch": kern,
                          "bound_ms": {"bytes": round(t_bytes, 4), "flop": round(t_flop, 4)},
                          "kernel_share_of_bound": round(max(t_bytes, t_flop) / kms, 3) if kms else None,
                          "loss_abs_diff": abs(vals["fused"] - vals["torch"]),
                          "grad_max_abs_diff_over_max": float((grads["fused"] - grads["torch"]).abs().max() / grads["torch"].abs().max()),
                          "steps": args.steps, "statistic": "median step time", "gpu": gpu}), flush=True)
        del bodies, fns, x, y, grads, win
        torch.cuda.empty_cache()
    # the term's cost inside a Stage-3 step
    P, RES, M = args.surfels, 512, 8
    scene = object_scene(P, seed=0, opacity="trained", center=(0.0, 0.0, 0.0))
    cams = []
    for f in range(M):
        R, t = orbit_view(f, 64)
        cams.append(make_camera(RES, RES, 2 * np.arctan(0.5), 2 * np.arctan(0.5), R=R.T, T=t, device=dev))
    bc = stack_cameras(cams)
    g = torch.Generator(device=dev).manual_seed(99)
    rgb = torch.rand((M, 3, RES, RES), device=dev, generator=g)
    cloud = SurfelCloud(scene, dev)
    bkgd = torch.tensor([0.2, 0.3, 0.4], device=dev, requires_grad=True)
    pipe, bg = PipelineParams(), torch.zeros(3, device=dev)

    def make_step(w):
        def body():
            out = render_loss_batch(bc, cloud, pipe, bg, rgb, learnable_bkgd=bkgd, w_rgb=1.0 - w, w_ssim=w, lambda_dist=10.0)
            out["loss"].backward()
        return body
    med, steps = _alternate({"w_ssim_0": make_step(0.0), "w_ssim_0.2": make_step(0.2)}, args, flush)
    for s_ in steps.values():
        s_.arm(); RZ.check_overflow(keep=True)
    print(json.dumps({"workload": "render_loss_batch step (fwd + bwd)", "surfels": P, "resolution": RES, "frames": M,
                      "ms_per_step": {k: round(v, 4) for k, v in med.items()},
                      "library_launches_per_step": {k: s_.launches for k, s_ in steps.items()},
                      "steps": args.steps, "statistic": "median step time", "gpu": gpu}), flush=True)
    RZ.set_sync_mode(True)
    RZ._pending.clear()


def _torch_mask_term(acc, mask, vis, det, w):
    """lab4d/engine/model.py:587-611,648-650,950-967,1000-1012 as the reference writes them, on (M,H,W) planes."""
    vd = vis * det[:, None, None]
    if mask.sum() > 0 and (1 - mask).sum() > 0:
        pos_wt = vd.sum() / mask[vd > 0].sum()
        neg_wt = vd.sum() / (1 - mask[vd > 0]).sum()
        bw = 0.5 * pos_wt * mask + 0.5 * neg_wt * (1 - mask)
    else:
        bw = 1
    v = (acc - mask).pow(2) * bw * vis * det[:, None, None]
    v = v.mean() if (v > 0).sum() == 0 else v[v > 0].mean()
    return v * w


def _count_syncs(fn):
    """torch-level host synchronisations of one call of fn (torch.cuda.set_sync_debug_mode)."""
    import warnings
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode("default")
    return sum("synchroniz" in str(r.message) for r in rec)


def bench_mask(args):
    from vidu4d_b200 import _capi, rasterizer as RZ
    from vidu4d_b200.graph import GraphedStep
    from vidu4d_b200.renderer import PipelineParams, make_camera, render_loss_batch, stack_cameras
    from vidu4d_b200.synthetic import SurfelCloud, object_scene, orbit_view
    assert torch.cuda.is_available(), "this measurement needs a GPU"
    dev = torch.device("cuda:0")
    _capi.load()
    gpu = _gpu_name()
    P = args.surfels
    scene = object_scene(P, seed=0, opacity="trained", center=(0.0, 0.0, 0.0))
    flush = torch.empty((256 << 20,), dtype=torch.uint8, device=dev)
    pipe, bg = PipelineParams(), torch.zeros(3, device=dev)
    for RES, M in ((256, 2), (512, 8)):
        cams = []
        for f in range(M):
            R, t = orbit_view(f, 64)
            cams.append(make_camera(RES, RES, 2 * np.arctan(0.5), 2 * np.arctan(0.5), R=R.T, T=t, device=dev))
        bc = stack_cameras(cams)
        g = torch.Generator(device=dev).manual_seed(99)
        rgb = torch.rand((M, 3, RES, RES), device=dev, generator=g)
        mask = (torch.rand((M, RES, RES), device=dev, generator=g) > 0.6).float()
        vis = (torch.rand((M, RES, RES), device=dev, generator=g) > 0.1).float()
        det = torch.ones(M, device=dev)
        w = torch.tensor([0.1], device=dev)
        cloud = SurfelCloud(scene, dev)
        kw = dict(vis2d=vis, mask_gt=mask, lambda_normal=0.05, lambda_dist=10.0)

        def fused():
            out = render_loss_batch(bc, cloud, pipe, bg, rgb, is_detected=det, mask_loss_weight=w, **kw)
            out["loss"].backward()
            return out["loss"]

        def eager():
            # the statements' own forward and autograd backward to dL/dalpha; the rasterizer backward that dL/dalpha feeds
            # runs for the other terms either way, at a cost independent of the values it is handed
            out = render_loss_batch(bc, cloud, pipe, bg, rgb, **kw)
            alpha = out["allmap"][:, 1].detach().requires_grad_(True)
            loss = out["loss"] + _torch_mask_term(alpha, mask, vis, det, w[0])
            loss.backward()
            eager.alpha = alpha
            return loss
        RZ.set_sync_mode(True)
        fused(); eager()                                               # warm-up: learns the instance capacity
        torch.cuda.synchronize()
        peak, loss = {}, {}
        for k, b in (("fused", fused), ("torch", eager)):
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            cloud.zero_grad()
            loss[k] = float(b().detach())
            torch.cuda.synchronize()
            peak[k] = round((torch.cuda.max_memory_allocated() - base) / 2**20, 1)
        # dL/dalpha of the term: the fused kernels on the torch arm's alpha against its autograd gradient
        from vidu4d_b200.renderer import _mask_term
        am = torch.zeros((M, 8, RES, RES), device=dev)
        am[:, 1] = eager.alpha.detach()
        dla = torch.zeros_like(am)
        _mask_term(M, RES, RES, am, mask, vis, det, w, dla)
        ga = eager.alpha.grad
        compare = {"loss_rel_diff": abs(loss["fused"] - loss["torch"]) / abs(loss["torch"]),
                   "dL_dalpha_max_abs_diff_over_max": float((dla[:, 1] - ga).abs().max() / ga.abs().max())}
        RZ.set_sync_mode(False)
        syncs = {"fused": _count_syncs(fused), "torch": _count_syncs(eager)}
        torch.cuda.synchronize()
        RZ._pending.clear()
        step = GraphedStep(fused, device=dev)
        step()
        for _ in range(args.warmup):
            step(check=False)
            eager()
        torch.cuda.synchronize()
        RZ._pending.clear()
        ms = {"fused": [], "torch": []}
        for i in range(args.steps):
            for k in ("fused", "torch"):
                flush.fill_(i & 255)
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                step.graph.replay() if k == "fused" else eager()
                b.record()
                b.synchronize()
                RZ._pending.clear()
                ms[k].append(a.elapsed_time(b))
        step.arm(); RZ.check_overflow(keep=True)
        RZ._pending.clear()
        RZ.set_sync_mode(True)
        fused()
        torch.cuda.synchronize()
        _capi.get_profile()
        _capi.set_profiling(True)
        for _ in range(5):
            fused()
        prof = _capi.get_profile()
        _capi.set_profiling(False)
        kern = {k: round(v["ms"] / max(v["count"], 1), 4) for k, v in prof.items()
                if k in ("mask_stats", "mask_loss", "mask_loss_scale", "loss_grad")}
        print(json.dumps({"workload": "render_loss_batch step with the silhouette term (fwd + bwd)", "surfels": P,
                          "resolution": RES, "frames": M, "ms_per_step": {k: round(float(np.median(v)), 4) for k, v in ms.items()},
                          "capture": {"fused": "one CUDA graph", "torch": "eager"}, "peak_mem_mb_above_inputs": peak,
                          "kernel_ms_per_launch": kern, "torch_host_syncs_per_eager_step": syncs,
                          "library_launches_per_step_fused": step.launches, "outputs": compare, "steps": args.steps,
                          "statistic": "median step time", "gpu": gpu}), flush=True)
        del step
        torch.cuda.empty_cache()
    RZ.set_sync_mode(True)
    RZ._pending.clear()


if __name__ == "__main__":
    main()
