"""Timing of the fused delta-skinning MLP (csrc/skin_mlp.cu via vidu4d_b200.warp.delta_skin) against the reference's
statements in fp32 torch (tests/delta_skin_model.unfolded: xyz_bone, the expanded conditioning code, cat, three Linear
layers through cuBLAS with TF32 off, relu * 0.1), forward + backward of sum(delta * w).

The three call shapes of one Stage-3 step at B = 25 bones, M = 2 frames:
    warp    (P,3) surfels, rest bones, the mean code              forward warp (warping.py:412-425)
    cycle   (M,P,3) points, each frame's bones and code           backward warp of cycle_loss (deformable_gaussian.py:1517-1574)
    reproj  (M,R,R,3) matched points, rest bones, the mean code   feat_reproj (deformable_gaussian.py:1305-1324)
and `step`, the three in one graph.  The protocol is tools/bench_features.py --cycle's: both paths alternate in one
process, each as one CUDA graph, a 256 MB fill flushes the L2 before every replay, the statistic is the median of CUDA-event
times; the kernels' own times come from sr_set_profiling in a separate eager pass; peak memory is an eager pass's
max_memory_allocated above the inputs.  The GPU's name, power limit and maximum SM clock are read in the same run and
printed with every line, and the SM clock seen under load is sampled once after the timed loop.

Operation counts (kept here, next to the times they divide): a point costs 3*64 + 64*64 + 64*B FMAs forward; the backward
recomputes that and adds the two backward GEMMs (64*B + 64*64 + 64*3) and the three weight-gradient GEMMs (the same
again).  The kernels pad B to 16 * ceil(B / 16) units; the counts below are the algorithm's, not the padded ones.

    python tools/bench_skin_mlp.py [--surfels 300000] [--res 256] [--steps 50] [--warmup 5]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

FP32_PEAK_TFLOPS = 67.0       # NVIDIA's data-sheet FP32 rate of the H100 SXM at its 700 W limit; never a measured figure
NAMES = {"W1": "linear_1.0.weight", "b1": "linear_1.0.bias", "W2": "linear_2.0.weight", "b2": "linear_2.0.bias",
         "W3": "linear_final.weight", "b3": "linear_final.bias"}


def _smi(query):
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={query}", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=20).stdout.strip().splitlines()[0]
    except Exception:
        return "unknown"


def fmas(points, B):
    fwd = points * (3 * 64 + 64 * 64 + 64 * B)
    return fwd, 3 * fwd


def make_inputs(P, R, B, M, dev, seed=0):
    from tests import delta_skin_model as dm
    g = torch.Generator().manual_seed(seed)
    rn = lambda *s: torch.randn(s, generator=g)  # noqa: E731

    def bones(*lead):
        r = torch.nn.functional.normalize(rn(*lead, B, 4), dim=-1)
        tr = torch.cat((torch.zeros(*lead, B, 1), 0.15 * rn(*lead, B, 3)), -1)
        return r, 0.5 * dm._qmul(tr, r)
    rest, art = bones(), bones(M)
    d = {"rest_r": rest[0], "rest_d": rest[1], "art_r": art[0], "art_d": art[1], "log_gauss": np.log(0.03) + 0.3 * rn(B, 3),
         "cond_mean": 0.5 * rn(160), "cond_frames": 0.5 * rn(M, 160),
         "xyz": 0.15 * rn(P, 3), "xyz_t": 0.15 * rn(M, P, 3), "xyz_m": 0.15 * rn(M, R, R, 3),
         "w_warp": rn(P, B), "w_cycle": rn(M, P, B), "w_reproj": rn(M, R, R, B)}
    return {k: v.to(dev).requires_grad_(not k.startswith("w_")) for k, v in d.items()}


CALLS = {"warp": ("xyz", "rest", "cond_mean"), "cycle": ("xyz_t", "art", "cond_frames"), "reproj": ("xyz_m", "rest", "cond_mean")}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--surfels", type=int, default=300_000)
    ap.add_argument("--res", type=int, default=256)
    ap.add_argument("--bones", type=int, default=25)
    ap.add_argument("--frames", type=int, default=2)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this measurement needs a GPU"
    from tests import delta_skin_model as dm
    from vidu4d_b200 import _capi, rasterizer as RZ
    from vidu4d_b200.graph import GraphedStep
    from vidu4d_b200.warp import DeltaSkinMLP, delta_skin
    dev = torch.device("cuda:0")
    _capi.load()
    torch.backends.cuda.matmul.allow_tf32 = False            # torch's default, stated: the torch path is FP32 cuBLAS
    gpu = _smi("name,power.limit,clocks.max.sm")
    P, R, B, M = args.surfels, args.res, args.bones, args.frames
    d = make_inputs(P, R, B, M, dev)
    torch.manual_seed(0)
    mlp = DeltaSkinMLP(B).to(dev)
    params = {k: mlp.get_parameter(v) for k, v in NAMES.items()}
    leaf_names = [k for k, v in d.items() if v.requires_grad] + list(NAMES)
    leaves = [d[k] for k in leaf_names[:-len(NAMES)]] + [params[k] for k in NAMES]
    flush = torch.empty((256 << 20,), dtype=torch.uint8, device=dev)

    def call(name, fused):
        pts, bones, cond = CALLS[name]
        r, dd = d[bones + "_r"], d[bones + "_d"]
        if fused:
            return delta_skin(d[pts], (r, dd), d["log_gauss"], mlp, d[cond])
        return dm.unfolded(d[pts], r, dd, d["log_gauss"], params, d[cond])

    def make_body(names, fused):
        def body():
            for v in leaves:
                v.grad = None
            loss = 0.0
            for n in names:
                loss = loss + (call(n, fused) * d["w_" + n]).sum()
            loss.backward()
        return body

    def grads64(names):
        """Every leaf's gradient from the reference's statements in float64: the yardstick both fp32 paths are held to."""
        d64 = {k: v.detach().double().requires_grad_(v.requires_grad) for k, v in d.items()}
        p64 = {k: v.detach().double().requires_grad_(True) for k, v in params.items()}
        loss = 0.0
        for n in names:
            pts, bones, cond = CALLS[n]
            loss = loss + (dm.unfolded(d64[pts], d64[bones + "_r"], d64[bones + "_d"], d64["log_gauss"], p64, d64[cond])
                           * d64["w_" + n]).sum()
        loss.backward()
        return {k: (d64[k] if k in d64 else p64[k]).grad for k in leaf_names}

    n_points = {"warp": P, "cycle": M * P, "reproj": M * R * R}
    workloads = {k: (k,) for k in CALLS}
    workloads["step"] = tuple(CALLS)
    for wl, names in workloads.items():
        bodies = {"fused": make_body(names, True), "torch": make_body(names, False)}
        peak, grads = {}, {}
        for k, b in bodies.items():                                  # eager: peak memory above the inputs, and the outputs
            b()
            torch.cuda.synchronize()
            for v in leaves:
                v.grad = None
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            b()
            torch.cuda.synchronize()
            peak[k] = round((torch.cuda.max_memory_allocated() - base) / 2**20, 1)
            grads[k] = {n: v.grad.clone() for n, v in zip(leaf_names, leaves) if v.grad is not None}
        with torch.no_grad():
            dv = max(float((call(n, True) - call(n, False)).abs().max()) for n in names)
        g64 = grads64(names)
        worst = {}
        for k, gk in grads.items():                                  # each path's worst leaf against float64
            err = {n: float((v.double() - g64[n]).abs().max() / g64[n].abs().max().clamp(min=1e-300)) for n, v in gk.items()}
            n = max(err, key=err.get)
            worst[k] = {"leaf": n, "max_abs_err_over_max": err[n]}
        compare = {"delta_max_abs_diff_fused_vs_torch": dv, "worst_gradient_vs_float64": worst}
        del grads, g64
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
        sm_clock = _smi("clocks.sm,power.draw")
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
        pts = sum(n_points[n] for n in names)
        f_fwd, f_bwd = fmas(pts, B)
        kern, rate = {}, {}
        for k, f in (("skin_mlp_fwd", f_fwd), ("skin_mlp_bwd", f_bwd), ("skin_mlp_reduce", 0)):
            if k in prof:
                per_step = prof[k]["ms"] / 5                          # all of the workload's launches of this kernel in one step
                kern[k] = round(per_step, 4)
                if f:
                    tf = 2 * f / (per_step * 1e-3) / 1e12
                    rate[k] = {"tflops_fp32": round(tf, 2), "share_of_data_sheet_67_tflops": round(tf / FP32_PEAK_TFLOPS, 3)}
        med = {k: round(float(np.median(v)), 4) for k, v in ms.items()}
        spread = {k: [round(float(np.percentile(v, 10)), 4), round(float(np.percentile(v, 90)), 4)] for k, v in ms.items()}
        print(json.dumps({"workload": f"delta_skin {wl} (fwd + bwd)", "points": pts, "surfels": P, "res": R, "frames": M, "bones": B,
                          "ms_per_step": med, "ms_p10_p90": spread, "peak_mem_mb_above_inputs": peak,
                          "kernel_ms_per_step": kern, "kernel_rate": rate, "fma_per_step": {"fwd": f_fwd, "bwd": f_bwd},
                          "launches_per_step": {k: s_.launches for k, s_ in steps.items()}, "outputs": compare,
                          "steps": args.steps, "statistic": "median step time", "gpu": gpu, "sm_clock_after_loop": sm_clock}),
              flush=True)
        del steps, bodies
        torch.cuda.empty_cache()
    RZ.set_sync_mode(True)
    RZ._pending.clear()


if __name__ == "__main__":
    main()
