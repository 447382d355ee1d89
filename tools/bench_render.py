"""Forward-only rendering of a sequence: render_frames against today's route (the training forward under no_grad, then
sr_post_forward per frame), two arms alternating in one process.

Workload: 300 K surfels (bench.py's object scene) on 64 orbiting cameras, frames_per_call 8, F in {0, 22}, at 512^2 and
at 128^2 (the reference's default render_res), with the scalar field of view and with a per-frame camera table.  Per arm:
frames/s (median over repeats of CUDA-event time, with min and max), per-kernel ms from sr_set_profiling in a separate
pass, and peak allocator bytes above the inputs.  The two arms' colour, feature planes, radii and maps are compared bit
for bit at every timed size.  Prints one JSON object; --out writes it too.

--contrib measures the per-surfel contribution statistics instead: render_frames without, with, and again without a
SurfelContributions accumulator (alternating, L2 flushed by a 256 MB write before every timed call), at 512^2 and F in
{0, 22}, scalar cameras; then the fraction of the scene prune_by_contribution's defaults remove (no frame blends them)
and render_frames' time before and after that prune, with the renders compared bit for bit.  Every timing is repeated in
--rounds rounds of one process.

--silhouette measures the background share of the statistics: render_frames without statistics, with a
SurfelContributions accumulator, with one that has the background words and the frames' silhouettes as masks, and
without statistics again (alternating, L2 flushed before every timed call), at 512^2 and F in {0, 22}, scalar cameras.
The silhouettes are the plain render's acc > 0.5.  Outputs and the four older words are compared bit for bit.

--lift measures lifting per-pixel maps onto the surfels: render_frames with a SurfelContributions accumulator alone,
with it and a SurfelLift of C = 1, 16 and 32 channels (uniform values in [-1, 1], value bound 1), and with the
accumulator alone again as the A/A control (alternating, L2 flushed before every timed call), at 512^2, F = 0, scalar
cameras.  Outputs and the statistics are compared bit for bit with the accumulator-only arm.

--anchors measures keeping each pixel's heaviest pairs: render_frames plain, with anchors=1, 4 and 8, and plain again
as the A/A control (alternating, L2 flushed before every timed call), at 512^2, F = 0, scalar cameras.  Outputs are
compared bit for bit with the plain arm.

Usage: python tools/bench_render.py [--frames 64] [--chunk 8] [--repeats 7] [--contrib | --silhouette | --lift |
                                    --anchors [--rounds 3]] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import math

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

TAN = 0.5
FOV = 2.0 * math.atan(TAN)
TANF = math.tan(FOV * 0.5)     # the tangent render() derives from FoV (renderer._cam_tans): both arms use it


def _cams(T, res, dev, table):
    from vidu4d_b200.renderer import BatchCameras
    from vidu4d_b200.synthetic import orbit_view, projection_matrix
    vms, cps = [], []
    for f in range(T):
        R, t = orbit_view(f, T)
        W2C = np.eye(4)
        W2C[:3, :3], W2C[:3, 3] = R, t
        vms.append(W2C.T.astype(np.float32))
        cps.append((-R.T @ t).astype(np.float32))
    vm = torch.from_numpy(np.stack(vms)).to(dev).contiguous()
    pm = (vm @ torch.from_numpy(projection_matrix(TAN, TAN)).to(dev)).contiguous()
    intr = None
    if table:       # per-frame tangents with off-centre principal points
        f = torch.arange(T, dtype=torch.float32)
        intr = torch.stack([torch.full((T,), TANF), torch.full((T,), TANF), 0.02 * res * torch.sin(f), 0.02 * res * torch.cos(f)],
                           1).to(dev).contiguous()
    return BatchCameras(res, res, FOV, FOV, vm, pm, torch.from_numpy(np.stack(cps)).to(dev).contiguous(), intr)


class _PC:
    def __init__(self, s):
        self.get_xyz, self.get_rotation, self.get_scaling = s["means3D"], s["rotations"], s["scales"]
        self.get_opacity, self.get_features, self.active_sh_degree = s["opacities"], s["shs"], 3


def today(cams, pc, bg, feat, chunk):
    """The training forward under no_grad per chunk of frames, then sr_post_forward per frame (table cameras: the loss
    pass's per-frame rays are not reachable from sr_post_forward, so the maps are skipped there)."""
    from vidu4d_b200 import _capi
    from vidu4d_b200.rasterizer import _C
    T, H, W = len(cams), cams.image_height, cams.image_width
    dev = pc.get_xyz.device
    e = torch.empty((0,), device=dev)
    outs = []
    with torch.no_grad():
        for t0 in range(0, T, chunk):
            c = slice(t0, min(T, t0 + chunk))
            kw = {} if feat is None else {"features": feat, "concat": False}
            if cams.intrinsics is not None:
                kw["intrinsics"] = cams.intrinsics[c]
            o = _C.rasterize_gaussians_batch(bg, pc.get_xyz, e, pc.get_opacity, pc.get_scaling, pc.get_rotation, 1.0,
                                             cams.world_view_transform[c], cams.full_proj_transform[c], TANF, TANF, H, W,
                                             pc.get_features, 3, cams.camera_center[c], **kw)
            maps = []
            if cams.intrinsics is None:
                for f in range(o[1].shape[0]):
                    m = [torch.empty((k, H, W), device=dev) for k in (1, 3, 1, 1, 1, 1, 3)]
                    _capi.call("sr_post_forward", dev, W, H, TANF, TANF, 0.0, o[2][f], cams.world_view_transform[c][f], *m)
                    maps.append(m)
            outs.append((o[1], o[3], o[7] if feat is not None else None, maps))
    return outs


def new(cams, pc, bg, feat, chunk):
    from vidu4d_b200.renderer import PipelineParams, render_frames
    return render_frames(cams, pc, PipelineParams(), bg, features=feat, frames_per_call=chunk)


def _same(a, b):
    return bool(torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32)))


def mismatches(o_today, o_new, chunk):
    """Names of the outputs whose bits differ between the arms (empty: identical)."""
    bad = set()
    keys = ("acc", "rend_normal", "rend_dist", "render_depth_median", "render_depth_expected", "surf_depth", "surf_normal")
    for i, (color, radii, feat, maps) in enumerate(o_today):
        c = slice(i * chunk, i * chunk + color.shape[0])
        for k, x, y in (("render", color, o_new["render"][c]), ("radii", radii, o_new["radii"][c]),
                        ("features", feat, o_new["features"][c] if feat is not None else None)):
            if x is not None and not _same(x, y):
                bad.add(k)
        for f, m in enumerate(maps):
            for k, x in zip(keys, m):
                y = o_new[k][c][f]
                if not _same(x, y if y.shape[0] == x.shape[0] else y[:1]):
                    bad.add(k)
    return sorted(bad)


def timed(fn, repeats):
    times = []
    for _ in range(repeats):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
        del out
    return times


def _flushed(fn, flush, repeats, i0=0):
    """CUDA-event ms of fn() per repeat, each after a 256 MB write that evicts L2."""
    times = []
    for i in range(repeats):
        flush.fill_((i0 + i) & 255)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
        del out
    return times


def _stat(t, frames):
    t = np.asarray(t)
    return {"ms_median": float(np.median(t)), "ms_min": float(t.min()), "ms_max": float(t.max()),
            "fps_median": frames / (float(np.median(t)) / 1e3)}


def contrib_main(args, gpu):
    """--contrib: `rounds` rounds in one process.  Each round times, for F = 0 and 22, three arms alternating -- plain,
    with the accumulator, plain again (an A/A control: the gap between the two plain arms is the noise floor of the
    paired comparison) -- then the prune pair (the scene before and after prune_by_contribution).  Every round's
    medians are reported, so drift over the process shows beside the paired differences."""
    from vidu4d_b200.renderer import SurfelContributions
    from vidu4d_b200.synthetic import object_scene
    dev = torch.device("cuda:0")
    s = object_scene(args.P, seed=0, opacity="trained", center=(0.0, 0.0, 0.0)).to_torch(dev)
    pc = _PC(s)
    g = torch.Generator(device=dev).manual_seed(0)
    flush = torch.empty((256 << 20,), dtype=torch.uint8, device=dev)
    res = 512
    cams = _cams(args.frames, res, dev, False)
    bg = torch.zeros(3, device=dev)
    feats = {0: None, 22: torch.rand((args.P, 22), device=dev, generator=g) * 2 - 1}
    acc = SurfelContributions.zeros(args.P, dev)

    def with_acc(feat):
        for t in (acc.weight_q, acc.max_weight, acc.pixels, acc.frames):
            t.zero_()
        return render_frames_contrib(cams, pc, bg, feat, args.chunk, acc)

    # what no frame blends, from one accumulated render (the statistics do not depend on F)
    with_acc(None)
    keep = ~acc.prune_mask()
    pruned = {"P_before": args.P, "P_after": int(keep.sum()), "pruned_fraction": float((~keep).sum()) / args.P,
              "kept_by_no_frame": int((acc.frames == 0).sum())}
    pcp = _PC({k: v[keep].contiguous() for k, v in s.items()})
    ident = {}
    for F, feat in feats.items():
        a, b = new(cams, pc, bg, feat, args.chunk), with_acc(feat)
        ident[F] = all(_same(a[k], b[k]) for k in a if k != "visibility_filter")
    a, b = new(cams, pc, bg, None, args.chunk), new(cams, pcp, bg, None, args.chunk)
    pruned["identical_images"] = all(_same(a[k], b[k]) for k in a if k not in ("visibility_filter", "radii"))
    del a, b
    rounds = []
    for rd in range(args.rounds):
        rows = []
        for F, feat in feats.items():
            arms = {"plain": lambda: new(cams, pc, bg, feat, args.chunk), "contrib": lambda: with_acc(feat),
                    "plain_again": lambda: new(cams, pc, bg, feat, args.chunk)}
            for fn in arms.values():          # warm-up
                fn()
            times = {k: [] for k in arms}
            for r in range(args.repeats):
                for k, fn in arms.items():
                    times[k] += _flushed(fn, flush, 1, r)
            row = {"round": rd, "res": res, "F": F, "identical_outputs": ident[F],
                   **{k: _stat(v, args.frames) for k, v in times.items()}}
            base = 0.5 * (row["plain"]["ms_median"] + row["plain_again"]["ms_median"])
            row["overhead"] = row["contrib"]["ms_median"] / base - 1.0
            row["plain_gap"] = row["plain_again"]["ms_median"] / row["plain"]["ms_median"] - 1.0
            print(json.dumps(row), flush=True)
            rows.append(row)
        arms = {"before": lambda: new(cams, pc, bg, None, args.chunk), "after": lambda: new(cams, pcp, bg, None, args.chunk)}
        for fn in arms.values():
            fn()
        times = {k: [] for k in arms}
        for r in range(args.repeats):
            for k, fn in arms.items():
                times[k] += _flushed(fn, flush, 1, r)
        prune = {"round": rd, **{k: _stat(v, args.frames) for k, v in times.items()}}
        prune["speedup"] = prune["before"]["ms_median"] / prune["after"]["ms_median"]
        print(json.dumps(prune), flush=True)
        rounds.append({"rows": rows, "prune": prune})
    out = {"gpu": gpu, "frames": args.frames, "frames_per_call": args.chunk, "P": args.P, "repeats": args.repeats,
           "pruned": pruned, "rounds": rounds}
    print(json.dumps(out))
    return out


def render_frames_contrib(cams, pc, bg, feat, chunk, acc, masks=None, lift=None, values=None):
    from vidu4d_b200.renderer import PipelineParams, render_frames
    return render_frames(cams, pc, PipelineParams(), bg, features=feat, frames_per_call=chunk, contributions=acc,
                         masks=masks, lift=lift, values=values)


def silhouette_main(args, gpu):
    """--silhouette: `rounds` rounds in one process; each times, for F = 0 and 22, four arms alternating -- plain, with
    the accumulator, with the accumulator and masks, plain again (the A/A control)."""
    from vidu4d_b200.renderer import SurfelContributions
    from vidu4d_b200.synthetic import object_scene
    dev = torch.device("cuda:0")
    s = object_scene(args.P, seed=0, opacity="trained", center=(0.0, 0.0, 0.0)).to_torch(dev)
    pc = _PC(s)
    g = torch.Generator(device=dev).manual_seed(0)
    flush = torch.empty((256 << 20,), dtype=torch.uint8, device=dev)
    res = 512
    cams = _cams(args.frames, res, dev, False)
    bg = torch.zeros(3, device=dev)
    feats = {0: None, 22: torch.rand((args.P, 22), device=dev, generator=g) * 2 - 1}
    acc = SurfelContributions.zeros(args.P, dev)
    acc_bg = SurfelContributions.zeros(args.P, dev, silhouettes=True)
    masks = new(cams, pc, bg, None, args.chunk)["acc"][:, 0] > 0.5          # (T, H, W) silhouettes

    def stats(feat, a, m=None):
        for t in (a.weight_q, a.max_weight, a.pixels, a.frames) + ((a.weight_bg_q, a.pixels_bg) if m is not None else ()):
            t.zero_()
        return render_frames_contrib(cams, pc, bg, feat, args.chunk, a, m)

    check = {}
    for F, feat in feats.items():
        a, b, c = new(cams, pc, bg, feat, args.chunk), stats(feat, acc), stats(feat, acc_bg, masks)
        check[F] = {"identical_outputs": all(_same(a[k], b[k]) and _same(a[k], c[k]) for k in a if k != "visibility_filter"),
                    "identical_words": all(torch.equal(getattr(acc, k), getattr(acc_bg, k))
                                           for k in ("weight_q", "max_weight", "pixels", "frames"))}
        del a, b, c
    frac = acc_bg.background_fraction
    scene = {"foreground_pixel_fraction": float(masks.float().mean()),
             "background_pair_fraction": float(acc_bg.pixels_bg.sum()) / max(1, int(acc_bg.pixels.sum())),
             "surfels_over_half_background": int((frac > 0.5).sum()), "surfels_all_background": int((frac == 1.0).sum())}
    print(json.dumps({"check": check, "scene": scene}), flush=True)
    rounds = []
    for rd in range(args.rounds):
        rows = []
        for F, feat in feats.items():
            arms = {"plain": lambda: new(cams, pc, bg, feat, args.chunk), "contrib": lambda: stats(feat, acc),
                    "masked": lambda: stats(feat, acc_bg, masks), "plain_again": lambda: new(cams, pc, bg, feat, args.chunk)}
            for fn in arms.values():          # warm-up
                fn()
            times = {k: [] for k in arms}
            for r in range(args.repeats):
                for k, fn in arms.items():
                    times[k] += _flushed(fn, flush, 1, r)
            row = {"round": rd, "res": res, "F": F, **check[F], **{k: _stat(v, args.frames) for k, v in times.items()}}
            base = 0.5 * (row["plain"]["ms_median"] + row["plain_again"]["ms_median"])
            row["contrib_overhead"] = row["contrib"]["ms_median"] / base - 1.0
            row["masked_overhead"] = row["masked"]["ms_median"] / base - 1.0
            row["masked_over_contrib"] = row["masked"]["ms_median"] / row["contrib"]["ms_median"] - 1.0
            row["plain_gap"] = row["plain_again"]["ms_median"] / row["plain"]["ms_median"] - 1.0
            print(json.dumps(row), flush=True)
            rows.append(row)
        rounds.append(rows)
    out = {"gpu": gpu, "frames": args.frames, "frames_per_call": args.chunk, "P": args.P, "repeats": args.repeats,
           "scene": scene, "rounds": rounds}
    print(json.dumps(out))
    return out


def lift_main(args, gpu):
    """--lift: `rounds` rounds in one process; each times five arms alternating -- the accumulator alone, with lifts of
    C = 1, 16 and 32 channels, and the accumulator alone again (the A/A control)."""
    from vidu4d_b200.renderer import SurfelContributions, SurfelLift
    from vidu4d_b200.synthetic import object_scene
    dev = torch.device("cuda:0")
    s = object_scene(args.P, seed=0, opacity="trained", center=(0.0, 0.0, 0.0)).to_torch(dev)
    pc = _PC(s)
    g = torch.Generator(device=dev).manual_seed(0)
    flush = torch.empty((256 << 20,), dtype=torch.uint8, device=dev)
    res = 512
    cams = _cams(args.frames, res, dev, False)
    bg = torch.zeros(3, device=dev)
    Cs = (1, 16, 32)
    values = {C: torch.rand((args.frames, C, res, res), device=dev, generator=g) * 2 - 1 for C in Cs}
    acc = SurfelContributions.zeros(args.P, dev)
    accs = {C: SurfelContributions.zeros(args.P, dev) for C in Cs}
    lifts = {C: SurfelLift.zeros(args.P, C, dev) for C in Cs}

    def stats(a, C=None):
        for t in (a.weight_q, a.max_weight, a.pixels, a.frames):
            t.zero_()
        if C is None:
            return render_frames_contrib(cams, pc, bg, None, args.chunk, a)
        lifts[C].sums.zero_()
        lifts[C].saturated.zero_()
        return render_frames_contrib(cams, pc, bg, None, args.chunk, a, lift=lifts[C], values=values[C])

    base = stats(acc)
    check = {}
    for C in Cs:
        out = stats(accs[C], C)
        check[C] = {"identical_outputs": all(_same(base[k], out[k]) for k in base if k != "visibility_filter"),
                    "identical_words": all(torch.equal(getattr(acc, k), getattr(accs[C], k))
                                           for k in ("weight_q", "max_weight", "pixels", "frames")),
                    "saturated": int(lifts[C].saturated), "nonzero_sums": int((lifts[C].sums != 0).sum())}
        del out
    del base
    print(json.dumps({"check": check, "pairs": int(acc.pixels.sum())}), flush=True)
    rounds = []
    for rd in range(args.rounds):
        arms = {"contrib": lambda: stats(acc), **{f"lift{C}": (lambda C=C: stats(accs[C], C)) for C in Cs},
                "contrib_again": lambda: stats(acc)}
        for fn in arms.values():          # warm-up
            fn()
        times = {k: [] for k in arms}
        for r in range(args.repeats):
            for k, fn in arms.items():
                times[k] += _flushed(fn, flush, 1, r)
        row = {"round": rd, "res": res, "F": 0, **{k: _stat(v, args.frames) for k, v in times.items()}}
        base_ms = 0.5 * (row["contrib"]["ms_median"] + row["contrib_again"]["ms_median"])
        for C in Cs:
            row[f"lift{C}_over_contrib"] = row[f"lift{C}"]["ms_median"] / base_ms - 1.0
        row["contrib_gap"] = row["contrib_again"]["ms_median"] / row["contrib"]["ms_median"] - 1.0
        print(json.dumps(row), flush=True)
        rounds.append(row)
    out = {"gpu": gpu, "frames": args.frames, "frames_per_call": args.chunk, "P": args.P, "repeats": args.repeats,
           "check": {str(C): v for C, v in check.items()}, "rounds": rounds}
    print(json.dumps(out))
    return out


def anchors_main(args, gpu):
    """--anchors: `rounds` rounds in one process; each times five arms alternating -- the plain render, with anchors of
    K = 1, 4 and 8 slots, and the plain render again (the A/A control)."""
    from vidu4d_b200.renderer import PipelineParams, render_frames
    from vidu4d_b200.synthetic import object_scene
    dev = torch.device("cuda:0")
    s = object_scene(args.P, seed=0, opacity="trained", center=(0.0, 0.0, 0.0)).to_torch(dev)
    pc = _PC(s)
    flush = torch.empty((256 << 20,), dtype=torch.uint8, device=dev)
    res = 512
    cams = _cams(args.frames, res, dev, False)
    bg = torch.zeros(3, device=dev)
    Ks = (1, 4, 8)

    def run(K=None):
        return render_frames(cams, pc, PipelineParams(), bg, frames_per_call=args.chunk, anchors=K)

    base = run()
    check = {}
    for K in Ks:
        out = run(K)
        check[K] = {"identical_outputs": all(_same(base[k], out[k]) for k in base if k != "visibility_filter"),
                    "filled_slots": int((out["anchor_ids"] >= 0).sum())}
        del out
    del base
    print(json.dumps({"check": check}), flush=True)
    rounds = []
    for rd in range(args.rounds):
        arms = {"plain": lambda: run(), **{f"anchors{K}": (lambda K=K: run(K)) for K in Ks}, "plain_again": lambda: run()}
        for fn in arms.values():          # warm-up
            fn()
        times = {k: [] for k in arms}
        for r in range(args.repeats):
            for k, fn in arms.items():
                times[k] += _flushed(fn, flush, 1, r)
        row = {"round": rd, "res": res, "F": 0, **{k: _stat(v, args.frames) for k, v in times.items()}}
        base_ms = 0.5 * (row["plain"]["ms_median"] + row["plain_again"]["ms_median"])
        for K in Ks:
            row[f"anchors{K}_over_plain"] = row[f"anchors{K}"]["ms_median"] / base_ms - 1.0
        row["plain_gap"] = row["plain_again"]["ms_median"] / row["plain"]["ms_median"] - 1.0
        print(json.dumps(row), flush=True)
        rounds.append(row)
    out = {"gpu": gpu, "frames": args.frames, "frames_per_call": args.chunk, "P": args.P, "repeats": args.repeats,
           "check": {str(K): v for K, v in check.items()}, "rounds": rounds}
    print(json.dumps(out))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=64)
    ap.add_argument("--chunk", type=int, default=8)
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--P", type=int, default=300_000)
    ap.add_argument("--contrib", action="store_true", help="measure the contribution statistics and the prune by them")
    ap.add_argument("--silhouette", action="store_true", help="measure the background share of the statistics")
    ap.add_argument("--lift", action="store_true", help="measure lifting per-pixel maps onto the surfels")
    ap.add_argument("--anchors", action="store_true", help="measure keeping each pixel's heaviest pairs")
    ap.add_argument("--rounds", type=int, default=3,
                    help="--contrib / --silhouette / --lift / --anchors: rounds of every measurement in one process")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_render needs a CUDA device")
    from vidu4d_b200 import _capi
    from vidu4d_b200.synthetic import object_scene
    dev = torch.device("cuda:0")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    if args.contrib or args.silhouette or args.lift or args.anchors:
        out = (contrib_main(args, gpu) if args.contrib else silhouette_main(args, gpu) if args.silhouette
               else lift_main(args, gpu) if args.lift else anchors_main(args, gpu))
        if args.out:
            os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
            with open(args.out, "w") as f:
                json.dump(out, f, indent=1)
        return
    s = object_scene(args.P, seed=0, opacity="trained", center=(0.0, 0.0, 0.0)).to_torch(dev)
    pc = _PC(s)
    g = torch.Generator(device=dev).manual_seed(0)
    results = []
    for res in (512, 128):
        for F in (0, 22):
            for table in (False, True):
                cams = _cams(args.frames, res, dev, table)
                feat = (torch.rand((args.P, F), device=dev, generator=g) * 2 - 1) if F else None
                bg = torch.zeros(3, device=dev)
                arms = {"render_frames": lambda: new(cams, pc, bg, feat, args.chunk),
                        "today": lambda: today(cams, pc, bg, feat, args.chunk)}
                for fn in arms.values():          # warm-up: capacity hints, module loads, allocator
                    fn()
                torch.cuda.synchronize()
                bad = mismatches(arms["today"](), arms["render_frames"](), args.chunk)
                times = {k: [] for k in arms}
                for _ in range(args.repeats):     # alternate the arms
                    for k, fn in arms.items():
                        times[k] += timed(fn, 1)
                row = {"res": res, "F": F, "cameras": "table" if table else "scalar", "identical": not bad, "mismatches": bad}
                base = torch.cuda.memory_allocated(dev)
                for k, fn in arms.items():
                    torch.cuda.synchronize()
                    torch.cuda.reset_peak_memory_stats(dev)
                    fn()
                    torch.cuda.synchronize()
                    peak = torch.cuda.max_memory_allocated(dev) - base
                    _capi.set_profiling(True)
                    fn()
                    prof = _capi.get_profile()
                    _capi.set_profiling(False)
                    t = np.asarray(times[k])
                    row[k] = {"fps_median": args.frames / (float(np.median(t)) / 1e3),
                              "fps_min": args.frames / (float(t.max()) / 1e3), "fps_max": args.frames / (float(t.min()) / 1e3),
                              "ms_median": float(np.median(t)), "peak_bytes_above_inputs": int(peak),
                              "kernels_ms": {n: round(v["ms"], 4) for n, v in prof.items()}}
                row["speedup"] = row["render_frames"]["fps_median"] / row["today"]["fps_median"]
                print(json.dumps(row), flush=True)
                results.append(row)
    out = {"gpu": gpu, "frames": args.frames, "frames_per_call": args.chunk, "P": args.P, "rows": results}
    print(json.dumps(out))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
