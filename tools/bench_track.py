"""Dense point tracking: track_pixels (csrc/track.cu) against the same math in chunked torch.

Workload: bench.py's object scene of 300 K surfels, moved per frame (a small rigid wobble, as the bob-warped copies of
Stage 3 would be), 64 orbiting cameras at 512^2.  Frame 0 is rendered with anchors=4 and every one of its 262 144 pixels is
tracked through the 64 frames.  Both arms are timed alternating, with CUDA events, L2 flushed by a 256 MB write before
every timed call; the torch arm processes --chunk queries at a time.  Reported per arm: median / min / max ms, peak
allocator bytes above the inputs; and the largest difference of xy and z between the arms over the valid queries.
Prints one JSON object; --out writes it too.

Usage: python tools/bench_track.py [--frames 64] [--P 300000] [--repeats 7] [--chunk 16384] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import math
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_render import _PC, _cams, _flushed, _stat  # noqa: E402


def _rotmat(q):
    """(.., 3, 3) rotation of unit-normalised quaternions (w, x, y, z); column 0 is t_u, column 1 t_v."""
    q = q / q.norm(dim=-1, keepdim=True)
    w, x, y, z = q.unbind(-1)
    return torch.stack([
        torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)], -1),
        torch.stack([2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)], -1),
        torch.stack([2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], -1)], -2)


def torch_track(anchors, queries, cams, means, rots, scales, chunk):
    """track_pixels' math in float32 torch, `chunk` queries at a time: (xy (N,T,2), z (N,T), coverage (N,))."""
    ids, w, uv = anchors
    S, K, H, W = ids.shape
    T = means.shape[0]
    N = queries.shape[0]
    f = torch.tensor([W / (2 * math.tan(cams.FoVx * 0.5)), H / (2 * math.tan(cams.FoVy * 0.5))], device=ids.device)
    c = torch.tensor([W / 2, H / 2], device=ids.device)
    vm = cams.world_view_transform                                       # (T,4,4), W2C transposed
    xy = torch.empty((N, T, 2), device=ids.device)
    z = torch.empty((N, T), device=ids.device)
    cov = torch.empty((N,), device=ids.device)
    for a in range(0, N, chunk):
        q = queries[a:a + chunk].long()
        s, x, y = q[:, 0], q[:, 1], q[:, 2]
        i = ids[s, :, y, x].long()                                       # (n,K)
        on = i >= 0
        ic = torch.where(on, i, torch.zeros_like(i))
        wk = torch.where(on, w[s, :, y, x], torch.zeros_like(w[s, :, y, x]))
        u, v = uv[s, :, 0, y, x], uv[s, :, 1, y, x]
        R = _rotmat(rots[:, ic])                                         # (T,n,K,3,3)
        sc = scales[ic]                                                  # (n,K,2)
        p = means[:, ic] + (u * sc[..., 0])[None, ..., None] * R[..., 0] + (v * sc[..., 1])[None, ..., None] * R[..., 1]
        sw = wk.sum(1)
        X = (wk[None, ..., None] * p).sum(2) / sw[None, :, None]         # (T,n,3)
        Xc = torch.einsum("tnj,tjk->tnk", X, vm[:, :3, :3]) + vm[:, None, 3, :3]
        xy[a:a + chunk] = (f * Xc[..., :2] / Xc[..., 2:3] + c).transpose(0, 1)
        z[a:a + chunk] = Xc[..., 2].transpose(0, 1)
        cov[a:a + chunk] = sw
    return xy, z, cov


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=64)
    ap.add_argument("--P", type=int, default=300_000)
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--chunk", type=int, default=16384)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_track needs a CUDA device")
    from vidu4d_b200.renderer import PipelineParams, render_frames
    from vidu4d_b200.synthetic import object_scene
    from vidu4d_b200.tracking import track_pixels
    dev = torch.device("cuda:0")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    s = object_scene(args.P, seed=0, opacity="trained", center=(0.0, 0.0, 0.0)).to_torch(dev)
    pc = _PC(s)
    T, res, K = args.frames, 512, 4
    cams = _cams(T, res, dev, False)
    # each frame's surfels: frame 0's, turned by a small angle about y and shifted
    means, rots = [], []
    for t in range(T):
        a = 0.1 * math.sin(2 * math.pi * t / T)
        Rt = torch.tensor([[math.cos(a), 0, math.sin(a)], [0, 1, 0], [-math.sin(a), 0, math.cos(a)]], device=dev)
        qt = torch.tensor([math.cos(a / 2), 0.0, math.sin(a / 2), 0.0], device=dev)
        means.append(s["means3D"] @ Rt.T + torch.tensor([0.02 * math.sin(a), 0.0, 0.0], device=dev))
        w1, x1, y1, z1 = qt.unbind(-1)
        w2, x2, y2, z2 = s["rotations"].unbind(-1)
        rots.append(torch.stack([w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2, w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2,
                                 w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2, w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2], -1))
    means, rots = torch.stack(means).contiguous(), torch.stack(rots).contiguous()
    first = type(cams)(res, res, cams.FoVx, cams.FoVy, cams.world_view_transform[:1].contiguous(),
                       cams.full_proj_transform[:1].contiguous(), cams.camera_center[:1].contiguous(), None)
    r = render_frames(first, pc, PipelineParams(), torch.zeros(3, device=dev), means3D=means[:1].contiguous(),
                      rotations=rots[:1].contiguous(), anchors=K)
    anchors = (r["anchor_ids"], r["anchor_weights"], r["anchor_uv"])
    yy, xx = torch.meshgrid(torch.arange(res, device=dev), torch.arange(res, device=dev), indexing="ij")
    queries = torch.stack([torch.zeros_like(xx), xx, yy], -1).reshape(-1, 3).int().contiguous()
    del r

    arms = {"track_pixels": lambda: track_pixels(anchors, queries, cams, pc, means3D=means, rotations=rots),
            "torch": lambda: torch_track(anchors, queries, cams, means, rots, s["scales"], args.chunk)}
    got, ref = arms["track_pixels"](), arms["torch"]()
    valid = got["coverage"] > 0
    check = {"queries": int(queries.shape[0]), "valid": int(valid.sum()),
             "max_abs_xy": float((got["xy"][valid] - ref[0][valid]).abs().max()),
             "max_abs_z": float((got["z"][valid] - ref[1][valid]).abs().max()),
             "max_abs_coverage": float((got["coverage"] - ref[2]).abs().max())}
    del got, ref
    print(json.dumps({"check": check}), flush=True)
    flush = torch.empty((256 << 20,), dtype=torch.uint8, device=dev)
    for fn in arms.values():              # warm-up
        fn()
    times = {k: [] for k in arms}
    for rep in range(args.repeats):
        for k, fn in arms.items():
            times[k] += _flushed(fn, flush, 1, rep)
    row = {k: _stat(v, T) for k, v in times.items()}
    base = torch.cuda.memory_allocated(dev)
    for k, fn in arms.items():
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats(dev)
        out = fn()
        torch.cuda.synchronize()
        row[k]["peak_bytes_above_inputs"] = int(torch.cuda.max_memory_allocated(dev) - base)
        del out
    row["speedup"] = row["torch"]["ms_median"] / row["track_pixels"]["ms_median"]
    out = {"gpu": gpu, "frames": T, "res": res, "K": K, "P": args.P, "torch_chunk": args.chunk, "repeats": args.repeats,
           "check": check, "timing": row}
    print(json.dumps(out))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
