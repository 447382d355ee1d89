"""Time and byte count of `preprocess_fwd` on the headline batch (300 K surfels, SH degree 3, 512^2, every per-surfel input
shared by the frames), at M = 1, 2 and 8 frames per launch.

Time: the library's per-kernel CUDA events (sr_set_profiling) over --launches batched forwards after one warm-up.
Bytes: what the kernel must move, from the shapes and frame strides of its arguments -- an input shared by every frame
(stride 0) once per launch, a per-frame input and every output once per frame.  Written outputs per frame: radius and
tiles_touched of every surfel, the 80-byte surfel record + depth + clamped bits of every surfel that touches a tile,
and one block sum per 256 surfels.  GB/s is set against the H100 SXM data-sheet 3.35 TB/s; the card's name, power
limit and SM clocks are read in the same run, since they are part of the number.

Usage: python tools/prof_preprocess.py [--frames 1,2,8] [--surfels 300000] [--res 512] [--launches 50] [--json out.json]
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
from vidu4d_b200 import _capi  # noqa: E402
from vidu4d_b200 import rasterizer as RZ  # noqa: E402
from vidu4d_b200.synthetic import object_scene, orbit_view, projection_matrix  # noqa: E402

DATASHEET_GBS = 3350.0


def card():
    out = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        out["power_limit"], out["sm_clock"], out["sm_clock_max"] = (s.strip() for s in q.split(","))
    except Exception as e:  # the numbers stay usable; the missing context is stated
        out["nvidia_smi"] = f"unavailable: {e}"
    return out


def views(M, dev):
    P = projection_matrix(0.5, 0.5).astype(np.float64)
    vms, pms, cps = [], [], []
    for f in range(M):
        Rm, tt = orbit_view(f, 64)
        W2C = np.eye(4); W2C[:3, :3] = Rm; W2C[:3, 3] = tt
        vms.append(W2C.T.astype(np.float32)); pms.append((W2C.T @ P).astype(np.float32)); cps.append((-Rm.T @ tt).astype(np.float32))
    return (torch.from_numpy(np.stack(a)).to(dev) for a in (vms, pms, cps))


def kernel_bytes(inputs, M, P, visible):
    """inputs: {name: (tensor, shared)}.  visible: per-frame count of surfels that touch a tile."""
    rd = 0
    for t, shared in inputs.values():
        per_frame = t.numel() * t.element_size() // (1 if shared else M)
        rd += per_frame * (1 if shared else M)
    wr = sum(P * (4 + 4) + v * (80 + 4 + 1) for v in visible) + M * ((P + 255) // 256) * 4
    reread = sum(t.numel() * t.element_size() * (M - 1) for t, shared in inputs.values() if shared)
    return rd, wr, reread


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", default="1,2,8")
    ap.add_argument("--surfels", type=int, default=300_000)
    ap.add_argument("--res", type=int, default=512)
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--json", default=None, help="also write the result lines to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("prof_preprocess: no CUDA device; kernel times are only measured on the GPU")
    dev = torch.device("cuda:0")
    sc = object_scene(a.surfels, seed=0, opacity="trained", center=(0, 0, 0))
    t = sc.to_torch(dev)
    e = torch.empty((0,), device=dev)
    bg = torch.zeros(3, device=dev)
    C = RZ._C
    rows = []
    info = card()
    for M in (int(s) for s in a.frames.split(",")):
        vms, pms, cps = views(M, dev)

        def fwd():
            return C.rasterize_gaussians_batch(bg, t["means3D"], e, t["opacities"], t["scales"], t["rotations"], 1.0, vms, pms, 0.5,
                                               0.5, a.res, a.res, t["shs"], 3, cps)
        o = fwd()
        torch.cuda.synchronize()
        visible = [int(v) for v in (o[3] > 0).sum(dim=1).tolist()]
        _capi.get_profile()
        _capi.set_profiling(True)
        for _ in range(a.launches):
            fwd()
        prof = _capi.get_profile()
        _capi.set_profiling(False)
        RZ.check_overflow()
        k = prof["preprocess_fwd"]
        ms = k["ms"] / max(k["count"], 1)
        inputs = {n: (t[n], True) for n in ("means3D", "shs", "opacities", "scales", "rotations")}
        rd, wr, reread = kernel_bytes(inputs, M, a.surfels, visible)
        row = {"kernel": "preprocess_fwd", "frames": M, "P": a.surfels, "res": a.res, "launches": k["count"],
               "ms_per_launch": round(ms, 5), "ms_per_frame": round(ms / M, 5),
               "MB_read": round(rd / 1e6, 2), "MB_written": round(wr / 1e6, 2),
               "MB_if_shared_inputs_reread_per_frame": round((rd + wr + reread) / 1e6, 2),
               "GBps": round((rd + wr) / 1e9 / (ms * 1e-3), 1), "frac_of_3350": round((rd + wr) / 1e9 / (ms * 1e-3) / DATASHEET_GBS, 3),
               "visible_per_frame": visible, "card": info}
        rows.append(row)
        print(json.dumps(row), flush=True)
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
