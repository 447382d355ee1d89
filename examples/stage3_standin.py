#!/usr/bin/env python
"""Stage-3 stand-in (BASELINE.json configs[2]): the warp -> rasterize -> loss -> Adam inner loop of
`lab4d/train.py --fg_motion gs-bob` on synthetic data, with this rasterizer dropped in.

What is mirrored from the reference (behaviour, not code):
  * canonical surfels warped per frame by a bag-of-bones dual-quaternion skinning field, kept in PyTorch as
    north_star asks: Gaussian skin logits -(dist^2) -> softmax -> sign-aligned DQ blend -> (q, t) per surfel ->
    x' = q x + t, r' = q (x) r        (lab4d/utils/geom_utils.py:48-92, lab4d/nnutils/skinning.py:89-124,
    lab4d/nnutils/deformable_gaussian.py:1033-1046,1395-1434)
  * the warped surfels are ALREADY in camera space and rendered with the identity KCamera
    (gs/scene/cameras.py:84-87,160-162, deformable_gaussian.py:1170-1188); inputs to the rasterizer are non-leaf
  * M = 2 frames per optimisation step (lab4d/engine/trainer.py:453-468), L1 on colour + normal-consistency +
    distortion regularisers (lab4d/engine/model.py:674-692,817-842), Adam on the surfel parameters
    (trainer.py:240-255), learnable-background in-place edit of the render (deformable_gaussian.py:188-190)

    python examples/stage3_standin.py --surfels 300000 --res 256 --frames 32 --steps 200
"""
from __future__ import annotations

import argparse
import json
import math
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from vidu4d_b200 import rasterizer as RZ  # noqa: E402
from vidu4d_b200.distributed import FlatGrads  # noqa: E402
from vidu4d_b200.renderer import PipelineParams, make_camera, render_fused  # noqa: E402
from vidu4d_b200.synthetic import SurfelCloud, object_scene  # noqa: E402


# ---- quaternion helpers (w, x, y, z) -----------------------------------------------------------
def qmul(a, b):
    aw, ax, ay, az = a.unbind(-1)
    bw, bx, by, bz = b.unbind(-1)
    return torch.stack([aw * bw - ax * bx - ay * by - az * bz, aw * bx + ax * bw + ay * bz - az * by,
                        aw * by - ax * bz + ay * bw + az * bx, aw * bz + ax * by - ay * bx + az * bw], -1)


def qconj(q):
    return q * q.new_tensor([1.0, -1.0, -1.0, -1.0])


def qrot(q, v):
    qv = torch.cat([torch.zeros_like(v[..., :1]), v], -1)
    return qmul(qmul(q, qv), qconj(q))[..., 1:]


class BobWarp(torch.nn.Module):
    """B bones with rest centres; per frame a rigid motion per bone; Gaussian skinning + DQ blending."""

    def __init__(self, n_bones, n_frames, center, radius, seed=0, amplitude=0.15, device="cuda"):
        super().__init__()
        g = torch.Generator().manual_seed(seed)
        d = torch.randn((n_bones, 3), generator=g)
        d = d / d.norm(dim=1, keepdim=True)
        self.register_buffer("rest", (d * radius * 0.7 + torch.tensor(center)).to(device))
        self.log_scale = torch.nn.Parameter(torch.full((n_bones,), math.log(radius * 0.6), device=device))
        # smooth per-frame articulation: axis-angle and translation as low-frequency sinusoids
        ph = torch.rand((n_bones, 3), generator=g) * 2 * math.pi
        tt = torch.arange(n_frames).float()[:, None, None] / max(n_frames, 1) * 2 * math.pi
        aa = amplitude * torch.sin(tt + ph[None])                    # (F,B,3)
        tr = 0.1 * radius * torch.cos(tt * 0.5 + ph[None])
        self.axis_angle = torch.nn.Parameter(aa.to(device))
        self.trans = torch.nn.Parameter(tr.to(device))

    def bone_dq(self, frame):
        aa = self.axis_angle[frame]
        ang = aa.norm(dim=-1, keepdim=True).clamp_min(1e-8)
        qr = torch.cat([torch.cos(ang / 2), torch.sin(ang / 2) * aa / ang], -1)          # (B,4)
        # rotate about the bone's rest centre, then translate:  x' = q (x - c) + c + t
        t = self.rest - qrot(qr, self.rest) + self.trans[frame]
        qd = 0.5 * qmul(torch.cat([torch.zeros_like(t[:, :1]), t], -1), qr)
        return qr, qd

    def forward(self, xyz, rot, frame):
        qr, qd = self.bone_dq(frame)
        d2 = ((xyz[:, None, :] - self.rest[None]) ** 2).sum(-1) / torch.exp(2 * self.log_scale)[None]   # (P,B)
        w = torch.softmax(-d2, dim=1)
        sign = torch.where((qr * qr[:1]).sum(-1, keepdim=True) < 0, -1.0, 1.0)          # sign-align to bone 0
        br = w @ (qr * sign)
        bd = w @ (qd * sign)
        n = br.norm(dim=-1, keepdim=True)
        br, bd = br / n, bd / n
        t = 2.0 * qmul(bd, qconj(br))[..., 1:]
        return qrot(br, xyz) + t, qmul(br, rot)


class WarpedView:
    """What render() reads from `pc`, for one frame: warped (non-leaf) xyz / rotation, shared other attributes."""

    def __init__(self, cloud, xyz, rot):
        self._c, self._xyz, self._rot = cloud, xyz, rot
        self.active_sh_degree = cloud.active_sh_degree

    get_xyz = property(lambda s: s._xyz)
    get_rotation = property(lambda s: torch.nn.functional.normalize(s._rot))
    get_opacity = property(lambda s: s._c.get_opacity)
    get_scaling = property(lambda s: s._c.get_scaling)
    get_features = property(lambda s: s._c.get_features)


def loss_fn(out, target, learnable_bg):
    out["render"][:3] = out["render"][:3] + (1 - out["acc"]) * learnable_bg       # in-place, as the reference does
    l1 = (out["render"] - target).abs().mean()
    normal = (1.0 - (out["rend_normal"] * out["surf_normal"]).sum(0)).mean()
    return l1 + 0.05 * normal + 0.01 * out["rend_dist"].mean()


def run(surfels=300_000, res=256, frames=32, steps=100, bones=25, device="cuda", seed=0, log_every=20, quiet=False):
    dev = torch.device(device)
    center = (0.0, 0.0, 1.0)
    gt_scene = object_scene(surfels, seed=seed, center=center)
    gt_cloud = SurfelCloud(gt_scene, dev)
    warp = BobWarp(bones, frames, center, 0.35, seed=seed, device=dev)
    cam = make_camera(res, res, 2 * math.atan(0.5), 2 * math.atan(0.5), device=dev)      # identity KCamera
    bg = torch.zeros(3, device=dev)
    pipe = PipelineParams()
    with torch.no_grad():   # targets: the ground-truth cloud under the ground-truth articulation
        targets = []
        for f in range(frames):
            x, r = warp(gt_cloud.get_xyz, gt_cloud._rotation, f)
            targets.append(render_fused(cam, WarpedView(gt_cloud, x, r), pipe, bg)["render"].clone())
    # the model starts from perturbed colours / opacities / positions and has to recover the targets
    init = object_scene(surfels, seed=seed, center=center)
    rng = np.random.default_rng(seed + 1)
    init.shs[:, 0] = init.shs[:, 0] * 0.3
    init.means3D += (0.003 * rng.normal(size=init.means3D.shape)).astype(np.float32)
    cloud = SurfelCloud(init, dev)
    learnable_bg = torch.zeros((3, 1, 1), device=dev, requires_grad=True)
    params = cloud.flat_params()
    fg = FlatGrads(params)
    opt = torch.optim.Adam([{"params": [cloud._xyz], "lr": 1.6e-5}, {"params": [cloud._features_dc], "lr": 2.5e-2},
                            {"params": [cloud._features_rest], "lr": 1.25e-3}, {"params": [cloud._opacity], "lr": 5e-2},
                            {"params": [cloud._scaling], "lr": 5e-3}, {"params": [cloud._rotation], "lr": 1e-3},
                            {"params": [learnable_bg], "lr": 1e-3}], fused=True)
    RZ.set_sync_mode(False)
    losses, t0 = [], None
    try:
        for step in range(steps):
            if step == 5:
                torch.cuda.synchronize(); t0 = time.perf_counter()
            fg.zero_()
            if learnable_bg.grad is not None:
                learnable_bg.grad.zero_()
            tot = 0.0
            for m in range(2):                                   # M = 2 frames per step
                f = (2 * step + m) % frames
                x, r = warp(cloud.get_xyz, cloud._rotation, f)
                out = render_fused(cam, WarpedView(cloud, x, r), pipe, bg)
                loss = loss_fn(out, targets[f], learnable_bg)
                loss.backward()
                tot = tot + loss.detach()
            opt.step()
            RZ.check_overflow()
            if step % log_every == 0 or step == steps - 1:
                losses.append((step, float(tot) / 2))
                if not quiet:
                    print(f"step {step:5d}  loss {losses[-1][1]:.5f}", flush=True)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0 if t0 else float("nan")
    finally:
        RZ.set_sync_mode(True)
    return {"surfels": surfels, "res": res, "frames": frames, "bones": bones, "steps": steps, "losses": losses,
            "steps_per_s": round((steps - 5) / dt, 2) if t0 else None, "frames_per_s": round(2 * (steps - 5) / dt, 2) if t0 else None}


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--surfels", type=int, default=300_000)
    ap.add_argument("--res", type=int, default=256)
    ap.add_argument("--frames", type=int, default=32)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--bones", type=int, default=25)
    a = ap.parse_args()
    print(json.dumps(run(a.surfels, a.res, a.frames, a.steps, a.bones)))
