#!/usr/bin/env python
"""BASELINE.json configs[2] (C3): the full Stage-3 gs-bob inner loop -- bob-skinning warp -> rasterize -> image losses ->
backward -> Adam -- on a synthetic 32-frame sequence, 300 K surfels, 256x256, M = 2 frames per optimisation step
(lab4d/engine/trainer.py:453-468), timed with three backends IN THE SAME LOOP on one GPU:

  reference   PyTorch warp (the reference's expressions: lab4d/utils/geom_utils.py:48-92, lab4d/nnutils/skinning.py:89-142,
              lab4d/nnutils/deformable_gaussian.py:1033-1046,1395-1434) + the UNMODIFIED reference rasterizer
              (oracle/_ref/_C.so through render()) frame by frame + torch losses
  ours        the same PyTorch warp + render_loss_batch (batched rasterizer, fused post-processing + losses)
  ours_fused  fused warp kernel (csrc/warp.cu) + render_loss_batch
  ours_full   ours_graph + FlatSurfelModel: flat parameter buffer, one-kernel Adam, densification statistics in the captured step
              (`ours_full_densify`: one densify_and_prune + graph re-capture in the middle of the timed loop)
  ours_graph  ours_fused with the WHOLE step (bone tables -> warp -> rasterize -> losses -> backward -> Adam) captured in a
              CUDA graph (vidu4d_b200.graph.GraphedStep): the step is ~25 kernels of this library plus ~100 tiny torch
              kernels for the B x M bone tables, so eager launch overhead is most of what is left

It reports steps/s of each and the warp's share of a step (CUDA events around the warp's forward and backward), which is
the number that says whether SURVEY.md 8(f) row N2 pays.

    python examples/stage3_step.py --surfels 300000 --res 256 --frames 32 --steps 60 [--backends ours_fused,ours,reference]
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
from vidu4d_b200 import renderer as RN  # noqa: E402
from vidu4d_b200.renderer import BatchCameras, PipelineParams, make_camera, render, render_loss_batch  # noqa: E402
from vidu4d_b200.synthetic import SurfelCloud, object_scene, projection_matrix  # noqa: E402
from vidu4d_b200.warp import bob_warp  # noqa: E402


from vidu4d_b200.warp import _qconj as qconj, _qmul as _qmul_small  # noqa: E402


def qmul(a, b):
    """Hamilton product.  Small operands (bone tables) take the 4-kernel gather form; the big (M,P,B,4) blends of the
    PyTorch warp take the component form, which is the faster of the two there (no 4x intermediate) -- the reference
    backend gets whichever PyTorch formulation is quickest for its tensor sizes."""
    if max(a.numel(), b.numel()) <= (1 << 16):
        return _qmul_small(a, b)
    aw, ax, ay, az = a.unbind(-1)
    bw, bx, by, bz = b.unbind(-1)
    return torch.stack((aw * bw - ax * bx - ay * by - az * bz, aw * bx + ax * bw + ay * bz - az * by,
                        aw * by - ax * bz + ay * bw + az * bx, aw * bz + ax * by - ay * bx + az * bw), -1)


def qapply(q, p):
    p4 = torch.cat((torch.zeros_like(p[..., :1]), p), -1)
    return qmul(qmul(q, p4), qconj(q))[..., 1:]


def q2dq(q, t):
    t4 = torch.cat((torch.zeros_like(t[..., :1]), t), -1)
    return q, 0.5 * qmul(t4, q)


def torch_warp(xyz, rot, rest, art, log_gauss, field2cam):
    """The reference's PyTorch chain, tensor shapes included: (M,P,B,4) blends, per-frame skinning weights."""
    M, B = art[0].shape[:2]
    P = xyz.shape[0]
    rr, rd = rest[0][None].expand(M, -1, -1), rest[1][None].expand(M, -1, -1)
    ir, idq = qconj(rr), qconj(rd)
    se3 = (qmul(art[0], ir), qmul(art[0], idq) + qmul(art[1], ir))
    xyz4 = xyz[None].expand(M, -1, -1)
    oq, ot = ir, 2.0 * qmul(idq, qconj(ir))[..., 1:]
    xb = qapply(oq[:, None], xyz4[:, :, None, :].expand(-1, -1, B, -1)) + ot[:, None]       # (M,P,B,3)
    skin = -((xb / log_gauss.exp()[None, None]) ** 2).sum(-1)
    w = skin.softmax(-1)
    qr = se3[0][:, None].repeat(1, P, 1, 1)
    qd = se3[1][:, None].repeat(1, P, 1, 1)
    anchor = w.argmax(-1).view(M, P, 1, 1).repeat(1, 1, 1, 4)
    sign = ((torch.gather(qr, 2, anchor) * qr).sum(-1) > 0)[..., None].float() * 2 - 1
    qr, qd = sign * qr, sign * qd
    qr_w = torch.einsum("bnk,bnkl->bnl", w, qr)
    qd_w = torch.einsum("bnk,bnkl->bnl", w, qd)
    inv = qr_w.norm(p=2, dim=-1, keepdim=True).reciprocal()
    qr_w, qd_w = qr_w * inv, qd_w * inv
    t = 2 * qmul(qd_w, qconj(qr_w))[..., 1:]
    xt = qapply(qr_w, xyz4) + t
    rt = qmul(qr_w, rot[None].expand(M, -1, -1))
    qc, tc = field2cam
    return qapply(qc[:, None], xt) + tc[:, None], qmul(qc[:, None].expand_as(rt), rt)


class Sequence(torch.nn.Module):
    """Learnable articulation of B bones over F frames + field2cam, parametrised like the reference: quaternion +
    translation per bone (rest and per frame), log Gaussian scales."""

    def __init__(self, B, F, radius, dev, seed=0):
        super().__init__()
        g = torch.Generator().manual_seed(seed)
        d = torch.randn((B, 3), generator=g); d = d / d.norm(dim=1, keepdim=True)
        self.rest_t = torch.nn.Parameter((d * radius * 0.7).to(dev))
        self.rest_q = torch.nn.Parameter(torch.tensor([[1.0, 0, 0, 0]]).repeat(B, 1).to(dev))
        self.log_gauss = torch.nn.Parameter(torch.full((B, 3), math.log(radius * 0.4)).to(dev))
        ph = torch.rand((B, 3), generator=g) * 2 * math.pi
        tt = torch.arange(F).float()[:, None, None] / max(F, 1) * 2 * math.pi
        aa = 0.15 * torch.sin(tt + ph[None])
        ang = aa.norm(dim=-1, keepdim=True).clamp_min(1e-8)
        self.art_q = torch.nn.Parameter(torch.cat([torch.cos(ang / 2), torch.sin(ang / 2) * aa / ang], -1).to(dev))   # (F,B,4)
        self.art_t = torch.nn.Parameter((d[None] * radius * 0.7 + 0.03 * radius * torch.cos(tt * 0.5 + ph[None])).to(dev))
        self.cam_q = torch.nn.Parameter(torch.tensor([[1.0, 0, 0, 0]]).repeat(F, 1).to(dev))
        self.cam_t = torch.nn.Parameter(torch.tensor([[0.0, 0.0, 1.0]]).repeat(F, 1).to(dev))

    def tables(self, frames):
        nq = torch.nn.functional.normalize
        return (q2dq(nq(self.rest_q, dim=-1), self.rest_t), q2dq(nq(self.art_q[frames], dim=-1), self.art_t[frames]),
                self.log_gauss, (nq(self.cam_q[frames], dim=-1), self.cam_t[frames]))


class WarpedView:
    def __init__(self, cloud, xyz, rot):
        self._c, self._xyz, self._rot = cloud, xyz, rot
        self.active_sh_degree = cloud.active_sh_degree
    get_xyz = property(lambda s: s._xyz)
    get_rotation = property(lambda s: torch.nn.functional.normalize(s._rot))
    get_opacity = property(lambda s: s._c.get_opacity)
    get_scaling = property(lambda s: s._c.get_scaling)
    get_features = property(lambda s: s._c.get_features)


def run_graph(surfels, res, frames, steps, bones, warm=5, seed=0):
    """ours_fused, whole step in one CUDA graph.  The frame pair of a step is a device tensor the graph reads."""
    from vidu4d_b200.graph import GraphedStep
    dev = torch.device("cuda:0")
    M = 2
    cloud = SurfelCloud(object_scene(surfels, seed=seed, center=(0.0, 0.0, 0.0)), dev)
    seq = Sequence(bones, frames, 0.35, dev, seed)
    tan = 0.5
    fov = 2 * math.atan(tan)
    eye = torch.eye(4, device=dev)[None].expand(M, -1, -1).contiguous()
    pm = torch.from_numpy(projection_matrix(tan, tan)).to(dev)[None].expand(M, -1, -1).contiguous()
    bc = BatchCameras(res, res, fov, fov, eye, pm, torch.zeros((M, 3), device=dev))
    bg = torch.zeros(3, device=dev)
    pipe = PipelineParams()
    targets = torch.rand((frames, 3, res, res), generator=torch.Generator().manual_seed(1)).to(dev)
    params = cloud.flat_params() + list(seq.parameters())
    opt = torch.optim.Adam(params, lr=1e-5, fused=True, capturable=True)
    fr = torch.zeros((M,), dtype=torch.int64, device=dev)
    loss_out = torch.zeros((), device=dev)

    def body():
        opt.zero_grad(set_to_none=False)
        rest, art, lg, f2c = seq.tables(fr)
        xc, rc, ent = bob_warp(cloud.get_xyz, cloud._rotation, rest, art, lg, f2c)
        loss = render_loss_batch(bc, cloud, pipe, bg, targets.index_select(0, fr), w_rgb=1.0, lambda_normal=0.05, lambda_dist=0.01,
                                 means3D=xc, rotations=torch.nn.functional.normalize(rc, dim=-1))["loss"]
        loss.backward()
        opt.step()
        loss_out.copy_(loss.detach())
        fr.add_(2).remainder_(frames)
    fr.copy_(torch.tensor([0, 1], device=dev))
    step = GraphedStep(body, device=dev)
    t0 = None
    for i in range(steps + warm):
        if i == warm:
            torch.cuda.synchronize(); t0 = time.perf_counter()
        step()
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    RZ.set_sync_mode(True); RZ._pending.clear()
    return {"backend": "ours_graph", "steps_per_s": round(steps / dt, 2), "frames_per_s": round(M * steps / dt, 2),
            "ms_per_step": round(dt / steps * 1e3, 3), "loss": float(loss_out), "graph_launches_of_this_library": step.launches}


def run_full(surfels, res, frames, steps, bones, warm=5, seed=0, densify_at=None):
    """Everything on the fast path: FlatSurfelModel (flat parameter buffer, one-kernel Adam, one-gather densify / prune),
    fused warp, render_loss_batch, the step as one CUDA graph that is re-captured when densification changes P."""
    from vidu4d_b200.graph import GraphedStep
    from vidu4d_b200.surfel_store import FlatSurfelModel
    dev = torch.device("cuda:0")
    M = 2
    sc = object_scene(surfels, seed=seed, center=(0.0, 0.0, 0.0))
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    op = np.clip(sc.opacities, 1e-6, 1 - 1e-6)
    model = FlatSurfelModel(t(sc.means3D), t(sc.shs[:, :1]), t(sc.shs[:, 1:]), t(np.log(op / (1 - op))), t(np.log(sc.scales)), t(sc.rotations),
                            lrs={"xyz": 1e-5, "f_dc": 1e-5, "f_rest": 1e-5, "opacity": 1e-5, "scaling": 1e-5, "rotation": 1e-5})
    seq = Sequence(bones, frames, 0.35, dev, seed)
    tan = 0.5
    fov = 2 * math.atan(tan)
    eye = torch.eye(4, device=dev)[None].expand(M, -1, -1).contiguous()
    pm = torch.from_numpy(projection_matrix(tan, tan)).to(dev)[None].expand(M, -1, -1).contiguous()
    bc = BatchCameras(res, res, fov, fov, eye, pm, torch.zeros((M, 3), device=dev))
    bg = torch.zeros(3, device=dev)
    pipe = PipelineParams()
    targets = torch.rand((frames, 3, res, res), generator=torch.Generator().manual_seed(1)).to(dev)
    opt = torch.optim.Adam(list(seq.parameters()), lr=1e-5, fused=True, capturable=True)
    fr = torch.zeros((M,), dtype=torch.int64, device=dev)
    loss_out = torch.zeros((), device=dev)
    stats = {}

    def body():
        opt.zero_grad(set_to_none=False)
        model.zero_grad_flat()
        rest, art, lg, f2c = seq.tables(fr)
        xc, rc, ent = bob_warp(model.get_xyz, model._rotation, rest, art, lg, f2c)
        out = render_loss_batch(bc, model, pipe, bg, targets.index_select(0, fr), w_rgb=1.0, lambda_normal=0.05, lambda_dist=0.01,
                                means3D=xc, rotations=torch.nn.functional.normalize(rc, dim=-1))
        out["loss"].backward()
        # densification statistics (trainer.py:553-560), inside the graph: all M frames in one kernel, on device
        model.add_densification_stats(out["viewspace_points"].grad, out["visibility_filter"], out["radii"])
        model.adam_step()
        opt.step()
        loss_out.copy_(out["loss"].detach())
        fr.add_(2).remainder_(frames)
    fr.copy_(torch.tensor([0, 1], device=dev))
    step = GraphedStep(body, key=lambda: model.P, device=dev)
    t0 = None
    for i in range(steps + warm):
        if i == warm:
            torch.cuda.synchronize(); t0 = time.perf_counter()
        if densify_at is not None and i == warm + densify_at:
            stats = model.densify_and_prune(2e-4, 0.005, 1.0, None)      # P changes: the next step() re-captures
        step()
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    RZ.set_sync_mode(True); RZ._pending.clear()
    return {"backend": "ours_full", "steps_per_s": round(steps / dt, 2), "frames_per_s": round(M * steps / dt, 2),
            "ms_per_step": round(dt / steps * 1e3, 3), "loss": float(loss_out), "graph_captures": step.captures, "densify": stats,
            "note": "flat-buffer Adam + densification statistics inside the captured step" + ("; wall time includes one densify_and_prune + re-capture" if densify_at is not None else "")}


def run(backend, surfels, res, frames, steps, bones, warm=5, seed=0):
    if backend == "ours_graph":
        return run_graph(surfels, res, frames, steps, bones, warm, seed)
    if backend == "ours_full":
        return run_full(surfels, res, frames, steps, bones, warm, seed)
    if backend == "ours_full_densify":
        r = run_full(surfels, res, frames, steps, bones, warm, seed, densify_at=steps // 2)
        r["backend"] = "ours_full_densify"
        return r
    dev = torch.device("cuda:0")
    M = 2
    cloud = SurfelCloud(object_scene(surfels, seed=seed, center=(0.0, 0.0, 0.0)), dev)
    seq = Sequence(bones, frames, 0.35, dev, seed)
    tan = 0.5
    fov = 2 * math.atan(tan)
    cam1 = make_camera(res, res, fov, fov, device=dev)                      # Stage 3's identity KCamera
    eye = torch.eye(4, device=dev)[None].expand(M, -1, -1).contiguous()
    pm = torch.from_numpy(projection_matrix(tan, tan)).to(dev)[None].expand(M, -1, -1).contiguous()
    bc = BatchCameras(res, res, fov, fov, eye, pm, torch.zeros((M, 3), device=dev))
    bg = torch.zeros(3, device=dev)
    pipe = PipelineParams()
    targets = torch.rand((frames, 3, res, res), generator=torch.Generator().manual_seed(1)).to(dev)
    params = cloud.flat_params() + list(seq.parameters())
    opt = torch.optim.Adam(params, lr=1e-5, fused=True)
    if backend == "reference":
        from oracle import ref_ext
        ref_ext.load()
        RN.GaussianRasterizer = ref_ext.RefGaussianRasterizer
    else:
        RN.GaussianRasterizer = RZ.GaussianRasterizer
        RZ.set_sync_mode(False)
    ev = lambda: torch.cuda.Event(enable_timing=True)  # noqa: E731
    warp_ms = 0.0
    t0 = None
    for step in range(steps + warm):
        if step == warm:
            torch.cuda.synchronize(); t0 = time.perf_counter(); warp_ms = 0.0
        fr = torch.tensor([(2 * step) % frames, (2 * step + 1) % frames], device=dev)
        opt.zero_grad(set_to_none=False)
        rest, art, lg, f2c = seq.tables(fr)
        e0, e1 = ev(), ev()
        e0.record()
        if backend == "ours_fused":
            xc, rc, ent = bob_warp(cloud.get_xyz, cloud._rotation, rest, art, lg, f2c)
        else:
            xc, rc = torch_warp(cloud.get_xyz, cloud._rotation, rest, art, lg, f2c)
        e1.record()
        # the rasterizer sees detached copies, so that the warp's backward can be timed on its own (one pass through each)
        xw, rw = xc, rc
        xc, rc = xw.detach().requires_grad_(True), rw.detach().requires_grad_(True)
        if backend == "reference":
            loss = 0.0
            for m in range(M):
                out = render(cam1, WarpedView(cloud, xc[m], rc[m]), pipe, bg)
                loss = loss + (out["render"] - targets[fr[m]]).abs().mean() \
                    + 0.05 * (1.0 - (out["rend_normal"] * out["surf_normal"]).sum(0)).mean() + 0.01 * out["rend_dist"].mean()
        else:
            loss = render_loss_batch(bc, cloud, pipe, bg, targets[fr], w_rgb=1.0, lambda_normal=0.05, lambda_dist=0.01, means3D=xc,
                                     rotations=torch.nn.functional.normalize(rc, dim=-1))["loss"]
        loss.backward()
        e2, e3 = ev(), ev()
        e2.record()
        torch.autograd.backward([xw, rw], [xc.grad, rc.grad])
        e3.record()
        opt.step()
        if backend != "reference":
            RZ.check_overflow()
        else:
            torch.cuda.synchronize()
        warp_ms += e0.elapsed_time(e1) + e2.elapsed_time(e3)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    RZ.set_sync_mode(True)
    return {"backend": backend, "steps_per_s": round(steps / dt, 2), "frames_per_s": round(M * steps / dt, 2),
            "ms_per_step": round(dt / steps * 1e3, 3), "warp_ms_per_step": round(warp_ms / steps, 3),
            "warp_share": round(warp_ms / steps / (dt / steps * 1e3), 3), "loss": float(loss)}


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--surfels", type=int, default=300_000)
    ap.add_argument("--res", type=int, default=256)
    ap.add_argument("--frames", type=int, default=32)
    ap.add_argument("--steps", type=int, default=60)
    ap.add_argument("--bones", type=int, default=25)
    ap.add_argument("--backends", default="ours_full,ours_graph,ours_fused,ours,reference")
    a = ap.parse_args()
    out = {"config": f"C3: {a.surfels} surfels, {a.frames}-frame sequence, {a.res}x{a.res}, M=2 frames/step, B={a.bones} bones, 1 GPU", "results": []}
    for b in a.backends.split(","):
        r = run(b, a.surfels, a.res, a.frames, a.steps, a.bones)
        out["results"].append(r)
        print(json.dumps(r), flush=True)
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    json.dump(out, open(os.path.join(ROOT, "gpurun_out", "stage3_c3.json"), "w"), indent=1)
