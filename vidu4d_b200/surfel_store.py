"""Flat-buffer surfel model: parameters, gradients and Adam moments of all surfel parameter groups in ONE fp32 buffer
each, with a single-kernel Adam step and a single-kernel densify / prune (SURVEY.md section 8(f) row N4).

Mirrors the slice of the reference the Stage-3 loop uses (same names and argument meaning):
    gs/scene/gaussian_model.py:98-118      get_xyz / get_scaling / get_rotation / get_opacity / get_features
    gs/scene/gaussian_model.py:291-356     _prune_optimizer / prune_points / cat_tensors_to_optimizer / densification_postfix
    gs/scene/gaussian_model.py:376-446     densify_and_split / densify_and_clone / densify_and_prune
    gs/scene/gaussian_model.py:450-452     add_densification_stats
    lab4d/engine/trainer.py:243-253        the gs_optimizer: torch.optim.Adam, one param group per tensor, eps = 1e-15
    lab4d/engine/trainer.py:550-568        max_radii2D bookkeeping + when densify_and_prune is called
The layout is the one the gradient all-reduce uses (distributed.FlatGrads): groups back to back, each (P, k) row-major.
"""
from __future__ import annotations

import ctypes as C
import math

import torch

from . import _capi

GROUPS = (("xyz", 3), ("f_dc", 3), ("f_rest", 45), ("opacity", 1), ("scaling", 2), ("rotation", 4))
# the optional seventh group: Stage 3's per-surfel registration feature (lab4d/engine/trainer.py:250, lr feature_lr)
REGIST_FEAT = ("regist_feat", 16)
_ATTR = {"xyz": "_xyz", "f_dc": "_features_dc", "f_rest": "_features_rest", "opacity": "_opacity", "scaling": "_scaling",
         "rotation": "_rotation", "regist_feat": "_regist_feat"}


def build_rotation(r):
    """gs/utils/general_utils.py build_rotation: (N,4) (w,x,y,z) -> (N,3,3), normalising first."""
    q = r / r.norm(dim=1, keepdim=True)
    w, x, y, z = q.unbind(1)
    R = torch.stack((1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y),
                     2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x),
                     2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)), 1)
    return R.view(-1, 3, 3)


class FlatSurfelModel(torch.nn.Module):
    """Surfel parameters as views of one flat buffer.  Duck-types what render() / render_loss_batch() read from `pc`.

    regist_feat (P,16), optional: the registration feature the reference optimises with the surfels
    (gs/scene/gaussian_model.py:324-325,358-378,405-406,427-428), as a seventh group after the other six (whose layout
    is then unchanged) -- `_regist_feat`, lr key "regist_feat" (default 0.0025, config.py feature_lr).  Densification
    carries it along: clones and split children copy their parent's row, pruned surfels drop theirs."""

    def __init__(self, xyz, features_dc, features_rest, opacity, scaling, rotation, sh_degree=3, percent_dense=0.01,
                 lrs=None, betas=(0.9, 0.999), eps=1e-15, regist_feat=None):
        super().__init__()
        dev = xyz.device
        self.max_sh_degree = 3
        self.active_sh_degree = sh_degree
        self.percent_dense = percent_dense
        self.betas, self.eps, self.step_count = betas, eps, 0
        # trainer.py:243-251 defaults (config.py: position_lr_init 1.6e-4 ... ); callers pass their own
        self.lrs = dict(lrs or {"xyz": 1.6e-4, "f_dc": 2.5e-3, "f_rest": 2.5e-3 / 20.0, "opacity": 5e-2, "scaling": 5e-3, "rotation": 1e-3})
        self.groups = GROUPS if regist_feat is None else GROUPS + (REGIST_FEAT,)
        if regist_feat is not None:
            self.lrs.setdefault("regist_feat", 2.5e-3)
        tensors = [xyz, features_dc.reshape(len(xyz), -1), features_rest.reshape(len(xyz), -1), opacity, scaling, rotation]
        self._install(tensors + ([] if regist_feat is None else [regist_feat]), dev)
        self.exp_avg = torch.zeros_like(self.flat)
        self.exp_avg_sq = torch.zeros_like(self.flat)
        self._reset_stats()

    # ---- layout -------------------------------------------------------------------------------------------------
    def _offsets(self, P):
        off, o = [], 0
        for _, k in self.groups:
            off.append(o); o += P * k
        return off, o

    def _install(self, tensors, dev):
        P = int(tensors[0].shape[0])
        off, total = self._offsets(P)
        if P % 4 != 0:
            # rotations / SH rows are read with 128-bit loads: every group must start 16-byte aligned
            pass
        self.P = P
        self.flat = torch.empty((total,), dtype=torch.float32, device=dev)
        for (name, k), o, t in zip(self.groups, off, tensors):
            self.flat[o:o + P * k].view(P, k).copy_(t.reshape(P, k))
        self._bind()

    def _bind(self):
        """(Re)create the nn.Parameter views and the flat gradient buffer after the flat buffer changed."""
        P = self.P
        off, total = self._offsets(P)
        self.grad_flat = torch.zeros((total,), dtype=torch.float32, device=self.flat.device)
        shapes = {"xyz": (P, 3), "f_dc": (P, 1, 3), "f_rest": (P, 15, 3), "opacity": (P, 1), "scaling": (P, 2), "rotation": (P, 4),
                  "regist_feat": (P, 16)}
        for (name, k), o in zip(self.groups, off):
            p = torch.nn.Parameter(self.flat[o:o + P * k].view(shapes[name]))
            p.grad = self.grad_flat[o:o + P * k].view(shapes[name])
            setattr(self, _ATTR[name], p)

    def _reset_stats(self):
        dev = self.flat.device
        self.xyz_gradient_accum = torch.zeros((self.P, 1), device=dev)
        self.denom = torch.zeros((self.P, 1), device=dev)
        self.max_radii2D = torch.zeros((self.P,), device=dev)

    # ---- what render() reads (gaussian_model.py:98-118) -------------------------------------------------------------
    get_xyz = property(lambda s: s._xyz)
    get_scaling = property(lambda s: torch.exp(s._scaling))
    get_rotation = property(lambda s: torch.nn.functional.normalize(s._rotation))
    get_opacity = property(lambda s: torch.sigmoid(s._opacity))
    get_features = property(lambda s: torch.cat((s._features_dc, s._features_rest), dim=1))

    def flat_params(self):
        return [getattr(self, _ATTR[name]) for name, _ in self.groups]

    def zero_grad_flat(self):
        self.grad_flat.zero_()

    # ---- one-kernel Adam (trainer.py:253 + 585-586) ---------------------------------------------------------------
    def adam_step(self, grad_scale: float = 1.0):
        lib = _capi.load()
        off, total = self._offsets(self.P)
        begin = (C.c_int64 * (len(self.groups) + 1))(*off, total)
        lr = (C.c_float * len(self.groups))(*[self.lrs[n] for n, _ in self.groups])
        self.step_count += 1
        with torch.cuda.device(self.flat.device):
            rc = lib.sr_adam_flat(len(self.groups), begin, lr, self.betas[0], self.betas[1], self.eps, self.step_count, float(grad_scale),
                                  self.flat.data_ptr(), self.grad_flat.data_ptr(), self.exp_avg.data_ptr(), self.exp_avg_sq.data_ptr(),
                                  torch.cuda.current_stream(self.flat.device).cuda_stream)
        _capi.check(rc, "sr_adam_flat")

    # ---- densification statistics (gaussian_model.py:450-452, trainer.py:553-560) ----------------------------------
    @torch.no_grad()
    def add_densification_stats(self, viewspace_grad, update_filter, radii=None):
        """Same values as the reference's boolean-mask updates, written with masks and in-place ops: fixed shapes and
        stable addresses, so the call can sit inside a captured CUDA graph (a boolean index would need a host sync)."""
        f = update_filter.unsqueeze(-1).to(torch.float32)
        self.xyz_gradient_accum.add_(torch.norm(viewspace_grad, dim=-1, keepdim=True) * f)
        self.denom.add_(f)
        if radii is not None:
            self.max_radii2D.copy_(torch.where(update_filter, torch.max(self.max_radii2D, radii.float()), self.max_radii2D))

    # ---- densify / prune in one gather (gaussian_model.py:376-446) ------------------------------------------------
    @torch.no_grad()
    def _compact(self, src, kind, child_slot=None, child_xyz=None, child_scaling=None):
        """New model = rows `src` of the old one.  kind 0: survivor (Adam state kept), 1: clone, 2: split child."""
        lib = _capi.load()
        dev = self.flat.device
        P_new = int(src.numel())
        old_off, _ = self._offsets(self.P)
        new_off, new_total = self._offsets(P_new)
        p_new = torch.empty((new_total,), dtype=torch.float32, device=dev)
        m_new, v_new = torch.empty_like(p_new), torch.empty_like(p_new)
        n = len(self.groups)
        width = (C.c_int32 * n)(*[k for _, k in self.groups])
        ob, nb = (C.c_int64 * n)(*old_off), (C.c_int64 * n)(*new_off)
        src = src.to(torch.int32).contiguous(); kind = kind.to(torch.uint8).contiguous()
        ptr = lambda t: None if t is None else t.contiguous().data_ptr()  # noqa: E731
        if child_slot is not None:
            child_slot = child_slot.to(torch.int32).contiguous(); child_xyz = child_xyz.float().contiguous(); child_scaling = child_scaling.float().contiguous()
        with torch.cuda.device(dev):
            rc = lib.sr_surfel_compact(n, width, ob, nb, 0, 4, P_new, src.data_ptr(), kind.data_ptr(), ptr(child_slot), ptr(child_xyz),
                                       ptr(child_scaling), self.flat.data_ptr(), self.exp_avg.data_ptr(), self.exp_avg_sq.data_ptr(),
                                       p_new.data_ptr(), m_new.data_ptr(), v_new.data_ptr(), torch.cuda.current_stream(dev).cuda_stream)
        _capi.check(rc, "sr_surfel_compact")
        self.flat, self.exp_avg, self.exp_avg_sq, self.P = p_new, m_new, v_new, P_new
        self._bind()

    @torch.no_grad()
    def prune_points(self, mask):
        keep = torch.nonzero(~mask, as_tuple=False).squeeze(1)
        stats = (self.xyz_gradient_accum[keep], self.denom[keep], self.max_radii2D[keep])
        self._compact(keep, torch.zeros_like(keep, dtype=torch.uint8))
        self.xyz_gradient_accum, self.denom, self.max_radii2D = stats

    @torch.no_grad()
    def remove_radius_outliers(self, nb_points: int = 20, radius: float = 0.004) -> int:
        """lab4d/engine/trainer.py:573-588 (Open3D's remove_radius_outlier, then prune_points) on the device: prunes every
        surfel with at most nb_points surfels, itself included, strictly closer than `radius` (knn.radius_outlier_mask).
        Returns the number pruned.  When none is, the buffers are left as they are (same addresses for a captured step)."""
        from .knn import radius_outlier_mask
        mask = radius_outlier_mask(self._xyz, nb_points, radius)
        n = int(mask.sum())
        if n:
            self.prune_points(mask)
        return n

    @torch.no_grad()
    def densify_and_prune(self, max_grad, min_opacity, extent, max_screen_size, generator=None):
        """gaussian_model.py:431-446 in ONE pass over the buffers.  The reference builds the result in four steps (clone ->
        cat; split -> cat, prune the split parents; prune by opacity / size), re-creating every parameter and both Adam
        moments each time; the final set and its order are a pure function of the masks, so it is assembled here as one
        source-index list:  [survivors that are not split] + [clones] + [split children], then filtered by the prune mask."""
        dev = self.flat.device
        P = self.P
        grads = self.xyz_gradient_accum / self.denom
        grads[grads.isnan()] = 0.0
        gn = torch.norm(grads, dim=-1)
        big = torch.max(self.get_scaling, dim=1).values > self.percent_dense * extent
        clone = (gn >= max_grad) & ~big
        # densify_and_split sees the post-clone set with zero-padded gradients: clones are never split
        split = (grads.squeeze(-1) >= max_grad) & big
        N = 2
        idx = torch.arange(P, device=dev)
        ci, si = idx[clone], idx[split]
        stds = torch.cat([self.get_scaling[si].repeat(N, 1), torch.zeros((N * si.numel(), 1), device=dev)], dim=-1)
        samples = torch.normal(mean=torch.zeros_like(stds), std=stds, generator=generator)
        rots = build_rotation(self._rotation[si]).repeat(N, 1, 1)
        child_xyz = torch.bmm(rots, samples.unsqueeze(-1)).squeeze(-1) + self._xyz[si].repeat(N, 1)
        child_scaling = torch.log(self.get_scaling[si].repeat(N, 1) / (0.8 * N))
        survivors = idx[~split]
        src = torch.cat([survivors, ci, si.repeat(N)])
        kind = torch.cat([torch.zeros_like(survivors), torch.ones_like(ci), torch.full((N * si.numel(),), 2, device=dev)]).to(torch.uint8)
        child_slot = torch.cat([torch.zeros(survivors.numel() + ci.numel(), dtype=torch.int64, device=dev), torch.arange(N * si.numel(), device=dev)])
        # prune on the assembled set (statistics were reset by densification_postfix: max_radii2D = 0 there)
        opac = torch.sigmoid(self._opacity[src, 0])
        prune = opac < min_opacity
        if max_screen_size:
            scal = torch.where((kind == 2)[:, None], child_scaling[child_slot.clamp(max=max(child_scaling.shape[0] - 1, 0))] if child_scaling.numel() else self._scaling[src],
                               self._scaling[src])
            prune = prune | (torch.exp(scal).max(dim=1).values > 0.1 * extent)
        keep = ~prune
        self._compact(src[keep], kind[keep], child_slot[keep], child_xyz, child_scaling)
        self._reset_stats()
        return {"cloned": int(clone.sum()), "split": int(split.sum()), "pruned": int(prune.sum()), "P": self.P}

    @torch.no_grad()
    def reset_opacity(self):
        """gaussian_model.py reset_opacity: opacity <- min(opacity, 0.01), Adam state of the group cleared."""
        off, _ = self._offsets(self.P)
        o = off[3]
        new = torch.log(torch.clamp(torch.sigmoid(self._opacity), max=0.01) / (1 - torch.clamp(torch.sigmoid(self._opacity), max=0.01)))
        self._opacity.data.copy_(new)
        self.exp_avg[o:o + self.P].zero_(); self.exp_avg_sq[o:o + self.P].zero_()
