"""Flat-buffer surfel model: parameters, gradients and Adam moments of all surfel parameter groups in ONE fp32 buffer
each, with a single-kernel Adam step and a single-kernel densify / prune (SURVEY.md section 8(f) row N4).

Mirrors the slice of the reference the Stage-3 loop uses (same names and argument meaning):
    gs/scene/gaussian_model.py:98-118      get_xyz / get_scaling / get_rotation / get_opacity / get_features
    gs/scene/gaussian_model.py:291-356     _prune_optimizer / prune_points / cat_tensors_to_optimizer / densification_postfix
    gs/scene/gaussian_model.py:376-446     densify_and_split / densify_and_clone / densify_and_prune
    gs/scene/gaussian_model.py:450-452     add_densification_stats
    lab4d/engine/trainer.py:243-253        the gs_optimizer: torch.optim.Adam, one param group per tensor, eps = 1e-15
    lab4d/engine/trainer.py:550-568        max_radii2D bookkeeping + when densify_and_prune is called
    lab4d/engine/trainer.py:386-396        load_checkpoint: fresh nn.Parameters assigned to the groups, then load_state_dict
    gs/scene/gaussian_model.py:189-268     save_ply / load_ply (vidu4d_b200/ply.py)
The layout is the one the gradient all-reduce uses (allreduce_grads_): groups back to back, each (P, k) row-major.
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
_GROUP_OF = {a: n for n, a in _ATTR.items()}
# each group's parameter shape after its row count (the reference's shapes)
_TAIL = {"xyz": (3,), "f_dc": (1, 3), "f_rest": (15, 3), "opacity": (1,), "scaling": (2,), "rotation": (4,), "regist_feat": (16,)}
# state_dict keys of the store-only state, next to the reference's parameter keys (DESIGN.md section 3.7)
_ALL_GROUPS = tuple(n for n, _ in GROUPS + (REGIST_FEAT,))
STORE_KEYS = ("store_groups", "store_exp_avg", "store_exp_avg_sq", "store_device_step", "store_lr", "store_step_count",
              "store_active_sh_degree", "store_densify_stats", "store_max_radii2D", "store_betas", "store_eps",
              "store_percent_dense")


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
        self._foreign = set()                 # groups assigned a tensor of another surfel count, not yet re-homed
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
        tensors = [xyz, features_dc.reshape(len(xyz), 3), features_rest.reshape(len(xyz), 45), opacity, scaling, rotation]
        self._install(tensors + ([] if regist_feat is None else [regist_feat]), dev)
        self.exp_avg = torch.zeros_like(self.flat)
        self.exp_avg_sq = torch.zeros_like(self.flat)
        # step()'s state, on the device at fixed addresses so that a captured step reads the current values on every
        # replay: the step count (shared by the groups, kept across densification and reset_opacity as the reference
        # keeps each group's `step`), the per-group rates, and the coefficient clip_grad_norm_ leaves for step()
        self.device_step = torch.zeros((), dtype=torch.int64, device=dev)
        self.device_lr = torch.tensor([self.lrs[n] for n, _ in self.groups], dtype=torch.float32, device=dev)
        self.clip_coef = torch.ones((), dtype=torch.float32, device=dev)
        self._clip_pending = False
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

    def _bind(self, names=None):
        """(Re)create the nn.Parameter views and the flat gradient buffer after the flat buffer changed.  With `names`,
        only those groups' views, over the current flat buffer and gradient buffer (same P: addresses kept)."""
        P = self.P
        off, total = self._offsets(P)
        if names is None:
            self.grad_flat = torch.zeros((total,), dtype=torch.float32, device=self.flat.device)
        for (name, k), o in zip(self.groups, off):
            if names is None or name in names:
                p = torch.nn.Parameter(self.flat[o:o + P * k].view((P,) + _TAIL[name]))
                p.grad = self.grad_flat[o:o + P * k].view((P,) + _TAIL[name])
                self._parameters[_ATTR[name]] = p
        self._foreign.clear()
        self._clip_pending = False            # a clip coefficient belongs to the gradients it was computed from

    def _reset_stats(self):
        dev = self.flat.device
        # xyz_gradient_accum and denom are the two rows of one buffer, so that one SUM all-reduce covers both
        self.densify_stats = torch.zeros((2, self.P), device=dev)
        self.max_radii2D = torch.zeros((self.P,), device=dev)

    # (P,1) views of densify_stats' rows; assigning one copies into the row (`accum += x` stays in place)
    def _stats_row(i):
        def get(self):
            return self.densify_stats[i].unsqueeze(-1)

        def set_(self, value):
            self.densify_stats[i].copy_(value.reshape(self.P))
        return property(get, set_)
    xyz_gradient_accum = _stats_row(0)
    denom = _stats_row(1)
    del _stats_row

    # ---- what render() reads (gaussian_model.py:98-118) -------------------------------------------------------------
    get_xyz = property(lambda s: s._live("render")._xyz)
    get_scaling = property(lambda s: torch.exp(s._live("render")._scaling))
    get_rotation = property(lambda s: torch.nn.functional.normalize(s._live("render")._rotation))
    get_opacity = property(lambda s: torch.sigmoid(s._live("render")._opacity))
    get_features = property(lambda s: torch.cat((s._live("render")._features_dc, s._features_rest), dim=1))

    def flat_params(self):
        self._live("flat_params")
        return [getattr(self, _ATTR[name]) for name, _ in self.groups]

    def zero_grad_flat(self):
        self.grad_flat.zero_()
        self._clip_pending = False

    # ---- group assignment: the reference's load_checkpoint (trainer.py:386-396) ---------------------------------------
    def __setattr__(self, name, value):
        group = _GROUP_OF.get(name)
        if group is None or "flat" not in self.__dict__:
            return super().__setattr__(name, value)
        if group not in [n for n, _ in self.groups]:
            raise AttributeError(f"this store has no {group} group: {name} would be a parameter outside the flat buffer, "
                                 f"never stepped; build the store with {group}=")
        self._assign(group, value)

    @torch.no_grad()
    def _assign(self, group, value):
        """`store._xyz = nn.Parameter(t)` (any group): the tensor's values are re-homed into the flat buffer instead of
        replacing the view, so that the store keeps rendering, differentiating and stepping one set of surfels.

        Same surfel count: copied into the group's rows in place (every address kept, Adam state kept, as an in-place
        `param.data.copy_` keeps it).  Another count: the tensor is held as it is until every group has been assigned
        one of that count -- the reference assigns them one at a time -- and the store is then rebuilt at the new count
        with zero moments and statistics (rows of another count have no Adam state to keep; load_state_dict restores
        it).  Until then every use of the store raises."""
        if not isinstance(value, torch.Tensor):
            raise TypeError(f"{_ATTR[group]} must be a tensor, got {type(value).__name__}")
        tail = _TAIL[group]
        if tuple(value.shape[1:]) != tail:
            raise ValueError(f"{_ATTR[group]} must be (P,{','.join(map(str, tail))}), got {tuple(value.shape)}")
        self._parameters[_ATTR[group]] = value if isinstance(value, torch.nn.Parameter) else torch.nn.Parameter(value.detach())
        self._foreign.add(group)
        rows = self._rows()
        if len(set(rows.values())) != 1:
            return
        P = next(iter(rows.values()))
        src = {n: self._parameters[_ATTR[n]].detach() for n in self._foreign}
        if P == self.P:
            for n, t in src.items():
                self._group_view(n).copy_(t)
            self._bind(list(src))
            return
        dev = self.flat.device
        self.P = P
        self.flat = torch.cat([src[n].reshape(-1).to(dev, torch.float32) for n, _ in self.groups])
        self.exp_avg = torch.zeros_like(self.flat)
        self.exp_avg_sq = torch.zeros_like(self.flat)
        self._bind()
        self._reset_stats()

    def _rows(self):
        return {n: (int(self._parameters[_ATTR[n]].shape[0]) if n in self._foreign else self.P) for n, _ in self.groups}

    def _group_view(self, name):
        off, _ = self._offsets(self.P)
        i = [n for n, _ in self.groups].index(name)
        k = self.groups[i][1]
        return self.flat[off[i]:off[i] + self.P * k].view((self.P,) + _TAIL[name])

    def _live(self, what):
        """self, once every group is a view of the flat buffer; raises while assigned groups disagree on P."""
        if self._foreign:
            rows = ", ".join(f"{_ATTR[n]}: {r}" for n, r in self._rows().items())
            raise RuntimeError(f"FlatSurfelModel.{what}: the surfel groups disagree on the surfel count ({rows}); assign "
                               f"every group a tensor of the same count, or load_state_dict, before using the store")
        return self

    # ---- one-kernel Adam (trainer.py:253 + 585-586) ---------------------------------------------------------------
    def adam_step(self, grad_scale: float = 1.0):
        self._live("adam_step")
        off, total = self._offsets(self.P)
        begin = (C.c_int64 * (len(self.groups) + 1))(*off, total)
        lr = (C.c_float * len(self.groups))(*[self.lrs[n] for n, _ in self.groups])
        self.step_count += 1
        _capi.call("sr_adam_flat", self.flat.device, len(self.groups), begin, lr, self.betas[0], self.betas[1], self.eps,
                   self.step_count, float(grad_scale), self.flat, self.grad_flat, self.exp_avg, self.exp_avg_sq)

    # ---- clip + Adam with the per-step state on the device (trainer.py:547, 589-591) -----------------------------------
    def _begin(self):
        off, total = self._offsets(self.P)
        return (C.c_int64 * (len(self.groups) + 1))(*off, total)

    def set_lr(self, name: str, value: float):
        """Set group `name`'s learning rate for step() (written in place: a captured step picks it up) and adam_step()."""
        i = [n for n, _ in self.groups].index(name)
        self.lrs[name] = float(value)
        self.device_lr[i].fill_(float(value))

    @torch.no_grad()
    def clip_grad_norm_(self, max_norm: float, extra_params=(), grad_scale: float = 1.0):
        """torch.nn.utils.clip_grad_norm_(self.flat_params() + extra_params, max_norm) (trainer.py:547, check_grad) for a
        step whose surfel gradients are grad_flat * grad_scale.  The extras' gradients (None ones skipped) are scaled
        here, with torch._foreach_mul_; the surfel gradients are scaled inside the next step(), which must get the same
        grad_scale.  Returns the total norm as a device tensor, without a host synchronisation."""
        self._live("clip_grad_norm_")
        dev = self.flat.device
        grads = [p.grad for p in extra_params if p.grad is not None]
        _capi.check_tensors([(f"extra_params[{i}].grad", g) for i, g in enumerate(grads)], "the surfel buffer", self.flat)
        norms = torch.stack(torch._foreach_norm(grads)) if grads else None
        n = len(self.groups)
        scratch = torch.empty((int(_capi.load().sr_grad_norm_scratch_bytes(n)),), dtype=torch.uint8, device=dev)
        total = torch.empty((), dtype=torch.float32, device=dev)
        _capi.call("sr_grad_norm_flat", dev, n, self._begin(), self.grad_flat, float(grad_scale), norms, len(grads),
                   float(max_norm), total, self.clip_coef, None, scratch, scratch.numel())
        if grads:
            torch._foreach_mul_(grads, self.clip_coef)
        self._clip_pending = True
        return total

    @torch.no_grad()
    def step(self, grad_scale: float = 1.0):
        """One Adam step (the gs_optimizer.step() of trainer.py:589-591) with its step count and rates read from the
        device, and the surfel gradients multiplied by grad_scale, then by the coefficient of a clip_grad_norm_ made
        since the last zero_grad_flat() / step().  device_step advances by one, also with no surfels.  Capturable: each
        replay of a graph holding this call steps with the current count and rates.  step_count is adam_step()'s."""
        self._live("step")
        coef = self.clip_coef if self._clip_pending else None
        self._clip_pending = False
        _capi.call("sr_adam_flat_state", self.flat.device, len(self.groups), self._begin(), self.device_lr, self.betas[0],
                   self.betas[1], self.eps, self.device_step, float(grad_scale), coef, self.flat, self.grad_flat,
                   self.exp_avg, self.exp_avg_sq)

    # ---- densification statistics (gaussian_model.py:450-452, trainer.py:553-560) ----------------------------------
    @torch.no_grad()
    def add_densification_stats(self, viewspace_grad, update_filter, radii=None, grad_scale: float = 1.0):
        """Same values as the reference's boolean-mask updates, written with masks and in-place ops: fixed shapes and
        stable addresses, so the call can sit inside a captured CUDA graph (a boolean index would need a host sync).

        One frame: viewspace_grad (P,3), update_filter (P,) bool, radii (P,) or None -- torch ops.
        A batch of M frames: viewspace_grad (M,P,3) float32 (render_loss_batch's out["viewspace_points"].grad),
        update_filter (M,P) or None, radii (M,P) int32 -- one kernel (sr_densify_stats) that applies the frames in order,
        with the same bits as M one-frame calls.  A frame sees a surfel where radii > 0; update_filter, when given, must
        be that mask (render_loss_batch's visibility_filter is).
        The norm is taken of grad_scale * viewspace_grad: the per-frame gradient of a loss that sums its frames, scaled
        as the step scales the parameter gradients (1 / frames, over all ranks)."""
        self._live("add_densification_stats")
        if viewspace_grad.dim() == 3:
            self._add_densification_stats_batch(viewspace_grad, update_filter, radii, grad_scale)
            return
        if grad_scale != 1.0:
            viewspace_grad = viewspace_grad * grad_scale
        f = update_filter.unsqueeze(-1).to(torch.float32)
        self.xyz_gradient_accum.add_(torch.norm(viewspace_grad, dim=-1, keepdim=True) * f)
        self.denom.add_(f)
        if radii is not None:
            self.max_radii2D.copy_(torch.where(update_filter, torch.max(self.max_radii2D, radii.float()), self.max_radii2D))

    def _add_densification_stats_batch(self, viewspace_grad, update_filter, radii, grad_scale):
        M, P = int(viewspace_grad.shape[0]), self.P
        if tuple(viewspace_grad.shape) != (M, P, 3):
            raise RuntimeError(f"viewspace_grad must be (M,P,3) with P = {P}, got {tuple(viewspace_grad.shape)}")
        if radii is None or tuple(radii.shape) != (M, P):
            raise RuntimeError(f"the batched form needs radii (M,P) = ({M},{P}), got "
                               f"{None if radii is None else tuple(radii.shape)}")
        if update_filter is not None and tuple(update_filter.shape) != (M, P):
            raise RuntimeError(f"update_filter must be (M,P) = ({M},{P}) or None, got {tuple(update_filter.shape)}")
        if viewspace_grad.dtype != torch.float32:
            raise RuntimeError(f"viewspace_grad must be float32, got {viewspace_grad.dtype}")
        if radii.dtype != torch.int32:
            raise RuntimeError(f"radii must be int32, got {radii.dtype}")
        ref = self.densify_stats
        _capi.check_tensors([("viewspace_grad", viewspace_grad), ("radii", radii), ("the statistics", ref)],
                            "the surfel buffer", self.flat, floats=[])
        if not math.isfinite(grad_scale):
            raise RuntimeError(f"grad_scale must be finite, got {grad_scale}")
        _capi.call("sr_densify_stats", self.flat.device, M, P, viewspace_grad.contiguous(), radii.contiguous(),
                   float(grad_scale), ref[0], ref[1], self.max_radii2D)

    # ---- multi-GPU: every rank keeps the same surfels (DESIGN.md section 4) -----------------------------------------
    @staticmethod
    def _world(group):
        import torch.distributed as dist
        if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
            return None
        return dist

    @torch.no_grad()
    def sync_densification_stats(self, group=None):
        """Make every rank's statistics those of all the ranks' frames: SUM over densify_stats (accum and denom, one
        collective), MAX over max_radii2D.  Call it right before densify_and_prune.  No-op on one rank."""
        self._live("sync_densification_stats")
        dist = self._world(group)
        if dist is None:
            return
        dist.all_reduce(self.densify_stats, op=dist.ReduceOp.SUM, group=group)
        dist.all_reduce(self.max_radii2D, op=dist.ReduceOp.MAX, group=group)

    @torch.no_grad()
    def allreduce_grads_(self, average_over: int | None = None, group=None):
        """Sum grad_flat over the ranks (one collective), then multiply by 1 / average_over if given.  Reads the current
        buffer, so it stays right after densification re-binds the gradients.  Returns grad_flat."""
        self._live("allreduce_grads_")
        dist = self._world(group)
        if dist is not None:
            dist.all_reduce(self.grad_flat, op=dist.ReduceOp.SUM, group=group)
        if average_over:
            self.grad_flat.mul_(1.0 / float(average_over))
        return self.grad_flat

    def replica_state(self) -> dict:
        """What must be equal on every rank between steps, by name (distributed.check_replicas' argument).  The
        statistics are each rank's own until sync_densification_stats."""
        self._live("replica_state")
        return {"P": self.P, "flat": self.flat, "exp_avg": self.exp_avg, "exp_avg_sq": self.exp_avg_sq,
                "device_step": self.device_step, "densify_stats": self.densify_stats, "max_radii2D": self.max_radii2D}

    # ---- densify / prune in one gather (gaussian_model.py:376-446) ------------------------------------------------
    @torch.no_grad()
    def _compact(self, src, kind, child_slot=None, child_xyz=None, child_scaling=None):
        """New model = rows `src` of the old one.  kind 0: survivor (Adam state kept), 1: clone, 2: split child."""
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
        if child_slot is not None:
            child_slot = child_slot.to(torch.int32).contiguous(); child_xyz = child_xyz.float().contiguous(); child_scaling = child_scaling.float().contiguous()
        _capi.call("sr_surfel_compact", dev, n, width, ob, nb, 0, 4, P_new, src, kind, child_slot, child_xyz, child_scaling, self.flat,
                   self.exp_avg, self.exp_avg_sq, p_new, m_new, v_new)
        self.flat, self.exp_avg, self.exp_avg_sq, self.P = p_new, m_new, v_new, P_new
        self._bind()

    @torch.no_grad()
    def prune_points(self, mask):
        self._live("prune_points")
        keep = torch.nonzero(~mask, as_tuple=False).squeeze(1)
        stats = (self.densify_stats[:, keep], self.max_radii2D[keep])
        self._compact(keep, torch.zeros_like(keep, dtype=torch.uint8))
        self.densify_stats, self.max_radii2D = stats

    @torch.no_grad()
    def remove_radius_outliers(self, nb_points: int = 20, radius: float = 0.004) -> int:
        """lab4d/engine/trainer.py:573-588 (Open3D's remove_radius_outlier, then prune_points) on the device: prunes every
        surfel with at most nb_points surfels, itself included, strictly closer than `radius` (knn.radius_outlier_mask).
        Returns the number pruned.  When none is, the buffers are left as they are (same addresses for a captured step)."""
        from .knn import radius_outlier_mask
        self._live("remove_radius_outliers")
        mask = radius_outlier_mask(self._xyz, nb_points, radius)
        n = int(mask.sum())
        if n:
            self.prune_points(mask)
        return n

    @torch.no_grad()
    def prune_by_contribution(self, contrib, min_weight: float = 0.0, min_pixels: int = 1,
                              max_background_fraction=None) -> int:
        """Prune every surfel whose summed blending weight over the rendered frames is below min_weight, or that
        contributed to fewer than min_pixels (frame, pixel) pairs: with the defaults, every surfel no frame blends (each
        view sees it behind opaque ones, or culls it).  With max_background_fraction f, also every surfel whose share of
        weight on the frames' background pixels (contrib.background_fraction, gathered by render_frames(...,
        masks=)) is above f: a clump that floats off the object, which every view blends over background.  The default
        None leaves the decision to the first two tests.  contrib: a renderer.SurfelContributions of this store's P surfels,
        filled by render_frames(contributions=) -- on several ranks, after distributed.allreduce_contributions, so that
        every rank prunes the same surfels.  Goes through prune_points: the Adam moments, statistics and regist_feat
        follow.  Returns the number pruned.  When none is, the buffers are left as they are (same addresses)."""
        self._live("prune_by_contribution")
        if contrib.P != self.P:
            raise RuntimeError(f"contributions are for {contrib.P} surfels, the store has {self.P}")
        mask = contrib.prune_mask(min_weight, min_pixels, max_background_fraction).to(self.flat.device)
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
        self._live("densify_and_prune")
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
        self._live("reset_opacity")
        off, _ = self._offsets(self.P)
        o = off[3]
        new = torch.log(torch.clamp(torch.sigmoid(self._opacity), max=0.01) / (1 - torch.clamp(torch.sigmoid(self._opacity), max=0.01)))
        self._opacity.data.copy_(new)
        self.exp_avg[o:o + self.P].zero_(); self.exp_avg_sq[o:o + self.P].zero_()

    # ---- checkpoints: the reference's parameter keys + the store-only state (DESIGN.md section 3.7) -----------------------
    def _save_to_state_dict(self, destination, prefix, keep_vars):
        """The reference's keys and shapes (_xyz (P,3), _features_dc (P,1,3), ..., _regist_feat (P,16)), which load into
        its GaussianModel / DeformableGaussian with strict=False, plus the store-only state under STORE_KEYS: both Adam
        moments as flat buffers in the group layout, the step counts, the rates (float64: device_lr is their float32
        rounding), SH degree, densification statistics, Adam's
        constants, percent_dense and the group list."""
        self._live("state_dict")
        super()._save_to_state_dict(destination, prefix, keep_vars)
        f64 = lambda v: torch.tensor(v, dtype=torch.float64)  # noqa: E731
        i64 = lambda v: torch.tensor(v, dtype=torch.int64)  # noqa: E731
        state = {"store_groups": i64([_ALL_GROUPS.index(n) for n, _ in self.groups]),
                 "store_exp_avg": self.exp_avg, "store_exp_avg_sq": self.exp_avg_sq, "store_device_step": self.device_step,
                 "store_lr": f64([self.lrs[n] for n, _ in self.groups]), "store_step_count": i64(self.step_count),
                 "store_active_sh_degree": i64(self.active_sh_degree), "store_densify_stats": self.densify_stats,
                 "store_max_radii2D": self.max_radii2D, "store_betas": f64(list(self.betas)), "store_eps": f64(self.eps),
                 "store_percent_dense": f64(self.percent_dense)}
        for k in STORE_KEYS:
            destination[prefix + k] = state[k] if keep_vars else state[k].detach()

    @torch.no_grad()
    def _load_from_state_dict(self, state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys, error_msgs):
        """Loads a checkpoint of any surfel count, this store's or the reference's.

        Same P: every tensor is copied into the existing buffers in place, so a GraphedStep captured on this store
        (keyed on P) keeps replaying on the right addresses.  Another P: fresh buffers, and the parameter views and
        grad_flat re-bound, as densification does.  A reference checkpoint (the parameter keys only) gives zero moments,
        step 0 and zero statistics, which is what the reference's own resume amounts to: its save_checkpoint keeps no
        gs_optimizer state; the rates, Adam's constants and active_sh_degree are then left as they are.

        Every other key -- a parameter or buffer the module has beside the surfel groups, such as the reference's
        `logscale` (trainer.py:387-388) -- goes through nn.Module's own loading, which also reports unknown keys."""
        names = [n for n, _ in self.groups]
        ours = {prefix + _ATTR[n] for n in names} | {prefix + k for k in STORE_KEYS}
        n_missing = len(missing_keys)
        super()._load_from_state_dict({k: v for k, v in state_dict.items() if k not in ours}, prefix, local_metadata,
                                      strict, missing_keys, unexpected_keys, error_msgs)
        missing_keys[n_missing:] = [k for k in missing_keys[n_missing:] if k not in ours]   # the groups are handled below
        mine = {k[len(prefix):]: v for k, v in state_dict.items() if k in ours}
        store = "store_exp_avg" in mine
        if store:
            absent = [k for k in STORE_KEYS if k not in mine]
            if absent:
                error_msgs.append(f"the checkpoint holds part of the surfel store's state only: {absent} missing")
                return
            theirs = tuple(_ALL_GROUPS[int(i)] for i in mine["store_groups"].tolist())
            if theirs != tuple(names):
                error_msgs.append(f"the checkpoint's surfel groups {list(theirs)} are not this store's {names}")
                return
        src = {}
        for n in names:
            v = mine.get(_ATTR[n])
            if v is None:
                missing_keys.append(prefix + _ATTR[n])
            elif tuple(v.shape[1:]) != _TAIL[n] or v.dim() != 1 + len(_TAIL[n]):
                error_msgs.append(f"size mismatch for {prefix + _ATTR[n]}: the checkpoint's {tuple(v.shape)} is not "
                                  f"(P,{','.join(map(str, _TAIL[n]))})")
                return
            else:
                src[n] = v
        if not src:
            return
        rows = {int(v.shape[0]) for v in src.values()}
        if len(rows) != 1:
            error_msgs.append(f"the checkpoint's surfel groups disagree on the surfel count: "
                              f"{ {_ATTR[n]: int(v.shape[0]) for n, v in src.items()} }")
            return
        P = rows.pop()
        if P != self.P and len(src) != len(names):
            error_msgs.append(f"the checkpoint has {P} surfels, the store {self.P}: every group is needed to change the "
                              f"surfel count, {[prefix + _ATTR[n] for n in names if n not in src]} missing")
            return
        if store:
            _, total = self._offsets(P)
            for k, shape in (("store_exp_avg", (total,)), ("store_exp_avg_sq", (total,)), ("store_densify_stats", (2, P)),
                             ("store_max_radii2D", (P,)), ("store_lr", (len(names),))):
                if tuple(mine[k].shape) != shape:
                    error_msgs.append(f"size mismatch for {prefix + k}: {tuple(mine[k].shape)}, expected {shape}")
                    return
        for n in names:                       # groups the checkpoint lacks keep their current rows (same P only)
            if n not in src:
                held = self._parameters[_ATTR[n]].detach()
                if int(held.shape[0]) != P:
                    error_msgs.append(f"{prefix + _ATTR[n]} is missing from the checkpoint and the tensor assigned to it "
                                      f"has {int(held.shape[0])} rows, the checkpoint's surfels {P}")
                    return
                src[n] = held
        dev = self.flat.device
        if P == self.P:
            foreign = list(self._foreign)
            for n in names:
                self._group_view(n).copy_(src[n])
            if foreign:
                self._bind(foreign)
            for buf, k in ((self.exp_avg, "store_exp_avg"), (self.exp_avg_sq, "store_exp_avg_sq"),
                           (self.densify_stats, "store_densify_stats"), (self.max_radii2D, "store_max_radii2D")):
                if store:
                    buf.copy_(mine[k])
                else:
                    buf.zero_()
            self.grad_flat.zero_()
        else:
            self.P = P
            self.flat = torch.cat([src[n].reshape(-1).to(dev, torch.float32) for n in names])
            self._bind()
            if store:
                cp = lambda k: mine[k].to(dev, torch.float32, copy=True).contiguous()  # noqa: E731
                self.exp_avg, self.exp_avg_sq = cp("store_exp_avg"), cp("store_exp_avg_sq")
                self.densify_stats, self.max_radii2D = cp("store_densify_stats"), cp("store_max_radii2D")
            else:
                self.exp_avg, self.exp_avg_sq = torch.zeros_like(self.flat), torch.zeros_like(self.flat)
                self._reset_stats()
        self._clip_pending = False
        if not store:
            self.device_step.zero_()
            self.step_count = 0
            return
        self.device_step.copy_(mine["store_device_step"])
        self.step_count = int(mine["store_step_count"])
        for n, r in zip(names, mine["store_lr"].tolist()):
            self.set_lr(n, r)
        self.active_sh_degree = int(mine["store_active_sh_degree"])
        self.betas = tuple(float(b) for b in mine["store_betas"].tolist())
        self.eps = float(mine["store_eps"])
        self.percent_dense = float(mine["store_percent_dense"])

    # ---- torch.optim.Adam interop: the reference's gs_optimizer (trainer.py:243-253) ----------------------------------
    @classmethod
    @torch.no_grad()
    def from_gaussian_model(cls, gm, optimizer=None, lrs=None, device=None):
        """A store holding `gm`'s surfels (any module with the reference's _xyz ... _rotation and optional _regist_feat),
        its active_sh_degree and percent_dense, and its max_radii2D / xyz_gradient_accum / denom when they have one row
        per surfel.  With `optimizer` -- the reference's gs_optimizer, a torch.optim.Adam with one param group per
        tensor named as in trainer.py:243-253 -- each group's rate, exp_avg, exp_avg_sq and step are imported, and
        Adam's betas and eps (which must be the same for every surfel group).  The store keeps one step count: the
        surfel groups must all have the same `step` (a group without state counts as step 0), or this raises.  Groups
        that are not surfel groups (bg_rgb) are left to the optimizer."""
        dev = torch.device(device) if device is not None else gm._xyz.device
        t = lambda name: getattr(gm, name).detach().to(dev, torch.float32)  # noqa: E731
        regist = getattr(gm, "_regist_feat", None)
        kw = {"sh_degree": int(getattr(gm, "active_sh_degree", 3)), "percent_dense": float(getattr(gm, "percent_dense", 0.01)),
              "regist_feat": None if regist is None else t("_regist_feat"), "lrs": lrs}
        if optimizer is not None:
            groups = {g.get("name"): g for g in optimizer.param_groups}
            names = [n for n, _ in GROUPS] + ([REGIST_FEAT[0]] if regist is not None else [])
            lost = [n for n in names if n not in groups or len(groups[n]["params"]) != 1]
            if lost:
                raise ValueError(f"the optimizer needs one param group of one tensor named {lost} (trainer.py:243-253)")
            for n in names:
                g = groups[n]
                if g.get("amsgrad") or g.get("maximize") or g.get("weight_decay", 0.0) != 0.0:
                    raise ValueError(f"param group {n!r}: the store's Adam has no amsgrad, maximize or weight decay")
            consts = {(tuple(groups[n]["betas"]), float(groups[n]["eps"])) for n in names}
            if len(consts) != 1:
                raise ValueError(f"the surfel groups' Adam betas / eps differ: {consts}; the store has one pair")
            (betas, eps), = consts
            kw.update(betas=tuple(float(b) for b in betas), eps=eps, lrs={n: float(groups[n]["lr"]) for n in names})
        m = cls(t("_xyz"), t("_features_dc"), t("_features_rest"), t("_opacity"), t("_scaling"), t("_rotation"), **kw)
        P = m.P
        for name in ("max_radii2D", "xyz_gradient_accum", "denom"):
            v = getattr(gm, name, None)
            if isinstance(v, torch.Tensor) and v.numel() == P:
                getattr(m, name).copy_(v.reshape(getattr(m, name).shape))
        if optimizer is not None:
            m._import_adam(optimizer)
        return m

    def _import_adam(self, optimizer):
        groups = {g.get("name"): g for g in optimizer.param_groups}
        steps, off = {}, self._offsets(self.P)[0]
        for (n, k), o in zip(self.groups, off):
            st = optimizer.state.get(groups[n]["params"][0], {})
            steps[n] = int(st["step"]) if "step" in st else 0
            for buf, key in ((self.exp_avg, "exp_avg"), (self.exp_avg_sq, "exp_avg_sq")):
                seg = buf[o:o + self.P * k]
                if key in st:
                    seg.copy_(st[key].reshape(-1))
                else:
                    seg.zero_()
        if len(set(steps.values())) > 1:
            raise ValueError(f"the surfel groups' Adam steps differ ({steps}); the store keeps one step count for all")
        step = next(iter(steps.values()))
        self.device_step.fill_(step)
        self.step_count = step

    def adam_state_dict(self, optimizer=None) -> dict:
        """The moments and step in torch.optim.Adam's state_dict() format, one param group per surfel group in the
        store's order (the order of trainer.py:243-253), for optimizer.load_state_dict / GaussianModel.restore.  With
        `optimizer` (one whose param groups are named as there, bg_rgb and others included), its own state_dict() with
        the surfel groups' state and rates replaced: the groups it has beyond the surfels keep theirs."""
        self._live("adam_state_dict")
        off, _ = self._offsets(self.P)
        per = {}
        for (n, k), o in zip(self.groups, off):
            view = lambda b: b[o:o + self.P * k].view((self.P,) + _TAIL[n]).clone()  # noqa: E731
            per[n] = {"step": torch.tensor(float(int(self.device_step)), dtype=torch.float32),
                      "exp_avg": view(self.exp_avg), "exp_avg_sq": view(self.exp_avg_sq)}
        if optimizer is None:
            base = {"weight_decay": 0.0, "amsgrad": False, "maximize": False, "foreach": None, "capturable": False,
                    "differentiable": False, "fused": None}
            groups = [dict(base, lr=self.lrs[n], betas=tuple(self.betas), eps=self.eps, params=[i], name=n)
                      for i, (n, _) in enumerate(self.groups)]
            return {"state": {i: per[n] for i, (n, _) in enumerate(self.groups)}, "param_groups": groups}
        sd = optimizer.state_dict()
        for g in sd["param_groups"]:
            n = g.get("name")
            if n in per:
                g.update(lr=self.lrs[n], betas=tuple(self.betas), eps=self.eps)
                sd["state"][g["params"][0]] = per[n]
        return sd

    # ---- 2DGS's vertex PLY (gaussian_model.py:189-268; vidu4d_b200/ply.py) -----------------------------------------------
    def save_ply(self, path, regist_feat: bool = True):
        """gaussian_model.py save_ply's file, plus regist_feat_0..15 when the store has the group and `regist_feat`."""
        from . import ply
        self._live("save_ply")
        ply.write_surfels(path, {n: self._parameters[_ATTR[n]].detach() for n, _ in self.groups
                                 if n != "regist_feat" or regist_feat})

    def load_ply(self, path):
        """gaussian_model.py load_ply: the file's surfels replace the store's, as a checkpoint without the store's state
        does (load_state_dict: in place at the same P; zero moments, step 0 and zero statistics), and active_sh_degree =
        max_sh_degree.  regist_feat is read when the file has it and the store has the group; otherwise the store's rows
        are kept at the same P and zero at another."""
        from . import ply
        got = ply.read_surfels(path)
        P = int(got["xyz"].shape[0])
        if "regist_feat" in [n for n, _ in self.groups] and "regist_feat" not in got and P != self.P:
            got["regist_feat"] = torch.zeros((P, 16))
        self.load_state_dict({_ATTR[n]: t for n, t in got.items() if n in [g for g, _ in self.groups]}, strict=False)
        self.active_sh_degree = self.max_sh_degree
