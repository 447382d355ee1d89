"""Frame sharding and the one collective of the hot path.

The reference expresses multi-GPU Stage 3 as DDP + DistributedSampler over frame pairs
(lab4d/dataloader/data_utils.py:56-61, lab4d/engine/train_utils.py:15-28, lab4d/train.py:28-36).  Frames are
independent units: every rank holds the canonical surfels, renders its own frames (warp -> rasterize -> loss ->
backward) and the canonical-surfel gradients are summed across ranks once per optimizer step.

    shard_frames()   which global frame indices this rank renders (rank r takes r, r+G, ...)
    FlatGrads        one flat fp32 buffer that *is* the .grad of every surfel parameter, so the exchange is a
                     single NCCL all-reduce over NVLink (gloo on CPU in the tests), no per-tensor buckets.
                     A FlatSurfelModel, whose size changes with densification, uses its own allreduce_grads_.
    shared_generator()   the same random stream on every rank (densify_and_prune's split noise)
    check_replicas()     raise if the ranks' copies of some tensors differ in any bit (a debugging and test aid)
    allreduce_contributions()   every rank's per-surfel contribution statistics summed over the ranks, exactly
    allreduce_lift()            every rank's lifted per-surfel sums summed over the ranks, exactly
"""
from __future__ import annotations

import os
from typing import List, Sequence

import torch
import torch.distributed as dist


def env_rank_world():
    return int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("LOCAL_RANK", "0"))


def init_distributed(backend: str | None = None, device: torch.device | None = None) -> tuple[int, int]:
    """Initialise torch.distributed from the torchrun environment (env://).  No-op for world size 1."""
    rank, world, _ = env_rank_world()
    if world > 1 and not dist.is_initialized():
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29500")
        if backend is None:
            backend = "nccl" if torch.cuda.is_available() else "gloo"
        kw = {}
        if backend == "nccl" and device is not None:
            kw["device_id"] = device
        if backend == "nccl":
            # the collective's CTAs must be resident on every rank before it can progress: a high-priority communication
            # stream lets them in ahead of the queued compute CTAs when an all-reduce overlaps the next step's kernels
            opts = dist.ProcessGroupNCCL.Options()
            opts.is_high_priority_stream = True
            kw["pg_options"] = opts
        dist.init_process_group(backend=backend, init_method="env://", rank=rank, world_size=world, **kw)
    return rank, world


def shard_frames(num_frames: int, rank: int, world: int) -> List[int]:
    """Round-robin frame assignment: rank r renders frames r, r+world, ... (SURVEY.md section 8(e))."""
    return list(range(rank, num_frames, world))


def _multi_rank(group) -> bool:
    return dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1


def shared_generator(device, seed: int | None = None, group=None) -> torch.Generator:
    """A generator on `device` seeded with the group's rank 0's seed (its `seed`, or a fresh random one), so that every
    rank draws the same numbers.  Pass it to FlatSurfelModel.densify_and_prune(generator=).  On one rank: seeded with
    `seed` (or a fresh one)."""
    device = torch.device(device)
    if seed is None:
        seed = int.from_bytes(os.urandom(8), "little") >> 1
    if _multi_rank(group):
        t = torch.tensor([int(seed)], dtype=torch.int64, device=device)
        dist.broadcast(t, src=dist.get_global_rank(group, 0) if group is not None else 0, group=group)
        seed = int(t.item())
    return torch.Generator(device=device).manual_seed(int(seed))


_P31 = (1 << 31) - 1


def _checksum(t: torch.Tensor) -> torch.Tensor:
    """A 64-bit checksum of t's raw bits, on t's device, as a 0-d int64 tensor: the low 31 bits of the sum of its 32-bit
    words (any single changed word shows) in the high half, and the position-weighted sum of the words modulo 2^31 - 1
    (moved words show) in the low half.  Every intermediate stays below 2^63 for tensors of up to 2^31 words."""
    b = t.detach().contiguous().reshape(-1).view(torch.uint8)
    if b.numel() % 4:
        b = torch.cat([b, b.new_zeros(4 - b.numel() % 4)])
    w = b.view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    pos = torch.arange(1, w.numel() + 1, dtype=torch.int64, device=w.device) % _P31
    weighted = (w % _P31) * pos % _P31
    return (w.sum() & 0x7FFFFFFF) * (1 << 32) + weighted.sum() % _P31


def check_replicas(named_tensors: dict, group=None) -> None:
    """Raise RuntimeError unless every rank holds the same bits in each tensor of `named_tensors` (name -> tensor, or
    name -> int such as the surfel count P), naming the first entry that differs and the ranks whose copy differs from
    the group's rank 0.  All-gathers one checksum and one size per entry (a debugging and test aid: one host sync; not
    meant for the step).  No-op on one rank."""
    if not _multi_rank(group):
        return
    names = list(named_tensors)
    dev = next((v.device for v in named_tensors.values() if isinstance(v, torch.Tensor)), torch.device("cpu"))
    rows = []
    for name in names:
        v = named_tensors[name]
        if isinstance(v, torch.Tensor):
            rows.append(torch.stack([torch.tensor(v.numel(), device=dev), _checksum(v.to(dev))]))
        else:
            rows.append(torch.tensor([int(v), 0], dtype=torch.int64, device=dev))
    mine = torch.stack(rows)
    world = dist.get_world_size(group)
    got = [torch.empty_like(mine) for _ in range(world)]
    dist.all_gather(got, mine, group=group)
    got = torch.stack(got).cpu()
    for k, name in enumerate(names):
        bad = [r for r in range(1, world) if not torch.equal(got[r, k], got[0, k])]
        if bad:
            what = "value or size" if int(got[bad[0], k, 0]) != int(got[0, k, 0]) else "bits"
            raise RuntimeError(f"replicas differ in {name!r} ({what}): ranks {bad} of the group differ from its rank 0")


def allreduce_contributions(contrib, group=None):
    """Make every rank's renderer.SurfelContributions those of all the ranks' frames: SUM over weight_q, pixels and
    frames, and over weight_bg_q and pixels_bg when present (int64 words; the totals stay below 2^63), MAX over
    max_weight (the float bits as int32, which order as the non-negative floats do).  Integer collectives are exact, so every rank ends with the same bits, those one rank
    rendering every frame would have, and FlatSurfelModel.prune_by_contribution prunes the same surfels everywhere.
    In place; returns contrib.  No-op on one rank."""
    if _multi_rank(group):
        sums = [contrib.weight_q, contrib.pixels, contrib.frames]
        if contrib.silhouettes:
            sums += [contrib.weight_bg_q, contrib.pixels_bg]
        for t in sums:
            dist.all_reduce(t, op=dist.ReduceOp.SUM, group=group)
        dist.all_reduce(contrib.max_weight, op=dist.ReduceOp.MAX, group=group)
    return contrib


def allreduce_lift(lift, group=None):
    """Make every rank's renderer.SurfelLift that of all the ranks' frames: SUM over sums and saturated (int64, two's
    complement: exact, whatever the order).  With allreduce_contributions over the same frames, every rank's
    lift.mean(contrib) has the same bits.  Every rank must use the same scale_log2 (checked).  In place; returns lift.
    No-op on one rank."""
    if _multi_rank(group):
        s = torch.tensor([lift.scale_log2, -lift.scale_log2], dtype=torch.int64, device=lift.sums.device)
        dist.all_reduce(s, op=dist.ReduceOp.MAX, group=group)
        if int(s[0]) != lift.scale_log2 or -int(s[1]) != lift.scale_log2:
            raise RuntimeError(f"lift scales differ across ranks: scale_log2 from {-int(s[1])} to {int(s[0])}")
        dist.all_reduce(lift.sums, op=dist.ReduceOp.SUM, group=group)
        dist.all_reduce(lift.saturated, op=dist.ReduceOp.SUM, group=group)
    return lift


class FlatGrads:
    """Gradients of a list of parameters laid out back to back in ONE fp32 buffer; each p.grad is a view."""

    def __init__(self, params: Sequence[torch.nn.Parameter]):
        self.params = list(params)
        dev = self.params[0].device
        n = sum(p.numel() for p in self.params)
        self.flat = torch.zeros((n,), dtype=torch.float32, device=dev)
        o = 0
        for p in self.params:
            p.grad = self.flat[o:o + p.numel()].view_as(p)
            o += p.numel()

    def zero_(self):
        self.flat.zero_()

    def allreduce_(self, average_over: int | None = None):
        """Sum over ranks (one collective); optionally divide by the global number of frames."""
        if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
            dist.all_reduce(self.flat, op=dist.ReduceOp.SUM)
        if average_over:
            self.flat.mul_(1.0 / float(average_over))
        return self.flat

    @property
    def nbytes(self) -> int:
        return self.flat.numel() * 4
