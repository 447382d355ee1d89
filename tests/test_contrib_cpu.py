"""CPU tests of the per-surfel contribution statistics: sr_render_forward_contrib's entry in the header, library and binding;
its argument checks, made before any device work; SurfelContributions' prune mask and render_frames' checks of it;
FlatSurfelModel.prune_by_contribution's bookkeeping; distributed.allreduce_contributions over two gloo ranks."""
import ctypes as C
import os
import re
import sys

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from .conftest import ROOT
from .test_render_cpu import _PC, _cams, _render_args

D = 1 << 20      # placeholder DEVICE pointer: never dereferenced (the calls fail before any device work)


def test_contrib_entry_point_in_header_library_and_binding(built):
    """The new entry point is sr_render_forward's parameter list with `const sr_contrib* contrib` before the stream; the
    binding's struct has the header's three pointer fields in order."""
    from vidu4d_b200 import _capi
    lib = _capi.load()
    assert hasattr(lib, "sr_render_forward_contrib") and "sr_render_forward_contrib" in _capi.RENDER_SYMBOLS
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "surfel_render.h")).read(), flags=re.S)
    protos = {name: [p.strip() for p in params.split(",")]
              for name, params in re.findall(r"SR_API\s+[\w\s\*]+?\b(sr_\w+)\s*\(([^)]*)\)", hdr)}
    base, new = protos["sr_render_forward"], protos["sr_render_forward_contrib"]
    assert new[:-2] == base[:-1] and new[-1] == base[-1] == "void* stream"
    assert new[-2] == "const sr_contrib* contrib"
    rt, args = _capi.RENDER_PROTOTYPES["sr_render_forward_contrib"]
    assert rt == C.c_int and args[:-2] == _capi.RENDER_PROTOTYPES["sr_render_forward"][1][:-1]
    assert args[-2:] == [C.c_void_p, C.c_void_p]
    fields = re.search(r"typedef struct sr_contrib \{(.*?)\} sr_contrib;", hdr, flags=re.S).group(1)
    assert re.findall(r"(\w+)\s*\*\s*(\w+);", fields) == [("uint64_t", "weight_q"), ("uint32_t", "max_weight"),
                                                          ("uint64_t", "pixels")]
    assert [n for n, _ in _capi.SrContrib._fields_] == ["weight_q", "max_weight", "pixels"]
    assert C.sizeof(_capi.SrContrib) == 24


def _contrib_args(fr, bt, contrib, **kw):
    return _render_args(fr, bt, **kw)[:-1] + [contrib, None]


@pytest.mark.parametrize("case, msg", [
    ("null_weight_q", b"contribution statistics pointer is NULL"),
    ("null_max_weight", b"contribution statistics pointer is NULL"),
    ("null_pixels", b"contribution statistics pointer is NULL"),
    ("weight_q_align", b"weight_q / pixels must be 8-byte aligned, max_weight 4-byte aligned"),
    ("pixels_align", b"weight_q / pixels must be 8-byte aligned, max_weight 4-byte aligned"),
    ("max_weight_align", b"weight_q / pixels must be 8-byte aligned, max_weight 4-byte aligned"),
    ("null_arena", b"arena is NULL"),
    ("capacity_0", b"capacity must be in (0, 2^30)"),
    ("F_33", b"F must be in [1, 32], got 33"),
    ("bg_F0", b"background must have 3 channels when F = 0, got 4"),
    ("frames_0", b"frames must be in [1, 65535]"),
    ("null_frame", b"frame descriptor is NULL"),
])
def test_render_forward_contrib_rejects_bad_arguments(built, case, msg):
    """sr_render_forward's checks (it shares them) and the statistics' own, all before any device work."""
    from vidu4d_b200 import _capi
    lib = _capi.load()
    fr = _capi.SrFrame(100, 3, 16, 64, 48, 0.5, 0.5, 1.0, 0, 0, 0)
    bt = _capi.SrBatch(2, 0, 0, 0, 0, 0, 0, 0)
    ct = _capi.SrContrib(D, D + 4096, D + 8192)
    kw = {}
    if case == "null_weight_q":
        ct.weight_q = None
    elif case == "null_max_weight":
        ct.max_weight = None
    elif case == "null_pixels":
        ct.pixels = None
    elif case == "weight_q_align":
        ct.weight_q = D + 4
    elif case == "pixels_align":
        ct.pixels = D + 8196
    elif case == "max_weight_align":
        ct.max_weight = D + 4098
    elif case == "null_arena":
        kw["arena"] = None
    elif case == "capacity_0":
        kw["cap"] = 0
    elif case == "F_33":
        kw.update(F=33, features=D, bg_ch=36)
    elif case == "bg_F0":
        kw["bg_ch"] = 4
    elif case == "frames_0":
        bt = _capi.SrBatch(0, 0, 0, 0, 0, 0, 0, 0)
    args = _contrib_args(fr, bt, C.byref(ct), **kw)
    if case == "null_frame":
        args[0] = None
    assert lib.sr_render_forward_contrib(*args) == -1
    assert msg in lib.sr_last_error(), (case, lib.sr_last_error())


def _contrib(wq, mw, px, fr=None):
    from vidu4d_b200.renderer import SurfelContributions
    wq = torch.tensor(wq, dtype=torch.int64)
    return SurfelContributions(wq, torch.tensor(mw, dtype=torch.int32), torch.tensor(px, dtype=torch.int64),
                               torch.zeros_like(wq) if fr is None else torch.tensor(fr, dtype=torch.int64))


def test_weight_and_prune_mask():
    from vidu4d_b200.renderer import SurfelContributions
    z = SurfelContributions.zeros(5, "cpu")
    assert z.P == 5 and [t.dtype for t in (z.weight_q, z.max_weight, z.pixels, z.frames)] == \
        [torch.int64, torch.int32, torch.int64, torch.int64]
    assert bool(z.prune_mask().all())                                   # nothing blended: everything goes
    q = [0, 1, 2 ** 31, 3 * 2 ** 32 + 5, 2 ** 62]
    c = _contrib(q, [0, 1, 2, 3, 4], [0, 1, 1, 7, 2 ** 40])
    assert c.weight.dtype == torch.float64
    assert c.weight.tolist() == [x / 2.0 ** 32 for x in q]
    assert c.prune_mask().tolist() == [True, False, False, False, False]
    assert c.prune_mask(min_weight=0.5).tolist() == [True, True, False, False, False]       # 2^31 / 2^32 = 0.5 stays
    assert c.prune_mask(min_weight=0.5000001).tolist() == [True, True, True, False, False]
    assert c.prune_mask(min_pixels=2).tolist() == [True, True, True, False, False]
    assert c.prune_mask(min_weight=0.0, min_pixels=0).tolist() == [False] * 5


@pytest.mark.parametrize("bad, msg", [
    ("P", r"contributions.weight_q must be a contiguous torch.int64 \(P,\) = \(10,\) tensor, got \(11,\)"),
    ("dtype", r"contributions.max_weight must be a contiguous torch.int32"),
    ("strided", r"contributions.pixels must be a contiguous"),
    ("device", r"contributions.weight_q must be on the rasterizer's device meta, got cpu"),
    ("type", r"contributions must be a SurfelContributions, got dict"),
])
def test_render_frames_rejects_bad_contributions_before_any_launch(bad, msg):
    from vidu4d_b200.renderer import PipelineParams, SurfelContributions, render_frames
    c = SurfelContributions.zeros(10, "cpu")
    pc = _PC(10)
    if bad == "P":
        c = SurfelContributions.zeros(11, "cpu")
    elif bad == "dtype":
        c.max_weight = torch.zeros(10, dtype=torch.float32)
    elif bad == "strided":
        c.pixels = torch.zeros(20, dtype=torch.int64)[::2]
    elif bad == "device":
        pc = _PC(10, dev="meta")           # the surfels' device is the rasterizer's
    elif bad == "type":
        c = {}
    with pytest.raises(RuntimeError, match=msg):
        render_frames(_cams(4), pc, PipelineParams(), torch.zeros(3), contributions=c)


def _cpu_store(P):
    from vidu4d_b200.surfel_store import FlatSurfelModel
    g = torch.Generator().manual_seed(0)
    r = lambda *s: torch.rand(s, generator=g)  # noqa: E731
    return FlatSurfelModel(r(P, 3), r(P, 1, 3), r(P, 15, 3), r(P, 1), r(P, 2), r(P, 4), regist_feat=r(P, 16))


def test_prune_by_contribution_bookkeeping(monkeypatch):
    """The mask reaches prune_points unchanged and the count is returned; no prune_points call when nothing goes; a
    statistics set of another P is refused."""
    from vidu4d_b200.surfel_store import FlatSurfelModel
    m = _cpu_store(5)
    seen = []
    monkeypatch.setattr(FlatSurfelModel, "prune_points", lambda self, mask: seen.append(mask.clone()))
    c = _contrib([0, 2 ** 32, 2 ** 30, 0, 7], [0, 5, 5, 0, 1], [0, 40, 3, 0, 1])
    assert m.prune_by_contribution(c) == 2
    assert seen[-1].tolist() == [True, False, False, True, False]
    assert m.prune_by_contribution(c, min_weight=0.25, min_pixels=2) == 3
    assert seen[-1].tolist() == [True, False, False, True, True]
    n = len(seen)
    assert m.prune_by_contribution(c, min_weight=0.0, min_pixels=0) == 0 and len(seen) == n
    with pytest.raises(RuntimeError, match="contributions are for 4 surfels, the store has 5"):
        m.prune_by_contribution(_contrib([1] * 4, [1] * 4, [1] * 4))


def _synthetic(rank, P=1000):
    """Rank `rank`'s statistics: large, distinct integer sums and float bits whose maximum is on either rank."""
    rng = np.random.default_rng(100 + rank)
    wq = rng.integers(0, 2 ** 52, P, dtype=np.int64)
    mw = (rng.random(P, dtype=np.float32) * 0.99).view(np.int32)
    px = rng.integers(0, 2 ** 40, P, dtype=np.int64)
    fr = rng.integers(0, 1000, P, dtype=np.int64)
    return _contrib(wq, mw, px, fr)


def _worker(rank, world, port, out):
    sys.path.insert(0, ROOT)
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1",
                      MASTER_PORT=str(port))
    import torch.distributed as dist
    from vidu4d_b200 import distributed as D
    D.init_distributed("gloo")
    c = _synthetic(rank)
    assert D.allreduce_contributions(c) is c
    D.check_replicas({"weight_q": c.weight_q, "max_weight": c.max_weight, "pixels": c.pixels, "frames": c.frames})
    torch.save({k: getattr(c, k) for k in ("weight_q", "max_weight", "pixels", "frames")}, f"{out}.{rank}")
    dist.destroy_process_group()


def test_allreduce_contributions_over_two_gloo_ranks(tmp_path):
    """Both ranks end with the same bits, those of the single-rank total: integer sums, and the maximum of the float
    bits, which is the bits of the maximum float."""
    import socket
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    out = str(tmp_path / "c")
    mp.start_processes(_worker, args=(2, port, out), nprocs=2, join=True, start_method="spawn")
    got = [torch.load(f"{out}.{r}") for r in range(2)]
    a, b = _synthetic(0), _synthetic(1)
    want = {"weight_q": a.weight_q + b.weight_q, "pixels": a.pixels + b.pixels, "frames": a.frames + b.frames,
            "max_weight": torch.maximum(a.max_weight, b.max_weight)}
    fmax = torch.maximum(a.max_weight.view(torch.float32), b.max_weight.view(torch.float32))
    assert torch.equal(want["max_weight"].view(torch.float32), fmax)
    for r in range(2):
        for k, v in want.items():
            assert torch.equal(got[r][k], v), (r, k)
    # one rank: a no-op that returns its argument
    from vidu4d_b200.distributed import allreduce_contributions
    c = _synthetic(0)
    assert allreduce_contributions(c) is c and torch.equal(c.weight_q, a.weight_q)
