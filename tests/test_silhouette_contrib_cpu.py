"""CPU tests of the silhouette share of the contribution statistics: sr_render_forward_contrib_masked's entry in the
header, library and binding, and its argument checks, made before any device work; SurfelContributions' background
words, background_fraction and prune mask; render_frames' checks of masks; FlatSurfelModel.prune_by_contribution's
max_background_fraction; distributed.allreduce_contributions of the background words over two gloo ranks."""
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


def _header_protos():
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "surfel_render.h")).read(), flags=re.S)
    protos = {name: [p.strip() for p in params.split(",")]
              for name, params in re.findall(r"SR_API\s+[\w\s\*]+?\b(sr_\w+)\s*\(([^)]*)\)", hdr)}
    return hdr, protos


def test_masked_entry_point_in_header_library_and_binding(built):
    """sr_render_forward_contrib_masked is sr_render_forward_contrib's parameter list with `const sr_contrib_mask* mask`
    before the stream; sr_render_forward_contrib and sr_contrib keep their prototype and layout; the binding's struct
    has the header's four fields in order."""
    from vidu4d_b200 import _capi
    lib = _capi.load()
    assert hasattr(lib, "sr_render_forward_contrib_masked") and "sr_render_forward_contrib_masked" in _capi.RENDER_SYMBOLS
    hdr, protos = _header_protos()
    base, new = protos["sr_render_forward_contrib"], protos["sr_render_forward_contrib_masked"]
    assert base[-2:] == ["const sr_contrib* contrib", "void* stream"]
    assert new[:-2] == base[:-1] and new[-2] == "const sr_contrib_mask* mask" and new[-1] == "void* stream"
    rt, args = _capi.RENDER_PROTOTYPES["sr_render_forward_contrib_masked"]
    assert rt == C.c_int and args[:-2] == _capi.RENDER_PROTOTYPES["sr_render_forward_contrib"][1][:-1]
    assert args[-2:] == [C.c_void_p, C.c_void_p]
    fields = re.search(r"typedef struct sr_contrib_mask \{(.*?)\} sr_contrib_mask;", hdr, flags=re.S).group(1)
    assert [tuple(x.split()) for x in re.findall(r"([\w ]+?\**\s*\w+);", fields)] == [
        ("const", "uint8_t*", "mask"), ("int64_t", "mask_stride"), ("uint64_t*", "weight_bg_q"), ("uint64_t*", "pixels_bg")]
    assert [n for n, _ in _capi.SrContribMask._fields_] == ["mask", "mask_stride", "weight_bg_q", "pixels_bg"]
    assert C.sizeof(_capi.SrContribMask) == 32
    old = re.search(r"typedef struct sr_contrib \{(.*?)\} sr_contrib;", hdr, flags=re.S).group(1)
    assert re.findall(r"(\w+)\s*\*\s*(\w+);", old) == [("uint64_t", "weight_q"), ("uint32_t", "max_weight"),
                                                       ("uint64_t", "pixels")]


def _masked_args(fr, bt, contrib, mask, **kw):
    return _render_args(fr, bt, **kw)[:-1] + [contrib, mask, None]


@pytest.mark.parametrize("case, msg", [
    ("no_contrib", b"a silhouette mask needs the contribution statistics (contrib is NULL)"),
    ("no_contrib_P0", b"a silhouette mask needs the contribution statistics (contrib is NULL)"),
    ("stride", b"silhouette mask frame stride must be >= H*W bytes"),
    ("stride_P0", b"silhouette mask frame stride must be >= H*W bytes"),
    ("null_weight_bg_q", b"silhouette statistics pointer is NULL"),
    ("null_pixels_bg", b"silhouette statistics pointer is NULL"),
    ("weight_bg_q_align", b"weight_bg_q / pixels_bg must be 8-byte aligned"),
    ("pixels_bg_align", b"weight_bg_q / pixels_bg must be 8-byte aligned"),
    ("null_pixels", b"contribution statistics pointer is NULL"),
    ("null_arena", b"arena is NULL"),
    ("F_33", b"F must be in [1, 32], got 33"),
    ("null_frame", b"frame descriptor is NULL"),
])
def test_render_forward_contrib_masked_rejects_bad_arguments(built, case, msg):
    """sr_render_forward_contrib's checks (it shares them) and the mask's own, all before any device work."""
    from vidu4d_b200 import _capi
    lib = _capi.load()
    P = 0 if case.endswith("_P0") else 100
    fr = _capi.SrFrame(P, 3, 16, 64, 48, 0.5, 0.5, 1.0, 0, 0, 0)
    bt = _capi.SrBatch(2, 0, 0, 0, 0, 0, 0, 0)
    ct = _capi.SrContrib(D, D + 4096, D + 8192)
    mk = _capi.SrContribMask(D + 12288, 64 * 48, D + 16384, D + 20480)
    contrib, kw = C.byref(ct), {}
    if case.startswith("no_contrib"):
        contrib = None
    elif case.startswith("stride"):
        mk.mask_stride = 64 * 48 - 1
    elif case == "null_weight_bg_q":
        mk.weight_bg_q = None
    elif case == "null_pixels_bg":
        mk.pixels_bg = None
    elif case == "weight_bg_q_align":
        mk.weight_bg_q = D + 16388
    elif case == "pixels_bg_align":
        mk.pixels_bg = D + 20482
    elif case == "null_pixels":
        ct.pixels = None
    elif case == "null_arena":
        kw["arena"] = None
    elif case == "F_33":
        kw.update(F=33, features=D, bg_ch=36)
    args = _masked_args(fr, bt, contrib, C.byref(mk), **kw)
    if case == "null_frame":
        args[0] = None
    assert lib.sr_render_forward_contrib_masked(*args) == -1
    assert msg in lib.sr_last_error(), (case, lib.sr_last_error())


def test_null_mask_is_the_unmasked_call(built):
    """A NULL mask struct, or one whose mask is NULL, is sr_render_forward_contrib: its output words are not checked, and
    a NULL contrib is then sr_render_forward (which fails here on the arena, the first check it reaches)."""
    from vidu4d_b200 import _capi
    lib = _capi.load()
    fr = _capi.SrFrame(100, 3, 16, 64, 48, 0.5, 0.5, 1.0, 0, 0, 0)
    bt = _capi.SrBatch(2, 0, 0, 0, 0, 0, 0, 0)
    ct = _capi.SrContrib(D, D + 4096, D + 8192)
    for mask in (None, C.byref(_capi.SrContribMask(None, 0, None, None))):
        for contrib in (C.byref(ct), None):
            assert lib.sr_render_forward_contrib_masked(*_masked_args(fr, bt, contrib, mask, arena=None)) == -1
            assert b"arena is NULL" in lib.sr_last_error()


def _contrib(wq, mw, px, wbg=None, pbg=None):
    from vidu4d_b200.renderer import SurfelContributions
    t = lambda v, dt=torch.int64: None if v is None else torch.tensor(v, dtype=dt)  # noqa: E731
    wq = t(wq)
    return SurfelContributions(wq, t(mw, torch.int32), t(px), torch.zeros_like(wq), t(wbg), t(pbg))


def test_zeros_background_fraction_and_prune_mask():
    from vidu4d_b200.renderer import SurfelContributions
    z = SurfelContributions.zeros(4, "cpu")
    assert z.weight_bg_q is None and z.pixels_bg is None and not z.silhouettes
    with pytest.raises(RuntimeError, match="background_fraction needs the background words"):
        z.background_fraction
    with pytest.raises(RuntimeError, match="background_fraction needs the background words"):
        z.prune_mask(max_background_fraction=0.5)
    z = SurfelContributions.zeros(4, "cpu", silhouettes=True)
    assert z.silhouettes and z.weight_bg_q.dtype == torch.int64 and z.pixels_bg.dtype == torch.int64
    assert z.weight_bg_q.shape == (4,) and z.pixels_bg.shape == (4,)
    # weight_q == 0: fraction 0, not NaN
    assert z.background_fraction.dtype == torch.float64 and z.background_fraction.tolist() == [0.0] * 4

    q = [0, 2 ** 32, 3 * 2 ** 32, 2 ** 40, 7, 2 ** 62]
    bq = [0, 2 ** 31, 3 * 2 ** 32, 2 ** 38, 0, 3 * 2 ** 60]
    c = _contrib(q, [0, 1, 2, 3, 4, 5], [0, 5, 9, 100, 1, 2 ** 40], bq, [0, 2, 9, 30, 0, 2 ** 39])
    assert c.background_fraction.tolist() == [0.0, 0.5, 1.0, 0.25, 0.0, 0.75]
    base = c.prune_mask().tolist()
    assert base == [True, False, False, False, False, False]
    assert c.prune_mask(max_background_fraction=None).tolist() == base
    assert c.prune_mask(max_background_fraction=0.5).tolist() == [True, False, True, False, False, True]
    assert c.prune_mask(max_background_fraction=0.25).tolist() == [True, True, True, False, False, True]
    assert c.prune_mask(max_background_fraction=0).tolist() == [True, True, True, True, False, True]
    assert c.prune_mask(max_background_fraction=1.0).tolist() == base
    assert c.prune_mask(min_pixels=6, max_background_fraction=0.9).tolist() == [True, True, True, False, True, False]
    for bad in (-0.1, 1.5, float("nan"), "0.5", True):
        with pytest.raises(RuntimeError, match="max_background_fraction must be a number in"):
            c.prune_mask(max_background_fraction=bad)
    # four-field construction keeps working
    old = _contrib([1, 2], [0, 0], [1, 1])
    assert not old.silhouettes and old.prune_mask().tolist() == [False, False]


@pytest.mark.parametrize("bad, msg", [
    ("masks_without_words", r"masks need contributions with the background words"),
    ("masks_without_contrib", r"masks need contributions with the background words"),
    ("words_without_masks", r"contributions has the background words \(weight_bg_q, pixels_bg\) but no masks"),
    ("one_word", r"weight_bg_q and contributions.pixels_bg must both be tensors or both None"),
    ("word_dtype", r"contributions.pixels_bg must be a contiguous torch.int64"),
    ("word_P", r"contributions.weight_bg_q must be a contiguous torch.int64 \(P,\) = \(10,\) tensor, got \(11,\)"),
    ("shape", r"masks must be \(T,H,W\) or \(T,1,H,W\) = \(4,24,32\), got \(4, 32, 24\)"),
    ("frames", r"masks must be \(T,H,W\) or \(T,1,H,W\) = \(4,24,32\), got \(3, 24, 32\)"),
    ("channels", r"masks must be \(T,H,W\) or \(T,1,H,W\) = \(4,24,32\), got \(4, 3, 24, 32\)"),
    ("dtype", r"masks must be bool, uint8 or floating point, got torch.int32"),
    ("device", r"masks must be on the rasterizer's device meta, got cpu"),
    ("type", r"masks must be a tensor, got ndarray"),
])
def test_render_frames_rejects_bad_masks_before_any_launch(bad, msg):
    from vidu4d_b200.renderer import PipelineParams, SurfelContributions, render_frames
    dev = "meta" if bad == "device" else "cpu"
    c = SurfelContributions.zeros(10, dev, silhouettes=True)
    masks = torch.ones((4, 24, 32), dtype=torch.bool)
    if bad == "masks_without_words":
        c = SurfelContributions.zeros(10, "cpu")
    elif bad == "masks_without_contrib":
        c = None
    elif bad == "words_without_masks":
        masks = None
    elif bad == "one_word":
        c.pixels_bg = None
    elif bad == "word_dtype":
        c.pixels_bg = torch.zeros(10, dtype=torch.int32)
    elif bad == "word_P":
        c.weight_bg_q = torch.zeros(11, dtype=torch.int64)
    elif bad == "shape":
        masks = torch.ones((4, 32, 24), dtype=torch.bool)
    elif bad == "frames":
        masks = torch.ones((3, 24, 32), dtype=torch.bool)
    elif bad == "channels":
        masks = torch.ones((4, 3, 24, 32))
    elif bad == "dtype":
        masks = torch.ones((4, 24, 32), dtype=torch.int32)
    elif bad == "type":
        masks = np.ones((4, 24, 32), dtype=bool)
    with pytest.raises(RuntimeError, match=msg):
        render_frames(_cams(4), _PC(10, dev=dev), PipelineParams(), torch.zeros(3), contributions=c, masks=masks)


def test_mask_conversion():
    """bool and uint8 pass as bytes (nonzero = foreground), floats are foreground where > 0.5; (T,1,H,W) is (T,H,W)."""
    from vidu4d_b200.renderer import _silhouette_masks
    g = torch.Generator().manual_seed(0)
    f = torch.rand((3, 1, 5, 7), generator=g)
    f[0, 0, 0, :3] = torch.tensor([0.5, 0.5000001, 1.0])
    got = _silhouette_masks(f, 3, 5, 7, "cpu")
    assert got.dtype == torch.uint8 and got.shape == (3, 5, 7) and got.is_contiguous()
    assert torch.equal(got.bool(), (f > 0.5).reshape(3, 5, 7)) and got[0, 0, :3].tolist() == [0, 1, 1]
    u = (torch.rand((3, 5, 7), generator=g) * 4).to(torch.uint8)
    assert torch.equal(_silhouette_masks(u, 3, 5, 7, "cpu"), u)
    b = u > 1
    assert torch.equal(_silhouette_masks(b, 3, 5, 7, "cpu"), b.to(torch.uint8))
    # a strided mask is made contiguous
    s = torch.ones((3, 5, 14), dtype=torch.bool)[:, :, ::2]
    assert _silhouette_masks(s, 3, 5, 7, "cpu").is_contiguous()


def test_prune_by_contribution_background_fraction(monkeypatch):
    """The fraction reaches the mask, None leaves today's decision, and without the background words a fraction is
    refused."""
    from vidu4d_b200.surfel_store import FlatSurfelModel
    from .test_contrib_cpu import _cpu_store
    m = _cpu_store(5)
    seen = []
    monkeypatch.setattr(FlatSurfelModel, "prune_points", lambda self, mask: seen.append(mask.clone()))
    c = _contrib([0, 2 ** 32, 2 ** 32, 2 ** 32, 2 ** 32], [0] * 5, [0, 4, 4, 4, 4],
                 [0, 0, 2 ** 31, 2 ** 31 + 1, 2 ** 32], [0, 0, 2, 2, 4])
    assert m.prune_by_contribution(c) == 1 and seen[-1].tolist() == [True, False, False, False, False]
    assert m.prune_by_contribution(c, max_background_fraction=0.5) == 3
    assert seen[-1].tolist() == [True, False, False, True, True]
    n = len(seen)
    assert m.prune_by_contribution(c, min_pixels=0, max_background_fraction=1.0) == 0 and len(seen) == n
    with pytest.raises(RuntimeError, match="background_fraction needs the background words"):
        m.prune_by_contribution(_contrib([1] * 5, [1] * 5, [1] * 5), max_background_fraction=0.5)


def _synthetic(rank, P=1000, silhouettes=True):
    rng = np.random.default_rng(200 + rank)
    wq = rng.integers(0, 2 ** 52, P, dtype=np.int64)
    mw = (rng.random(P, dtype=np.float32) * 0.99).view(np.int32)
    px = rng.integers(0, 2 ** 40, P, dtype=np.int64)
    wbg = (wq // rng.integers(1, 9, P)).astype(np.int64) if silhouettes else None
    pbg = (px // rng.integers(1, 9, P)).astype(np.int64) if silhouettes else None
    c = _contrib(wq, mw, px, wbg, pbg)
    c.frames = torch.from_numpy(rng.integers(0, 1000, P, dtype=np.int64))
    return c


_NAMES = ("weight_q", "max_weight", "pixels", "frames", "weight_bg_q", "pixels_bg")


def _worker(rank, world, port, out):
    sys.path.insert(0, ROOT)
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1",
                      MASTER_PORT=str(port))
    import torch.distributed as dist
    from vidu4d_b200 import distributed as D
    D.init_distributed("gloo")
    c = _synthetic(rank)
    assert D.allreduce_contributions(c) is c
    D.check_replicas({k: getattr(c, k) for k in _NAMES})
    plain = _synthetic(rank, silhouettes=False)
    D.allreduce_contributions(plain)
    assert plain.weight_bg_q is None and plain.pixels_bg is None
    torch.save({"sil": {k: getattr(c, k) for k in _NAMES},
                "plain": {k: getattr(plain, k) for k in _NAMES[:4]}}, f"{out}.{rank}")
    dist.destroy_process_group()


def test_allreduce_sums_the_background_words_over_two_gloo_ranks(tmp_path):
    """The background words are summed like weight_q and pixels; the four older words reduce as they did, with and
    without the background words present."""
    import socket
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    out = str(tmp_path / "c")
    mp.start_processes(_worker, args=(2, port, out), nprocs=2, join=True, start_method="spawn")
    got = [torch.load(f"{out}.{r}") for r in range(2)]
    for sil in (True, False):
        a, b = _synthetic(0, silhouettes=sil), _synthetic(1, silhouettes=sil)
        want = {"weight_q": a.weight_q + b.weight_q, "pixels": a.pixels + b.pixels, "frames": a.frames + b.frames,
                "max_weight": torch.maximum(a.max_weight, b.max_weight)}
        if sil:
            want.update(weight_bg_q=a.weight_bg_q + b.weight_bg_q, pixels_bg=a.pixels_bg + b.pixels_bg)
        for r in range(2):
            for k, v in want.items():
                assert torch.equal(got[r]["sil" if sil else "plain"][k], v), (sil, r, k)
