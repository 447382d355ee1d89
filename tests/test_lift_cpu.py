"""CPU tests of lifting per-pixel maps onto the surfels: sr_render_forward_lift's entry in the header, library and
binding, and its argument checks, made before any device work; SurfelLift's scale, mean and checks; render_frames'
checks of lift and values; distributed.allreduce_lift over two gloo ranks."""
import ctypes as C
import math
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


def _header():
    return re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "surfel_render.h")).read(), flags=re.S)


def test_lift_entry_point_in_header_library_and_binding(built):
    """sr_render_forward_lift is sr_render_forward_contrib's parameter list with `const sr_lift* lift` before the stream;
    the binding's struct has the header's six fields in order, with C's padding; the constants agree."""
    from vidu4d_b200 import _capi
    lib = _capi.load()
    assert hasattr(lib, "sr_render_forward_lift") and "sr_render_forward_lift" in _capi.RENDER_SYMBOLS
    hdr = _header()
    protos = {name: [p.strip() for p in params.split(",")]
              for name, params in re.findall(r"SR_API\s+[\w\s\*]+?\b(sr_\w+)\s*\(([^)]*)\)", hdr)}
    base, new = protos["sr_render_forward_contrib"], protos["sr_render_forward_lift"]
    assert new[:-2] == base[:-1] and new[-2] == "const sr_lift* lift" and new[-1] == "void* stream"
    rt, args = _capi.RENDER_PROTOTYPES["sr_render_forward_lift"]
    assert rt == C.c_int and args[:-2] == _capi.RENDER_PROTOTYPES["sr_render_forward_contrib"][1][:-1]
    assert args[-2:] == [C.c_void_p, C.c_void_p]
    fields = re.search(r"typedef struct sr_lift \{(.*?)\} sr_lift;", hdr, flags=re.S).group(1)
    assert [tuple(x.split()) for x in re.findall(r"([\w ]+?\**\s*\w+);", fields)] == [
        ("const", "float*", "values"), ("int32_t", "C"), ("int64_t", "values_stride"), ("int32_t", "scale_log2"),
        ("int64_t*", "sums"), ("uint64_t*", "saturated")]
    assert [n for n, _ in _capi.SrLift._fields_] == ["values", "C", "values_stride", "scale_log2", "sums", "saturated"]
    assert C.sizeof(_capi.SrLift) == 48
    assert [_capi.SrLift.values_stride.offset, _capi.SrLift.sums.offset] == [16, 32]
    consts = dict(re.findall(r"#define (SR_LIFT_\w+) \(?(-?\d+)\)?", hdr))
    assert int(consts["SR_LIFT_MAX_CHANNELS"]) == 32
    assert (int(consts["SR_LIFT_SCALE_MIN"]), int(consts["SR_LIFT_SCALE_MAX"])) == (_capi.LIFT_SCALE_MIN,
                                                                                  _capi.LIFT_SCALE_MAX) == (-64, 64)


def _lift_args(fr, bt, contrib, lift, **kw):
    return _render_args(fr, bt, **kw)[:-1] + [contrib, lift, None]


@pytest.mark.parametrize("case, msg", [
    ("no_contrib", b"a lift needs the contribution statistics (contrib is NULL)"),
    ("no_contrib_P0", b"a lift needs the contribution statistics (contrib is NULL)"),
    ("C_0", b"lift: C must be in [1, 32], got 0"),
    ("C_33", b"lift: C must be in [1, 32], got 33"),
    ("C_33_P0", b"lift: C must be in [1, 32], got 33"),
    ("F_1", b"lift: feature channels cannot be composited in the same call (F must be 0)"),
    ("F_1_P0", b"lift: feature channels cannot be composited in the same call (F must be 0)"),
    ("stride", b"lift: values frame stride must be >= C*H*W floats"),
    ("stride_P0", b"lift: values frame stride must be >= C*H*W floats"),
    ("stride_negative", b"lift: values frame stride must be >= C*H*W floats"),
    ("scale_low", b"lift: scale_log2 must be in [-64, 64], got -65"),
    ("scale_high", b"lift: scale_log2 must be in [-64, 64], got 65"),
    ("scale_high_P0", b"lift: scale_log2 must be in [-64, 64], got 65"),
    ("null_values", b"lift: values / sums / saturated pointer is NULL"),
    ("null_sums", b"lift: values / sums / saturated pointer is NULL"),
    ("null_saturated", b"lift: values / sums / saturated pointer is NULL"),
    ("values_align", b"lift: values must be 4-byte aligned"),
    ("sums_align", b"lift: sums / saturated must be 8-byte aligned"),
    ("saturated_align", b"lift: sums / saturated must be 8-byte aligned"),
    ("null_weight_q", b"contribution statistics pointer is NULL"),
    ("null_arena", b"arena is NULL"),
    ("null_frame", b"frame descriptor is NULL"),
])
def test_render_forward_lift_rejects_bad_arguments(built, case, msg):
    """sr_render_forward_contrib's checks (it shares them) and the lift's own, all before any device work.  The C, F,
    stride and scale checks hold at P = 0 too; the pointers are only checked when there are surfels to add."""
    from vidu4d_b200 import _capi
    lib = _capi.load()
    P = 0 if case.endswith("_P0") else 100
    W, H = 64, 48
    fr = _capi.SrFrame(P, 3, 16, W, H, 0.5, 0.5, 1.0, 0, 0, 0)
    bt = _capi.SrBatch(2, 0, 0, 0, 0, 0, 0, 0)
    ct = _capi.SrContrib(D, D + 4096, D + 8192)
    lf = _capi.SrLift(D + 12288, 7, 7 * W * H, 32, D + 16384, D + 20480)
    contrib, kw = C.byref(ct), {}
    if case.startswith("no_contrib"):
        contrib = None
    elif case == "C_0":
        lf.C = 0
    elif case.startswith("C_33"):
        lf.C = 33
        lf.values_stride = 33 * W * H
    elif case.startswith("F_1"):
        kw.update(F=1, features=D, bg_ch=3)
    elif case.startswith("stride"):
        lf.values_stride = -1 if case == "stride_negative" else 7 * W * H - 1
    elif case == "scale_low":
        lf.scale_log2 = -65
    elif case.startswith("scale_high"):
        lf.scale_log2 = 65
    elif case == "null_values":
        lf.values = None
    elif case == "null_sums":
        lf.sums = None
    elif case == "null_saturated":
        lf.saturated = None
    elif case == "values_align":
        lf.values = D + 12290
    elif case == "sums_align":
        lf.sums = D + 16388
    elif case == "saturated_align":
        lf.saturated = D + 20484
    elif case == "null_weight_q":
        ct.weight_q = None
    elif case == "null_arena":
        kw["arena"] = None
    args = _lift_args(fr, bt, contrib, C.byref(lf), **kw)
    if case == "null_frame":
        args[0] = None
    assert lib.sr_render_forward_lift(*args) == -1
    assert msg in lib.sr_last_error(), (case, lib.sr_last_error())


def test_null_lift_is_the_contrib_call(built):
    """lift = NULL is sr_render_forward_contrib: no lift check runs (it fails here on the arena, the first check it
    reaches), and with contrib NULL as well it is sr_render_forward."""
    from vidu4d_b200 import _capi
    lib = _capi.load()
    fr = _capi.SrFrame(100, 3, 16, 64, 48, 0.5, 0.5, 1.0, 0, 0, 0)
    bt = _capi.SrBatch(2, 0, 0, 0, 0, 0, 0, 0)
    ct = _capi.SrContrib(D, D + 4096, D + 8192)
    for contrib in (C.byref(ct), None):
        assert lib.sr_render_forward_lift(*_lift_args(fr, bt, contrib, None, arena=None)) == -1
        assert b"arena is NULL" in lib.sr_last_error()
    # the lift's extreme scales and C pass its checks
    for c, s in ((1, -64), (32, 64), (8, 0)):
        lf = _capi.SrLift(D, c, c * 64 * 48, s, D, D)
        assert lib.sr_render_forward_lift(*_lift_args(fr, bt, C.byref(ct), C.byref(lf), arena=None)) == -1
        assert b"arena is NULL" in lib.sr_last_error()


@pytest.mark.parametrize("B, s", [
    (1.0, 32), (1, 32), (0.75, 32), (0.5, 33), (0.5000001, 32), (2.0, 31), (2.0000002, 30), (3.0, 30), (255.0, 24),
    (256.0, 24), (257.0, 23), (2.0 ** 96, -64), (2.0 ** -32, 64), (1.5 * 2.0 ** -33, 64), (math.pi, 30),
])
def test_scale_from_value_bound(B, s):
    """s = 32 - ceil(log2 B), exactly: |v| <= B keeps |v| 2^s <= 2^32, and a B one ulp above a power of two takes the
    next smaller scale."""
    from vidu4d_b200.renderer import SurfelLift
    assert SurfelLift.scale_for(B) == s
    assert abs(float(B)) * 2.0 ** s <= 2.0 ** 32 < abs(float(B)) * 2.0 ** (s + 1)
    lf = SurfelLift.zeros(5, 3, "cpu", value_bound=B)
    assert lf.scale_log2 == s and lf.sums.shape == (5, 3) and lf.sums.dtype == torch.int64
    assert lf.saturated.shape == (1,) and lf.saturated.dtype == torch.int64 and lf.P == 5 and lf.C == 3


@pytest.mark.parametrize("B, msg", [
    (0.0, "value_bound must be a finite positive number"), (-1.0, "value_bound must be a finite positive number"),
    (float("inf"), "value_bound must be a finite positive number"),
    (float("nan"), "value_bound must be a finite positive number"), (True, "value_bound must be a finite positive number"),
    ("1", "value_bound must be a finite positive number"),
    (2.0 ** 96 * 1.0000001, r"gives scale_log2 -65, outside \[-64, 64\]"),
    (2.0 ** -33, r"gives scale_log2 65, outside \[-64, 64\]"),
])
def test_scale_rejects_bad_bounds(B, msg):
    from vidu4d_b200.renderer import SurfelLift
    with pytest.raises(RuntimeError, match=msg):
        SurfelLift.scale_for(B)


def test_zeros_rejects_bad_channel_counts():
    from vidu4d_b200.renderer import SurfelLift
    for c in (0, 33, 2.0, True):
        with pytest.raises(RuntimeError, match="C must be an int in"):
            SurfelLift.zeros(4, c, "cpu")


def test_mean():
    """(sums 2^-s) / (weight_q 2^-32) per channel in float64; 0 where weight_q is 0, negative sums stay negative."""
    from vidu4d_b200.renderer import SurfelContributions, SurfelLift
    c = SurfelContributions.zeros(4, "cpu")
    c.weight_q.copy_(torch.tensor([0, 2 ** 32, 2 ** 31, 3 * 2 ** 33]))
    lf = SurfelLift.zeros(4, 2, "cpu", value_bound=4.0)
    assert lf.scale_log2 == 30
    lf.sums.copy_(torch.tensor([[5, -5], [2 ** 30, -(2 ** 29)], [3 * 2 ** 28, 0], [-(2 ** 33), 2 ** 34]]))
    m = lf.mean(c)
    assert m.dtype == torch.float64 and m.shape == (4, 2)
    assert m.tolist() == [[0.0, 0.0], [1.0, -0.5], [1.5, 0.0], [-8 / 6, 16 / 6]]
    with pytest.raises(RuntimeError, match="contributions are for 3 surfels, the lift for 4"):
        lf.mean(SurfelContributions.zeros(3, "cpu"))


@pytest.mark.parametrize("bad, msg", [
    ("not_a_lift", r"lift must be a SurfelLift, got dict"),
    ("no_contrib", r"lift needs contributions: SurfelContributions.zeros\(P, device\)"),
    ("masks", r"lift and masks cannot be combined in one call"),
    ("features", r"lift renders colour only: features must be None"),
    ("no_values", r"lift needs values: the \(T,C,H,W\) maps to lift"),
    ("values_without_lift", r"values are lifted into a SurfelLift"),
    ("sums_dtype", r"lift.sums must be a contiguous torch.int64 \(P,C\) tensor with P = 10"),
    ("sums_P", r"lift.sums must be a contiguous torch.int64 \(P,C\) tensor with P = 10 and 1 <= C <= 32, got \(11, 3\)"),
    ("sums_C", r"lift.sums must be a contiguous torch.int64 \(P,C\) tensor with P = 10 and 1 <= C <= 32, got \(10, 33\)"),
    ("saturated", r"lift.saturated must be a \(1,\) torch.int64 tensor"),
    ("scale", r"lift.scale_log2 must be an int in \[-64, 64\], got 70"),
    ("shape", r"values must be \(T,C,H,W\) = \(4,3,24,32\), got \(4, 24, 32, 3\)"),
    ("frames", r"values must be \(T,C,H,W\) = \(4,3,24,32\), got \(3, 3, 24, 32\)"),
    ("dtype", r"values must be float32, got torch.float64"),
    ("device", r"values must be on the rasterizer's device cpu, got meta"),
    ("strided", r"values must be contiguous; a channels-last \(T,H,W,C\) map passes as maps.permute\(0, 3, 1, 2\)"),
    ("type", r"values must be a tensor, got ndarray"),
])
def test_render_frames_rejects_bad_lift_and_values_before_any_launch(bad, msg):
    from vidu4d_b200.renderer import PipelineParams, SurfelContributions, SurfelLift, render_frames
    T, P, Cn, H, W = 4, 10, 3, 24, 32
    c = SurfelContributions.zeros(P, "cpu")
    lf = SurfelLift.zeros(P, Cn, "cpu")
    values = torch.zeros((T, Cn, H, W))
    kw = {}
    if bad == "not_a_lift":
        lf = {}
    elif bad == "no_contrib":
        c = None
    elif bad == "masks":
        c = SurfelContributions.zeros(P, "cpu", silhouettes=True)
        kw["masks"] = torch.ones((T, H, W), dtype=torch.bool)
    elif bad == "features":
        kw["features"] = torch.zeros((P, 4))
    elif bad == "no_values":
        values = None
    elif bad == "values_without_lift":
        lf = None
    elif bad == "sums_dtype":
        lf.sums = torch.zeros((P, Cn), dtype=torch.int32)
    elif bad == "sums_P":
        lf.sums = torch.zeros((P + 1, Cn), dtype=torch.int64)
    elif bad == "sums_C":
        lf.sums = torch.zeros((P, 33), dtype=torch.int64)
    elif bad == "saturated":
        lf.saturated = torch.zeros((2,), dtype=torch.int64)
    elif bad == "scale":
        lf.scale_log2 = 70
    elif bad == "shape":
        values = torch.zeros((T, H, W, Cn))
    elif bad == "frames":
        values = torch.zeros((T - 1, Cn, H, W))
    elif bad == "dtype":
        values = values.double()
    elif bad == "device":
        values = torch.zeros((T, Cn, H, W), device="meta")
    elif bad == "strided":
        values = torch.zeros((T, H, W, Cn)).permute(0, 3, 1, 2)
    elif bad == "type":
        values = np.zeros((T, Cn, H, W), dtype=np.float32)
    with pytest.raises(RuntimeError, match=msg):
        render_frames(_cams(T), _PC(P), PipelineParams(), torch.zeros(3), contributions=c, lift=lf, values=values, **kw)


def _synthetic(rank, P=1000, Cn=7, s=30):
    from vidu4d_b200.renderer import SurfelLift
    rng = np.random.default_rng(300 + rank)
    return SurfelLift(torch.from_numpy(rng.integers(-2 ** 60, 2 ** 60, (P, Cn), dtype=np.int64)),
                      torch.tensor([int(rng.integers(0, 2 ** 40))], dtype=torch.int64), s)


def _worker(rank, world, port, out):
    sys.path.insert(0, ROOT)
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1",
                      MASTER_PORT=str(port))
    import torch.distributed as dist
    from vidu4d_b200 import distributed as D
    D.init_distributed("gloo")
    lf = _synthetic(rank)
    assert D.allreduce_lift(lf) is lf
    D.check_replicas({"sums": lf.sums, "saturated": lf.saturated})
    bad = _synthetic(rank, s=30 + rank)
    try:
        D.allreduce_lift(bad)
        refused = False
    except RuntimeError as e:
        refused = "lift scales differ across ranks: scale_log2 from 30 to 31" in str(e)
    torch.save({"sums": lf.sums, "saturated": lf.saturated, "refused": refused,
                "untouched": torch.equal(bad.sums, _synthetic(rank, s=30 + rank).sums)}, f"{out}.{rank}")
    dist.destroy_process_group()


def test_allreduce_lift_over_two_gloo_ranks(tmp_path):
    """sums and saturated are summed (int64, wrapping as two's complement does); ranks with different scales are
    refused before anything is summed."""
    import socket
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    out = str(tmp_path / "l")
    mp.start_processes(_worker, args=(2, port, out), nprocs=2, join=True, start_method="spawn")
    got = [torch.load(f"{out}.{r}") for r in range(2)]
    a, b = _synthetic(0), _synthetic(1)
    for r in range(2):
        assert torch.equal(got[r]["sums"], a.sums + b.sums)
        assert torch.equal(got[r]["saturated"], a.saturated + b.saturated)
        assert got[r]["refused"] and got[r]["untouched"]
