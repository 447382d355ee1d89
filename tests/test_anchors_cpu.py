"""CPU tests of pixel anchors and tracking: sr_render_forward_anchors and sr_track_pixels in their headers, the library
and the bindings; every argument check, made before any device work; render_frames' and track_pixels' checks of shapes,
types and combinations; the anchor slot rule; the float64 tracking model on a case with a closed form."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

from .conftest import ROOT
from .test_render_cpu import _PC, _cams, _render_args
from .track_model import slot_rule, slot_rule_sorted, track, within

D = 1 << 20      # placeholder DEVICE pointer: never dereferenced (the calls fail before any device work)


def _protos(header):
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", header)).read(), flags=re.S)
    return hdr, {name: [p.strip() for p in params.split(",")]
                 for name, params in re.findall(r"SR_API\s+[\w\s\*]+?\b(sr_\w+)\s*\(([^)]*)\)", hdr)}


def test_anchor_entry_point_in_header_library_and_binding(built):
    """sr_render_forward_anchors is sr_render_forward's parameter list with `const sr_anchors* anchors` before the
    stream; the binding's struct has the header's five fields in order, with C's padding."""
    from vidu4d_b200 import _capi
    lib = _capi.load()
    assert hasattr(lib, "sr_render_forward_anchors") and "sr_render_forward_anchors" in _capi.RENDER_SYMBOLS
    hdr, protos = _protos("surfel_render.h")
    base, new = protos["sr_render_forward"], protos["sr_render_forward_anchors"]
    assert new[:-2] == base[:-1] and new[-2] == "const sr_anchors* anchors" and new[-1] == "void* stream"
    rt, args = _capi.RENDER_PROTOTYPES["sr_render_forward_anchors"]
    assert rt == C.c_int and args[:-2] == _capi.RENDER_PROTOTYPES["sr_render_forward"][1][:-1]
    assert args[-2:] == [C.c_void_p, C.c_void_p]
    fields = re.search(r"typedef struct sr_anchors \{(.*?)\} sr_anchors;", hdr, flags=re.S).group(1)
    assert [tuple(x.split()) for x in re.findall(r"([\w ]+?\**\s*\w+);", fields)] == [
        ("int32_t", "K"), ("int64_t", "stride"), ("int32_t*", "ids"), ("float*", "weights"), ("float*", "uv")]
    assert [n for n, _ in _capi.SrAnchors._fields_] == ["K", "stride", "ids", "weights", "uv"]
    assert C.sizeof(_capi.SrAnchors) == 40 and _capi.SrAnchors.stride.offset == 8
    assert int(re.search(r"#define SR_ANCHORS_MAX (\d+)", hdr).group(1)) == max(_capi.ANCHOR_SLOTS) == 8


def test_track_header_library_and_binding_agree(built):
    """include/surfel_track.h <-> libsurfel_raster.so <-> _capi.TRACK_PROTOTYPES, kind for kind; the table is disjoint
    from every other table."""
    from vidu4d_b200 import _capi
    lib = _capi.load()
    _, protos = _protos("surfel_track.h")
    assert set(protos) == set(_capi.TRACK_SYMBOLS) == {"sr_track_pixels"}
    kinds = {"int32_t": C.c_int32, "int64_t": C.c_int64, "float": C.c_float}
    for name, params in protos.items():
        assert hasattr(lib, name)
        want = [C.c_void_p if "*" in p else kinds[p.replace("const", "").split()[0]] for p in params]
        assert _capi.TRACK_PROTOTYPES[name] == (C.c_int, want), name
    others = set()
    for t in (_capi.SYMBOLS, _capi.SSIM_SYMBOLS, _capi.OPTIM_SYMBOLS, _capi.SKIN_MLP_SYMBOLS, _capi.MASK_LOSS_SYMBOLS,
              _capi.CAMERA_SYMBOLS, _capi.DET_SYMBOLS, _capi.RENDER_SYMBOLS):
        others |= set(t)
    assert not set(_capi.TRACK_SYMBOLS) & others


@pytest.mark.parametrize("case, msg", [
    ("null", b"anchors is NULL"),
    ("K_0", b"anchors: K must be 1, 2, 4 or 8, got 0"),
    ("K_3", b"anchors: K must be 1, 2, 4 or 8, got 3"),
    ("K_16_P0", b"anchors: K must be 1, 2, 4 or 8, got 16"),
    ("F_1", b"anchors: feature channels cannot be composited in the same call (F must be 0)"),
    ("stride", b"anchors: frame stride must be >= K*H*W elements"),
    ("stride_P0", b"anchors: frame stride must be >= K*H*W elements"),
    ("null_ids", b"anchors: ids / weights / uv pointer is NULL"),
    ("null_weights_P0", b"anchors: ids / weights / uv pointer is NULL"),
    ("null_uv", b"anchors: ids / weights / uv pointer is NULL"),
    ("ids_align", b"anchors: ids / weights / uv must be 4-byte aligned"),
    ("uv_align", b"anchors: ids / weights / uv must be 4-byte aligned"),
    ("null_arena", b"arena is NULL"),
    ("null_frame", b"frame descriptor is NULL"),
])
def test_render_forward_anchors_rejects_bad_arguments(built, case, msg):
    """The anchors' own checks, then sr_render_forward's (it shares them), all before any device work."""
    from vidu4d_b200 import _capi
    lib = _capi.load()
    P = 0 if case.endswith("_P0") else 100
    W, H = 64, 48
    fr = _capi.SrFrame(P, 3, 16, W, H, 0.5, 0.5, 1.0, 0, 0, 0)
    bt = _capi.SrBatch(2, 0, 0, 0, 0, 0, 0, 0)
    an = _capi.SrAnchors(4, 4 * W * H, D, D + 65536, D + 131072)
    kw = {}
    if case.startswith("K_"):
        an.K = int(case.split("_")[1])
    elif case == "F_1":
        kw.update(F=1, features=D, bg_ch=3)
    elif case.startswith("stride"):
        an.stride = 4 * W * H - 1
    elif case == "null_ids":
        an.ids = None
    elif case.startswith("null_weights"):
        an.weights = None
    elif case == "null_uv":
        an.uv = None
    elif case == "ids_align":
        an.ids = D + 2
    elif case == "uv_align":
        an.uv = D + 131073
    elif case == "null_arena":
        kw["arena"] = None
    args = _render_args(fr, bt, **kw)[:-1] + [None if case == "null" else C.byref(an), None]
    if case == "null_frame":
        args[0] = None
    assert lib.sr_render_forward_anchors(*args) == -1
    assert msg in lib.sr_last_error(), (case, lib.sr_last_error())


def _track_args(**kw):
    a = dict(N=5, T=3, S=2, P=100, K=4, W=64, H=48, queries=D, ids=D, w=D, uv=D, stride=4 * 64 * 48, means=D, ms=0,
             scales=D, rots=D, rs=0, vm=D, tx=0.5, ty=0.5, cams=None, depth=None, tol=0.05, xy=D, z=D, vis=D, cov=D)
    a.update(kw)
    return list(a.values()) + [None]


@pytest.mark.parametrize("kw, msg", [
    (dict(N=-1), b"track: N, T, S and P must be >= 0"),
    (dict(T=65536), b"track: T must be <= 65535, got 65536"),
    (dict(K=3), b"track: K must be 1, 2, 4 or 8, got 3"),
    (dict(W=0), b"track: image size must be in [1, 65535]"),
    (dict(stride=4 * 64 * 48 - 1), b"track: anchor frame stride must be >= K*H*W"),
    (dict(ms=299), b"track: means3D frame stride must be 0 or >= 3*P floats"),
    (dict(rs=402), b"track: rotations frame stride must be 0 or a multiple of 4 that is >= 4*P floats"),
    (dict(tol=-1.0), b"track: depth_tolerance must be >= 0"),
    (dict(tx=0.0), b"track: tan_fovx and tan_fovy must be positive without a camera table"),
    (dict(queries=None), b"track: query or output pointer is NULL"),
    (dict(cov=None), b"track: query or output pointer is NULL"),
    (dict(uv=None), b"track: anchor pointer is NULL"),
    (dict(rots=None), b"track: surfel pointer is NULL"),
    (dict(vm=None), b"track: viewmatrix is NULL"),
    (dict(w=D + 2), b"track: float and int32 arrays must be 4-byte aligned"),
    (dict(xy=D + 4), b"track: scales and xy must be 8-byte aligned"),
    (dict(rots=D + 8), b"track: rotations must be 16-byte aligned"),
])
def test_track_pixels_rejects_bad_arguments(built, kw, msg):
    from vidu4d_b200 import _capi
    lib = _capi.load()
    assert lib.sr_track_pixels(*_track_args(**kw)) == -1
    assert msg in lib.sr_last_error(), (kw, lib.sr_last_error())


def test_track_pixels_without_queries_or_targets_launches_nothing(built):
    from vidu4d_b200 import _capi
    lib = _capi.load()
    before = lib.sr_launch_count()
    assert lib.sr_track_pixels(*_track_args(N=0, queries=None, xy=None)) == 0
    assert lib.sr_track_pixels(*_track_args(T=0)) == 0
    assert lib.sr_launch_count() == before


@pytest.mark.parametrize("kw, msg", [
    (dict(anchors=3), r"anchors must be a slot count in \(1, 2, 4, 8\), got 3"),
    (dict(anchors=True), r"anchors must be a slot count in \(1, 2, 4, 8\), got True"),
    (dict(anchors=4.0), r"anchors must be a slot count in \(1, 2, 4, 8\), got 4.0"),
    (dict(anchors=4, features=torch.zeros((10, 4))), "anchors render colour only and gather no statistics: features"),
    (dict(anchors=4, contributions=object()), "anchors render colour only and gather no statistics: contributions"),
    (dict(anchors=4, masks=torch.zeros((4, 24, 32))), "anchors render colour only and gather no statistics: masks"),
    (dict(anchors=4, lift=object()), "anchors render colour only and gather no statistics: lift"),
])
def test_render_frames_rejects_bad_anchor_arguments_before_any_launch(kw, msg):
    from vidu4d_b200.renderer import PipelineParams, render_frames
    with pytest.raises(RuntimeError, match=msg):
        render_frames(_cams(4), _PC(10), PipelineParams(), torch.zeros(3), **kw)


def _anchors(S=2, K=4, H=24, W=32):
    return (torch.zeros((S, K, H, W), dtype=torch.int32), torch.zeros((S, K, H, W)), torch.zeros((S, K, 2, H, W)))


@pytest.mark.parametrize("kw, msg", [
    (dict(anchors=_anchors()[:2]), "anchors must be render_frames' \\(anchor_ids, anchor_weights, anchor_uv\\)"),
    (dict(anchors=(_anchors()[0].float(),) + _anchors()[1:]), "anchor_ids must be an int32 \\(S,K,H,W\\) tensor"),
    (dict(anchors=_anchors(K=3)), r"anchor_ids must have K in \(1, 2, 4, 8\) slots, got 3"),
    (dict(anchors=(_anchors()[0], torch.zeros((2, 4, 24, 31)), _anchors()[2])), "anchor_weights must be a float32"),
    (dict(anchors=_anchors()[:2] + (torch.zeros((2, 4, 24, 32)),)), "anchor_uv must be a float32"),
    (dict(anchors=_anchors()[:2] + (torch.zeros((2, 4, 2, 32, 24)).transpose(3, 4),)), "anchor_uv must be contiguous"),
    (dict(anchors=_anchors(H=20)), "cameras are 32x24, the anchors 32x20"),
    (dict(queries=torch.zeros((5, 3))), r"queries must be an \(N,3\) int32 tensor"),
    (dict(queries=torch.zeros((5, 2), dtype=torch.int32)), r"queries must be an \(N,3\) int32 tensor"),
    (dict(means3D=torch.zeros((3, 10, 3))), r"means3D must be \(T,P,3\) = \(4,10,3\)"),
    (dict(rotations=torch.zeros((4, 10, 3))), r"rotations must be \(T,P,4\) = \(4,10,4\)"),
    (dict(depth=torch.zeros((4, 24, 31))), r"depth must be a float32 \(T,H,W\) = \(4,24,32\) tensor"),
    (dict(depth_tolerance=-0.1), "depth_tolerance must be >= 0"),
])
def test_track_pixels_rejects_malformed_inputs_before_any_launch(kw, msg):
    from vidu4d_b200.tracking import track_pixels
    a = dict(anchors=_anchors(), queries=torch.zeros((5, 3), dtype=torch.int32))
    a.update(kw)
    with pytest.raises(RuntimeError, match=msg):
        track_pixels(a.pop("anchors"), a.pop("queries"), _cams(4), _PC(10), **a)


def test_slot_rule_is_a_stable_descending_sort():
    """The kernel's insertion (a pair enters only above a strictly smaller last slot) keeps the K heaviest pairs sorted
    by weight, the earlier pair first among equal weights: a stable sort on descending weight."""
    rng = np.random.default_rng(0)
    for trial in range(2000):
        n = int(rng.integers(0, 20))
        # few distinct values, so that ties are common
        w = rng.choice(np.array([0.5, 0.25, 0.125, 0.3, 0.01], np.float32), size=n)
        for K in (1, 2, 4, 8):
            assert slot_rule(list(w), K) == slot_rule_sorted(list(w), K), (trial, K, w)
    assert slot_rule([0.5, 0.5, 0.7, 0.5], 2) == [2, 0]
    assert slot_rule([0.1, 0.2, 0.3], 8) == [2, 1, 0]


def test_track_model_moves_with_a_rigid_translation():
    """One surfel facing an identity camera, shifted by (dx, dy) in frame 1: the model's projection moves by the focal
    length times the shift over the depth, within its bound, and its bound is a few units in the last place."""
    W = H = 32
    P = 1
    ids = np.zeros((1, 1, H, W), np.int32)
    w = np.full((1, 1, H, W), 0.5, np.float32)
    uv = np.zeros((1, 1, 2, H, W), np.float32)
    uv[0, 0, 0], uv[0, 0, 1] = 0.25, -0.5
    means = np.array([[[0.0, 0.0, 2.0]], [[0.125, -0.0625, 2.0]]], np.float32)
    rots = np.tile(np.array([1.0, 0.0, 0.0, 0.0], np.float32), (2, P, 1))
    scales = np.array([[0.1, 0.2]], np.float32)
    vms = np.tile(np.eye(4, dtype=np.float32).reshape(16), (2, 1))
    q = np.array([[0, 3, 4], [0, 31, 0]])
    m = track(ids, w, uv, q, means, rots, scales, vms, W, H, tans=(0.5, 0.5))
    f = W / (2 * 0.5)
    for t in range(2):
        X = means[t, 0].astype(np.float64) + np.array([0.25 * float(np.float32(0.1)), -0.5 * float(np.float32(0.2)), 0.0])
        ex, ey = f * X[0] / X[2] + W / 2, f * X[1] / X[2] + H / 2
        assert np.all(np.abs(m["x"].v[:, t] - ex) < 1e-9) and np.all(np.abs(m["y"].v[:, t] - ey) < 1e-9)
        assert np.all(m["x"].b[:, t] * 2.0 ** -24 < 1e-4)
        assert np.all(within(np.float32(m["x"].v[:, t]), m["x"][:, t]))
    assert m["valid"].all() and np.all(m["coverage"].v == 0.5)
