"""CPU tests of forward-only rendering (include/surfel_render.h): the header, library and binding agree; every entry point
rejects bad arguments with its own message before any device work; the arena is sr_forward's three buffers less exactly
the arrays only a backward reads; render_frames rejects malformed shapes before any launch."""
import ctypes as C
import os
import re

import pytest
import torch

from .conftest import ROOT

D = 1 << 20      # placeholder DEVICE pointer: never dereferenced (the calls fail before any device work)


def test_render_header_library_and_binding_agree(built):
    """include/surfel_render.h <-> libsurfel_raster.so <-> _capi.RENDER_PROTOTYPES, kind for kind; the table is disjoint
    from every other table; SR_ABI_VERSION is unchanged."""
    from vidu4d_b200 import _capi
    lib = _capi.load()
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "surfel_render.h")).read(), flags=re.S)
    protos = re.findall(r"SR_API\s+([\w\s\*]+?)\b(sr_\w+)\s*\(([^)]*)\)", hdr)
    assert {name for _, name, _ in protos} == set(_capi.RENDER_SYMBOLS)
    kinds = {"int32_t": C.c_int32, "int64_t": C.c_int64, "float": C.c_float}
    rets = {"int": C.c_int, "size_t": C.c_size_t}
    frame, batch = C.POINTER(_capi.SrFrame), C.POINTER(_capi.SrBatch)
    for ret, name, params in protos:
        assert hasattr(lib, name)
        want = []
        for p in params.split(","):
            p = p.replace("const", "").strip()
            want.append(frame if p.startswith("sr_frame") else batch if p.startswith("sr_batch")
                        else C.c_void_p if "*" in p else kinds[p.split()[0]])
        assert _capi.RENDER_PROTOTYPES[name] == (rets[ret.strip()], want), name
    others = set()
    for t in (_capi.SYMBOLS, _capi.SSIM_SYMBOLS, _capi.OPTIM_SYMBOLS, _capi.SKIN_MLP_SYMBOLS, _capi.MASK_LOSS_SYMBOLS,
              _capi.CAMERA_SYMBOLS, _capi.DET_SYMBOLS):
        others |= set(t)
    assert not set(_capi.RENDER_SYMBOLS) & others
    raster = open(os.path.join(ROOT, "include", "surfel_raster.h")).read()
    assert lib.sr_abi_version() == _capi.ABI_VERSION == int(re.search(r"#define SR_ABI_VERSION (\d+)", raster).group(1)) == 12


def _render_args(fr, bt, bg_ch=3, F=0, features=None, rot=D, scales=D, shs=None, colors=D, arena=D, cap=4096, cstride=0):
    return [C.byref(fr), C.byref(bt), D, bg_ch, D, shs, colors, D, scales, rot, features, F, 0, D, D, D, D, cstride,
            D if F else None, 0, D, D, arena, cap, D, None, None]


def _post_args(M=2, bkgd=None, color=None, color_stride=0, allmap=D):
    return [M, 64, 48, 0.5, 0.5, None, 0.0, allmap, D, bkgd, color, color_stride] + [D] * 7 + [None]


@pytest.mark.parametrize("case, msg", [
    ("null_arena", b"arena is NULL"),
    ("misaligned_arena", b"arena must be 16-byte aligned"),
    ("null_means", b"surfel attribute pointer is NULL"),
    ("null_outputs", b"output pointer is NULL"),
    ("F_33", b"F must be in [1, 32], got 33"),
    ("F_neg", b"F must be in [1, 32], got -1"),
    ("features_without_F", b"got 0"),
    ("bg_F", b"background must have 3 or 3+F = 7 channels, got 5"),
    ("bg_F0", b"background must have 3 channels when F = 0, got 4"),
    ("rotations", b"rotations / shs must be 16-byte aligned"),
    ("scales", b"scales 8-byte aligned"),
    ("shs", b"rotations / shs must be 16-byte aligned"),
    ("capacity_0", b"capacity must be in (0, 2^30)"),
    ("capacity_big", b"capacity must be in (0, 2^30)"),
    ("frames_0", b"frames must be in [1, 65535]"),
])
def test_render_forward_rejects_bad_arguments(built, case, msg):
    from vidu4d_b200 import _capi
    lib = _capi.load()
    fr = _capi.SrFrame(100, 3, 16, 64, 48, 0.5, 0.5, 1.0, 0, 0, 0)
    bt = _capi.SrBatch(2, 0, 0, 0, 0, 0, 0, 0)
    kw = {}
    if case == "null_arena":
        kw["arena"] = None
    elif case == "misaligned_arena":
        kw["arena"] = D + 8
    elif case == "F_33":
        kw.update(F=33, features=D, bg_ch=36)
    elif case == "F_neg":
        kw.update(F=-1, features=D)
    elif case == "features_without_F":
        kw.update(features=D)
    elif case == "bg_F":
        kw.update(F=4, features=D, bg_ch=5, cstride=7 * 64 * 48)
    elif case == "bg_F0":
        kw.update(bg_ch=4)
    elif case == "rotations":
        kw["rot"] = D + 4
    elif case == "scales":
        kw["scales"] = D + 4
    elif case == "shs":
        kw.update(shs=D + 4, colors=None)
    elif case == "capacity_0":
        kw["cap"] = 0
    elif case == "capacity_big":
        kw["cap"] = 1 << 30
    elif case == "frames_0":
        bt = _capi.SrBatch(0, 0, 0, 0, 0, 0, 0, 0)
    args = _render_args(fr, bt, **kw)
    if case == "null_means":
        args[4] = None
    if case == "null_outputs":
        args[16] = None
    if case == "shs":
        fr.sh_coeffs = 16
    assert lib.sr_render_forward(*args) == -1
    assert msg in lib.sr_last_error(), (case, lib.sr_last_error())
    assert lib.sr_render_forward(None, C.byref(bt), *_render_args(fr, bt)[2:]) == -1
    assert b"frame descriptor is NULL" in lib.sr_last_error()


@pytest.mark.parametrize("case, msg", [
    ("M_0", b"M must be in [1, 65535], got 0"),
    ("M_neg", b"M must be in [1, 65535], got -3"),
    ("null_allmap", b"sr_post_forward_frames: a required pointer is NULL"),
    ("bkgd_without_color", b"learnable_bkgd is given but color is NULL"),
    ("color_stride", b"color frame stride must be >= 3*H*W"),
])
def test_post_forward_frames_rejects_bad_arguments(built, case, msg):
    from vidu4d_b200 import _capi
    lib = _capi.load()
    kw = {"M_0": dict(M=0), "M_neg": dict(M=-3), "null_allmap": dict(allmap=None), "bkgd_without_color": dict(bkgd=D),
          "color_stride": dict(bkgd=D, color=D, color_stride=3 * 64 * 48 - 1)}[case]
    assert lib.sr_post_forward_frames(*_post_args(**kw)) == -1
    assert msg in lib.sr_last_error(), (case, lib.sr_last_error())


@pytest.mark.parametrize("P, cap, W, H", [(0, 256, 16, 16), (1, 4096, 75, 53), (1000, 8192, 80, 48),
                                          (300_000, 1_200_128, 512, 512), (12_345, 99_840, 128, 128)])
def test_render_bytes_is_the_three_buffers_less_the_backward_state(built, P, cap, W, H):
    """sr_render_bytes = sr_geom_bytes + sr_binning_bytes + sr_image_bytes less exactly: the geometry's gradient
    accumulator (80 B per surfel, its last array), the binning's contribution masks, and the image's final_T, n_contrib and
    sub_last -- each measured between the offsets sr_debug_view reports."""
    from vidu4d_b200 import _capi
    lib = _capi.load()
    L = _capi.SrDebugLayout()
    assert lib.sr_debug_view(P, W, H, cap, C.byref(L)) == 0
    align = lambda x: (x + 255) // 256 * 256  # noqa: E731
    sgrad = align(max(P, 1) * 80)
    contrib = L.sort_ctl - L.contrib
    final_T, n_contrib, sub_last = L.n_contrib - L.final_T, L.ranges - L.n_contrib, L.tile_order - L.sub_last
    assert contrib > 0 and final_T == align(3 * W * H * 4) and n_contrib == align(2 * W * H * 4) and sub_last > 0
    full = lib.sr_geom_bytes(P) + lib.sr_binning_bytes(cap, W, H) + lib.sr_image_bytes(W, H)
    assert lib.sr_render_bytes(P, cap, W, H) == full - sgrad - contrib - final_T - n_contrib - sub_last


class _PC:
    def __init__(self, P, dev="cpu"):
        self.get_xyz = torch.zeros((P, 3), device=dev)
        self.get_rotation = torch.zeros((P, 4), device=dev)
        self.get_scaling = torch.zeros((P, 2), device=dev)
        self.get_opacity = torch.zeros((P, 1), device=dev)
        self.get_features = torch.zeros((P, 1, 3), device=dev)
        self.active_sh_degree = 0


def _cams(T, W=32, H=24, intrinsics=None):
    from vidu4d_b200.renderer import BatchCameras
    eye = torch.eye(4).expand(T, 4, 4).contiguous()
    return BatchCameras(W, H, 1.0, 1.0, eye, eye, torch.zeros((T, 3)), intrinsics)


@pytest.mark.parametrize("kw, msg", [
    (dict(frames_per_call=0), "frames_per_call must be an int >= 1"),
    (dict(frames_per_call=2.0), "frames_per_call must be an int >= 1"),
    (dict(means3D=torch.zeros((3, 10, 3))), r"means3D must be \(T,P,3\) = \(4,10,3\)"),
    (dict(rotations=torch.zeros((4, 10, 3))), r"rotations must be \(T,P,4\) = \(4,10,4\)"),
    (dict(features=torch.zeros((10, 33))), "features must have 1..32 channels"),
    (dict(features=torch.zeros((11, 4))), r"features must have dimensions \(P,F\) or \(M,P,F\) with P = 10"),
    (dict(features=torch.zeros((3, 10, 4))), r"features must be \(P,F\) or \(T,P,F\) with T = 4"),
    (dict(features=torch.zeros((10, 4)), bg_color=torch.zeros(5)), "background must have 3 or 3\\+F = 7 values"),
    (dict(bg_color=torch.zeros(4)), "bg_color must have 3 values without features"),
    (dict(learnable_bkgd=torch.zeros(4)), "learnable_bkgd must have 3 elements"),
    (dict(learnable_bkgd=torch.zeros(3)), "learnable_bkgd must be a CUDA tensor"),
    (dict(intrinsics=torch.zeros((3, 4))), r"intrinsics must be a float32 \(M,4\) = \(4, 4\)"),
])
def test_render_frames_rejects_malformed_shapes_before_any_launch(kw, msg):
    """Every check runs on the host before a kernel is queued, so these CPU tensors never reach the library."""
    from vidu4d_b200.renderer import PipelineParams, render_frames
    intr = kw.pop("intrinsics", None)
    bg = kw.pop("bg_color", torch.zeros(3))
    with pytest.raises(RuntimeError, match=msg):
        render_frames(_cams(4, intrinsics=intr), _PC(10), PipelineParams(), bg, **kw)
