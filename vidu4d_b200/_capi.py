"""ctypes binding of vidu4d_b200/lib/libsurfel_raster.so (include/surfel_raster.h).

The CUDA library is the product; there is NO fallback.  If the library is missing or does not
export the declared ABI this module raises at first use -- it never routes to a CPU path.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libsurfel_raster.so")

ABI_VERSION = 10
SR_STATUS_OVERFLOW = 1
SR_STATUS_PREFILTER = 4
SR_BATCH_SUM_SHARED = 1
FEATURES_MAX = 32          # channels per call (SR_FEAT_MAX); also the widest feature row sr_feature_rows_* writes


class SrFrame(C.Structure):
    _fields_ = [
        ("P", C.c_int32), ("sh_degree", C.c_int32), ("sh_coeffs", C.c_int32),
        ("width", C.c_int32), ("height", C.c_int32),
        ("tan_fovx", C.c_float), ("tan_fovy", C.c_float), ("scale_modifier", C.c_float),
        ("prefiltered", C.c_int32), ("debug", C.c_int32), ("flags", C.c_uint32),
    ]


class SrBatch(C.Structure):
    """sr_batch: frames + per-frame strides (in floats; 0 = shared by all frames) of the per-surfel inputs."""
    _fields_ = [("frames", C.c_int32), ("flags", C.c_uint32), ("means3D", C.c_int64), ("shs", C.c_int64), ("colors_precomp", C.c_int64),
                ("opacities", C.c_int64), ("scales", C.c_int64), ("rotations", C.c_int64)]


class SrDebugLayout(C.Structure):
    _fields_ = [
        ("surfel_rec", C.c_size_t), ("depths", C.c_size_t), ("tiles_touched", C.c_size_t),
        ("point_offsets", C.c_size_t), ("clamped", C.c_size_t),
        ("keys", C.c_size_t * 2), ("values", C.c_size_t * 2), ("sort_ctl", C.c_size_t),
        ("inst_rec", C.c_size_t), ("contrib", C.c_size_t),
        ("final_T", C.c_size_t), ("n_contrib", C.c_size_t), ("ranges", C.c_size_t), ("sub_last", C.c_size_t),
    ]


class SurfelRasterError(RuntimeError):
    pass


# restype and argtypes of every entry point, in include/surfel_raster.h's order (tests/test_host_cpu.py checks them against
# the header).  Device pointers are c_void_p; the trailing c_void_p of most entry points is the stream.
_p, _i32, _i64, _f32, _f64 = C.c_void_p, C.c_int32, C.c_int64, C.c_float, C.c_double
_FRAME, _BATCH = C.POINTER(SrFrame), C.POINTER(SrBatch)
PROTOTYPES = {
    "sr_geom_bytes": (C.c_size_t, [_i32]),
    "sr_image_bytes": (C.c_size_t, [_i32, _i32]),
    "sr_binning_bytes": (C.c_size_t, [_i64, _i32, _i32]),
    "sr_forward": (C.c_int, [_FRAME, _BATCH, _p, _i32] + [_p] * 7 + [_i32, _i64] + [_p] * 3 + [_p, _i64, _p, _i64] + [_p] * 5
                   + [_i64, _p, _p, _p]),
    "sr_backward": (C.c_int, [_FRAME, _BATCH, _p, _i32] + [_p] * 6 + [_i32, _i64] + [_p] * 4 + [_p, _i64, _p, _i64] + [_p] * 6
                    + [_i64] + [_p] * 10),
    "sr_mark_visible": (C.c_int, [_i32] + [_p] * 5),
    "sr_debug_view": (C.c_int, [_i32, _i32, _i32, _i64, C.POINTER(SrDebugLayout)]),
    "sr_post_forward": (C.c_int, [_i32, _i32, _f32, _f32, _f32] + [_p] * 10),
    "sr_post_backward": (C.c_int, [_i32, _i32, _f32, _f32, _f32] + [_p] * 12),
    "sr_render_loss_batch": (C.c_int, [_i32, _i32, _i32, _f32, _f32, _f32] + [_p] * 8 + [_f32] * 4 + [_p] * 6),
    "sr_feature_loss_batch": (C.c_int, [_i32] * 6 + [_p] * 10),
    "sr_bob_warp_table_floats": (C.c_size_t, [_i32, _i32]),
    "sr_bob_warp_forward": (C.c_int, [_i32] * 3 + [_p] * 14),
    "sr_bob_warp_backward": (C.c_int, [_i32] * 3 + [_p] * 18),
    "sr_global_match_forward": (C.c_int, [_i32] * 6 + [_p] * 10),
    "sr_global_match_backward": (C.c_int, [_i32] * 6 + [_p] * 13),
    "sr_reproj_loss_forward": (C.c_int, [_i32] * 5 + [_f32] + [_p] * 20),
    "sr_reproj_loss_backward": (C.c_int, [_i32] * 5 + [_p] * 19),
    "sr_cycle_loss_table_floats": (C.c_size_t, [_i32, _i32]),
    "sr_cycle_loss_forward": (C.c_int, [_i32] * 3 + [_p] * 16),
    "sr_cycle_loss_backward": (C.c_int, [_i32] * 3 + [_p] * 17),
    "sr_feature_rows_forward": (C.c_int, [_i32] * 4 + [_p] * 14),
    "sr_feature_rows_backward": (C.c_int, [_i32] * 4 + [_p] * 19),
    "sr_adam_flat": (C.c_int, [_i32, _p, _p, _f32, _f32, _f32, _i64, _f32] + [_p] * 5),
    "sr_surfel_compact": (C.c_int, [_i32, _p, _p, _p, _i32, _i32, _i32] + [_p] * 12),
    "sr_knn_cells": (C.c_int64, [_i32, _p, _p, _p, _p]),
    "sr_knn_mean_dist2": (C.c_int, [_i32] + [_p] * 6),
    "sr_radius_outlier_scratch_bytes": (C.c_int64, [_i32]),
    "sr_radius_outlier_mask": (C.c_int, [_i32, _p, _f64, _i32, _p, _p, _p, _i64, _p]),
    "sr_abi_version": (C.c_int, []),
    "sr_last_error": (C.c_char_p, []),
    "sr_launch_count": (C.c_uint64, []),
    "sr_set_profiling": (None, [C.c_int]),
    "sr_get_profile": (C.c_char_p, []),
}
SYMBOLS = tuple(PROTOTYPES)

# the fused SSIM loss, declared in include/surfel_ssim.h: same library, same error path, its own header (and so its own
# table) because surfel_raster.h is the rasterizer's drop-in boundary
SSIM_PROTOTYPES = {
    "sr_ssim_scratch_bytes": (C.c_int64, [_i32] * 4),
    "sr_ssim_forward": (C.c_int, [_i32] * 4 + [_p] * 3 + [_i64] + [_p] * 5 + [_i64, _p]),
    "sr_ssim_backward": (C.c_int, [_i32] * 4 + [_p] * 3 + [_i64] + [_p] * 3 + [_i32, _p, _i32] + [_p] * 3 + [_i64, _p]),
}
SSIM_SYMBOLS = tuple(SSIM_PROTOTYPES)

# gradient-norm clipping and the Adam step with its state on the device, declared in include/surfel_optim.h (own header
# and table for the same reason)
OPTIM_PROTOTYPES = {
    "sr_grad_norm_scratch_bytes": (C.c_int64, [_i32]),
    "sr_grad_norm_flat": (C.c_int, [_i32, _p, _p, _f32, _p, _i32, _f32] + [_p] * 4 + [_i64, _p]),
    "sr_adam_flat_state": (C.c_int, [_i32, _p, _p, _f32, _f32, _f32, _p, _f32] + [_p] * 6),
}
OPTIM_SYMBOLS = tuple(OPTIM_PROTOTYPES)

# the fused delta-skinning MLP, declared in include/surfel_skin_mlp.h (own header and table for the same reason)
SKIN_MLP_PROTOTYPES = {
    "sr_delta_skin_scratch_bytes": (C.c_int64, [_i32] * 3),
    "sr_delta_skin_forward": (C.c_int, [_i32] * 6 + [_p] * 8),
    "sr_delta_skin_backward": (C.c_int, [_i32] * 6 + [_p] * 14 + [_i64, _p]),
}
SKIN_MLP_SYMBOLS = tuple(SKIN_MLP_PROTOTYPES)

# Stage 3's silhouette loss with the reference's balance weights, declared in include/surfel_mask_loss.h (own header and
# table for the same reason)
MASK_LOSS_PROTOTYPES = {
    "sr_mask_loss_scratch_bytes": (C.c_int64, [_i32] * 3),
    "sr_mask_loss_batch": (C.c_int, [_i32] * 3 + [_p, _i64] + [_p] * 9 + [_i64, _p]),
}
MASK_LOSS_SYMBOLS = tuple(MASK_LOSS_PROTOTYPES)


_lib = None


def load():
    """Load the CUDA library; raise loudly if it is absent (run `python -m vidu4d_b200.build`)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise SurfelRasterError(
            f"{LIB_PATH} not found: the CUDA extension is not built. Run `python -m vidu4d_b200.build` "
            "(or __graft_entry__.build()). There is no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    for s in SYMBOLS + SSIM_SYMBOLS + OPTIM_SYMBOLS + SKIN_MLP_SYMBOLS + MASK_LOSS_SYMBOLS:
        if not hasattr(lib, s):
            raise SurfelRasterError(f"{LIB_PATH} does not export {s}")
    for name, (restype, argtypes) in (list(PROTOTYPES.items()) + list(SSIM_PROTOTYPES.items()) + list(OPTIM_PROTOTYPES.items())
                                      + list(SKIN_MLP_PROTOTYPES.items()) + list(MASK_LOSS_PROTOTYPES.items())):
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = restype, argtypes
    if lib.sr_abi_version() != ABI_VERSION:
        raise SurfelRasterError(f"ABI mismatch: library {lib.sr_abi_version()} != binding {ABI_VERSION}")
    _lib = lib
    return lib


def check(rc: int, what: str):
    if rc != 0:
        msg = load().sr_last_error().decode("utf-8", "replace")
        raise SurfelRasterError(f"{what} failed (code {rc}): {msg}")


def call(name: str, device, *args):
    """Run entry point `name` on `device`'s current stream, which is passed as the last argument.  A tensor argument
    passes as its data_ptr(); ints, floats, None (NULL) and ctypes objects pass unchanged.  Raises SurfelRasterError
    with the library's message if the call fails."""
    import torch
    fn = getattr(load(), name)
    args = [a.data_ptr() if isinstance(a, torch.Tensor) else a for a in args]
    with torch.cuda.device(device):
        check(fn(*args, torch.cuda.current_stream(device).cuda_stream), name)


def check_tensors(named, ref_name: str, ref, floats=None):
    """Raise RuntimeError unless every tensor of `floats` ((name, tensor) pairs; default `named`) is float32 and every
    tensor of `named` is a CUDA tensor on `ref`'s device."""
    import torch
    for name, t in named if floats is None else floats:
        if t.dtype != torch.float32:
            raise RuntimeError(f"{name} must be float32, got {t.dtype}")
    for name, t in named:
        if not t.is_cuda:
            raise RuntimeError(f"{name} must be a CUDA tensor (there is no CPU fallback)")
        if t.device != ref.device:
            raise RuntimeError(f"{name} is on {t.device}, {ref_name} on {ref.device}")


def launch_count() -> int:
    return int(load().sr_launch_count())


def set_profiling(on: bool):
    load().sr_set_profiling(1 if on else 0)


def get_profile() -> dict:
    """{"kernel": {"ms": total, "count": n}} since the previous call (synchronises the device)."""
    import json
    return json.loads(load().sr_get_profile().decode())
