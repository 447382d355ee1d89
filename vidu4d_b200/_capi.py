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

SYMBOLS = (
    "sr_geom_bytes", "sr_image_bytes", "sr_binning_bytes", "sr_forward", "sr_backward",
    "sr_mark_visible", "sr_debug_view", "sr_abi_version", "sr_last_error", "sr_launch_count",
    "sr_set_profiling", "sr_get_profile", "sr_post_forward", "sr_post_backward", "sr_render_loss_batch", "sr_bob_warp_table_floats", "sr_bob_warp_forward", "sr_bob_warp_backward", "sr_adam_flat", "sr_surfel_compact", "sr_knn_cells", "sr_knn_mean_dist2",
    "sr_feature_loss_batch", "sr_global_match_forward", "sr_global_match_backward", "sr_reproj_loss_forward", "sr_reproj_loss_backward",
    "sr_cycle_loss_table_floats", "sr_cycle_loss_forward", "sr_cycle_loss_backward",
    "sr_radius_outlier_scratch_bytes", "sr_radius_outlier_mask", "sr_feature_rows_forward", "sr_feature_rows_backward",
)
FEATURES_MAX = 32          # channels per call (SR_FEAT_MAX)


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
    for s in SYMBOLS:
        if not hasattr(lib, s):
            raise SurfelRasterError(f"{LIB_PATH} does not export {s}")
    vp, i32, i64, f32p = C.c_void_p, C.c_int32, C.c_int64, C.c_void_p
    lib.sr_abi_version.restype = C.c_int
    lib.sr_last_error.restype = C.c_char_p
    lib.sr_launch_count.restype = C.c_uint64
    lib.sr_geom_bytes.restype = C.c_size_t
    lib.sr_geom_bytes.argtypes = [i32]
    lib.sr_image_bytes.restype = C.c_size_t
    lib.sr_image_bytes.argtypes = [i32, i32]
    lib.sr_binning_bytes.restype = C.c_size_t
    lib.sr_binning_bytes.argtypes = [i64, i32, i32]
    lib.sr_forward.restype = C.c_int
    lib.sr_forward.argtypes = ([C.POINTER(SrFrame), C.POINTER(SrBatch), f32p, i32] + [f32p] * 7 + [i32, i64]
                               + [f32p] * 3 + [vp, i64, vp, i64] + [vp] * 5 + [i64, vp, vp, vp])
    lib.sr_backward.restype = C.c_int
    lib.sr_backward.argtypes = ([C.POINTER(SrFrame), C.POINTER(SrBatch), f32p, i32] + [f32p] * 6 + [i32, i64]
                                + [f32p] * 3 + [vp] + [f32p, i64, f32p, i64] + [f32p] * 3 + [vp] * 3 + [i64]
                                + [f32p] * 9 + [vp])
    lib.sr_mark_visible.restype = C.c_int
    lib.sr_mark_visible.argtypes = [i32, f32p, f32p, f32p, vp, vp]
    lib.sr_debug_view.restype = C.c_int
    lib.sr_debug_view.argtypes = [i32, i32, i32, i64, C.POINTER(SrDebugLayout)]
    lib.sr_post_forward.restype = C.c_int
    lib.sr_post_forward.argtypes = [i32, i32, C.c_float, C.c_float, C.c_float] + [vp] * 10
    lib.sr_post_backward.restype = C.c_int
    lib.sr_post_backward.argtypes = [i32, i32, C.c_float, C.c_float, C.c_float] + [vp] * 12
    lib.sr_render_loss_batch.restype = C.c_int
    lib.sr_render_loss_batch.argtypes = [i32, i32, i32, C.c_float, C.c_float, C.c_float] + [vp] * 8 + [C.c_float] * 4 + [vp] * 6
    lib.sr_feature_loss_batch.restype = C.c_int
    lib.sr_feature_loss_batch.argtypes = [i32] * 6 + [vp] * 10
    lib.sr_bob_warp_table_floats.restype = C.c_size_t
    lib.sr_bob_warp_table_floats.argtypes = [i32, i32]
    lib.sr_bob_warp_forward.restype = C.c_int
    lib.sr_bob_warp_forward.argtypes = [i32, i32, i32] + [vp] * 14
    lib.sr_bob_warp_backward.restype = C.c_int
    lib.sr_bob_warp_backward.argtypes = [i32, i32, i32] + [vp] * 18
    lib.sr_global_match_forward.restype = C.c_int
    lib.sr_global_match_forward.argtypes = [i32] * 6 + [vp] * 10
    lib.sr_global_match_backward.restype = C.c_int
    lib.sr_global_match_backward.argtypes = [i32] * 6 + [vp] * 13
    lib.sr_reproj_loss_forward.restype = C.c_int
    lib.sr_reproj_loss_forward.argtypes = [i32] * 5 + [C.c_float] + [vp] * 20
    lib.sr_reproj_loss_backward.restype = C.c_int
    lib.sr_reproj_loss_backward.argtypes = [i32] * 5 + [vp] * 19
    lib.sr_cycle_loss_table_floats.restype = C.c_size_t
    lib.sr_cycle_loss_table_floats.argtypes = [i32, i32]
    lib.sr_cycle_loss_forward.restype = C.c_int
    lib.sr_cycle_loss_forward.argtypes = [i32] * 3 + [vp] * 16
    lib.sr_cycle_loss_backward.restype = C.c_int
    lib.sr_cycle_loss_backward.argtypes = [i32] * 3 + [vp] * 17
    lib.sr_feature_rows_forward.restype = C.c_int
    lib.sr_feature_rows_forward.argtypes = [i32] * 4 + [vp] * 14
    lib.sr_feature_rows_backward.restype = C.c_int
    lib.sr_feature_rows_backward.argtypes = [i32] * 4 + [vp] * 19
    lib.sr_adam_flat.restype = C.c_int
    lib.sr_adam_flat.argtypes = [i32, vp, vp, C.c_float, C.c_float, C.c_float, i64, C.c_float, vp, vp, vp, vp, vp]
    lib.sr_surfel_compact.restype = C.c_int
    lib.sr_surfel_compact.argtypes = [i32, vp, vp, vp, i32, i32, i32] + [vp] * 12
    lib.sr_knn_cells.restype = C.c_int64
    lib.sr_knn_cells.argtypes = [i32, vp, vp, vp, vp]
    lib.sr_knn_mean_dist2.restype = C.c_int
    lib.sr_knn_mean_dist2.argtypes = [i32, vp, vp, vp, vp, vp, vp]
    lib.sr_radius_outlier_scratch_bytes.restype = C.c_int64
    lib.sr_radius_outlier_scratch_bytes.argtypes = [i32]
    lib.sr_radius_outlier_mask.restype = C.c_int
    lib.sr_radius_outlier_mask.argtypes = [i32, vp, C.c_double, i32, vp, vp, vp, i64, vp]
    lib.sr_set_profiling.restype = None
    lib.sr_set_profiling.argtypes = [C.c_int]
    lib.sr_get_profile.restype = C.c_char_p
    if lib.sr_abi_version() != ABI_VERSION:
        raise SurfelRasterError(f"ABI mismatch: library {lib.sr_abi_version()} != binding {ABI_VERSION}")
    _lib = lib
    return lib


def check(rc: int, what: str):
    if rc != 0:
        msg = load().sr_last_error().decode("utf-8", "replace")
        raise SurfelRasterError(f"{what} failed (code {rc}): {msg}")


def launch_count() -> int:
    return int(load().sr_launch_count())


def set_profiling(on: bool):
    load().sr_set_profiling(1 if on else 0)


def get_profile() -> dict:
    """{"kernel": {"ms": total, "count": n}} since the previous call (synchronises the device)."""
    import json
    return json.loads(load().sr_get_profile().decode())
