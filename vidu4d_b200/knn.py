"""`distCUDA2` of the reference's simple-knn submodule (gs/submodules/simple-knn/simple_knn.cu, ext.cpp): mean squared
distance of every point to its three nearest neighbours, used once to initialise the surfel scales
(gs/scene/gaussian_model.py:139-140: `scales = log(sqrt(clamp_min(distCUDA2(points), 1e-7)))`).

`radius_outlier_mask`: the fixed-radius neighbour count behind Stage 3's periodic outlier filter."""
from __future__ import annotations

import ctypes as C

import torch

from . import _capi


def distCUDA2(points: torch.Tensor) -> torch.Tensor:
    """points (P,3) float32 CUDA tensor -> (P,) float32: (d0 + d1 + d2) / 3 over the three nearest OTHER points."""
    lib = _capi.load()
    if not points.is_cuda:
        raise RuntimeError("points must be a CUDA tensor")      # the reference's extension has no CPU path either
    pts = points.detach().to(torch.float32).contiguous()
    P = int(pts.shape[0])
    out = torch.empty((P,), dtype=torch.float32, device=pts.device)
    if P == 0:
        return out
    lo, hi = pts.amin(0).cpu(), pts.amax(0).cpu()                # one host sync: this is an initialisation-time routine
    bmin = (C.c_float * 3)(*[float(v) for v in lo]); bmax = (C.c_float * 3)(*[float(v) for v in hi])
    cells = int(lib.sr_knn_cells(P, bmin, bmax, None, None))
    scratch = torch.empty((2 * P + 3 * cells,), dtype=torch.int32, device=pts.device)
    _capi.call("sr_knn_mean_dist2", pts.device, P, pts, bmin, bmax, out, scratch)
    return out


def radius_outlier_mask(points: torch.Tensor, nb_points: int = 20, radius: float = 0.004, return_counts: bool = False):
    """Stage 3's `pcd.remove_radius_outlier(nb_points, radius)` (lab4d/engine/trainer.py:573-588) on the device.

    points (P,3) CUDA tensor (any layout; converted to contiguous float32) -> (P,) bool PRUNE mask, True where fewer than
    nb_points + 1 points, the point itself included, lie strictly closer than `radius` (float64 distances; see
    sr_radius_outlier_mask in include/surfel_raster.h).  With return_counts, also the (P,) int32 counts capped at
    nb_points + 1.  Runs on torch's current stream without a host synchronisation, so it can be captured in a CUDA graph."""
    lib = _capi.load()
    if not points.is_cuda:
        raise RuntimeError("points must be a CUDA tensor")
    if points.dim() != 2 or points.shape[1] != 3:
        raise ValueError(f"points must be (P,3), got {tuple(points.shape)}")
    pts = points.detach().to(torch.float32).contiguous()
    P = int(pts.shape[0])
    keep = torch.empty((P,), dtype=torch.uint8, device=pts.device)
    counts = torch.empty((P,), dtype=torch.int32, device=pts.device) if return_counts else None
    nbytes = int(lib.sr_radius_outlier_scratch_bytes(P))
    scratch = torch.empty((max(nbytes, 1),), dtype=torch.uint8, device=pts.device)
    _capi.call("sr_radius_outlier_mask", pts.device, P, pts, float(radius), int(nb_points), keep, counts, scratch, nbytes)
    prune = keep == 0
    return (prune, counts) if return_counts else prune
