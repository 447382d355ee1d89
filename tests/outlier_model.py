"""Float64 model of the radius outlier filter (csrc/outlier.cu, include/surfel_raster.h sr_radius_outlier_mask):

    count_i = #{ j : d2(i,j) < r2 }, j = i included,  d2 = ((xi-xj)^2 + (yi-yj)^2) + (zi-zj)^2,  r2 = r * r,

every coordinate a float32 widened to float64 and every difference, product and sum rounded on its own (numpy's
elementwise operations are single IEEE operations, never fused).  A point is kept iff count > nb_points.  No fixture of
the reference exists for this op (its Open3D call cannot run here), so this model is the oracle."""
import numpy as np


def radius_counts(points, radius: float, chunk: int = 1024) -> np.ndarray:
    """(P,) int64 exact counts, brute force over all pairs in row chunks."""
    x = np.asarray(points, dtype=np.float32).astype(np.float64)
    r2 = float(radius) * float(radius)
    P = x.shape[0]
    out = np.zeros((P,), dtype=np.int64)
    with np.errstate(invalid="ignore", over="ignore"):
        for s in range(0, P, chunk):
            a = x[s:s + chunk]
            acc = a[:, None, 0] - x[None, :, 0]
            acc = acc * acc
            t = a[:, None, 1] - x[None, :, 1]
            acc = acc + t * t
            t = a[:, None, 2] - x[None, :, 2]
            acc = acc + t * t
            out[s:s + chunk] = (acc < r2).sum(1)
    return out


def keep_and_capped(counts: np.ndarray, nb_points: int):
    """keep mask (count > nb_points) and the counts capped at nb_points + 1, as the kernel reports them."""
    return counts > nb_points, np.minimum(counts, nb_points + 1).astype(np.int32)
