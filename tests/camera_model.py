"""TEST INFRASTRUCTURE -- per-frame principal-point offsets (include/surfel_camera.h) on top of the centred oracles.

The CPU oracles (oracle/surfel_oracle.c, oracle/post_oracle.py) put the principal point at the image centre, as the
reference does.  An offset (ox, oy) enters the rasterizer linearly, in two places only, so the centred oracles give it
exactly, with no restatement of their arithmetic:

  * forward: T = (K [M0 M1 p_view])^T, whose first two rows get cx * (third row); moving cx by ox adds ox * T_w to
    T_u, and oy * T_w to T_v (T_w = the third row, unchanged).  The AABB centre moves by (ox, oy).  The composite reads
    only T and pixel coordinates, so it needs no change at all: the oracle composites from the GPU's own records.
  * backward: dL/dM = K^T dT, whose z component gets cx * dT_u + cy * dT_v + dT_w.  Moving (cx, cy) by (ox, oy) is
    therefore the same as adding ox * dT_u + oy * dT_v to dT_w, where dT is the transMat gradient after the AABB vjp,
    which only ADDS to the accumulator (surfel_oracle.c chain_one).  So the offset chain is the centred chain run on
    accumulators whose dT_w slots carry that sum.  dL/dtransMat itself (before K^T) and the mean2D proxy (a W/2 scale
    of dT_u, dT_v) do not depend on the offset.
  * the loss pass: depth_to_normal's ray grid, K^-1 (x, y, 1) with K's principal point at (W/2 + ox, H/2 + oy).
"""
import numpy as np

from oracle import post_oracle as po
from oracle import surfel_oracle as so

_TW = slice(so.ACC_T + 6, so.ACC_T + 9)


def offset_records(st, ox, oy):
    """(P,9) transMat and (P,2) AABB centres of the centred forward state st with the principal point moved by (ox, oy),
    float64 (the kernel rounds each of its own operations; compare with a rounding tolerance)."""
    T = st.transMat.reshape(-1, 9).astype(np.float64)
    T[:, 0:3] += ox * T[:, 6:9]
    T[:, 3:6] += oy * T[:, 6:9]
    return T, st.means2D.reshape(-1, 2).astype(np.float64) + np.array([ox, oy])


def offset_chain(st, acc, tm, ox, oy):
    """backward()'s per-surfel gradients with K's principal point moved by (ox, oy): st is the forward state (its records
    carry the offset already when they are the GPU's), acc the (P,18) accumulators, tm the (P,9) transMat gradient the
    centred chain returns for them (dT after the AABB vjp)."""
    tm = np.asarray(tm, np.float64).reshape(-1, 9)
    a = np.array(acc, np.float64, copy=True).reshape(-1, so.NACC)
    a[:, _TW] += ox * tm[:, 0:3] + oy * tm[:, 3:6]
    out = so.chain(st, a)
    out["dL_dtransMat"] = np.asarray(tm, np.float32).reshape(out["dL_dtransMat"].shape)
    return out


def offset_bound_sums(st, B, acc, tm, ox, oy):
    """The accumulator-level bound sums B (P,18, in units of u = 2^-24) for offset_chain: the dT_w slots also carry
    |ox| |dT_u| + |oy| |dT_v| times the error dT already has (so chain_bound's |cx| becomes |cx| + |ox|), the rounding of
    the sum added there, and the magnitude of the terms that sum brings in."""
    B = np.array(B, np.float64, copy=True).reshape(-1, so.NACC)
    b_tm = np.asarray(so.chain_bound(st, B)["dL_dtransMat"], np.float64).reshape(-1, 9)
    tm = np.abs(np.asarray(tm, np.float64).reshape(-1, 9))
    shifted = np.abs(np.asarray(acc, np.float64).reshape(-1, so.NACC)[:, _TW]) + abs(ox) * tm[:, 0:3] + abs(oy) * tm[:, 3:6]
    B[:, _TW] += abs(ox) * b_tm[:, 0:3] + abs(oy) * b_tm[:, 3:6] + 3.0 * shifted
    return B


def rays(ox, oy):
    """post_oracle.rays with K's principal point at (W/2 + ox, H/2 + oy): the same integer pixel grid, K^-1, c2w."""
    def offset_rays(wvt, W, H, tanx, tany):
        wvt = np.asarray(wvt, np.float64)
        c2w = np.linalg.inv(wvt.T)
        fx, fy = W / (2.0 * tanx), H / (2.0 * tany)
        K = np.array([[fx, 0.0, W / 2.0 + ox], [0.0, fy, H / 2.0 + oy], [0.0, 0.0, 1.0]])
        gx, gy = np.meshgrid(np.arange(W, dtype=np.float64), np.arange(H, dtype=np.float64), indexing="xy")
        pts = np.stack([gx, gy, np.ones_like(gx)], -1).reshape(-1, 3)
        d = pts @ np.linalg.inv(K).T @ c2w[:3, :3].T
        return d.reshape(H, W, 3), c2w[:3, 3].copy()
    return offset_rays


def stage3_losses(ox, oy, *args, **kw):
    """post_oracle.stage3_losses with the ray grid's principal point moved by (ox, oy)."""
    return _with_rays(ox, oy, po.stage3_losses, *args, **kw)


def stage3_losses_backward(ox, oy, *args, **kw):
    """post_oracle.stage3_losses_backward with the ray grid's principal point moved by (ox, oy)."""
    return _with_rays(ox, oy, po.stage3_losses_backward, *args, **kw)


def _with_rays(ox, oy, fn, *args, **kw):
    saved = po.rays
    po.rays = rays(ox, oy)            # post_forward / post_backward look the name up at call time
    try:
        return fn(*args, **kw)
    finally:
        po.rays = saved
