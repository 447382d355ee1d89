"""TEST INFRASTRUCTURE -- float64 torch restatement of Stage 3's per-surfel feature rows (csrc/feature_rows.cu,
vidu4d_b200.warp.feature_rows), built on the quaternion algebra of oracle/warp_oracle.py:

    lab4d/nnutils/deformable_gaussian.py:1106-1182   query_field: normal, flow scale, [regist | flow / s | normal | density]
    lab4d/nnutils/deformable_gaussian.py:817-883     compute_flow with flip_pair (:789-805)
    lab4d/nnutils/deformable_gaussian.py:1742-1769   compute_gauss_density (warping.py:463-495, transforms.py:28-40)

Autograd of these expressions is the gradient oracle; torch's max / min / maximum / abs backward is the routing of the
flow scale's gradient over tied elements that the kernel reproduces.  Pinned to tests/golden/frows_*.npz by
tests/test_feature_rows_cpu.py.
"""
from __future__ import annotations

import torch

from oracle import warp_oracle as wo


def flow(xyz_cam, Kmat):
    """(M,P,2): pi(K[m'], x[m']) - pi(K[m], x[m]), m' = m xor 1 (M = 1: m' = m); pi(K,x) = (Kx)[:2] / (Kx)[2]."""
    M = xyz_cam.shape[0]
    if M > 1 and M % 2:
        raise ValueError(f"M must be 1 or even (flip_pair pairs frames 2k, 2k+1), got {M}")
    v = torch.einsum("mij,mpj->mpi", Kmat, xyz_cam)
    uv = (v / v[..., 2:])[..., :2]
    partner = torch.arange(M, device=xyz_cam.device) ^ 1 if M > 1 else torch.zeros(1, dtype=torch.long, device=xyz_cam.device)
    return uv[partner] - uv


def gauss_density(xyz, rest_dq, logibeta):
    """(P,1): exp(logibeta) * max_b exp(-0.5 |xyz - c_b|^2 / 0.01^2), c_b the translation of the rest bone b."""
    _, centres = wo.dq_to_qt(*rest_dq)
    d2 = ((xyz[:, None, :] - centres[None]) ** 2).sum(-1) / 0.01 ** 2
    return torch.exp(-0.5 * d2).max(-1).values[:, None] * logibeta.exp()


def normal(scaling, rot_cam, cam_q):
    """(M,P,3): cam_q[m] applied to rot_cam[m,p] applied to e_x or e_y, the arg-min of the two tangent scales (the first
    on ties, as torch.min(dim) returns it; written without one_hot, which synchronises with the host on CUDA)."""
    y = scaling[:, 1] < scaling[:, 0]
    axis = torch.stack((~y, y, torch.zeros_like(y)), -1).to(rot_cam.dtype)
    return wo.qapply(cam_q[:, None], wo.qapply(rot_cam, axis[None]))


def feature_rows(regist, xyz, scaling, xyz_cam, rot_cam, Kmat, field2cam, rest_dq, logibeta):
    """rows (M,P,Cf+6), flow scale s (0-d), gauss_density (P,1), flow (M,P,2)."""
    M, P = xyz_cam.shape[:2]
    f = flow(xyz_cam, Kmat)
    s = torch.max(f.max(), torch.abs(f.min())) + 1e-6
    dens = gauss_density(xyz, rest_dq, logibeta)
    rows = torch.cat([regist[None].expand(M, -1, -1), f / s, normal(scaling, rot_cam, field2cam[0]),
                      dens[None].expand(M, -1, -1)], -1)
    return rows, s, dens, f
