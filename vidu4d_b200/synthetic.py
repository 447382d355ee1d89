"""Seeded synthetic surfel scenes (SURVEY.md section 8(d)) and a minimal surfel-parameter container.

Scenes are generated with numpy on the CPU (deterministic across machines) and moved to a device by the
caller.  `object_scene` is the Stage-3-like case: a noisy sphere of mesh-sampled surfels in CAMERA space in
front of an identity camera (lab4d/nnutils/deformable_gaussian.py:1170-1188, gs/scene/cameras.py:72-162);
`orbit_camera` supplies rigid cameras that exercise the non-identity view-matrix arithmetic.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import numpy as np
import torch

C0 = 0.28209479177387814


def _quat_from_rotmat(R: np.ndarray) -> np.ndarray:
    """(N,3,3) rotation matrices -> (N,4) quaternions (w,x,y,z), numerically safe branch selection."""
    N = R.shape[0]
    q = np.zeros((N, 4), dtype=np.float64)
    tr = R[:, 0, 0] + R[:, 1, 1] + R[:, 2, 2]
    c0 = tr > 0
    c1 = (~c0) & (R[:, 0, 0] >= R[:, 1, 1]) & (R[:, 0, 0] >= R[:, 2, 2])
    c2 = (~c0) & (~c1) & (R[:, 1, 1] >= R[:, 2, 2])
    c3 = ~(c0 | c1 | c2)
    s = np.sqrt(np.maximum(tr[c0] + 1.0, 1e-12)) * 2
    q[c0] = np.stack([0.25 * s, (R[c0, 2, 1] - R[c0, 1, 2]) / s, (R[c0, 0, 2] - R[c0, 2, 0]) / s,
                      (R[c0, 1, 0] - R[c0, 0, 1]) / s], 1)
    s = np.sqrt(np.maximum(1.0 + R[c1, 0, 0] - R[c1, 1, 1] - R[c1, 2, 2], 1e-12)) * 2
    q[c1] = np.stack([(R[c1, 2, 1] - R[c1, 1, 2]) / s, 0.25 * s, (R[c1, 0, 1] + R[c1, 1, 0]) / s,
                      (R[c1, 0, 2] + R[c1, 2, 0]) / s], 1)
    s = np.sqrt(np.maximum(1.0 + R[c2, 1, 1] - R[c2, 0, 0] - R[c2, 2, 2], 1e-12)) * 2
    q[c2] = np.stack([(R[c2, 0, 2] - R[c2, 2, 0]) / s, (R[c2, 0, 1] + R[c2, 1, 0]) / s, 0.25 * s,
                      (R[c2, 1, 2] + R[c2, 2, 1]) / s], 1)
    s = np.sqrt(np.maximum(1.0 + R[c3, 2, 2] - R[c3, 0, 0] - R[c3, 1, 1], 1e-12)) * 2
    q[c3] = np.stack([(R[c3, 1, 0] - R[c3, 0, 1]) / s, (R[c3, 0, 2] + R[c3, 2, 0]) / s,
                      (R[c3, 1, 2] + R[c3, 2, 1]) / s, 0.25 * s], 1)
    return q


@dataclass
class Scene:
    means3D: np.ndarray      # (P,3) float32
    scales: np.ndarray       # (P,2)  activated (exp applied)
    rotations: np.ndarray    # (P,4)  (w,x,y,z), unit norm up to fp32 rounding
    opacities: np.ndarray    # (P,1)  activated (sigmoid applied)
    shs: np.ndarray          # (P,16,3)
    sh_degree: int = 3

    @property
    def P(self):
        return self.means3D.shape[0]

    def to_torch(self, device, requires_grad=False):
        out = {}
        for k in ("means3D", "scales", "rotations", "opacities", "shs"):
            t = torch.from_numpy(getattr(self, k)).to(device)
            if requires_grad:
                t.requires_grad_(True)
            out[k] = t
        return out


def object_scene(P: int, seed: int = 0, radius: float = 0.35, center=(0.0, 0.0, 1.0), opacity: str = "trained",
                 sh_degree: int = 3, noise: float = 0.02) -> Scene:
    """Noisy sphere of P surfels, mesh-sampling-like scales (mean-3NN spacing), radial normals."""
    rng = np.random.default_rng(seed)
    d = rng.normal(size=(P, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    r = radius * (1.0 + noise * rng.normal(size=(P, 1)))
    xyz = d * r + np.asarray(center, dtype=np.float64)[None]
    # tangent frame: third column = (noisy) radial normal
    n = d + 0.1 * rng.normal(size=(P, 3))
    n /= np.linalg.norm(n, axis=1, keepdims=True)
    a = rng.normal(size=(P, 3))
    t1 = a - (a * n).sum(1, keepdims=True) * n
    t1 /= np.linalg.norm(t1, axis=1, keepdims=True)
    t2 = np.cross(n, t1)
    R = np.stack([t1, t2, n], axis=2)                      # columns
    q = _quat_from_rotmat(R)
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    spacing = math.sqrt(4.0 * math.pi * radius * radius / max(P, 1))
    # sqrt(mean squared 3-NN distance) of a Poisson surface sampling ~ 0.78 * spacing (gaussian_model.py:139-140)
    scales = 0.78 * spacing * (1.0 + 0.2 * (2.0 * rng.random(size=(P, 2)) - 1.0))
    if opacity == "trained":
        op = rng.uniform(0.2, 1.0, size=(P, 1))
    elif opacity == "init":
        op = 1.0 / (1.0 + np.exp(-rng.normal(-2.2, 1.0, size=(P, 1))))   # inverse_sigmoid(0.1)-centred
    else:
        raise ValueError("opacity must be 'trained' or 'init'")
    rgb = rng.uniform(0.0, 1.0, size=(P, 3))
    shs = np.zeros((P, 16, 3))
    shs[:, 0] = (rgb - 0.5) / C0
    shs[:, 1:] = 0.05 * rng.normal(size=(P, 15, 3))
    f32 = lambda x: np.ascontiguousarray(x, dtype=np.float32)  # noqa: E731
    return Scene(f32(xyz), f32(scales), f32(q), f32(op), f32(shs), sh_degree)


def shell_with_strays(P: int, seed: int = 0, radius: float = 0.15, thickness: float = 0.002, stray_frac: float = 0.01,
                      center=(0.0, 0.0, 1.0)) -> np.ndarray:
    """(P,3) float32 surfel centres like a densified Stage-3 object: a thin noisy sphere dense enough that a point has ~50
    others within 0.004 (the reference's outlier radius), plus stray_frac of the points scattered uniformly over a box
    three radii wide, far from the surface (lab4d/engine/trainer.py:573-588 exists to prune those)."""
    rng = np.random.default_rng(seed)
    n_stray = int(round(P * stray_frac))
    d = rng.normal(size=(P - n_stray, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    shell = d * (radius + thickness * rng.normal(size=(P - n_stray, 1)))
    strays = rng.uniform(-3 * radius, 3 * radius, size=(n_stray, 3))
    xyz = np.concatenate([shell, strays])[rng.permutation(P)] + np.asarray(center, dtype=np.float64)[None]
    return np.ascontiguousarray(xyz, dtype=np.float32)


def random_rotation(rng) -> np.ndarray:
    q = rng.normal(size=4)
    q /= np.linalg.norm(q)
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def rigid_view(scene_cam: Scene, R_wc: np.ndarray, t_wc: np.ndarray):
    """Given a scene expressed in CAMERA space and a world->camera rigid map x_c = R_wc x_w + t_wc, return the
    same scene expressed in WORLD space plus the (viewmatrix, campos) in the reference's convention
    (viewmatrix = W2C transposed, stored row-major; gs/scene/cameras.py:54-57)."""
    R = np.asarray(R_wc, np.float64)
    t = np.asarray(t_wc, np.float64)
    xw = (scene_cam.means3D.astype(np.float64) - t[None]) @ R      # R^T (x_c - t)
    # surfel orientation: R_c = R_wc R_w  ->  R_w = R_wc^T R_c ; do it on quaternions via matrices
    q = scene_cam.rotations.astype(np.float64)
    w, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    Rc = np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)], 1),
                   np.stack([2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)], 1),
                   np.stack([2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], 1)], 1)
    Rw = np.einsum('ji,njk->nik', R, Rc)
    qw = _quat_from_rotmat(Rw)
    qw /= np.linalg.norm(qw, axis=1, keepdims=True)
    W2C = np.eye(4)
    W2C[:3, :3] = R
    W2C[:3, 3] = t
    viewmatrix = W2C.T.astype(np.float32).copy()               # row-vector convention
    campos = (-R.T @ t).astype(np.float32)
    world = Scene(np.ascontiguousarray(xw, np.float32), scene_cam.scales, np.ascontiguousarray(qw, np.float32),
                  scene_cam.opacities, scene_cam.shs, scene_cam.sh_degree)
    return world, viewmatrix, campos


def projection_matrix(tanfovx, tanfovy, znear=0.01, zfar=100.0) -> np.ndarray:
    """gs/utils/graphics_utils.py:53-76, transposed like the reference stores it."""
    P = np.zeros((4, 4), np.float32)
    P[0, 0] = 1.0 / tanfovx
    P[1, 1] = 1.0 / tanfovy
    P[3, 2] = 1.0
    P[2, 2] = zfar / (zfar - znear)
    P[2, 3] = -(zfar * znear) / (zfar - znear)
    return P.T.copy()


def orbit_view(frame: int, nframes: int, tilt: float = 0.3):
    """World->camera rigid map of an orbiting camera that keeps the object at camera-space (0,0,1):
    the object sits at the world origin, the camera circles it at distance 1."""
    ang = 2.0 * math.pi * frame / max(nframes, 1)
    ca, sa = math.cos(ang), math.sin(ang)
    ct, st = math.cos(tilt), math.sin(tilt)
    Ry = np.array([[ca, 0, sa], [0, 1, 0], [-sa, 0, ca]])
    Rx = np.array([[1, 0, 0], [0, ct, -st], [0, st, ct]])
    R_wc = Rx @ Ry
    t_wc = np.array([0.0, 0.0, 1.0])
    return R_wc, t_wc


class SurfelCloud(torch.nn.Module):
    """The slice of gs/scene/gaussian_model.py::GaussianModel that render() reads (gaussian_model.py:98-118):
    raw parameters + activations.  Parameter list and order follow the Stage-3 gs_optimizer
    (lab4d/engine/trainer.py:243-251)."""

    def __init__(self, scene: Scene, device="cuda", fused_features: bool = False):
        """fused_features: keep the SH rows as ONE (P, 16, 3) parameter instead of the reference's _features_dc /
        _features_rest pair (gaussian_model.py:98-118 concatenates the pair on every get_features; a model that stores
        the rows the way the rasterizer reads them skips that copy and the split of its gradient)."""
        super().__init__()
        t = lambda a: torch.nn.Parameter(torch.from_numpy(np.ascontiguousarray(a)).to(device))  # noqa: E731
        self.max_sh_degree = 3
        self.active_sh_degree = scene.sh_degree
        self._xyz = t(scene.means3D)
        self.fused_features = bool(fused_features)
        if self.fused_features:
            self._features = t(scene.shs)
        else:
            self._features_dc = t(scene.shs[:, :1])
            self._features_rest = t(scene.shs[:, 1:])
        self._scaling = t(np.log(scene.scales))
        self._rotation = t(scene.rotations)
        op = np.clip(scene.opacities, 1e-6, 1 - 1e-6)
        self._opacity = t(np.log(op / (1 - op)))

    @property
    def get_xyz(self):
        return self._xyz

    @property
    def get_scaling(self):
        return torch.exp(self._scaling)

    @property
    def get_rotation(self):
        return torch.nn.functional.normalize(self._rotation)

    @property
    def get_opacity(self):
        return torch.sigmoid(self._opacity)

    @property
    def get_features(self):
        if self.fused_features:
            return self._features
        return torch.cat((self._features_dc, self._features_rest), dim=1)

    def get_covariance(self, scaling_modifier=1.0):
        raise NotImplementedError("precomputed covariance is not supported (see rasterizer.py)")

    def flat_params(self):
        if self.fused_features:
            return [self._xyz, self._features, self._opacity, self._scaling, self._rotation]
        return [self._xyz, self._features_dc, self._features_rest, self._opacity, self._scaling, self._rotation]
