"""GPU parity of the BENCHMARKED kernels at the BENCHMARKED configuration (300 K surfels, 512x512, bench.py's scene
and cameras) against stored records of the unmodified reference extension's outputs (tests/golden/ref_headline_*.npz,
tests/golden/make_reference_records.py): tile assignment / sort / ranges / contributor counts bit-exact, rendered planes
and all eight gradient tensors within 1e-4 (north_star).
"""
import numpy as np
import pytest
import torch

from .conftest import load_golden
from .test_gpu_parity import _assert_matches_record, _run_ours

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev(built):
    from vidu4d_b200 import _capi
    _capi.load()
    return torch.device("cuda:0")


def bench_inputs(view, P=300_000, res=512):
    """The exact inputs bench.py renders: object_scene(seed 0, trained opacities) at the world origin, orbit camera
    `view` of 64 (view=None: the Stage-3 identity camera with the object at z = 1)."""
    from vidu4d_b200.synthetic import object_scene, orbit_view, projection_matrix
    tan = 0.5
    Pm = projection_matrix(tan, tan).astype(np.float64)
    if view is None:
        sc = object_scene(P, seed=0, opacity="trained", center=(0.0, 0.0, 1.0))
        vm = np.eye(4, dtype=np.float32); cp = np.zeros(3, np.float32)
    else:
        sc = object_scene(P, seed=0, opacity="trained", center=(0.0, 0.0, 0.0))
        R, t = orbit_view(view, 64)
        W2C = np.eye(4); W2C[:3, :3] = R; W2C[:3, 3] = t
        vm = W2C.T.astype(np.float32); cp = (-R.T @ t).astype(np.float32)
    pm = (vm.astype(np.float64) @ Pm).astype(np.float32)
    rng = np.random.default_rng(1234)
    return dict(means3D=sc.means3D, scales=sc.scales, rotations=sc.rotations, opacities=sc.opacities, shs=sc.shs,
                colors_precomp=np.zeros((0,), np.float32), viewmatrix=vm, projmatrix=pm, campos=cp,
                bg=np.zeros(3, np.float32), dL_dcolor=rng.normal(size=(3, res, res)).astype(np.float32),
                dL_dallmap=(0.1 * rng.normal(size=(8, res, res))).astype(np.float32),
                meta=np.array([P, res, res, 3, 0], np.int64), tanfov=np.array([tan, tan], np.float32))


@pytest.mark.parametrize("view", [None, 0, 17], ids=["identity", "orbit0", "orbit17"])
def test_headline_against_reference_record(view, dev):
    rec = load_golden("ref_headline_" + ("identity" if view is None else f"orbit{view}"))
    assert int(rec["num_rendered"][0]) > 300_000
    # rendered planes: 1e-4 relative (north_star).  The depth / alpha / normal / median planes and the colour, which match
    # the sm_100a reference build bit for bit, are held to XBUILD_TOL against this record; distortion (fp32 depth mapping,
    # DESIGN.md 3.1) and the eight gradient tensors to TOL of each tensor's max magnitude
    near = ("color",) + tuple(f"allmap{ch}" for ch in (0, 1, 2, 3, 4, 5, 7))
    _assert_matches_record(_run_ours(bench_inputs(view), dev), rec, 512, 512, near=near)
