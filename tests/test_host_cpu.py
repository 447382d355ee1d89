"""CPU: the C-ABI library loads and exports everything include/surfel_raster.h declares; host-side logic
(argument validation, capacity policy, buffer sizing, drop-in API surface, scene generators)."""
import ctypes as C
import inspect
import os
import re

import numpy as np
import pytest
import torch

from .conftest import ROOT


def test_library_exports_declared_abi(built):
    from vidu4d_b200 import _capi
    lib = _capi.load()
    hdr = open(os.path.join(ROOT, "include", "surfel_raster.h")).read()
    declared = set(re.findall(r"SR_API\s+[\w\s\*]+?\b(sr_\w+)\s*\(", hdr))
    assert declared, "no SR_API declarations parsed"
    for sym in declared:
        assert hasattr(lib, sym), f"{sym} declared in the header but not exported"
    assert declared == set(_capi.SYMBOLS)
    assert lib.sr_abi_version() == _capi.ABI_VERSION


def test_buffer_sizing_monotonic_and_invertible(built):
    from vidu4d_b200 import _capi
    from vidu4d_b200.rasterizer import _capacity_from_bytes, _round_cap
    lib = _capi.load()
    assert lib.sr_geom_bytes(0) > 0 and lib.sr_geom_bytes(1000) < lib.sr_geom_bytes(100000)
    assert lib.sr_image_bytes(512, 512) >= 512 * 512 * 20
    prev = 0
    for cap in (256, 512, 4096, 100_096, 1_000_192, 3_000_064):
        assert cap == _round_cap(cap)
        b = lib.sr_binning_bytes(cap, 512, 512)
        assert b > prev
        assert _capacity_from_bytes(b, 512, 512) == cap
        # the per-stage contribution masks make the size depend on the tile count too
        assert lib.sr_binning_bytes(cap, 1024, 1024) > b
        prev = b
    with pytest.raises(_capi.SurfelRasterError):
        _capacity_from_bytes(prev + 1, 512, 512)


def test_debug_layout_is_aligned(built):
    from vidu4d_b200 import _capi
    lib = _capi.load()
    L = _capi.SrDebugLayout()
    assert lib.sr_debug_view(1000, 96, 64, 4096, C.byref(L)) == 0
    for name, _ in L._fields_:
        v = getattr(L, name)
        vals = list(v) if hasattr(v, "__len__") else [v]
        for x in vals:
            assert x % 256 == 0, (name, x)


def test_argument_validation_without_gpu(built):
    """Bad arguments are rejected before any CUDA call (so this runs on a CPU-only box)."""
    from vidu4d_b200 import _capi
    lib = _capi.load()
    nul = [None] * 16 + [0] + [None] * 3      # 16 pointers, capacity, 3 pointers
    fr = _capi.SrFrame(10, 3, 16, -5, 64, 0.5, 0.5, 1.0, 0, 0, 0)
    rc = lib.sr_forward(C.byref(fr), *nul)
    assert rc == -1 and b"image size" in lib.sr_last_error()
    fr = _capi.SrFrame(10, 5, 16, 64, 64, 0.5, 0.5, 1.0, 0, 0, 0)
    assert lib.sr_forward(C.byref(fr), *nul) == -1 and b"sh_degree" in lib.sr_last_error()
    fr = _capi.SrFrame(10, 3, 4, 64, 64, 0.5, 0.5, 1.0, 0, 0, 0)
    assert lib.sr_forward(C.byref(fr), *nul) == -1 and b"coefficients" in lib.sr_last_error()
    assert lib.sr_mark_visible(-1, None, None, None, None, None) == -1


def test_api_surface_matches_reference_names():
    import diff_surfel_rasterization as drop
    from vidu4d_b200 import rasterizer as R
    assert drop.GaussianRasterizer is R.GaussianRasterizer
    assert R.GaussianRasterizationSettings._fields == (
        "image_height", "image_width", "tanfovx", "tanfovy", "bg", "scale_modifier", "viewmatrix", "projmatrix",
        "sh_degree", "campos", "prefiltered", "debug")
    sig = inspect.signature(R.GaussianRasterizer.forward)
    assert list(sig.parameters) == ["self", "means3D", "means2D", "opacities", "shs", "colors_precomp", "scales",
                                    "rotations", "cov3D_precomp"]
    assert list(inspect.signature(R._C.rasterize_gaussians).parameters) == [
        "background", "means3D", "colors", "opacity", "scales", "rotations", "scale_modifier", "transMat_precomp",
        "viewmatrix", "projmatrix", "tan_fovx", "tan_fovy", "image_height", "image_width", "sh", "degree", "campos",
        "prefiltered", "debug"]
    assert len(inspect.signature(R._C.rasterize_gaussians_backward).parameters) == 22
    assert hasattr(R.GaussianRasterizer, "markVisible")


def test_C_is_an_importable_submodule():
    """`from diff_surfel_rasterization import _C` and `import diff_surfel_rasterization._C` both work, as with the
    reference's pybind extension (RAST/setup.py:18-23, RAST/diff_surfel_rasterization/__init__.py:14)."""
    import importlib
    m = importlib.import_module("diff_surfel_rasterization._C")
    from diff_surfel_rasterization import _C
    assert m is _C
    for fn in ("rasterize_gaussians", "rasterize_gaussians_backward", "mark_visible"):
        assert callable(getattr(m, fn))


def test_rasterizer_argument_errors_match_reference():
    from vidu4d_b200.rasterizer import GaussianRasterizationSettings, GaussianRasterizer
    rs = GaussianRasterizationSettings(8, 8, 0.5, 0.5, torch.zeros(3), 1.0, torch.eye(4), torch.eye(4), 0,
                                       torch.zeros(3), False, False)
    r = GaussianRasterizer(rs)
    x = torch.zeros(4, 3)
    with pytest.raises(Exception, match="excatly one of either SHs or precomputed colors"):
        r(x, x, torch.zeros(4, 1), scales=torch.zeros(4, 2), rotations=torch.zeros(4, 4))
    with pytest.raises(Exception, match="excatly one of either SHs or precomputed colors"):
        r(x, x, torch.zeros(4, 1), shs=torch.zeros(4, 1, 3), colors_precomp=torch.zeros(4, 3), scales=torch.zeros(4, 2),
          rotations=torch.zeros(4, 4))
    with pytest.raises(Exception, match="scale/rotation pair or precomputed 3D covariance"):
        r(x, x, torch.zeros(4, 1), shs=torch.zeros(4, 1, 3))
    # CPU tensors are rejected like CHECK_INPUT does (rasterize_points.cu:27-28) -- there is no CPU fallback
    with pytest.raises(RuntimeError, match="must be a CUDA tensor"):
        r(x, x, torch.zeros(4, 1), shs=torch.zeros(4, 1, 3), scales=torch.zeros(4, 2), rotations=torch.zeros(4, 4))


def test_product_does_not_import_oracle():
    """The product path must never route through the oracle (or any CPU fallback)."""
    pkg = os.path.join(ROOT, "vidu4d_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dirpath, f)).read()
                assert "surfel_oracle" not in src and "from oracle" not in src and "import oracle" not in src, f
    assert "oracle" not in open(os.path.join(ROOT, "diff_surfel_rasterization", "__init__.py")).read().replace("H100-native", "")


def test_missing_library_fails_loudly(monkeypatch, tmp_path):
    from vidu4d_b200 import _capi
    monkeypatch.setattr(_capi, "_lib", None)
    monkeypatch.setattr(_capi, "LIB_PATH", str(tmp_path / "nope.so"))
    with pytest.raises(_capi.SurfelRasterError, match="no CPU fallback"):
        _capi.load()


def test_scene_generators_are_seeded():
    from vidu4d_b200.synthetic import object_scene, orbit_view, random_rotation, rigid_view
    a, b = object_scene(500, seed=7), object_scene(500, seed=7)
    for k in ("means3D", "scales", "rotations", "opacities", "shs"):
        np.testing.assert_array_equal(getattr(a, k), getattr(b, k))
    assert np.allclose(np.linalg.norm(a.rotations, axis=1), 1.0, atol=1e-6)
    assert (a.opacities > 0).all() and (a.opacities <= 1).all() and (a.scales > 0).all()
    R, t = orbit_view(3, 16)
    assert np.allclose(R @ R.T, np.eye(3), atol=1e-12)
    w, vm, cp = rigid_view(a, random_rotation(np.random.default_rng(0)), np.array([0.1, 0.2, 0.3]))
    # camera-space positions are preserved: x_c = W2C x_w
    W2C = vm.T.astype(np.float64)
    xc = w.means3D.astype(np.float64) @ W2C[:3, :3].T + W2C[:3, 3]
    assert np.abs(xc - a.means3D).max() < 1e-5


def test_render_twin_on_cpu_reference_glue():
    """depth_to_normal restatement agrees with gs/utils/point_utils.py on a fronto-parallel plane (its normals face the camera: -z)."""
    from vidu4d_b200.renderer import depth_to_normal, make_camera
    cam = make_camera(32, 24, 2 * np.arctan(0.5), 2 * np.arctan(0.375), device="cpu")
    depth = torch.full((1, 24, 32), 2.0)
    n = depth_to_normal(cam, depth)
    assert n.shape == (24, 32, 3)
    inner = n[1:-1, 1:-1]
    assert torch.allclose(inner, torch.tensor([0.0, 0.0, -1.0]).expand_as(inner), atol=1e-5)
    assert (n[0] == 0).all() and (n[:, 0] == 0).all()


def test_contribution_mask_stage_slots_never_overlap():
    """common.cuh bin_layout: stage s of tile t (32 instances of its sorted list) keeps its per-pixel contribution
    masks in slot (range.x >> 5) + t + s of a buffer with (capacity >> 5) + tiles + 1 slots.  The composite kernels rely on
    those slots being disjoint between tiles and inside the buffer for ANY list lengths (no prefix sum of stage counts
    is ever computed)."""
    rng = np.random.default_rng(7)
    for trial in range(200):
        tiles = int(rng.integers(1, 400))
        kind = trial % 4
        if kind == 0:
            lens = rng.integers(0, 4, size=tiles)                       # mostly tiny / empty tiles
        elif kind == 1:
            lens = rng.integers(0, 3000, size=tiles)
        elif kind == 2:
            lens = np.where(rng.random(tiles) < 0.7, 0, rng.integers(1, 100, size=tiles))
        else:
            lens = rng.choice([0, 1, 31, 32, 33, 63, 64, 65], size=tiles)
        start = np.concatenate([[0], np.cumsum(lens)[:-1]])
        R = int(lens.sum())
        nslots = (R >> 5) + tiles + 1
        prev_end = 0
        for t in range(tiles):
            if lens[t] == 0:
                continue
            base = (int(start[t]) >> 5) + t
            nst = (int(lens[t]) + 31) // 32
            assert base >= prev_end, (trial, t)
            assert base + nst <= nslots, (trial, t)
            prev_end = base + nst


def test_check_overflow_bookkeeping_without_a_gpu(built, monkeypatch):
    """nosync mode's once-per-step check: capacity hints follow the largest num_rendered seen, an overflowed or
    prefilter-violating frame raises, keep=True leaves the watch list for the next CUDA-graph replay."""
    from vidu4d_b200 import _capi, rasterizer as R
    class _Stream:                      # stands in for the torch.cuda.Stream a forward ran on (no .device: CPU-only box)
        synced = 0

        def synchronize(self):
            _Stream.synced += 1
    st = _Stream()
    saved = (list(R._pending), dict(R._cap_hint), R._host_next)
    try:
        R._pending.clear(); R._cap_hint.clear()
        key = (0, 64, 64)
        R._pending.append((torch.tensor([[1000, 0]], dtype=torch.int32), key, 4096, st))
        R._pending.append((torch.tensor([[500, 0], [3000, 0], [2000, 0]], dtype=torch.int32), key, 4096, st))   # a batch of 3 frames
        R.check_overflow(keep=True)
        assert R._cap_hint[key] == 3000 and len(R._pending) == 2
        assert _Stream.synced >= 1           # the pending forwards' own stream / device is synchronised, not "the current device"
        R.check_overflow()
        assert not R._pending and R._host_next == 0
        assert R._pick_capacity(key, 10) == R._round_cap(int(3000 * 1.5) + 4096)
        R._pending.append((torch.tensor([[100, 0], [9000, _capi.SR_STATUS_OVERFLOW]], dtype=torch.int32), key, 4096, st))
        with pytest.raises(_capi.SurfelRasterError, match="overflow"):
            R.check_overflow()
        assert R._cap_hint[key] == 9000 and not R._pending          # hints updated: the re-run will fit
        R._pending.append((torch.tensor([[10, _capi.SR_STATUS_PREFILTER]], dtype=torch.int32), key, 4096, st))
        with pytest.raises(RuntimeError, match="prefiltered"):
            R.check_overflow()
    finally:
        R._pending[:] = saved[0]; R._cap_hint.clear(); R._cap_hint.update(saved[1]); R._host_next = saved[2]


def test_batch_descriptor_and_validation_without_gpu(built):
    """The batched entry points validate their descriptor before any CUDA call; sr_batch's ctypes layout matches the C one."""
    from vidu4d_b200 import _capi
    lib = _capi.load()
    assert C.sizeof(_capi.SrBatch) == 8 + 6 * 8                      # int32 frames, uint32 flags, six int64 strides
    fr = _capi.SrFrame(10, 3, 16, 64, 64, 0.5, 0.5, 1.0, 0, 0, 0)
    nul = [None] * 16 + [0] + [None] * 3
    for frames in (0, -3, 70000):
        bt = _capi.SrBatch(frames, 0, 0, 0, 0, 0, 0, 0)
        assert lib.sr_forward_batch(C.byref(fr), C.byref(bt), *nul) == -1 and b"frames" in lib.sr_last_error()
    assert lib.sr_forward_batch(C.byref(fr), None, *nul) == -1
    bt = _capi.SrBatch(2, 0, 0, 0, 0, 0, 0, 0)
    nulb = [None] * 13 + [None, None, None, 0] + [None] * 9
    assert lib.sr_backward_batch(C.byref(fr), C.byref(bt), *nulb) == -1 and b"NULL" in lib.sr_last_error()
    # pure host helpers
    assert lib.sr_bob_warp_table_floats(25, 2) == 25 * 10 + 2 * 25 * 8 + 2 * 7
    assert lib.sr_bob_warp_forward(10, 65, 1, *([None] * 14)) == -1                 # more than 64 bones
    assert lib.sr_adam_flat(0, None, None, 0.9, 0.999, 1e-15, 1, 1.0, None, None, None, None, None) == -1
    lo, hi = (C.c_float * 3)(0, 0, 0), (C.c_float * 3)(1, 2, 0.5)
    h, dims = C.c_float(), (C.c_int32 * 3)()
    cells = lib.sr_knn_cells(10000, lo, hi, C.byref(h), dims)
    assert cells == dims[0] * dims[1] * dims[2] and 1000 < cells < 100000 and 0.02 < h.value < 0.2


def test_batch_input_normalisation_on_cpu():
    """_batch_inputs: shared (single-frame shape) vs per-frame (leading M) inputs -> strides in floats; shape errors."""
    from vidu4d_b200 import rasterizer as R

    class _T:            # _f32c insists on CUDA tensors: stand-in with the attributes _batch_inputs reads
        pass
    orig = R._f32c
    R._f32c = lambda t, name: t
    try:
        ins, st = R._batch_inputs(3, means3D=(torch.zeros(3, 10, 3), (3,)), sh=(torch.zeros(10, 16, 3), None),
                                  rotations=(torch.zeros(10, 4), (4,)), colors=(torch.zeros(0), (3,)))
        assert st == {"means3D": 30, "sh": 0, "rotations": 0, "colors": 0} and ins["colors"] is None
        with pytest.raises(RuntimeError, match="leading dimension"):
            R._batch_inputs(3, means3D=(torch.zeros(2, 10, 3), (3,)))
        with pytest.raises(RuntimeError, match="trailing dimensions"):
            R._batch_inputs(3, scales=(torch.zeros(10, 3), (2,)))
        with pytest.raises(RuntimeError, match="dimensions"):
            R._batch_inputs(3, means3D=(torch.zeros(3), (3,)))
    finally:
        R._f32c = orig
    assert R.BatchRasterizationSettings._fields[:10] == R.GaussianRasterizationSettings._fields[:10]


def test_flat_surfel_layout_matches_flatgrads_order():
    """The flat store's group order and widths are the gs_optimizer's (lab4d/engine/trainer.py:243-251) and FlatGrads'."""
    from vidu4d_b200.surfel_store import GROUPS
    assert [n for n, _ in GROUPS] == ["xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation"]
    assert sum(k for _, k in GROUPS) == 58


def test_surfel_cloud_fused_features_on_cpu():
    """SurfelCloud(fused_features=True) keeps the SH rows as ONE leaf: get_features is that leaf (no torch.cat in the
    graph), the values equal the reference-style pair's concatenation, and flat_params / FlatGrads follow the 5-tensor list."""
    from vidu4d_b200 import distributed as D
    from vidu4d_b200.synthetic import SurfelCloud, object_scene
    scene = object_scene(257, seed=3)
    a, b = SurfelCloud(scene, "cpu"), SurfelCloud(scene, "cpu", fused_features=True)
    assert b.get_features is b._features and b.get_features.is_leaf and b.get_features.shape == (257, 16, 3)
    assert not a.get_features.is_leaf and torch.equal(a.get_features.detach(), b.get_features.detach())
    assert [tuple(p.shape) for p in b.flat_params()] == [(257, 3), (257, 16, 3), (257, 1), (257, 2), (257, 4)]
    assert len(a.flat_params()) == 6
    fg = D.FlatGrads(b.flat_params())
    (b.get_features.sum() * 2.0 + b.get_xyz.sum()).backward()
    assert fg.flat.numel() == 257 * 58 and float(fg.flat.sum()) == 257 * 48 * 2.0 + 257 * 3
