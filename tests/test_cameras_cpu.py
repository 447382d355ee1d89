"""CPU tests of per-frame intrinsics (include/surfel_camera.h): the sr_frame_cameras layout, the argument checks of the
three entry points that read the table, camera_table(), and tests/camera_model.py (the principal-point offsets derived
from the centred oracles)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

from .conftest import GOLDEN_CASES, ROOT, load_golden
from .test_host_cpu import _null_backward_args, _null_forward_args


def test_frame_cameras_layout_matches_c(built, tmp_path):
    """ctypes' SrFrameCameras against the C compiler's sr_frame_cameras: size and both member offsets."""
    from vidu4d_b200 import _capi
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "surfel_camera.h"\n'
                   'int main(void) { printf("%zu %zu %zu %u\\n", sizeof(sr_frame_cameras), offsetof(sr_frame_cameras, frame),'
                   ' offsetof(sr_frame_cameras, cameras), SR_FRAME_CAMERAS); return 0; }\n')
    exe = tmp_path / "layout"
    subprocess.check_call(["cc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    size, off_frame, off_cams, bit = (int(v) for v in subprocess.check_output([str(exe)]).split())
    assert size == C.sizeof(_capi.SrFrameCameras)
    assert off_frame == _capi.SrFrameCameras.frame.offset == 0
    assert off_cams == _capi.SrFrameCameras.cameras.offset
    assert bit == _capi.SR_FRAME_CAMERAS


def test_camera_header_and_abi_version_match_library_and_binding(built):
    """include/surfel_camera.h <-> libsurfel_raster.so <-> _capi.CAMERA_PROTOTYPES, and the ABI version: the
    SR_ABI_VERSION surfel_raster.h defines is the library's and the binding's."""
    import re
    from vidu4d_b200 import _capi
    lib = _capi.load()
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "surfel_camera.h")).read(), flags=re.S)
    protos = re.findall(r"SR_API\s+([\w\s\*]+?)\b(sr_\w+)\s*\(([^)]*)\)", hdr)
    assert {name for _, name, _ in protos} == set(_capi.CAMERA_SYMBOLS)
    kinds = {"int32_t": C.c_int32, "float": C.c_float}
    for _, name, params in protos:
        assert hasattr(lib, name)
        want = [C.c_void_p if "*" in p else kinds[p.replace("const", "").split()[0]] for p in params.split(",")]
        assert _capi.CAMERA_PROTOTYPES[name][1] == want, name
    raster = open(os.path.join(ROOT, "include", "surfel_raster.h")).read()
    assert lib.sr_abi_version() == _capi.ABI_VERSION == int(re.search(r"#define SR_ABI_VERSION (\d+)", raster).group(1))


def test_flag_with_null_table_is_einval_before_any_cuda_call(built):
    """SR_FRAME_CAMERAS with cameras == NULL fails in sr_forward, sr_backward and sr_render_loss_batch_cameras with its
    own message, before any device work (these calls would otherwise need a GPU)."""
    from vidu4d_b200 import _capi
    lib = _capi.load()
    fc = _capi.SrFrameCameras(_capi.SrFrame(10, 3, 16, 64, 64, 0.0, 0.0, 1.0, 0, 0, _capi.SR_FRAME_CAMERAS), None)
    bt = _capi.SrBatch(2, 0, 0, 0, 0, 0, 0, 0)
    fr = fc.frame                                               # shares fc's memory
    assert lib.sr_forward(*_null_forward_args(fr, bt)) == -1 and b"camera table is NULL" in lib.sr_last_error()
    assert lib.sr_backward(*_null_backward_args(fr, bt)) == -1 and b"camera table is NULL" in lib.sr_last_error()
    rc = lib.sr_render_loss_batch_cameras(2, 64, 64, None, 0.0, *([None] * 8), 1.0, 0.0, 0.0, 0.0, *([None] * 6))
    assert rc == -1 and b"camera table is NULL" in lib.sr_last_error()
    # with the table given the same calls get past that check to their own (other NULL pointers)
    fc.cameras = 16
    assert lib.sr_forward(*_null_forward_args(fr, bt)) == -1 and b"camera table" not in lib.sr_last_error()
    rc = lib.sr_render_loss_batch_cameras(2, 64, 64, 16, 0.0, *([None] * 8), 1.0, 0.0, 0.0, 0.0, *([None] * 6))
    assert rc == -1 and b"required pointer is NULL" in lib.sr_last_error()


def test_camera_table_from_K():
    from vidu4d_b200.renderer import camera_table
    W, H = 96, 64
    K = torch.tensor([[[120.0, 0.0, 48.0], [0.0, 110.0, 32.0], [0.0, 0.0, 1.0]],
                      [[80.5, 0.0, 51.25], [0.0, 79.0, 27.5], [0.0, 0.0, 1.0]]], dtype=torch.float64)
    t = camera_table(W, H, K)
    assert t.dtype == torch.float32 and tuple(t.shape) == (2, 4) and t.is_contiguous()
    k = K.to(torch.float32)
    want = torch.stack([torch.tensor(W, dtype=torch.float32) / (2 * k[:, 0, 0]), torch.tensor(H, dtype=torch.float32)
                        / (2 * k[:, 1, 1]), k[:, 0, 2] - W / 2, k[:, 1, 2] - H / 2], 1)
    assert torch.equal(t, want)
    assert t[0, 2] == 0 and t[0, 3] == 0 and t[1, 2] == 3.25 and t[1, 3] == -4.5
    # the round trip: the rasterizer's focal length W / (2 tan) is K's again
    assert torch.allclose(W / (2 * t[:, 0]), k[:, 0, 0], rtol=1e-6) and torch.allclose(H / (2 * t[:, 1]), k[:, 1, 1], rtol=1e-6)
    with pytest.raises(RuntimeError, match=r"\(M,3,3\)"):
        camera_table(W, H, K[:, :2])


def test_intrinsics_argument_checks_on_cpu():
    from vidu4d_b200.rasterizer import _check_intrinsics
    ref = torch.zeros(3)
    with pytest.raises(RuntimeError, match=r"\(M,4\)"):
        _check_intrinsics(torch.zeros((2, 3)), 2, ref)
    with pytest.raises(RuntimeError, match="float32"):
        _check_intrinsics(torch.zeros((2, 4), dtype=torch.float64), 2, ref)
    with pytest.raises(RuntimeError, match="CUDA"):
        _check_intrinsics(torch.zeros((2, 4)), 2, ref)
    assert _check_intrinsics(None, 2, ref) is None


def _oracle(g, **kw):
    from oracle import surfel_oracle as so
    P, W, H, deg, pre = [int(v) for v in g["in_meta"]]
    return so.forward(g["in_means3D"], g["in_opacities"], g["in_scales"], g["in_rotations"],
                      shs=None if pre else g["in_shs"], colors_precomp=g["in_colors_precomp"] if pre else None, sh_degree=deg,
                      W=W, H=H, tanfovx=float(g["in_tanfov"][0]), tanfovy=float(g["in_tanfov"][1]), bg=g["in_bg"],
                      viewmatrix=g["in_viewmatrix"], projmatrix=g["in_projmatrix"], campos=g["in_campos"], **kw)


@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_offset_model_with_zero_offsets_is_the_centred_oracle(name, built):
    """tests/camera_model.py with offsets 0 gives the centred oracles' records, gradients and rays bit for bit."""
    from oracle import post_oracle as po
    from oracle import surfel_oracle as so
    from . import camera_model as cm
    g = load_golden(name)
    st = _oracle(g)
    T, c = cm.offset_records(st, 0.0, 0.0)
    assert np.array_equal(T.astype(np.float32), st.transMat.reshape(-1, 9))
    assert np.array_equal(c.astype(np.float32), st.means2D.reshape(-1, 2))
    so.composite_ext(st)
    og = so.backward(st, g["in_dL_dcolor"], g["in_dL_dallmap"], bounds=True)
    ref, off = so.chain(st, og["acc"]), cm.offset_chain(st, og["acc"], og["dL_dtransMat"], 0.0, 0.0)
    for k in ref:
        assert np.array_equal(np.asarray(ref[k]).view(np.uint8), np.asarray(off[k]).view(np.uint8)), (name, k)
    W, H = st.W, st.H
    rd, ro = po.rays(g["in_viewmatrix"], W, H, 0.5, 0.4)
    rd2, ro2 = cm.rays(0.0, 0.0)(g["in_viewmatrix"], W, H, 0.5, 0.4)
    assert np.array_equal(rd, rd2) and np.array_equal(ro, ro2)


@pytest.mark.parametrize("name", ["rigid_bg_96x64", "ragged_80x48_deg1", "id_deg3_64"])
def test_offset_records_render_the_shifted_image(name, built):
    """Records moved by a principal point 16 px right of the centre (exactly one tile), composited by the oracle from the
    centred binning moved by one tile column, render the centred image shifted by 16 columns.  Interior pixels are
    compared outside either side's knife-edge pixels; the first tile column is left out (surfels that reach it from
    the left were clamped away from the centred binning)."""
    from oracle import surfel_oracle as so
    from . import camera_model as cm
    g = load_golden(name)
    a = _oracle(g)
    ka = so.composite_ext(a)["knife"]
    P, W, H = a.P, a.W, a.H
    T, c = cm.offset_records(a, 16.0, 0.0)
    tx, ty = (W + 15) // 16, (H + 15) // 16
    rg = a.ranges.reshape(ty, tx, 2).copy()
    shifted = np.zeros_like(rg)
    shifted[:, 1:] = rg[:, :-1]
    b, ext = so.from_records(g["in_means3D"], g["in_opacities"], g["in_scales"], g["in_rotations"], shs=g["in_shs"], sh_degree=int(
        g["in_meta"][3]), W=W, H=H, tanfovx=float(g["in_tanfov"][0]), tanfovy=float(g["in_tanfov"][1]), bg=g["in_bg"],
        viewmatrix=g["in_viewmatrix"], projmatrix=g["in_projmatrix"], campos=g["in_campos"], transMat=T.astype(np.float32),
        means2D=c.astype(np.float32), normal_opacity=a.normal_opacity.reshape(P, 4), rgb=a.rgb.reshape(P, 3), radii=a.radii,
        clamped=a.clamped.reshape(P, 3), point_list=a.point_list, ranges=shifted.reshape(-1, 2))
    src = (slice(1, H - 1), slice(1, W - 17))
    dst = (slice(1, H - 1), slice(17, W - 1))
    keep = ~(ka[src] | ext["knife"][dst])
    assert keep.mean() > 0.95
    for plane in ("color", "allmap"):
        x, y = getattr(a, plane)[(slice(None),) + src], getattr(b, plane)[(slice(None),) + dst]
        scale = np.abs(x).max() + 1e-12
        err = np.abs(x.astype(np.float64) - y) * keep
        assert err.max() <= 1e-4 * scale, (name, plane, float(err.max()), scale)
    assert not np.allclose(a.color, b.color)                   # the offset does move the image
