"""CPU tests of the fused silhouette loss (csrc/mask_loss.cu, include/surfel_mask_loss.h): the float64 model
(tests/mask_loss_model.py) against fixtures made by the reference's own loss code (tests/golden/maskloss_*.npz), the header
<-> library <-> binding match, each bad argument's own message, SR_ECUDA without a device, and render_loss_batch's
argument checks (every bad call is rejected before any CUDA work)."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from .conftest import ROOT, load_golden

CASES = ["maskloss_binary_48x40", "maskloss_fractional_48x40", "maskloss_undetected_48x40", "maskloss_none_detected_48x40",
         "maskloss_all_zero_48x40", "maskloss_all_one_48x40", "maskloss_outside_vis_48x40", "maskloss_acc_eq_gt_48x40",
         "maskloss_m8_37x23"]
D = 1 << 20      # placeholder DEVICE pointer: never dereferenced (the calls fail before any device work)


@pytest.mark.parametrize("name", CASES)
def test_model_matches_reference_fixture(name):
    from .mask_loss_model import mask_loss
    g = load_golden(name)
    r = mask_loss(g["in_alpha"], g["in_mask"], g["in_vis2d"], g["in_is_detected"], g["in_weight"][0])
    assert r["branch"] == bool(g["ref_branch"][0])
    binary = np.isin(g["in_mask"], (0.0, 1.0)).all()
    if r["branch"] and binary:      # exact integer sums: the weights, bw and v are torch's bit for bit
        assert np.array_equal([r["pos_wt"], r["neg_wt"]], [g["ref_pos_wt"][0], g["ref_neg_wt"][0]], equal_nan=True)
    if binary:
        assert np.array_equal(r["v"], g["ref_v"], equal_nan=True)
    assert np.array_equal(r["counts"], g["ref_counts"])
    loss, ref = r["terms"].sum(), float(g["ref_loss"][0])
    if np.isnan(ref):
        assert np.isnan(loss)
    else:
        assert abs(loss - ref) <= 1e-6 * abs(ref) + 1e-30, (loss, ref)
    rg = g["ref_grad_alpha"].astype(np.float64)
    assert np.array_equal(np.isnan(r["grad"]), np.isnan(rg)) and np.array_equal(np.isinf(r["grad"]), np.isinf(rg))
    fin = np.isfinite(rg)
    assert np.all(np.abs(r["grad"][fin] - rg[fin]) <= 1e-6 * np.abs(rg[fin]))
    if name == "maskloss_undetected_48x40":
        assert r["counts"][0] == 0 and np.abs(r["grad"][0]).max() == 0
    if name in ("maskloss_none_detected_48x40", "maskloss_outside_vis_48x40"):
        assert np.isnan(ref) and np.isnan(rg).all()
    if name == "maskloss_outside_vis_48x40":
        assert np.isinf(r["pos_wt"]) and r["neg_wt"] == 1.0
    if name == "maskloss_acc_eq_gt_48x40":           # no positive v: the fallback v.mean() is 0, and so is the gradient
        assert r["counts"].sum() == 0 and ref == 0.0 and np.abs(rg).max() == 0


def test_mask_loss_header_matches_library_and_binding(built):
    """include/surfel_mask_loss.h <-> libsurfel_raster.so <-> _capi.MASK_LOSS_PROTOTYPES, kind for kind."""
    from vidu4d_b200 import _capi
    lib = _capi.load()
    hdr = open(os.path.join(ROOT, "include", "surfel_mask_loss.h")).read()
    body = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    protos = re.findall(r"SR_API\s+([\w\s\*]+?)\b(sr_\w+)\s*\(([^)]*)\)", body)
    assert {name for _, name, _ in protos} == set(_capi.MASK_LOSS_SYMBOLS)
    others = (set(_capi.SYMBOLS) | set(_capi.SSIM_SYMBOLS) | set(_capi.OPTIM_SYMBOLS) | set(_capi.SKIN_MLP_SYMBOLS))
    assert not set(_capi.MASK_LOSS_SYMBOLS) & others
    c_kinds = {"int": "int32", "int32_t": "int32", "int64_t": "int64", "float": "float", "double": "double", "void": None}
    py_kinds = {C.c_int32: "int32", C.c_int64: "int64", C.c_float: "float", C.c_double: "double"}

    def c_kind(decl):
        return "pointer" if "*" in decl else c_kinds[decl.replace("const", "").split()[0]]

    def py_kind(t):
        return "pointer" if t in (C.c_void_p, C.c_char_p) else py_kinds[t]
    for ret, name, params in protos:
        assert hasattr(lib, name)
        params = [p for p in params.split(",") if p.strip() not in ("", "void")]
        restype, argtypes = _capi.MASK_LOSS_PROTOTYPES[name]
        assert py_kind(restype) == c_kind(ret), name
        assert [py_kind(t) for t in argtypes] == [c_kind(p) for p in params], name


def test_scratch_query(built):
    from vidu4d_b200 import _capi
    lib = _capi.load()
    for bad in ((0, 48, 40), (2, 0, 40), (2, 48, 0), (65536, 4, 4), (1, 4, 524281)):
        assert lib.sr_mask_loss_scratch_bytes(*bad) == -1, bad
    a, b = lib.sr_mask_loss_scratch_bytes(2, 256, 256), lib.sr_mask_loss_scratch_bytes(8, 512, 512)
    assert 5 * 2 * 256 * 256 < a < 6 * 2 * 256 * 256 and 5 * 8 * 512 * 512 < b < 6 * 8 * 512 * 512


def _good(lib, M=2, W=48, H=40):
    nb = int(lib.sr_mask_loss_scratch_bytes(M, W, H))
    return dict(M=M, W=W, H=H, alpha=D, alpha_stride=8 * W * H, mask_gt=D, vis2d=None, is_detected=None, weight=D,
                terms=D, counts=D, balance=D, dL_dalpha=D, scratch=D, scratch_bytes=nb, stream=None)


def test_bad_argument_sets_its_own_message(built):
    from vidu4d_b200 import _capi
    lib = _capi.load()
    g = _good(lib)
    cases = [(dict(M=0), b"M, W and H must be >= 1"), (dict(W=0), b"M, W and H must be >= 1"),
             (dict(H=-1), b"M, W and H must be >= 1"), (dict(M=65536), b"M must be <= 65535"),
             (dict(H=524281), b"H must be <= 524280"), (dict(alpha_stride=48 * 40 - 1), b"alpha_stride 1919 is below H*W"),
             (dict(alpha=None), b"alpha, mask_gt, weight and dL_dalpha must not be NULL"),
             (dict(mask_gt=None), b"alpha, mask_gt, weight and dL_dalpha must not be NULL"),
             (dict(weight=None), b"alpha, mask_gt, weight and dL_dalpha must not be NULL"),
             (dict(dL_dalpha=None), b"alpha, mask_gt, weight and dL_dalpha must not be NULL"),
             (dict(terms=None), b"terms, counts and balance must not be NULL"),
             (dict(counts=None), b"terms, counts and balance must not be NULL"),
             (dict(balance=None), b"terms, counts and balance must not be NULL"),
             (dict(scratch=None), b"scratch must not be NULL"), (dict(scratch=D + 8), b"256-byte aligned"),
             (dict(scratch_bytes=g["scratch_bytes"] - 1), b"fewer than sr_mask_loss_scratch_bytes(2, 48, 40)")]
    for kw, want in cases:
        assert lib.sr_debug_view(0, 0, 0, 0, None) == -1        # a sentinel message from a different failure
        sentinel = lib.sr_last_error()
        rc = lib.sr_mask_loss_batch(*dict(g, **kw).values())
        msg = lib.sr_last_error()
        assert rc == -1, (kw, rc, msg)
        assert msg != sentinel and b"sr_mask_loss_batch" in msg and want in msg, (kw, msg)


def _cuda_failures_child():
    """Run with no visible device: a call whose arguments pass every check returns SR_ECUDA with the CUDA error's text."""
    if torch.cuda.device_count() != 0:
        print("SKIP: a device is visible")
        return
    from vidu4d_b200 import _capi
    lib = _capi.load()
    cudart = C.CDLL("libcudart.so.12")
    cudart.cudaGetErrorString.restype = C.c_char_p
    texts = {cudart.cudaGetErrorString(e) for e in range(1, 1000)} - {cudart.cudaGetErrorString(999999)}
    for vis, det in ((None, None), (D, D)):
        assert lib.sr_debug_view(0, 0, 0, 0, None) == -1
        rc = lib.sr_mask_loss_batch(*dict(_good(lib), vis2d=vis, is_detected=det).values())
        msg = lib.sr_last_error()
        assert rc == -2, (rc, msg)
        assert b"CUDA error in sr_mask_loss_batch" in msg and any(msg.endswith(b": " + t) for t in texts), msg
    print("OK")


def test_cuda_failure_sets_its_own_message(built):
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    flags = ["-s"] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable] + flags + ["-c", "import tests.test_mask_loss_cpu as t; t._cuda_failures_child()"],
                       cwd=ROOT, env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.strip().splitlines()[-1] in ("OK", "SKIP: a device is visible"), r.stdout


def test_python_rejects_bad_mask_loss_arguments():
    from vidu4d_b200.renderer import _check_mask_loss
    M = 2
    mask, w = torch.zeros((M, 40, 48)), torch.ones(1)

    def chk(mask_gt=mask, mask_wt=None, w_mask=0.0, det=None, weight=w):
        return _check_mask_loss(M, torch.device("cuda:0"), mask_gt, mask_wt, w_mask, det, weight)
    with pytest.raises(RuntimeError, match="mask_loss_weight needs mask_gt"):
        chk(mask_gt=None)
    with pytest.raises(RuntimeError, match="neither mask_wt nor w_mask"):
        chk(mask_wt=torch.ones((M, 40, 48)))
    with pytest.raises(RuntimeError, match="neither mask_wt nor w_mask"):
        chk(w_mask=0.1)
    with pytest.raises(RuntimeError, match="mask_loss_weight must be a float32 \\(1,\\) tensor"):
        chk(weight=torch.ones(2))
    with pytest.raises(RuntimeError, match="mask_loss_weight must be a float32 \\(1,\\) tensor"):
        chk(weight=torch.ones(1, dtype=torch.float64))
    with pytest.raises(RuntimeError, match="is_detected must be"):
        chk(det=torch.ones(M + 1))
    with pytest.raises(RuntimeError, match="mask_loss_weight must be a CUDA tensor"):
        chk()
