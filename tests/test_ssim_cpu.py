"""CPU: the float64 SSIM model (tests/ssim_model.py) against the reference's own outputs and finite differences; ssim()'s
argument checks; and include/surfel_ssim.h given the checks tests/test_host_cpu.py and tests/test_abi_errors_cpu.py give
surfel_raster.h (header <-> library <-> binding, each entry point's own message, SR_ECUDA without a device)."""
import ctypes as C
import glob
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from . import ssim_model as sm
from .conftest import GOLDEN_DIR, ROOT, load_golden

CASES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLDEN_DIR, "ssim_*.npz")))
D = 1 << 20      # placeholder DEVICE pointer: never dereferenced (the calls fail before any device work)


def test_fixtures_present():
    assert len(CASES) == 8


@pytest.mark.parametrize("case", CASES)
def test_model_matches_reference(case):
    """The float64 model against the reference run in float64.  The reference's 2-D window is the float32-rounded outer
    product of the 1-D weights, the model's the exact product (as the separable CUDA op's): every 2-D weight differs by
    at most 2^-24 relative.  That moves the mean by ~1e-9 and, where sigma^2 cancels (near-constant images), the
    gradient by ~4e-6 of its largest element."""
    g = load_golden(case)
    x, y, gup = g["in_img1"], g["in_img2"], g["in_gup"]
    assert abs(sm.ssim(x, y) - float(g["ref64_mean"])) <= 1e-8
    if x.ndim == 4:
        np.testing.assert_allclose(sm.ssim(x, y, size_average=False), g["ref64_per_image"], rtol=0, atol=1e-8)
        grad = sm.vjp_mean(x, y, gup, size_average=False)
    else:
        grad = sm.vjp_mean(x, y, float(gup))
    ref = g["ref64_grad"]
    assert np.abs(grad - ref).max() <= 1e-5 * max(np.abs(ref).max(), 1e-12), case


def test_window_weights_are_the_references():
    """The 1-D weights equal, bit for bit, the float32 weights the reference's gaussian(11, 1.5) builds."""
    import math
    g = torch.Tensor([math.exp(-(i - 5) ** 2 / float(2 * 1.5 ** 2)) for i in range(11)])
    assert np.array_equal((g / g.sum()).numpy().astype(np.float64), sm.window())


def test_model_vjp_matches_finite_differences():
    rng = np.random.default_rng(0)
    x, y = rng.uniform(size=(2, 2, 9, 13)), rng.uniform(size=(2, 2, 9, 13))
    gm = rng.normal(size=x.shape)
    L = lambda a: float((sm.ssim_map(a, y) * gm).sum())  # noqa: E731
    grad = sm.vjp(x, y, gm)
    h = 1e-6
    for idx in [(0, 0, 0, 0), (1, 1, 8, 12), (0, 1, 4, 6), (1, 0, 0, 12), (0, 0, 5, 1)]:
        xp, xm = x.copy(), x.copy()
        xp[idx] += h
        xm[idx] -= h
        fd = (L(xp) - L(xm)) / (2 * h)
        assert abs(fd - grad[idx]) <= 1e-6 * max(1.0, abs(fd)), (idx, fd, grad[idx])


def test_ssim_validates_without_gpu():
    from vidu4d_b200.ssim import ssim
    a = torch.rand(3, 8, 8)
    with pytest.raises(RuntimeError, match="window_size"):
        ssim(a, a, window_size=7)
    with pytest.raises(RuntimeError, match="same shape"):
        ssim(a, torch.rand(3, 8, 9))
    with pytest.raises(RuntimeError, match="float32"):
        ssim(a.double(), a.double())
    with pytest.raises(RuntimeError, match="img2 requires grad"):
        ssim(a, a.clone().requires_grad_(True))
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        ssim(a, a)
    with pytest.raises(RuntimeError, match="dimension"):
        ssim(torch.rand(8, 8), torch.rand(8, 8))
    with pytest.raises(RuntimeError, match="dimension"):
        ssim(torch.rand(0, 3, 8, 8), torch.rand(0, 3, 8, 8))


def test_ssim_header_matches_library_and_binding(built):
    """include/surfel_ssim.h <-> libsurfel_raster.so <-> _capi.SSIM_PROTOTYPES, kind for kind."""
    from vidu4d_b200 import _capi
    lib = _capi.load()
    hdr = open(os.path.join(ROOT, "include", "surfel_ssim.h")).read()
    body = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    protos = re.findall(r"SR_API\s+([\w\s\*]+?)\b(sr_\w+)\s*\(([^)]*)\)", body)
    assert {name for _, name, _ in protos} == set(_capi.SSIM_SYMBOLS)
    assert not set(_capi.SSIM_SYMBOLS) & set(_capi.SYMBOLS)
    c_kinds = {"int": "int32", "int32_t": "int32", "int64_t": "int64", "float": "float", "double": "double", "void": None}
    py_kinds = {C.c_int32: "int32", C.c_int64: "int64", C.c_float: "float", C.c_double: "double"}

    def c_kind(decl):
        return "pointer" if "*" in decl else c_kinds[decl.replace("const", "").split()[0]]

    def py_kind(t):
        return "pointer" if t in (C.c_void_p, C.c_char_p) else py_kinds[t]
    for ret, name, params in protos:
        assert hasattr(lib, name)
        params = [p for p in params.split(",") if p.strip() not in ("", "void")]
        restype, argtypes = _capi.SSIM_PROTOTYPES[name]
        assert py_kind(restype) == c_kind(ret), name
        assert [py_kind(t) for t in argtypes] == [c_kind(p) for p in params], name


def test_scratch_query(built):
    from vidu4d_b200 import _capi
    lib = _capi.load()
    assert lib.sr_ssim_scratch_bytes(0, 3, 8, 8) == -1 and lib.sr_ssim_scratch_bytes(1, 3, 8, -1) == -1
    a, b = lib.sr_ssim_scratch_bytes(1, 3, 32, 32), lib.sr_ssim_scratch_bytes(8, 3, 512, 512)
    assert 0 < a < b and b >= 8 * 3 * 256 * 4 + 8 * 3 * 256 * 4
    assert lib.sr_ssim_scratch_bytes(70000, 1, 1, 1) >= 70000 * 4


def _calls(lib):
    """{entry point: (valid arguments, invalid arguments)}: the valid ones pass every argument check."""
    nb = int(lib.sr_ssim_scratch_bytes(2, 3, 16, 16))

    def fwd(C_=3, alpha=None, stride=0, bkgd=None, scratch_bytes=nb):
        return [2, C_, 16, 16, D, D, alpha, stride, bkgd, D, D, D, D, scratch_bytes, None]

    def bwd(per_image=1, alpha=D, bkgd=D, dalpha=D):
        return [2, 3, 16, 16, D, D, alpha, 8 * 256, bkgd, D, D, per_image, D, 1, dalpha, D, D, nb, None]
    return {"sr_ssim_forward": (fwd(), fwd(scratch_bytes=nb - 1)),
            "sr_ssim_backward": (bwd(), bwd(per_image=2))}


def test_bad_argument_sets_its_own_message(built):
    from vidu4d_b200 import _capi
    lib = _capi.load()
    nb = int(lib.sr_ssim_scratch_bytes(2, 3, 16, 16))
    bad = dict(_calls(lib))
    extra = [("sr_ssim_forward", [2, 1, 16, 16, D, D, D, 256, D, D, D, D, D, nb, None], b"C = 3"),
             ("sr_ssim_forward", [2, 3, 16, 16, D, D, D, 255, D, D, D, D, D, nb, None], b"alpha_stride"),
             ("sr_ssim_forward", [0, 3, 16, 16, D, D, None, 0, None, D, D, D, D, nb, None], b"must be >= 1"),
             ("sr_ssim_backward", [2, 3, 16, 16, D, D, D, 256, D, D, D, 1, D, 1, None, D, D, nb, None], b"dL_dalpha"),
             ("sr_ssim_backward", [2, 3, 16, 16, D, D, None, 0, None, None, D, 1, D, 0, None, None, D, nb, None], b"NULL")]
    cases = [(n, b, None) for n, (_, b) in bad.items()] + extra
    for name, args, want in cases:
        assert lib.sr_debug_view(0, 0, 0, 0, None) == -1        # a sentinel message from a different failure
        sentinel = lib.sr_last_error()
        rc = getattr(lib, name)(*args)
        msg = lib.sr_last_error()
        assert rc == -1, (name, rc, msg)
        assert msg and msg != sentinel and name.encode() in msg, (name, msg)
        assert want is None or want in msg, (name, msg)


def _cuda_failures_child():
    """Run with no visible device: each SSIM entry point returns SR_ECUDA with the CUDA error's text."""
    if torch.cuda.device_count() != 0:
        print("SKIP: a device is visible")
        return
    from vidu4d_b200 import _capi
    lib = _capi.load()
    cudart = C.CDLL("libcudart.so.12")
    cudart.cudaGetErrorString.restype = C.c_char_p
    texts = {cudart.cudaGetErrorString(e) for e in range(1, 1000)} - {cudart.cudaGetErrorString(999999)}
    for name, (good, _) in _calls(lib).items():
        assert lib.sr_debug_view(0, 0, 0, 0, None) == -1
        rc = getattr(lib, name)(*good)
        msg = lib.sr_last_error()
        assert rc == -2, (name, rc, msg)
        assert b"CUDA error in" in msg and any(msg.endswith(b": " + t) for t in texts), (name, msg)
    print("OK")


def test_cuda_failure_sets_its_own_message(built):
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    flags = ["-s"] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable] + flags + ["-c", "import tests.test_ssim_cpu as t; t._cuda_failures_child()"],
                       cwd=ROOT, env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.strip().splitlines()[-1] in ("OK", "SKIP: a device is visible"), r.stdout
