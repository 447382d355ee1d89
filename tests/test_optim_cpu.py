"""CPU: include/surfel_optim.h given the checks tests/test_host_cpu.py and tests/test_abi_errors_cpu.py give
surfel_raster.h (header <-> library <-> binding, each bad argument's own message, SR_ECUDA without a device); the clip
model (tests/optim_model.py) against torch.nn.utils.clip_grad_norm_; and the margin that lets the device's float64 pow
reproduce the host's fp32 Adam scalars."""
import ctypes as C
import math
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from . import optim_model as om
from .conftest import ROOT

D = 1 << 20      # placeholder DEVICE pointer: never dereferenced (the calls fail before any device work)


def test_optim_header_matches_library_and_binding(built):
    """include/surfel_optim.h <-> libsurfel_raster.so <-> _capi.OPTIM_PROTOTYPES, kind for kind."""
    from vidu4d_b200 import _capi
    lib = _capi.load()
    hdr = open(os.path.join(ROOT, "include", "surfel_optim.h")).read()
    body = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    protos = re.findall(r"SR_API\s+([\w\s\*]+?)\b(sr_\w+)\s*\(([^)]*)\)", body)
    assert {name for _, name, _ in protos} == set(_capi.OPTIM_SYMBOLS)
    assert not set(_capi.OPTIM_SYMBOLS) & (set(_capi.SYMBOLS) | set(_capi.SSIM_SYMBOLS))
    c_kinds = {"int": "int32", "int32_t": "int32", "int64_t": "int64", "float": "float", "double": "double", "void": None}
    py_kinds = {C.c_int32: "int32", C.c_int64: "int64", C.c_float: "float", C.c_double: "double"}

    def c_kind(decl):
        return "pointer" if "*" in decl else c_kinds[decl.replace("const", "").split()[0]]

    def py_kind(t):
        return "pointer" if t in (C.c_void_p, C.c_char_p) else py_kinds[t]
    for ret, name, params in protos:
        assert hasattr(lib, name)
        params = [p for p in params.split(",") if p.strip() not in ("", "void")]
        restype, argtypes = _capi.OPTIM_PROTOTYPES[name]
        assert py_kind(restype) == c_kind(ret), name
        assert [py_kind(t) for t in argtypes] == [c_kind(p) for p in params], name


def test_scratch_query(built):
    from vidu4d_b200 import _capi
    lib = _capi.load()
    assert lib.sr_grad_norm_scratch_bytes(0) == -1 and lib.sr_grad_norm_scratch_bytes(9) == -1
    assert 0 < lib.sr_grad_norm_scratch_bytes(1) < lib.sr_grad_norm_scratch_bytes(7) == 7 * lib.sr_grad_norm_scratch_bytes(1)


def _begin(*b):
    return (C.c_int64 * len(b))(*b)


def _calls(lib):
    """{entry point: (valid arguments, invalid arguments)}: the valid ones pass every argument check."""
    nb = int(lib.sr_grad_norm_scratch_bytes(2))

    def norm(n=2, begin=None, grads=D, extra=D, n_extra=3, scratch=D, scratch_bytes=nb):
        return [n, _begin(0, 5, 9) if begin is None else begin, grads, 1.0, extra, n_extra, 5.0, D, D, None, scratch,
                scratch_bytes, None]

    def adam(n=2, begin=None, step=D, params=D):
        return [n, _begin(0, 5, 9) if begin is None else begin, D, 0.9, 0.999, 1e-15, step, 1.0, None, params, D, D, D, None]
    return {"sr_grad_norm_flat": (norm(), norm(scratch_bytes=nb - 1)),
            "sr_adam_flat_state": (adam(), adam(step=D + 4))}


def test_bad_argument_sets_its_own_message(built):
    from vidu4d_b200 import _capi
    lib = _capi.load()
    nb = int(lib.sr_grad_norm_scratch_bytes(2))
    good = {n: g for n, (g, _) in _calls(lib).items()}

    def with_(name, **kw):
        a = list(good[name])
        idx = {"sr_grad_norm_flat": {"n": 0, "begin": 1, "grads": 2, "extra": 4, "n_extra": 5, "scratch": 10},
               "sr_adam_flat_state": {"n": 0, "begin": 1, "lr": 2, "step": 6, "params": 9}}[name]
        for k, v in kw.items():
            a[idx[k]] = v
        return a
    cases = [(n, b, None) for n, (_, b) in _calls(lib).items()]
    cases[0] = cases[0][:2] + (b"sr_grad_norm_scratch_bytes",)
    cases[1] = cases[1][:2] + (b"8-byte aligned",)
    for name in good:
        cases += [(name, with_(name, n=0), b"n_groups must be in [1, 8]"),
                  (name, with_(name, n=9), b"n_groups must be in [1, 8]"),
                  (name, with_(name, begin=None), b"begin is NULL"),
                  (name, with_(name, begin=_begin(1, 5, 9)), b"begin[0] must be 0"),
                  (name, with_(name, begin=_begin(0, 9, 5)), b"non-decreasing")]
    cases += [("sr_grad_norm_flat", with_("sr_grad_norm_flat", grads=None), b"must not be NULL"),
              ("sr_grad_norm_flat", with_("sr_grad_norm_flat", grads=D + 4), b"16-byte aligned"),
              ("sr_grad_norm_flat", with_("sr_grad_norm_flat", scratch=D + 4), b"scratch must be 8-byte aligned"),
              ("sr_grad_norm_flat", with_("sr_grad_norm_flat", n_extra=-1), b"n_extra must be >= 0"),
              ("sr_grad_norm_flat", with_("sr_grad_norm_flat", extra=None), b"extra_norms is NULL"),
              ("sr_adam_flat_state", with_("sr_adam_flat_state", lr=None), b"NULL"),
              ("sr_adam_flat_state", with_("sr_adam_flat_state", step=None), b"NULL"),
              ("sr_adam_flat_state", with_("sr_adam_flat_state", params=D + 8), b"16-byte aligned")]
    assert nb > 0
    for name, args, want in cases:
        assert lib.sr_debug_view(0, 0, 0, 0, None) == -1        # a sentinel message from a different failure
        sentinel = lib.sr_last_error()
        rc = getattr(lib, name)(*args)
        msg = lib.sr_last_error()
        assert rc == -1, (name, rc, msg)
        assert msg and msg != sentinel and name.encode() in msg, (name, msg)
        assert want is None or want in msg, (name, want, msg)


def _cuda_failures_child():
    """Run with no visible device: each entry point returns SR_ECUDA with the CUDA error's text -- also with no surfels
    (the clip coefficient is still written and the step count still advances)."""
    if torch.cuda.device_count() != 0:
        print("SKIP: a device is visible")
        return
    from vidu4d_b200 import _capi
    lib = _capi.load()
    cudart = C.CDLL("libcudart.so.12")
    cudart.cudaGetErrorString.restype = C.c_char_p
    texts = {cudart.cudaGetErrorString(e) for e in range(1, 1000)} - {cudart.cudaGetErrorString(999999)}
    calls = [(n, g) for n, (g, _) in _calls(lib).items()]
    calls += [(n, [a if i != 1 else _begin(0, 0, 0) for i, a in enumerate(g)]) for n, g in calls]
    for name, good in calls:
        assert lib.sr_debug_view(0, 0, 0, 0, None) == -1
        rc = getattr(lib, name)(*good)
        msg = lib.sr_last_error()
        assert rc == -2, (name, rc, msg)
        assert b"CUDA error in" in msg and any(msg.endswith(b": " + t) for t in texts), (name, msg)
    print("OK")


def test_cuda_failure_sets_its_own_message(built):
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    flags = ["-s"] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable] + flags + ["-c", "import tests.test_optim_cpu as t; t._cuda_failures_child()"],
                       cwd=ROOT, env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.strip().splitlines()[-1] in ("OK", "SKIP: a device is visible"), r.stdout


@pytest.mark.parametrize("scale", [1e-3, 0.3, 1.0, 7.0, 1e4, 0.0, math.inf, math.nan])
def test_clip_model_matches_torch(scale):
    """The model's total and coefficient against torch.nn.utils.clip_grad_norm_ on CPU tensors: norms below and above
    max_norm, a zero total, an Inf and a NaN gradient.  torch sums the per-tensor norms' squares in fp32, the model the
    squares in float64, so the totals agree to a few ulp; given torch's total, the coefficient agrees bit for bit."""
    g = torch.Generator().manual_seed(3)
    shapes = [(40, 3), (40, 45), (40, 1), (7,), (3,)]
    grads = [torch.randn(s, generator=g) * scale if math.isfinite(scale) and scale else torch.zeros(s) for s in shapes]
    if not math.isfinite(scale):
        grads[1][5, 7] = scale
    if scale != 0.0:
        grads[2][0, 0] = 1.0               # reads the applied coefficient back exactly
    params = [torch.zeros(s, requires_grad=True) for s in shapes]
    for p, gr in zip(params, grads):
        p.grad = gr.clone()
    total_t = torch.nn.utils.clip_grad_norm_(params, 5.0)
    # the first three stand for surfel groups (float64 sums of squares), the last two for extras (fp32 norms)
    sums = [float((gr.double() ** 2).sum()) for gr in grads[:3]]
    extra = [float(torch.linalg.vector_norm(gr)) for gr in grads[3:]]
    total, coef = om.clip(sums, extra, 5.0)
    tt = np.float32(total_t.item())
    if math.isnan(scale):
        assert math.isnan(total) and math.isnan(tt) and math.isnan(coef) and math.isnan(float(params[2].grad[0, 0]))
    elif math.isinf(scale):
        assert total == tt == np.inf and coef == 0.0 and float(params[2].grad[0, 0]) == 0.0
    elif scale == 0.0:
        assert total == tt == 0.0 and coef == 1.0 and all(float(p.grad.abs().max()) == 0.0 for p in params)
    else:
        assert abs(float(total) - float(tt)) <= 4 * float(np.spacing(tt)), (total, tt)
        applied = np.float32(params[2].grad[0, 0].item())
        assert om.clip([float(tt) ** 2], [], 5.0)[1] == applied, (scale, applied)
        assert (applied < 1.0) == (scale >= 0.3)


def test_bias_corrections_have_margin_for_device_pow():
    """For every step 2..100 000 at Adam's default betas (torch's doubles), every float64 value within 4 ulp of the host's
    pow(beta, t) gives the same fp32 scalars: sqrt(1 - beta2^t), and lr / (1 - beta1^t) for each of the Stage-3 rates
    as fp32 values.  The device's pow is within 2 ulp, so sr_adam_flat_state reproduces sr_adam_flat's scalars.  Step 1
    takes beta itself, no pow, on both sides: there 2.5e-3 / (1 - 0.9) and 5e-2 / (1 - 0.9) round differently 1 ulp
    below 0.9."""
    t = np.arange(2, 100001)
    lrs = np.float32([1.6e-4, 2.5e-3, 2.5e-3 / 20.0, 5e-2, 5e-3, 1e-3]).astype(np.float64)
    for beta in (0.9, 0.999):
        p = np.array([math.pow(beta, float(k)) for k in t])
        outs = []
        for shift in range(-4, 5):
            c = p.copy()
            for _ in range(abs(shift)):
                c = np.nextafter(c, 1.0 if shift > 0 else 0.0)
            if beta == 0.999:
                outs.append(np.sqrt(1.0 - c).astype(np.float32)[None])
            else:
                outs.append((lrs[:, None] / (1.0 - c)[None]).astype(np.float32))
        assert all(np.array_equal(o, outs[4]) for o in outs), beta
    bc1, sqrt_bc2 = om.bias_corrections(0.9, 0.999, 1)
    assert bc1 == 1.0 - 0.9 and sqrt_bc2 == np.float32(math.sqrt(1.0 - 0.999))
