"""CPU: the delta-skinning models (tests/delta_skin_model.py) against the reference's own outputs (tests/golden/dskin_*.npz),
the fold against the unfolded expression, DeltaSkinMLP's state dict, include/surfel_skin_mlp.h <-> library <-> binding, and
every argument check of the C entry points and of delta_skin()."""
import ctypes as C
import glob
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from . import delta_skin_model as dm
from .conftest import GOLDEN_DIR, ROOT, load_golden

CASES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLDEN_DIR, "dskin_*.npz")))
LEAVES = ("points", "art_r", "art_d", "log_gauss", "cond") + dm.PARAMS
D = 1 << 20      # placeholder DEVICE pointer: never dereferenced (the calls fail before any device work)


def test_fixtures_present():
    assert len(CASES) == 8


def frames(g):
    """The fixture's points as (M,n,3), its upstream gradient as (M,n,B)."""
    pts = g["in_points"]
    M = pts.shape[0] if pts.ndim > 2 else 1
    return pts.reshape(M, -1, 3), g["in_w_delta"].reshape(M, -1, g["in_W3"].shape[0])


@pytest.mark.parametrize("case", CASES)
def test_unfolded_model_matches_reference(case):
    """The torch restatement against the reference: float64 values and every gradient to ~1e-12, float32 values to 1e-5."""
    g = load_golden(case)
    t = {k: torch.from_numpy(g["in_" + k]).double().requires_grad_(True) for k in LEAVES}
    d = dm.unfolded(t["points"], t["art_r"], t["art_d"], t["log_gauss"], {k: t[k] for k in dm.PARAMS}, t["cond"])
    assert float((d.detach() - torch.from_numpy(g["ref64_delta"])).abs().max()) <= 1e-12
    (d * torch.from_numpy(g["in_w_delta"]).double()).sum().backward()
    for k in LEAVES:
        ref = g["ref64_grad_" + k]
        assert np.abs(t[k].grad.numpy() - ref).max() <= 1e-12 * max(1.0, np.abs(ref).max()), (case, k)
    t32 = {k: torch.from_numpy(g["in_" + k]) for k in LEAVES}
    d32 = dm.unfolded(t32["points"], t32["art_r"], t32["art_d"], t32["log_gauss"], {k: t32[k] for k in dm.PARAMS}, t32["cond"])
    assert np.abs(d32.numpy() - g["ref_delta"]).max() <= 1e-5


@pytest.mark.parametrize("case", CASES)
def test_folded_equals_unfolded_in_float64(case):
    g = load_golden(case)
    F = dm.fold_table(g["in_art_r"], g["in_art_d"], g["in_log_gauss"], g["in_W1"], g["in_b1"], g["in_cond"])
    d = dm.folded(g["in_points"], F, g["in_W2"], g["in_b2"], g["in_W3"], g["in_b3"])
    assert np.abs(d - g["ref64_delta"]).max() <= 1e-12


@pytest.mark.parametrize("case", CASES)
def test_chain_reproduces_fixture_and_bounds_its_shadow(case):
    """The kernel's chain on the float64 fold: its values are the reference's float64 delta, its fp32 shadow lies within
    the bound, and the reference's own fp32 delta lies within the bound plus the reference's own rounding (1e-6)."""
    g = load_golden(case)
    pts, gd = frames(g)
    F = dm.fold_table(g["in_art_r"], g["in_art_d"], g["in_log_gauss"], g["in_W1"], g["in_b1"], g["in_cond"])
    o = dm.chain_frames(pts, F, g["in_W2"], g["in_b2"], g["in_W3"], g["in_b3"], gd)
    ref = g["ref64_delta"].reshape(o["delta"].v.shape)
    assert np.abs(o["delta"].v - ref).max() <= 1e-12
    for k in ("delta", "g_x", "g_F", "g_W2", "g_b2", "g_W3", "g_b3"):
        assert dm.within(o[k].f, o[k]) <= 1.0, (case, k)
    assert o["knife"].mean() <= 0.02
    if case == "dskin_b25_clipped":
        assert not o["delta"].v.any() and not g["ref_delta"].any()
        assert all(not o[k].v.any() for k in ("g_x", "g_F", "g_W2", "g_b2", "g_W3", "g_b3"))
        assert all(not g["ref_grad_" + k].any() for k in LEAVES)
    # the gradients of the points and of the last two layers, knife points masked on both sides
    keep = ~o["knife"]
    o = dm.chain_frames(pts, F, g["in_W2"], g["in_b2"], g["in_W3"], g["in_b3"], gd * keep[..., None])
    t = {k: torch.from_numpy(g["in_" + k]).double().requires_grad_(True) for k in LEAVES}
    d = dm.unfolded(t["points"], t["art_r"], t["art_d"], t["log_gauss"], {k: t[k] for k in dm.PARAMS}, t["cond"])
    (d.reshape(gd.shape) * torch.from_numpy(gd * keep[..., None]).double()).sum().backward()
    for k, name in (("g_x", "points"), ("g_W2", "W2"), ("g_b2", "b2"), ("g_W3", "W3"), ("g_b3", "b3")):
        ref = t[name].grad.numpy().reshape(o[k].v.shape)
        assert np.abs(o[k].v - ref).max() <= 1e-11 * max(1.0, np.abs(ref).max()), (case, k)


def test_module_accepts_reference_state_dict():
    from vidu4d_b200.warp import DeltaSkinMLP
    g = load_golden("dskin_b7")
    names = {"W1": "linear_1.0.weight", "b1": "linear_1.0.bias", "W2": "linear_2.0.weight", "b2": "linear_2.0.bias",
             "W3": "linear_final.weight", "b3": "linear_final.bias"}
    mlp = DeltaSkinMLP(7)
    assert set(mlp.state_dict()) == set(names.values())
    mlp.load_state_dict({v: torch.from_numpy(g["in_" + k]) for k, v in names.items()})
    assert torch.equal(mlp.linear_1[0].weight, torch.from_numpy(g["in_W1"])) and mlp.linear_1[0].weight.shape == (64, 21 + 160)


def test_tables_match_the_model_fold():
    """delta_skin_tables (torch, differentiable) against fold_table (NumPy), shared and per frame."""
    from vidu4d_b200.warp import delta_skin_tables
    for case in ("dskin_b25_shared", "dskin_b25_m2_frames"):
        g = load_golden(case)
        t = {k: torch.from_numpy(g["in_" + k]) for k in LEAVES}
        F = delta_skin_tables((t["art_r"], t["art_d"]), t["log_gauss"], t["W1"], t["b1"], t["cond"])
        F64 = dm.fold_table(g["in_art_r"], g["in_art_d"], g["in_log_gauss"], g["in_W1"], g["in_b1"], g["in_cond"])
        assert F.dtype == torch.float32 and tuple(F.shape) == F64.shape
        assert np.abs(F.numpy() - F64).max() <= 2.0 ** -23 * np.abs(F64).max()


def test_header_matches_library_and_binding(built):
    """include/surfel_skin_mlp.h <-> libsurfel_raster.so <-> _capi.SKIN_MLP_PROTOTYPES, kind for kind."""
    from vidu4d_b200 import _capi
    lib = _capi.load()
    hdr = open(os.path.join(ROOT, "include", "surfel_skin_mlp.h")).read()
    body = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    protos = re.findall(r"SR_API\s+([\w\s\*]+?)\b(sr_\w+)\s*\(([^)]*)\)", body)
    assert {name for _, name, _ in protos} == set(_capi.SKIN_MLP_SYMBOLS)
    assert not set(_capi.SKIN_MLP_SYMBOLS) & (set(_capi.SYMBOLS) | set(_capi.SSIM_SYMBOLS) | set(_capi.OPTIM_SYMBOLS))
    c_kinds = {"int": "int32", "int32_t": "int32", "int64_t": "int64", "float": "float", "double": "double", "void": None}
    py_kinds = {C.c_int32: "int32", C.c_int64: "int64", C.c_float: "float", C.c_double: "double"}

    def c_kind(decl):
        return "pointer" if "*" in decl else c_kinds[decl.replace("const", "").split()[0]]

    def py_kind(t):
        return "pointer" if t in (C.c_void_p, C.c_char_p) else py_kinds[t]
    for ret, name, params in protos:
        assert hasattr(lib, name)
        params = [p for p in params.split(",") if p.strip() not in ("", "void")]
        restype, argtypes = _capi.SKIN_MLP_PROTOTYPES[name]
        assert py_kind(restype) == c_kind(ret), name
        assert [py_kind(t) for t in argtypes] == [c_kind(p) for p in params], name


def test_scratch_query(built):
    from vidu4d_b200 import _capi
    lib = _capi.load()
    q = lib.sr_delta_skin_scratch_bytes
    assert q(0, 10, 25) == -1 and q(1, 0, 25) == -1 and q(1, 10, 0) == -1 and q(1, 10, 65) == -1 and q(70000, 1, 1) == -1
    assert q(65535, 40000, 25) == -1                                  # M * N >= 2^31
    part = lambda B: 4 * (B * 65 + 64 * 65 + 256)  # noqa: E731
    assert q(1, 1, 25) == part(25) and q(1, 129, 64) == 2 * part(64)
    assert q(2, 300_000, 25) == 264 * part(25) and q(2, 300_000, 25) < 8 << 20      # a persistent grid: a few MB at any N
    assert q(300, 1000, 7) == 300 * part(7)


def _fwd(M=2, N=100, B=25, Mt=2, width=64, depth=2, null=None):
    ptrs = [None if i == null else D for i in range(7)]
    return [M, N, B, Mt, width, depth] + ptrs + [None]


def _bwd(M=2, N=100, B=25, Mt=2, width=64, depth=2, null=None, scratch_bytes=None):
    from vidu4d_b200 import _capi
    ptrs = [None if i == null else D for i in range(14)]
    nb = int(_capi.load().sr_delta_skin_scratch_bytes(2, 100, 25)) if scratch_bytes is None else scratch_bytes
    return [M, N, B, Mt, width, depth] + ptrs + [nb, None]


BAD = [(dict(width=128), b"width"), (dict(depth=3), b"depth"), (dict(B=0), b"B must be"), (dict(B=65), b"B must be"),
       (dict(M=0), b"M must be"), (dict(N=0), b"N >= 1"), (dict(M=65536, Mt=1), b"M must be"), (dict(Mt=3), b"Mt must be"),
       (dict(M=65535, N=40000, Mt=1), b"too large"), (dict(null=0), b"NULL"), (dict(null=6), b"NULL")]


def test_bad_argument_sets_its_own_message(built):
    from vidu4d_b200 import _capi
    lib = _capi.load()
    cases = [("sr_delta_skin_forward", _fwd(**kw), want) for kw, want in BAD]
    cases += [("sr_delta_skin_backward", _bwd(**kw), want) for kw, want in BAD]
    cases += [("sr_delta_skin_backward", _bwd(null=13), b"NULL"), ("sr_delta_skin_backward", _bwd(scratch_bytes=100), b"scratch")]
    for name, args, want in cases:
        assert lib.sr_debug_view(0, 0, 0, 0, None) == -1        # a sentinel message from a different failure
        sentinel = lib.sr_last_error()
        rc = getattr(lib, name)(*args)
        msg = lib.sr_last_error()
        assert rc == -1, (name, args, rc, msg)
        assert msg and msg != sentinel and name.encode() in msg and want in msg, (name, msg)


def _cuda_failures_child():
    """Run with no visible device: each entry point returns SR_ECUDA with the CUDA error's text."""
    if torch.cuda.device_count() != 0:
        print("SKIP: a device is visible")
        return
    from vidu4d_b200 import _capi
    lib = _capi.load()
    for name, good in (("sr_delta_skin_forward", _fwd(B=64)), ("sr_delta_skin_backward", _bwd(B=25))):
        assert lib.sr_debug_view(0, 0, 0, 0, None) == -1
        rc = getattr(lib, name)(*good)
        msg = lib.sr_last_error()
        assert rc == -2 and b"CUDA error in " + name.encode() in msg, (name, rc, msg)
    print("OK")


def test_cuda_failure_sets_its_own_message(built):
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    flags = ["-s"] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable] + flags + ["-c", "import tests.test_delta_skin_cpu as t; t._cuda_failures_child()"],
                       cwd=ROOT, env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.strip().splitlines()[-1] in ("OK", "SKIP: a device is visible"), r.stdout


def test_python_rejects_bad_arguments():
    from vidu4d_b200.warp import DeltaSkinMLP, delta_skin
    B, M, N = 5, 2, 10
    mlp = DeltaSkinMLP(B)
    ok = dict(points=torch.zeros(M, N, 3), articulation=(torch.zeros(B, 4), torch.zeros(B, 4)), log_gauss=torch.zeros(B, 3), mlp=mlp,
              cond=torch.zeros(160))
    bad = [(dict(points=torch.zeros(N, 2)), "points must be"), (dict(points=torch.zeros(M, 0, 3)), "points must be"),
           (dict(points=torch.zeros(1, 1, 1, 1, 3)), "points must be"), (dict(log_gauss=torch.zeros(B, 2)), "log_gauss must be"),
           (dict(log_gauss=torch.zeros(65, 3)), "log_gauss must be"), (dict(mlp=torch.nn.Linear(3, 3)), "mlp must be"),
           (dict(mlp=DeltaSkinMLP(6)), "mlp has 6 bones"), (dict(articulation=(torch.zeros(B, 4),)), "articulation must be"),
           (dict(articulation=(torch.zeros(3, B, 4), torch.zeros(3, B, 4))), "articulation must be"),
           (dict(articulation=(torch.zeros(B, 4), torch.zeros(M, B, 4))), "articulation must be"),
           (dict(cond=torch.zeros(159)), "cond must be"), (dict(cond=torch.zeros(3, 160)), "cond must be"),
           (dict(points=torch.zeros(M, N, 3, dtype=torch.float64)), "points must be float32"),
           (dict(cond=torch.zeros(160, dtype=torch.float64)), "cond must be float32"),
           (dict(mlp=DeltaSkinMLP(B).double()), r"mlp\.linear_1\.0\.weight must be float32"),
           (dict(), "points must be a CUDA tensor")]
    for kw, want in bad:
        with pytest.raises(RuntimeError, match=want):
            delta_skin(**dict(ok, **kw))
    with pytest.raises(RuntimeError, match="num_bones"):
        DeltaSkinMLP(65)
