"""The restated SSIM op and its bound (tests/ssim_bounds.py), on the CPU: its values equal the float64 model
(tests/ssim_model.py) far inside the bound; its fp32 shadow lies within K u B + FLOOR of its value for every case the
GPU test runs and every tests/golden/ssim_*.npz input; and the bound is not vacuous."""
import glob
import os

import numpy as np
import pytest

from . import ssim_bounds as sb
from . import ssim_model as sm
from .conftest import GOLDEN_DIR

FIXTURES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLDEN_DIR, "ssim_*.npz")))
MAPS = ("A", "B", "Cm")

# the largest tol / max |value| per tensor, measured on these inputs: about 1/2 to 1/10 of these ceilings.  The maps reach
# 0.06 on the near-constant case, where sigma^2 cancels to ~1e-6 and the 1/C2 factor amplifies it; the HDR cases are
# guarded on the backward only (their maps are well conditioned only up to the 1/64 rule, by construction).
CEIL = {"maps": 0.15, "means": 1e-2, "dimg1": 2e-3, "dalpha": 5e-6, "dbkgd": 2e-3}


def _tol(e):
    return sb.K * sb.U * e.b + sb.FLOOR


def _pin(what, e, ref, skip=None):
    """The restatement's value equals the model's far inside the bound: |v - ref| <= 1e-3 tol."""
    ref = np.broadcast_to(np.asarray(ref, np.float64), e.v.shape)
    bad = ~(np.abs(e.v - ref) <= 1e-3 * _tol(e))
    if skip is not None:
        bad &= ~skip
    assert not bad.any(), (what, np.argwhere(bad)[:4].tolist())


def _model_refs(c):
    """ssim_model's map, maps, means and the VJP of the op's backward (composite included) in float64."""
    x = sb.image_x(c["img1"], c["alpha"], c["bkgd"]).v
    y = c["img2"].astype(np.float64)
    N = x.shape[0]
    A, B, Cm = sm.maps(x, y)
    up = c["dL_dssim"].astype(np.float64)
    gx = sm.vjp_mean(x, y, up if c["per_image"] else up[0], size_average=not c["per_image"])
    r = dict(A=A, B=B, Cm=Cm, m=sm.ssim_map(x, y), ssim_img=sm.ssim(x, y, size_average=False), ssim_mean=sm.ssim(x, y),
             dimg1=gx if c["dimg1"] is None else c["dimg1"] + gx)
    if c["alpha"] is not None:
        bk = c["bkgd"].astype(np.float64)[None, :, None, None]
        r["dalpha"] = c["dalpha"] - (gx * bk).sum(1)
        r["dbkgd"] = c["dbkgd"] + (gx * (1.0 - c["alpha"][:, None].astype(np.float64))).sum((2, 3))
    assert r["ssim_img"].shape == (N,)
    return r, np.stack([A, B, Cm])


def check_case(c):
    """Pins the values, checks the shadow; returns (forward, backward, {tensor: tol / max |value|})."""
    ref, maps64 = _model_refs(c)
    fw = sb.forward(c["img1"], c["img2"], c["alpha"], c["bkgd"])
    ill = fw["ill"]
    bad_img = ill.reshape(ill.shape[0], -1).any(1)
    for k in MAPS + ("m",):
        _pin(k, fw[k], ref[k], ill)
    _pin("ssim_img", fw["ssim_img"], ref["ssim_img"], bad_img)
    if not bad_img.any():
        _pin("ssim_mean", fw["ssim_mean"], ref["ssim_mean"])
    # the backward's values on exact maps; its bound (and shadow) on the forward's fp32 maps
    args = (c["img1"], c["img2"])
    kw = dict(alpha=c["alpha"], bkgd=c["bkgd"], dimg1=c["dimg1"], dalpha=c.get("dalpha"), dbkgd=c.get("dbkgd"))
    bw64 = sb.backward(*args, maps64, c["dL_dssim"], c["per_image"], **kw)
    for k in ("dimg1", "dalpha", "dbkgd"):
        if k in bw64:
            _pin(k, bw64[k], ref[k])
    bw = sb.backward(*args, sb.fp32_maps(fw), c["dL_dssim"], c["per_image"], **kw)
    for k in MAPS + ("m",):
        assert sb.within(fw[k].f, fw[k], ill) <= 1.0, k
    assert sb.within(fw["ssim_img"].f, fw["ssim_img"], bad_img) <= 1.0
    if not bad_img.any():
        assert sb.within(fw["ssim_mean"].f, fw["ssim_mean"]) <= 1.0
    rel = {}
    for k, e in list(bw.items()) + [(k, fw[k]) for k in MAPS + ("ssim_img",)]:
        if k == "gxv":
            continue
        assert sb.within(e.f, e, ill if k in MAPS else None) <= 1.0, k
        keep = ~ill if k in MAPS else np.ones(e.v.shape, bool)
        if keep.any() and np.abs(e.v[keep]).max() > 0:
            rel[k] = float(_tol(e)[keep].max() / np.abs(e.v[keep]).max())
    return fw, bw, rel


@pytest.mark.parametrize("name", list(sb.CASES))
def test_restatement_equals_model_and_shadow_meets_bound(name):
    c = sb.make_case(name)
    fw, bw, rel = check_case(c)
    kind = sb.CASES[name][1]
    if kind != "hdr":
        assert not fw["ill"].any(), (name, int(fw["ill"].sum()))
    for k, r in rel.items():
        if kind == "hdr" and k not in ("dimg1", "dalpha", "dbkgd"):
            continue
        ceil = CEIL["maps" if k in MAPS else "means" if k == "ssim_img" else k]
        assert r < ceil, (name, k, r)


@pytest.mark.parametrize("name", FIXTURES)
def test_fixture_inputs_shadow_meets_bound(name):
    c = sb.fixture_case(name)
    fw, _, _ = check_case(c)
    assert not fw["ill"].any() or "hdr" in name


def test_upstream_spread():
    """Per-image upstream values 1 .. 1e-6 with one negative and one exactly 0; a scalar without per_image."""
    g = sb.upstream(5, 1, None)
    assert g[0] == 1 and g[1] < 0 and g[-1] == 0 and np.isclose(np.abs(g[-2]), 10 ** -4.5)
    assert sb.upstream(3, 0, None).shape == (1,)


def test_bound_catches_a_one_tap_shift():
    """A filter whose window is off by one pixel moves every map far outside the bound on textured input: the bound is
    tight enough to see a halo shifted by one."""
    c = sb.make_case("seam_31x33")
    fw = sb.forward(c["img1"], c["img2"], c["alpha"], c["bkgd"])
    x = np.roll(c["img1"], 1, -1)
    shifted = sb.forward(x, c["img2"], c["alpha"], c["bkgd"])
    assert sb.within(shifted["A"].v, fw["A"]) > 100


def test_kernel_constants():
    """The reduction depth follows csrc/ssim.cu's launch constants."""
    src = open(os.path.join(os.path.dirname(__file__), "..", "vidu4d_b200", "csrc", "ssim.cu")).read()
    for name, val in (("SS_T", sb.SS_T), ("SS_R", sb.SS_R), ("SS_THREADS", sb.SS_THREADS)):
        assert f"constexpr int {name} = {val};" in src, name
    assert sb.LEVELS == 3 + 5 + 7
