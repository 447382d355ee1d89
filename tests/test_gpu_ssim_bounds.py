"""Every element of the fused SSIM op (csrc/ssim.cu, sr_ssim_forward / sr_ssim_backward) -- the maps A, B, Cm, ssim_img,
ssim_mean, dL/dimg1, dL/dalpha and dL/dbkgd -- against the float64 restatement of its kernels (tests/ssim_bounds.py,
pinned to tests/ssim_model.py by tests/test_ssim_bounds_cpu.py), under the a-priori rounding-error bound
|gpu - value| <= K u B + FLOOR, with K = 2.

The entry points are driven through _capi.call, so the maps the backward reads are visible; the backward's bound is
evaluated on those fp32 maps as leaves.  Ill-conditioned pixels (ssim_bounds.py) are not compared in the maps, nor the
means of an image holding one; each case prints their count and the largest err / tol per tensor, and keeps the count
within a few times the count measured on an H100 (ILL_MEASURED).  The backward needs no exclusions.

The cases (ssim_bounds.CASES) put the image inside one window, on 32-px tile seams and one-pixel last tiles, at C = 1, 2,
3 and 5, and at render_loss_batch's M = 4, 3 x 120 x 160; the contents are textured, piecewise constant (sigma = 0),
near-constant, exactly 0 over a region, and HDR with negative values; per_image 0 and 1 with the per-image upstream
spread over 1 .. 1e-6, one negative and one exactly 0; accumulate 0 and 1 onto a random prefill; and the background
composite with alpha_stride = H W and with alpha as plane 1 of an 8-plane allmap.  Every output buffer has a sentinel
guard tail, the allmap's other seven planes hold a sentinel, and all of them must come back bit-identical.
"""
import numpy as np
import pytest
import torch

from . import ssim_bounds as sb
from .test_ssim_bounds_cpu import FIXTURES

pytestmark = pytest.mark.gpu

# ill-conditioned pixels per case, measured on an H100 80GB HBM3 (a property of the inputs and the bound: 0 on [0, 1])
ILL_MEASURED = {**{k: 0 for k in sb.CASES}, "seam_65x97": 728, "hdr_allmap": 268}
SENT = -1234.5          # sentinel of every byte the op must not write
GUARD = 97              # floats of guard tail after each output buffer


@pytest.fixture(scope="module")
def dev(built):
    from vidu4d_b200 import _capi
    _capi.load()
    return torch.device("cuda:0")


def _t(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def _guarded(n, dev, fill=None):
    """A float buffer of n floats plus a sentinel tail; the first n hold `fill` (flat) or the sentinel."""
    buf = torch.full((n + GUARD,), SENT, dtype=torch.float32, device=dev)
    if fill is not None:
        buf[:n] = _t(np.asarray(fill, np.float32).reshape(-1), dev)
    return buf


def _gpu(c, dev):
    """Forward with and without maps, then backward; returns numpy outputs and the sentinel checks' verdicts."""
    from vidu4d_b200 import _capi
    N, C, H, W = c["img1"].shape
    HW, NP = H * W, N * C * H * W
    img1, img2 = _t(c["img1"], dev), _t(c["img2"], dev)
    alpha = bk = dal = dbk = None
    stride = 0
    if c["composite"] == "allmap":
        stride = 8 * HW
        am = torch.full((N, 8, H, W), SENT, dtype=torch.float32, device=dev)
        am[:, 1] = _t(c["alpha"], dev)
        dam = torch.full((N, 8, H, W), SENT, dtype=torch.float32, device=dev)
        dam[:, 1] = _t(c["dalpha"], dev)
        am0, dam0 = am.clone(), dam.clone()
        alpha, dal = am[:, 1], dam[:, 1]          # strided views: data_ptr() is plane 1 of image 0
    elif c["composite"] == "hw":
        stride = HW
        alpha, dal = _guarded(N * HW, dev, c["alpha"]), _guarded(N * HW, dev, c["dalpha"])
    if c["composite"] is not None:
        bk, dbk = _t(c["bkgd"], dev), _guarded(N * 3, dev, c["dbkgd"])
    nbytes = int(_capi.load().sr_ssim_scratch_bytes(N, C, H, W))
    scratch = torch.empty((nbytes,), dtype=torch.uint8, device=dev)
    maps, simg, mean = _guarded(3 * NP, dev), _guarded(N, dev), _guarded(1, dev)
    _capi.call("sr_ssim_forward", dev, N, C, H, W, img1, img2, alpha, stride, bk, simg, mean, maps, scratch, nbytes)
    simg0, mean0 = _guarded(N, dev), _guarded(1, dev)
    _capi.call("sr_ssim_forward", dev, N, C, H, W, img1, img2, alpha, stride, bk, simg0, mean0, None, scratch, nbytes)
    d = _guarded(NP, dev, c["dimg1"])
    up = _t(c["dL_dssim"], dev)
    _capi.call("sr_ssim_backward", dev, N, C, H, W, img1, img2, alpha, stride, bk, maps, up, c["per_image"], d,
               c["accumulate"], dal, dbk, scratch, nbytes)
    torch.cuda.synchronize(dev)
    n = lambda t: t.cpu().numpy()  # noqa: E731
    out = dict(maps=n(maps[:3 * NP]).reshape(3, N, C, H, W), ssim_img=n(simg[:N]), ssim_mean=n(mean[:1]).reshape(()),
               dimg1=n(d[:NP]).reshape(N, C, H, W))
    tails = [maps, simg, mean, simg0, mean0, d]
    if c["composite"] == "allmap":
        out["dalpha"], out["dbkgd"] = n(dam[:, 1]), n(dbk[:N * 3]).reshape(N, 3)
        planes = [p for p in range(8) if p != 1]
        assert torch.equal(am, am0), "the allmap input changed"
        assert torch.equal(dam[:, planes], dam0[:, planes]), "dL/dallmap changed outside plane 1"
        tails.append(dbk)
    elif c["composite"] == "hw":
        out["dalpha"], out["dbkgd"] = n(dal[:N * HW]).reshape(N, H, W), n(dbk[:N * 3]).reshape(N, 3)
        tails += [dal, dbk]
    for i, t in enumerate(tails):
        assert (t[-GUARD:] == SENT).all(), ("guard tail written", i)
    assert torch.equal(simg0[:N], simg[:N]) and torch.equal(mean0[:1], mean[:1]), "the forward without maps differs"
    return out


def _cmp(name, what, mine, e, report, skip=None):
    r = sb.within(mine, e, skip)
    report[what] = max(report.get(what, 0.0), r)
    if r > 1.0:
        tol = sb.K * sb.U * e.b + sb.FLOOR
        ratio = np.abs(np.asarray(mine, np.float64) - e.v) / tol
        if skip is not None:
            ratio = np.where(skip, 0.0, ratio)
        ratio = np.where(np.isnan(mine), np.inf, ratio)
        i = int(np.argmax(ratio))
        idx = np.unravel_index(i, np.shape(mine))
        raise AssertionError((name, what, "element", idx, "gpu", np.asarray(mine).flat[i], "value", e.v.flat[i],
                              "bound", tol.flat[i]))


def run(name, c, dev, cap=None):
    """The GPU op, the model (its backward on the GPU's maps) and every element compared.  Returns (model fw, bw, gpu)."""
    g = _gpu(c, dev)
    fw = sb.forward(c["img1"], c["img2"], c["alpha"], c["bkgd"])
    bw = sb.backward(c["img1"], c["img2"], g["maps"], c["dL_dssim"], c["per_image"], c["alpha"], c["bkgd"], c["dimg1"],
                     c.get("dalpha"), c.get("dbkgd"))
    ill = fw["ill"]
    bad_img = ill.reshape(ill.shape[0], -1).any(1)
    report = {}
    for i, k in enumerate(("A", "B", "Cm")):
        _cmp(name, k, g["maps"][i], fw[k], report, ill)
    _cmp(name, "ssim_img", g["ssim_img"], fw["ssim_img"], report, bad_img)
    if not bad_img.any():
        _cmp(name, "ssim_mean", g["ssim_mean"], fw["ssim_mean"], report)
    for k in ("dimg1", "dalpha", "dbkgd"):
        if k in g:
            _cmp(name, k, g[k], bw[k], report)
    if c["per_image"]:             # an image whose upstream is exactly 0 contributes exactly nothing
        for i in np.flatnonzero(c["dL_dssim"] == 0):
            want = 0.0 if c["dimg1"] is None else c["dimg1"][i]
            assert np.array_equal(g["dimg1"][i], np.broadcast_to(want, g["dimg1"][i].shape)), (name, "zero upstream", i)
            if "dalpha" in g:
                assert np.array_equal(g["dalpha"][i], c["dalpha"][i]) and np.array_equal(g["dbkgd"][i], c["dbkgd"][i])
    n_ill = int(ill.sum())
    print(f"\n[{name}] {tuple(c['img1'].shape)}: ill-conditioned {n_ill}; "
          + ", ".join(f"{k} {v:.3g}" for k, v in report.items()))
    if cap is not None:
        assert n_ill <= cap, (name, "ill-conditioned pixels", n_ill)
    return fw, bw, g


@pytest.mark.parametrize("name", list(sb.CASES))
def test_elementwise(name, dev):
    c = sb.make_case(name)
    run(name, c, dev, cap=4 * ILL_MEASURED[name])
    if sb.CASES[name][1] != "hdr":
        assert ILL_MEASURED[name] == 0


@pytest.mark.parametrize("name", FIXTURES)
def test_fixture_inputs_elementwise(name, dev):
    run(name, sb.fixture_case(name), dev, cap=0)


def test_production_call(dev):
    """render_loss_batch's SSIM term (renderer._ssim_term) on constructed colour and allmap, no rasterizer: dL/dcolor,
    dL/dallmap and dL/dbkgd prefilled by sr_render_loss_batch.  The term runs the op with per_image = 1, accumulate = 1,
    g = -w_ssim and alpha = plane 1 of the allmap, returns (1 - ssim_f) w_ssim, and adds its gradient after the loss
    terms'."""
    from vidu4d_b200.renderer import _ssim_term
    from .test_gpu_loss_bounds import OPTS, TANX, TANY, _frames, _loss_gpu, _wvts
    M, H, W, w_ssim = 4, 120, 160, 0.2
    am, color, target, vis, _ = _frames(M, W, H, seed=31, with_vis=True, with_bk=True)
    am = np.nan_to_num(am, nan=2.0, posinf=2.0)
    o = OPTS["all_bkgd"]
    T = lambda a: _t(a, dev)  # noqa: E731
    colt, amt, tgt, vist = T(color), T(am), T(target), T(vis)
    rng = np.random.default_rng(5)
    mask, wt = T(rng.uniform(0, 1, (M, H, W)).astype(np.float32)), T(rng.uniform(0.5, 1.5, (M, H, W)).astype(np.float32))
    bk = T(sb.BKGD)
    wvt = _wvts(M, 3).contiguous().to(dev)
    _, dLc, dLa, dLb, _ = _loss_gpu(M, W, H, o, colt, amt, wvt, tgt, vist, mask, wt, bk, dev)
    c0, a0, b0 = dLc.cpu().numpy(), dLa.cpu().numpy(), dLb.cpu().numpy()
    assert np.isfinite(c0).all() and np.isfinite(a0[:, 1]).all() and np.isfinite(b0).all()
    terms = _ssim_term(M, H, W, colt, amt, tgt, bk, w_ssim, dLc, dLa, dLb)
    torch.cuda.synchronize(dev)
    # the op-level call it makes, with the loss pass's gradients as the prefill
    c = dict(img1=color, img2=target, per_image=1, accumulate=1, composite="allmap", alpha=am[:, 1], bkgd=sb.BKGD,
             dL_dssim=np.full(M, -w_ssim, np.float32), dimg1=c0, dalpha=a0[:, 1], dbkgd=b0)
    fw, bw, g = run("production_call", c, dev, cap=0)
    assert np.array_equal(dLc.cpu().numpy(), g["dimg1"]), "dL/dcolor is not the op's accumulate=1, g=-w_ssim result"
    got_a = dLa.cpu().numpy()
    assert np.array_equal(got_a[:, 1], g["dalpha"]) and np.array_equal(dLb.cpu().numpy(), g["dbkgd"])
    planes = [p for p in range(8) if p != 1]
    assert np.array_equal(got_a[:, planes], a0[:, planes]), "the SSIM term wrote outside dL/dalpha"
    w = sb._k(w_ssim, np.float32(w_ssim))
    want = (sb.ONE - fw["ssim_img"]) * w
    _cmp("production_call", "ssim_terms", terms.cpu().numpy(), want, {})
