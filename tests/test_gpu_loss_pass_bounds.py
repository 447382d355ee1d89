"""The whole Stage-3 loss pass of render_loss_batch, every term on at once, element by element under the rounding-error
bound: the loss kernel with per-frame cameras (csrc/loss.cu), SSIM with the learnable-background composite
(csrc/ssim.cu), the silhouette loss (csrc/mask_loss.cu) and the feature-plane losses (csrc/loss.cu) all write into the
planes the rasterizer backward consumes.

The rasterizer runs in the loop; the models start from its own forward outputs (render, allmap, feature planes), so
their inputs are exact, and the planes are taken where they enter _C.rasterize_gaussians_backward_batch.  Each shared
plane is modelled as the sum of its terms, in the order the kernels add into it, each add one more rounding:
    dL/dcolor  = loss kernel + SSIM
    dL/dalpha  = loss kernel + SSIM (only with a learnable background) + silhouette
    dL/dbkgd   = loss kernel + SSIM, then summed over frames and scaled by the upstream scalar (torch)
    features   = the feature losses' planes * upstream scalar + the caller's own gradient (addcmul)
The backward runs from 1.7 * loss + 0.3 * mean(features[:, 16:21]^2): the upstream scalar is not 1 and the caller's own
gradient lands on channels no fused term touches.  Each tensor prints its headroom, the largest err / (K u B + FLOOR).
"""
import numpy as np
import pytest
import torch

from . import feature_loss_bounds as fb
from . import ssim_bounds as sb
from .error_bound import TINY_U, _E
from .mask_loss_model import mask_loss
from .test_gpu_loss_bounds import _loss_model

pytestmark = pytest.mark.gpu

U, K, FLOOR = 2.0 ** -24, 2.0, float(np.finfo(np.float32).tiny)
F, CF, GM = 22, 16, 21
W_RGB, W_SSIM, LAM_N, LAM_D = 0.8, 0.2, 0.05, 10.0
UP = np.float32(1.7)                    # the upstream scalar of the fused loss
CALLER = np.float32(0.3)                # the caller's own loss on features[:, 16:21]

# name: (W, H, M, learnable background, vis2d)
CASES = {
    "97x41_m1": (97, 41, 1, True, True),
    "65x33_m3": (65, 33, 3, True, True),
    "97x41_m3_no_bkgd": (97, 41, 3, False, True),
    "65x33_m3_no_vis": (65, 33, 3, True, False),
    "256x160_m8": (256, 160, 8, True, True),
}


@pytest.fixture(scope="module")
def dev(built):
    from vidu4d_b200 import _capi
    _capi.load()
    return torch.device("cuda:0")


def _table(M, W, H):
    """Per-frame (tan_x, tan_y, cx_off, cy_off): both tangents differ between frames, non-integer offsets of either sign."""
    f = np.arange(M)
    sgn = np.where(f % 2, -1.0, 1.0)
    return np.stack([0.5 + 0.02 * f, 0.5 * H / W * (1.0 - 0.03 * f), sgn * (0.08 * W + 0.375),
                     -sgn * (0.08 * H + 0.3125)], 1).astype(np.float32)


def _ratio(x, e, skip=None):
    r = np.abs(np.asarray(x, np.float64) - e.v) / (K * U * e.b + FLOOR)
    r = np.where(np.isnan(x), np.inf, r)
    return r if skip is None else np.where(skip, 0.0, r)


def _cmp(name, what, x, e, report, skip=None):
    r = _ratio(x, e, skip)
    i = int(np.argmax(r))
    report[what] = max(report.get(what, 0.0), float(r.flat[i]))
    assert r.flat[i] <= 1.0, (name, what, np.unravel_index(i, r.shape), "gpu", np.asarray(x).flat[i], "model", e.v.flat[i],
                              "bound", K * U * e.b.flat[i] + FLOOR)


def _abs(v, bound):
    """An _E from a value and an absolute error bound."""
    return _E(v, np.asarray(bound, np.float64) / U)


def _run(name, W, H, M, with_bk, with_vis, dev, monkeypatch, hook=None, per_frame=False):
    """hook(args, kwargs, out, pc): called inside the spied rasterizer backward, before the real one, with its arguments,
    render_loss_batch's outputs and the surfel cloud; per_frame: Stage 3's per-frame positions and orientations (the
    cloud's own, moved per frame), as means3D / rotations overrides.  Returns (out, dL/dallmap, the spied call: its
    arguments and the real backward's gradients)."""
    from vidu4d_b200 import rasterizer as RZ
    from vidu4d_b200.renderer import PipelineParams, render_loss_batch
    from dataclasses import replace
    from .test_gpu_feature_loss import _scene
    P = 20000 if M < 8 else 60000
    bc, _, mk = _scene(P, W, H, M, dev, seed=W + H + M)
    rows = _table(M, W, H)
    bc = replace(bc, intrinsics=torch.from_numpy(rows).to(dev))
    g = torch.Generator(device=dev).manual_seed(W * H + M)
    rgb = torch.rand((M, 3, H, W), device=dev, generator=g)
    vis = None
    if with_vis:
        vis = (torch.rand((M, H, W), device=dev, generator=g) > 0.2) * (0.5 + torch.rand((M, H, W), device=dev, generator=g))
    mask = (torch.rand((M, H, W), device=dev, generator=g) > 0.5).float()
    ftgt = torch.randn((M, CF, H, W), device=dev, generator=g) * 0.3
    feat = torch.randn((P, F), device=dev, generator=g) * 0.3
    feat[:, GM] = torch.rand((P,), device=dev, generator=g)
    feat.requires_grad_(True)
    det = torch.ones(M, device=dev)
    if M > 1:
        det[1] = 0.0
    wf = torch.tensor([1e-2, 7e-3], device=dev)
    wm = torch.tensor([0.1], device=dev)
    bk = torch.tensor([0.3, 0.5, 0.2], device=dev, requires_grad=True) if with_bk else None
    seen, spied, held = [], {}, {}
    real = RZ._C.rasterize_gaussians_backward_batch
    pc = mk()
    over = {}
    if per_frame:
        f_ = torch.arange(M, device=dev, dtype=torch.float32)[:, None, None]
        dx = torch.randn((1, P, 3), device=dev, generator=g) * 0.002
        dq = torch.randn((1, P, 4), device=dev, generator=g) * 0.02
        over = dict(means3D=pc.get_xyz[None] + f_ * dx, rotations=torch.nn.functional.normalize(pc._rotation[None] + f_ * dq, dim=-1))

    def spy(*a, **k):
        seen.append((a[11].clone(), a[12].clone(), k["dL_dout_features"].clone(), k.get("grad_scale"),
                     k.get("features_grad_scale")))
        if hook is not None:
            hook(a, k, held["out"], pc)
        spied.update(args=a, kwargs=k, grads=real(*a, **k))
        return spied["grads"]
    monkeypatch.setattr(RZ._C, "rasterize_gaussians_backward_batch", staticmethod(spy))
    try:
        out = render_loss_batch(bc, pc, PipelineParams(), torch.zeros(3, device=dev), rgb, vis2d=vis, mask_gt=mask,
                                learnable_bkgd=bk, w_rgb=W_RGB, lambda_normal=LAM_N, lambda_dist=LAM_D, features=feat,
                                feature_target=ftgt, is_detected=det, gauss_mask_channel=GM, feature_loss_weights=wf,
                                w_ssim=W_SSIM, mask_loss_weight=wm, **over)
        held["out"] = out
        (float(UP) * out["loss"] + float(CALLER) * out["features"][:, 16:21].square().mean()).backward()
        torch.cuda.synchronize()
    finally:
        monkeypatch.undo()
    assert len(seen) == 1
    dLc, dLa, dLf, gscale, fgscale = seen[0]
    assert float(gscale) == float(UP) and fgscale is None       # the feature planes arrive scaled already
    n = lambda t: None if t is None else t.detach().cpu().numpy()  # noqa: E731
    color, am, planes = n(out["render"]), n(out["allmap"]), n(out["features"])
    dLc, dLa, dLf = n(dLc), n(dLa), n(dLf)
    tgt, visn, maskn, detn, ftn, wvt = n(rgb), n(vis), n(mask), n(det), n(ftgt), n(bc.world_view_transform)
    bkn = n(bk)
    alpha = np.ascontiguousarray(am[:, 1])
    report, knives = {}, {"rgb": 0, "stencil": 0, "feature": 0}
    nblocks = -(-W // 32) * -(-H // 8)
    depth = 5 + 8 + nblocks

    # ---- SSIM on the final colour, its backward on the forward's running-error maps (upstream -w_ssim per frame)
    fw = sb.forward(color, tgt, alpha if with_bk else None, bkn if with_bk else None)
    assert not fw["ill"].any(), name
    zeros_a, zeros_b = np.zeros((M, H, W), np.float32), np.zeros((M, 3), np.float32)
    bw = sb.backward(color, tgt, [fw["A"], fw["B"], fw["Cm"]], np.full(M, -W_SSIM, np.float32), 1,
                     alpha if with_bk else None, bkn if with_bk else None, None, zeros_a, zeros_b)
    ssim_want = (sb.ONE - fw["ssim_img"]) * sb._k(W_SSIM, np.float32(W_SSIM))
    _cmp(name, "ssim_terms", n(out["ssim_terms"]), ssim_want, report)

    # ---- the silhouette loss: added into dL/dalpha last
    ml = mask_loss(alpha, maskn, visn, detn, 0.1)
    assert np.array_equal(n(out["mask_counts"]), ml["counts"]), name
    mt = n(out["mask_terms"]).astype(np.float64)
    assert np.all(np.abs(mt - ml["terms"]) <= ml["terms_bound"] + 1e-30), (name, mt, ml["terms"], ml["terms_bound"])
    report["mask_terms"] = float((np.abs(mt - ml["terms"]) / (ml["terms_bound"] + 1e-30)).max())

    # ---- the loss kernel, frame by frame with its own camera row, and the planes it shares
    o = dict(w_rgb=W_RGB, w_mask=0.0, lambda_normal=LAM_N, lambda_dist=LAM_D, depth_ratio=0.0)
    inv_n = np.float32(1.0) / np.float32(H * W)
    dlb_parts = []
    term_want = np.zeros((M, 4))
    term_bound = np.zeros((M, 4))
    for f in range(M):
        tag = f"{name} frame {f}"
        mdl = _loss_model(color[f], am[f], wvt[f], tgt[f], o, None if visn is None else visn[f], maskn[f], None,
                          bkn, cam=tuple(float(x) for x in rows[f]))
        kn, own, nbk = mdl["rgb_knife"], mdl["st_own"], mdl["st_nb"]
        knives["rgb"] += int(kn.sum())
        knives["stencil"] += int(own.sum())
        for ch in range(3):
            _cmp(tag, "dL_dcolor", dLc[f, ch], mdl["gcol"][ch] + bw["gxv"][f, ch], report, skip=kn)
        p1 = mdl["planes"][1]
        if with_bk:
            p1 = p1 + bw["dalpha"][f]
        p1 = p1 + _abs(ml["grad"][f], ml["grad_bound"][f])
        _cmp(tag, "dL_dallmap[1]", dLa[f, 1], p1, report, skip=nbk | kn)
        for p in (0, 5):
            _cmp(tag, f"dL_dallmap[{p}]", dLa[f, p], mdl["planes"][p], report, skip=nbk)
        for p in (2, 3, 4):
            _cmp(tag, f"dL_dallmap[{p}]", dLa[f, p], mdl["planes"][p], report, skip=own)
        assert (dLa[f, 6] == np.float32(LAM_D) * inv_n).all() and (dLa[f, 7] == 0).all(), tag
        for k in range(4):
            t = mdl["part"][k]
            term_want[f, k], term_bound[f, k] = t.v.sum(), t.b.sum() + depth * np.abs(t.v).sum()
        if with_bk:
            a64 = 1.0 - am[f, 1].astype(np.float64)
            lb = []
            for ch in range(3):
                t = mdl["part"][4 + ch]
                # at an rgb knife the sign, so the pixel's part, may be any of -s, 0, s: its part's bound covers 2 s (1 - a)
                s = float(W_RGB * inv_n / 3.0)
                lb.append(_E(t.v.sum(), t.b.sum() + (2.0 * s * np.abs(a64[kn]).sum()) / (K * U)
                             + depth * np.abs(t.v).sum()))
            dlb_parts.append([lb[ch] + bw["dbkgd"][f, ch] for ch in range(3)])
    _cmp(name, "terms", n(out["terms"]), _E(term_want, term_bound), report)

    # ---- the feature losses on the rendered planes, with the GPU's counts; the planes handed to the rasterizer
    px = fb.pixel_terms(planes, ftn, maskn, detn, alpha, GM)
    fcounts, fterms = n(out["feature_counts"]), n(out["feature_terms"])
    knives["feature"] = sum(int(k.sum()) for k in px["knife"].values())
    frep = {}
    _, ftm, fg = fb.scaled(px, fcounts, n(wf), GM)
    for k in range(2):
        kn = px["knife"][k]
        want = ((px["v"][k].v > 0) & ~kn).reshape(M, -1).sum(1)
        assert np.all((fcounts[:, k] >= want) & (fcounts[:, k] <= want + kn.reshape(M, -1).sum(1))), (name, k)
        fb._within(name, f"feature_terms[{k}]", fterms[:, k], ftm[k], frep)
    report.update(frep)
    up = _E.leaf(UP)
    nf = float(M * 5 * H * W)
    for c in range(F):
        if c in fg:
            e = fg[c] * up
            skip = px["knife"][1 if c == GM else 0]
        elif 16 <= c < 21:      # the caller's 0.3 * mean(x^2): 0.3f / n, times 2 x; four roundings at most
            v = float(CALLER) / nf * 2.0 * planes[:, c].astype(np.float64)
            e, skip = _E(v, 4.0 * np.abs(v) + 4.0 * TINY_U), None
        else:
            assert (dLf[:, c] == 0).all(), (name, c)
            continue
        _cmp(name, "dL_dout_features", dLf[:, c], e, report, skip=skip)

    # ---- learnable_bkgd.grad = sum over frames of dL/dbkgd, times the upstream scalar
    if with_bk:
        gb = n(bk.grad).astype(np.float64)
        for ch in range(3):
            parts = [dlb_parts[f][ch] for f in range(M)]
            sv = sum(p.v for p in parts)
            sbnd = sum(p.b for p in parts) + M * sum(np.abs(p.v) for p in parts)
            e = _E(sv, sbnd) * up
            _cmp(name, "learnable_bkgd.grad", gb[ch], e, report)
    else:
        assert dlb_parts == []

    # ---- loss: the sum of every term, in fp32 by torch
    allt = [n(out[k]).astype(np.float64).ravel() for k in ("terms", "ssim_terms", "mask_terms", "feature_terms")]
    tv = np.concatenate(allt)
    mb = (term_bound.sum() + ssim_want.b.sum() + ml["terms_bound"].sum() / U + sum(ftm[k].b.sum() for k in ftm))
    lw = term_want.sum() + ssim_want.v.sum() + ml["terms"].sum() + sum(ftm[k].v.sum() for k in ftm)
    _cmp(name, "loss", float(out["loss"]), _E(lw, mb + len(tv) * np.abs(tv).sum()), report)
    _cmp(name, "loss = sum of terms", float(out["loss"]), _E(tv.sum(), len(tv) * np.abs(tv).sum()), report)
    print(f"\n[{name}] M={M} {W}x{H} bkgd={with_bk} vis={with_vis}: knife rgb {knives['rgb']} stencil "
          f"{knives['stencil']} feature {knives['feature']} of {M * W * H} px; "
          + ", ".join(f"{k} {v:.3g}" for k, v in report.items()))
    assert sum(knives.values()) <= 8 + 1e-3 * M * W * H, (name, knives)
    spied.update(feat=feat, over=over, pc=pc)
    return out, dLa, spied


@pytest.mark.parametrize("name", list(CASES))
def test_loss_pass_every_term_elementwise(name, dev, monkeypatch):
    W, H, M, with_bk, with_vis = CASES[name]
    out, dLa, _ = _run(name, W, H, M, with_bk, with_vis, dev, monkeypatch)
    assert float(out["mask_terms"].abs().sum()) > 0 and float(out["ssim_terms"].abs().min()) > 0
    if M > 1:                   # the undetected frame: no feature count, no silhouette count
        assert int(out["feature_counts"][1, 0]) == 0 and int(out["mask_counts"][1]) == 0
        assert int(out["feature_counts"][0, 0]) > 0
