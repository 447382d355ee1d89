"""GPU tests of the flat surfel store (SURVEY.md 8(f) row N4): the one-kernel Adam step against torch.optim.Adam, and the
one-gather densify / prune against a step-by-step restatement of the reference's procedure
(gs/scene/gaussian_model.py:291-446), same random draws -- parameters and Adam moments must come out identical."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev(built):
    from vidu4d_b200 import _capi
    _capi.load()
    return torch.device("cuda:0")


def _model(P, dev, seed=0):
    from vidu4d_b200.surfel_store import FlatSurfelModel
    from vidu4d_b200.synthetic import object_scene
    sc = object_scene(P, seed=seed)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    op = np.clip(sc.opacities, 1e-6, 1 - 1e-6)
    return FlatSurfelModel(t(sc.means3D), t(sc.shs[:, :1]), t(sc.shs[:, 1:]), t(np.log(op / (1 - op))), t(np.log(sc.scales)), t(sc.rotations))


def test_flat_adam_matches_torch_adam(dev):
    """adam_step() against torch.optim.Adam over four steps: both moments bit for bit, and each parameter within the
    rounding of the fp32 rate (tests/optim_model.py rate_rounding_ok), every step from torch's parameters."""
    from . import optim_model as om
    m = _model(5003, dev)           # odd size: groups start at unaligned offsets, the kernel's scalar tail is exercised
    ref = [p.detach().clone().requires_grad_(True) for p in m.flat_params()]
    names = ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation")
    opt = torch.optim.Adam([{"params": [p], "lr": m.lrs[n]} for p, n in zip(ref, names)], lr=0.0, eps=1e-15)
    g = torch.Generator(device=dev).manual_seed(1)
    for step in range(4):
        m.zero_grad_flat()
        with torch.no_grad():
            for p, r in zip(m.flat_params(), ref):
                p.copy_(r)
        before = [r.detach().clone() for r in ref]
        for p, r in zip(m.flat_params(), ref):
            gr = torch.randn(p.shape, device=dev, generator=g) * (10.0 ** (step - 2))
            p.grad.copy_(gr)
            r.grad = gr.clone() * 0.25
        m.adam_step(grad_scale=0.25)
        opt.step()
        off, total = m._offsets(m.P)
        for p, r, n, b, a, e in zip(m.flat_params(), ref, names, before, off, off[1:] + [total]):
            assert torch.equal(m.exp_avg[a:e], opt.state[r]["exp_avg"].flatten()), (step, n)
            assert torch.equal(m.exp_avg_sq[a:e], opt.state[r]["exp_avg_sq"].flatten()), (step, n)
            assert om.rate_rounding_ok(p.detach().cpu().numpy(), r.detach().cpu().numpy(), b.cpu().numpy()).all(), (step, n)


def _reference_densify(params, state, stats, percent_dense, max_grad, min_opacity, extent, max_screen_size, gen):
    """Plain-tensor restatement of GaussianModel.densify_and_prune (gaussian_model.py:431-446) with its helpers:
    params / state: dicts name -> tensor / (exp_avg, exp_avg_sq); returns the new dicts."""
    from vidu4d_b200.surfel_store import build_rotation
    names = list(params)

    def cat(new):        # cat_tensors_to_optimizer + densification_postfix (:331-374)
        for n in names:
            params[n] = torch.cat((params[n], new[n]), 0)
            state[n] = (torch.cat((state[n][0], torch.zeros_like(new[n])), 0), torch.cat((state[n][1], torch.zeros_like(new[n])), 0))

    def prune(mask):     # prune_points + _prune_optimizer (:297-329)
        keep = ~mask
        for n in names:
            params[n] = params[n][keep]
            state[n] = (state[n][0][keep], state[n][1][keep])

    grads = stats["accum"] / stats["denom"]
    grads[grads.isnan()] = 0.0
    scal = lambda: torch.exp(params["scaling"])  # noqa: E731
    # densify_and_clone (:407-429)
    sel = (torch.norm(grads, dim=-1) >= max_grad) & (scal().max(dim=1).values <= percent_dense * extent)
    cat({n: params[n][sel] for n in names})
    # densify_and_split (:376-405)
    n_init = params["xyz"].shape[0]
    padded = torch.zeros((n_init,), device=grads.device)
    padded[:grads.shape[0]] = grads.squeeze()
    sel = (padded >= max_grad) & (scal().max(dim=1).values > percent_dense * extent)
    N = 2
    stds = scal()[sel].repeat(N, 1)
    stds = torch.cat([stds, 0 * torch.ones_like(stds[:, :1])], dim=-1)
    samples = torch.normal(mean=torch.zeros_like(stds), std=stds, generator=gen)
    rots = build_rotation(params["rotation"][sel]).repeat(N, 1, 1)
    new = {n: params[n][sel].repeat(*([N] + [1] * (params[n].dim() - 1))) for n in names}
    new["xyz"] = torch.bmm(rots, samples.unsqueeze(-1)).squeeze(-1) + params["xyz"][sel].repeat(N, 1)
    new["scaling"] = torch.log(scal()[sel].repeat(N, 1) / (0.8 * N))
    cat(new)
    prune(torch.cat((sel, torch.zeros(N * int(sel.sum()), device=sel.device, dtype=torch.bool))))
    # final prune (:438-444); max_radii2D was reset to zero by densification_postfix
    pm = (torch.sigmoid(params["opacity"]) < min_opacity).squeeze()
    if max_screen_size:
        pm = pm | (scal().max(dim=1).values > 0.1 * extent)
    prune(pm)
    return params, state


@pytest.mark.parametrize("max_screen_size", [None, 20])
def test_densify_and_prune_matches_reference_procedure(max_screen_size, dev):
    m = _model(20000, dev, seed=3)
    g = torch.Generator(device=dev).manual_seed(5)
    # a few Adam steps so that the moments are non-trivial, then densification statistics
    for _ in range(2):
        for p in m.flat_params():
            p.grad.copy_(torch.randn(p.shape, device=dev, generator=g) * 1e-3)
        m.adam_step()
    with torch.no_grad():
        m._opacity[:500] = -8.0                                   # some surfels to prune (opacity < 0.005)
        m._scaling[500:800] += 2.5                                # some large ones (split candidates / size prune)
    vis = torch.rand((m.P,), device=dev, generator=g) > 0.3
    m.add_densification_stats(torch.randn((m.P, 3), device=dev, generator=g) * 3e-4, vis)
    names = ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation")
    off, _ = m._offsets(m.P)
    params = {n: p.detach().clone() for n, p in zip(names, m.flat_params())}
    state = {n: (m.exp_avg[o:o + p.numel()].view(p.shape).clone(), m.exp_avg_sq[o:o + p.numel()].view(p.shape).clone())
             for n, p, o in zip(names, m.flat_params(), off)}
    stats = {"accum": m.xyz_gradient_accum.clone(), "denom": m.denom.clone()}
    extent = 1.0
    want_p, want_s = _reference_densify(params, state, stats, m.percent_dense, 2e-4, 0.005, extent, max_screen_size,
                                        torch.Generator(device=dev).manual_seed(77))
    info = m.densify_and_prune(2e-4, 0.005, extent, max_screen_size, generator=torch.Generator(device=dev).manual_seed(77))
    assert info["cloned"] > 0 and info["split"] > 0 and info["pruned"] > 0
    assert m.P == want_p["xyz"].shape[0] == info["P"]
    off, _ = m._offsets(m.P)
    for n, p, o in zip(names, m.flat_params(), off):
        assert torch.equal(p.detach(), want_p[n].view(p.shape)), n
        assert torch.equal(m.exp_avg[o:o + p.numel()].view(p.shape), want_s[n][0].view(p.shape)), n
        assert torch.equal(m.exp_avg_sq[o:o + p.numel()].view(p.shape), want_s[n][1].view(p.shape)), n
    assert m.xyz_gradient_accum.shape == (m.P, 1) and float(m.max_radii2D.abs().sum()) == 0.0


def test_grown_model_renders_and_trains(dev):
    """P grows mid-run (densification): the rasterizer re-sizes its buffers, gradients land in the re-bound flat buffer,
    the Adam step runs on the new layout."""
    from vidu4d_b200.renderer import PipelineParams, make_camera, render_fused
    m = _model(20000, dev, seed=4)
    cam = make_camera(160, 128, 2 * np.arctan(0.5), 2 * np.arctan(0.4), device=dev)
    bg = torch.zeros(3, device=dev)
    sizes = []
    for it in range(4):
        m.zero_grad_flat()
        out = render_fused(cam, m, PipelineParams(), bg)
        (out["render"].mean() + 0.1 * out["rend_dist"].mean()).backward()
        assert float(m.grad_flat.abs().sum()) > 0
        m.add_densification_stats(out["viewspace_points"].grad, out["visibility_filter"], out["radii"])
        m.adam_step()
        if it == 1:
            m.xyz_gradient_accum += 1.0         # force densification
            info = m.densify_and_prune(2e-4, 0.005, 1.0, None)
            assert info["P"] > 20000
        sizes.append(m.P)
    assert sizes[-1] > sizes[0] and torch.isfinite(m.flat).all()


def test_graphed_step_recaptures_on_growth_and_on_overflow(dev):
    """A captured step survives (a) densification changing the surfel count and (b) the scene outgrowing the instance
    capacity baked into the graph: both re-capture transparently and give the same image as an eager render."""
    from vidu4d_b200 import rasterizer as RZ
    from vidu4d_b200.graph import GraphedStep
    from vidu4d_b200.renderer import PipelineParams, make_camera, render_fused
    m = _model(12000, dev, seed=6)
    cam = make_camera(128, 96, 2 * np.arctan(0.5), 2 * np.arctan(0.375), device=dev)
    bg = torch.zeros(3, device=dev)
    img = torch.zeros((3, 96, 128), device=dev)

    def body():
        m.zero_grad_flat()
        out = render_fused(cam, m, PipelineParams(), bg)
        out["render"].mean().backward()
        img.copy_(out["render"].detach())
    step = GraphedStep(body, key=lambda: m.P, device=dev)
    try:
        step(); step()
        assert step.captures == 1 and float(m.grad_flat.abs().sum()) > 0
        eager = render_fused(cam, m, PipelineParams(), bg)["render"].detach().clone()
        RZ.check_overflow()
        step()
        assert torch.equal(img, eager)
        # (a) densification: P changes -> re-capture
        m.xyz_gradient_accum += 1.0; m.denom += 1.0
        info = m.densify_and_prune(2e-4, 0.005, 1.0, None)
        assert info["P"] != 12000
        step()
        assert step.captures == 2 and m.grad_flat.numel() == m.flat.numel()
        # (b) the scene grows inside the same P: inflate the surfels so that num_rendered exceeds the baked capacity
        with torch.no_grad():
            m._scaling += 3.0
        step()                                       # overflow detected -> hints refreshed -> re-captured -> re-run
        assert step.captures == 3
        eager = render_fused(cam, m, PipelineParams(), bg)["render"].detach().clone()
        RZ.check_overflow()
        step()
        assert torch.equal(img, eager)
    finally:
        RZ.set_sync_mode(True)
        RZ._pending.clear()


def test_graphed_step_growth_200k_to_300k(dev):
    """The Stage-3 scale of the densification path (gs/scene/gaussian_model.py:291-356, lab4d/engine/trainer.py:562-568):
    a captured batched step over 200 K surfels, half of them densified (clone or split: +1 surfel each) -> 300 K, the
    step re-captured with re-sized buffers, image and gradient equal to an eager run on the grown model."""
    from vidu4d_b200 import rasterizer as RZ
    from vidu4d_b200.graph import GraphedStep
    from vidu4d_b200.renderer import PipelineParams, make_camera, render_fused
    m = _model(200000, dev, seed=8)
    cam = make_camera(256, 256, 2 * np.arctan(0.5), 2 * np.arctan(0.5), device=dev)
    bg = torch.zeros(3, device=dev)
    img = torch.zeros((3, 256, 256), device=dev)

    def body():
        m.zero_grad_flat()
        out = render_fused(cam, m, PipelineParams(), bg)
        (out["render"].mean() + 0.1 * out["rend_dist"].mean()).backward()
        img.copy_(out["render"].detach())
    step = GraphedStep(body, key=lambda: m.P, device=dev)
    try:
        step(); step()
        assert step.captures == 1
        with torch.no_grad():
            m._opacity.clamp_(min=-2.0)                    # nobody falls under the opacity prune threshold
        m.denom += 1.0
        m.xyz_gradient_accum[:100000] += 1.0                # exactly half of the surfels densify
        info = m.densify_and_prune(2e-4, 0.005, 1.0, None)
        assert info["cloned"] + info["split"] == 100000 and info["pruned"] == 0 and m.P == 300000
        m.adam_step()                                       # the optimizer state followed the new layout
        step()
        assert step.captures == 2 and m.grad_flat.numel() == m.flat.numel() == 300000 * 58
        g_graph = m.grad_flat.clone()
        i_graph = img.clone()
        RZ.check_overflow()
        RZ.set_sync_mode(True)
        m.zero_grad_flat()
        out = render_fused(cam, m, PipelineParams(), bg)
        (out["render"].mean() + 0.1 * out["rend_dist"].mean()).backward()
        assert torch.equal(i_graph, out["render"].detach())
        rel = float((g_graph - m.grad_flat).norm() / m.grad_flat.norm())
        assert rel < 1e-5, rel                              # atomics order differs run to run; nothing else does
    finally:
        RZ.set_sync_mode(True)
        RZ._pending.clear()


def _knn_cloud(P, kind, dev):
    g = torch.Generator(device=dev).manual_seed(P)
    blob = lambda n: torch.randn((n, 3), device=dev, generator=g) * torch.tensor([1.0, 0.2, 3.0], device=dev)  # noqa: E731
    if kind == "sphere":
        x = torch.randn((P, 3), device=dev, generator=g)
        return x / x.norm(dim=1, keepdim=True) * 0.35
    if kind == "dups":
        return torch.randn((P // 3, 3), device=dev, generator=g).repeat(3, 1)
    if kind == "lattice":                 # 20^3 points 0.125 apart: every distance exact, ties everywhere
        i = torch.arange(20, device=dev, dtype=torch.float32) * 0.125
        return torch.stack(torch.meshgrid(i, i, i, indexing="ij"), -1).reshape(-1, 3)[:P]
    if kind == "planar":                  # zero z extent
        x = blob(P)
        x[:, 2] = 0.0
        return x
    if kind == "collinear":               # zero y and z extent
        x = blob(P)
        x[:, 1:] = 0.0
        return x
    if kind == "stray":                   # one point far from the rest: a sparse grid, a long search for it
        x = blob(P)
        x[-1] = torch.tensor([1e3, -1e3, 1e3], device=dev)
        return x
    if kind == "offset":                  # coordinates near 1e4, where fp32 spacing is 1e-3
        return blob(P) * 0.1 + 1e4
    return blob(P)


KNN_CASES = [(20000, "sphere"), (5000, "blob"), (4, "tiny"), (3000, "dups"), (1, "tiny"), (2, "tiny"), (3, "tiny"),
             (8000, "lattice"), (5000, "planar"), (3000, "collinear"), (5001, "stray"), (4000, "offset")]


@pytest.mark.parametrize("P,kind", KNN_CASES)
def test_knn_mean_dist2_matches_brute_force(P, kind, dev):
    """distCUDA2 (simple_knn.cu:132-218): exact 3-NN mean squared distance, duplicates included, every element against
    float64 brute force on the same fp32 points under the fp32 rounding bound.  Each squared distance
    fl(ex*ex + ey*ey + ez*ez) with ex = fl(xj - xi) lies within 5u of the exact D (2u from the differences, one rounding
    per product and per sum, contracted or not); so the i-th smallest of them lies within 5u of the i-th smallest D
    whichever of tied or near-tied neighbours the kernel keeps, and the two sums and the divide add 3u:
    |out - (D1 + D2 + D3) / 3| <= 8u (D1 + D2 + D3) / 3, checked with K = 2.  With fewer than 3 other points the unused
    slots hold FLT_MAX, as in the reference: 3 points give fl(FLT_MAX / 3), 1 or 2 points Inf."""
    from vidu4d_b200.knn import distCUDA2
    x = _knn_cloud(P, kind, dev)
    got = distCUDA2(x)
    if P <= 3:
        fmax = np.float32(np.finfo(np.float32).max)
        want = np.float32(fmax / np.float32(3.0)) if P == 3 else np.float32(np.inf)
        assert (got.cpu().numpy() == want).all(), (P, got, want)
        return
    S = torch.empty(P, dtype=torch.float64, device=dev)
    xd = x.double()
    for s in range(0, P, 2000):
        d = torch.cdist(xd[s:s + 2000], xd, compute_mode="donot_use_mm_for_euclid_dist").pow(2)
        d[torch.arange(d.shape[0]), torch.arange(s, s + d.shape[0])] = float("inf")
        S[s:s + d.shape[0]] = torch.topk(d, 3, dim=1, largest=False).values.sum(1)
    err = (got.double() - S / 3).abs()
    lim = 2 * 8 * 2.0 ** -24 * S / 3 + float(np.finfo(np.float32).tiny)
    r = err / lim
    print(f"knn {kind} P={P}: largest err / bound {float(r.max()):.3g}")
    assert bool((r <= 1).all()), (kind, int((r > 1).sum()), float(r.max()), int(r.argmax()))
