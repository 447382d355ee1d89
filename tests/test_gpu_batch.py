"""GPU tests of batched calls (sr_forward / sr_backward with M frames, SURVEY.md 8(f) row N1): M frames in one
launch set must equal M single-frame calls -- forward planes, sorted lists and contributor counts bit for bit, gradients
up to the order of the atomic reductions -- for shared and for per-frame surfel sets, and through autograd."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev(built):
    from vidu4d_b200 import _capi
    _capi.load()
    return torch.device("cuda:0")


def _cams(M, dev):
    from vidu4d_b200.synthetic import orbit_view, projection_matrix
    Pm = projection_matrix(0.5, 0.5).astype(np.float64)
    vms, pms, cps = [], [], []
    for f in range(M):
        R, t = orbit_view(3 * f + 1, 64)
        W2C = np.eye(4); W2C[:3, :3] = R; W2C[:3, 3] = t
        vms.append(W2C.T.astype(np.float32)); pms.append((W2C.T @ Pm).astype(np.float32)); cps.append((-R.T @ t).astype(np.float32))
    return (torch.from_numpy(np.stack(vms)).to(dev), torch.from_numpy(np.stack(pms)).to(dev), torch.from_numpy(np.stack(cps)).to(dev))


@pytest.mark.parametrize("per_frame", [False, True], ids=["shared_surfels", "per_frame_surfels"])
def test_batch_equals_single_frame_calls(per_frame, dev):
    from vidu4d_b200 import rasterizer as RZ
    from vidu4d_b200.synthetic import object_scene
    M, P, W, H = 4, 20000, 208, 144         # ragged: 13 x 9 tiles
    sc = object_scene(P, seed=5, center=(0.0, 0.0, 0.0))
    t = sc.to_torch(dev)
    vms, pms, cps = _cams(M, dev)
    e = torch.empty((0,), device=dev)
    bg = torch.tensor([0.2, 0.1, 0.4], device=dev)
    g = torch.Generator(device=dev).manual_seed(2)
    dLc = torch.randn((M, 3, H, W), device=dev, generator=g)
    dLo = torch.randn((M, 8, H, W), device=dev, generator=g)
    if per_frame:   # Stage-3 like: every frame has its own (warped) positions and orientations
        means = torch.stack([t["means3D"] + 0.01 * f * torch.randn((P, 3), device=dev, generator=g) for f in range(M)])
        rots = torch.stack([torch.nn.functional.normalize(t["rotations"] + 0.05 * f * torch.randn((P, 4), device=dev, generator=g)) for f in range(M)])
    else:
        means, rots = t["means3D"], t["rotations"]
    C = RZ._C
    nr, color, allmap, radii, gb, bb, ib = C.rasterize_gaussians_batch(
        bg, means, e, t["opacities"], t["scales"], rots, 1.0, vms, pms, 0.5, 0.5, H, W, t["shs"], 3, cps)
    grads = C.rasterize_gaussians_backward_batch(bg, means, radii, e, t["scales"], rots, 1.0, vms, pms, 0.5, 0.5, dLc, dLo,
                                                 t["shs"], 3, cps, gb, bb, ib)
    assert len(nr) == M and color.shape == (M, 3, H, W) and radii.shape == (M, P)
    for f in range(M):
        m_f = means[f] if per_frame else means
        r_f = rots[f] if per_frame else rots
        o = C.rasterize_gaussians(bg, m_f, e, t["opacities"], t["scales"], r_f, 1.0, e, vms[f], pms[f], 0.5, 0.5, H, W,
                                  t["shs"], 3, cps[f], False, False)
        assert o[0] == nr[f]
        assert torch.equal(o[1], color[f]) and torch.equal(o[2], allmap[f]) and torch.equal(o[3], radii[f])
        gs = C.rasterize_gaussians_backward(bg, m_f, o[3], e, t["scales"], r_f, 1.0, e, vms[f], pms[f], 0.5, 0.5, dLc[f], dLo[f],
                                            t["shs"], 3, cps[f], o[4], o[0], o[5], o[6], False)
        for a, b in zip(gs, grads):
            assert a.shape == b[f].shape
            assert float((a - b[f]).abs().max()) <= 2e-5 * float(a.abs().max() + 1e-30)
    # SR_BATCH_SUM_SHARED: gradients of inputs shared by the frames come back summed over the frames, in the input's shape
    flat = torch.zeros((P * 48 + 64,), device=dev)
    gsum = C.rasterize_gaussians_backward_batch(bg, means, radii, e, t["scales"], rots, 1.0, vms, pms, 0.5, 0.5, dLc, dLo, t["shs"],
                                                3, cps, gb, bb, ib, sum_shared=True, want_transmat=False,
                                                outs={"dL_dsh": flat[64:64 + P * 48]})
    names = ("dL_dmeans2D", "dL_dcolors", "dL_dopacity", "dL_dmeans3D", "dL_dtransMat", "dL_dsh", "dL_dscales", "dL_drotations")
    per_frame_inputs = {"dL_dmeans2D"} | ({"dL_dmeans3D", "dL_drotations"} if per_frame else set())
    for nme, a, b in zip(names, grads, gsum):
        if nme == "dL_dtransMat":
            assert b is None
            continue
        want = a if nme in per_frame_inputs else a.sum(0)
        assert b.shape == want.shape, nme
        assert float((b - want).abs().max()) <= 2e-5 * float(want.abs().max() + 1e-30), nme
    assert gsum[5].data_ptr() == flat[64:].data_ptr()           # written in place into the caller's buffer
    # grad_scale: the backward is linear in dL_dout
    g2 = C.rasterize_gaussians_backward_batch(bg, means, radii, e, t["scales"], rots, 1.0, vms, pms, 0.5, 0.5, dLc, dLo, t["shs"],
                                              3, cps, gb, bb, ib, grad_scale=torch.tensor(-2.5, device=dev))
    for a, b in zip(grads, g2):
        assert float((b + 2.5 * a).abs().max()) <= 2e-5 * float((2.5 * a).abs().max() + 1e-30)


def test_batch_autograd_sums_shared_inputs(dev):
    """rasterize_gaussians_batch through autograd: gradients of inputs shared by the frames are the sums over frames of the
    single-frame op's gradients; per-frame inputs keep their leading M."""
    from vidu4d_b200 import rasterizer as RZ
    from vidu4d_b200.synthetic import SurfelCloud, object_scene
    M, P, W, H = 3, 8000, 128, 96
    vms, pms, cps = _cams(M, dev)
    bg = torch.zeros(3, device=dev)
    g = torch.Generator(device=dev).manual_seed(4)
    wc = torch.randn((M, 3, H, W), device=dev, generator=g)
    wa = torch.randn((M, 8, H, W), device=dev, generator=g)
    scene = object_scene(P, seed=9, center=(0.0, 0.0, 0.0))
    shift = 0.02 * torch.randn((M, P, 3), device=dev, generator=g)

    cloud = SurfelCloud(scene, dev)
    rs = RZ.BatchRasterizationSettings(H, W, 0.5, 0.5, bg, 1.0, vms, pms, 3, cps)
    means = cloud.get_xyz[None] + shift                                   # per frame (M,P,3); everything else shared
    m2d = torch.zeros((M, P, 3), device=dev, requires_grad=True)
    color, radii, allmap = RZ.rasterize_gaussians_batch(means, m2d, cloud.get_features, None, cloud.get_opacity,
                                                        cloud.get_scaling, cloud.get_rotation, rs)
    ((color * wc).sum() + (allmap * wa).sum()).backward()
    got = [p.grad.clone() for p in cloud.flat_params()]

    cloud2 = SurfelCloud(scene, dev)
    vp = []
    for f in range(M):
        rs1 = RZ.GaussianRasterizationSettings(H, W, 0.5, 0.5, bg, 1.0, vms[f], pms[f], 3, cps[f], False, False)
        m2 = torch.zeros((P, 3), device=dev, requires_grad=True)
        c1, r1, a1 = RZ.GaussianRasterizer(rs1)(means3D=cloud2.get_xyz + shift[f], means2D=m2, shs=cloud2.get_features,
                                                opacities=cloud2.get_opacity, scales=cloud2.get_scaling, rotations=cloud2.get_rotation)
        ((c1 * wc[f]).sum() + (a1 * wa[f]).sum()).backward()
        assert torch.equal(c1, color[f].detach()) and torch.equal(r1, radii[f])
        vp.append(m2.grad)
    for a, p in zip(got, cloud2.flat_params()):
        assert float((a - p.grad).abs().max()) <= 5e-5 * float(p.grad.abs().max() + 1e-30), tuple(p.shape)
    assert float((m2d.grad - torch.stack(vp)).abs().max()) <= 5e-5 * float(torch.stack(vp).abs().max() + 1e-30)
