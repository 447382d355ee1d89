"""GPU tests of the radius outlier filter (csrc/outlier.cu via vidu4d_b200.knn.radius_outlier_mask and
FlatSurfelModel.remove_radius_outliers): keep mask and capped counts EXACTLY equal to the float64 brute-force oracle
(tests/outlier_model.py's formula, evaluated here on the device in row chunks with one eager elementwise op per rounding,
not with torch.cdist, whose matmul form is a different formula)."""
import numpy as np
import pytest
import torch

from .outlier_model import keep_and_capped, radius_counts

pytestmark = pytest.mark.gpu
R, NB = 0.004, 20                              # the reference's call (lab4d/engine/trainer.py:580)


@pytest.fixture(scope="module")
def dev(built):
    from vidu4d_b200 import _capi
    _capi.load()
    return torch.device("cuda:0")


def oracle_counts(x: torch.Tensor, radius: float, chunk: int = 256) -> torch.Tensor:
    """outlier_model.radius_counts on the device: float32 rows widened to float64, each op rounded on its own."""
    xd = x.to(torch.float32).double()
    r2 = float(radius) * float(radius)
    out = torch.empty((xd.shape[0],), dtype=torch.int64, device=x.device)
    cols = [xd[:, k].contiguous()[None, :] for k in range(3)]
    for s in range(0, xd.shape[0], chunk):
        a = xd[s:s + chunk]
        acc = a[:, 0:1] - cols[0]
        acc.mul_(acc)
        for k in (1, 2):
            t = a[:, k:k + 1] - cols[k]
            t.mul_(t)
            acc.add_(t)
        out[s:s + chunk] = (acc < r2).sum(1)
    return out


def check(x: torch.Tensor, nb_points: int, radius: float):
    from vidu4d_b200.knn import radius_outlier_mask
    prune, capped = radius_outlier_mask(x, nb_points, radius, return_counts=True)
    c = oracle_counts(x, radius)
    assert prune.dtype == torch.bool and prune.shape == (x.shape[0],)
    assert torch.equal(prune, ~(c > nb_points))
    assert torch.equal(capped.long(), c.clamp(max=nb_points + 1))
    return prune, c


def _shell(P, dev, seed=0):
    from vidu4d_b200.synthetic import shell_with_strays
    return torch.from_numpy(shell_with_strays(P, seed=seed)).to(dev)


def test_device_oracle_is_the_numpy_model(dev):
    x = _shell(3000, dev, seed=1)
    x[:50] = x[100:150]
    assert np.array_equal(oracle_counts(x, 0.02).cpu().numpy(), radius_counts(x.cpu().numpy(), 0.02))


def test_reference_call_on_300k_shell(dev):
    x = _shell(300_000, dev, seed=2)
    prune, c = check(x, NB, R)
    n = int(prune.sum())
    assert 3000 <= n < 150_000, n              # every stray and the thin edges of the shell
    assert int((c == NB).sum()) + int((c == NB + 1).sum()) > 0     # knife-edge counts occur at this density


def test_clone_duplicates(dev):
    x = _shell(50_000, dev, seed=3)
    g = torch.Generator(device=dev).manual_seed(3)
    src = torch.randint(0, x.shape[0], (20_000,), device=dev, generator=g)
    x = torch.cat([x, x[src], x[src[:5000]]])           # clone densification copies rows exactly, some twice
    check(x, NB, R)
    check(x, 0, R)


@pytest.mark.parametrize("far", [1e2, 1e6, 1e30])
def test_single_stray_far_away(far, dev):
    x = _shell(20_000, dev, seed=4)
    strays = torch.tensor([[far, 0.5, 1.0], [-far, -far, far], [0.0, far, -far]], device=dev)
    x = torch.cat([x[:10_000], strays, x[10_000:]])
    prune, _ = check(x, NB, R)
    assert bool(prune[10_000:10_003].all())
    # a clamped cluster: 30 copies of a far point (distance 0 to each other) are each other's neighbours
    x = torch.cat([x, torch.tensor([[far, -far, far]], device=dev).repeat(30, 1)])
    prune, _ = check(x, NB, R)
    assert not bool(prune[-30:].any())


def test_pairs_at_exactly_the_radius(dev):
    """Pairs (p, p + (3s, 4s, 0)) with s = 2^-10: d2 = 25 s^2 exactly = r2 for r = 5s -> not neighbours; at r one ulp
    above 5s they are."""
    from vidu4d_b200.knn import radius_outlier_mask
    s = 2.0 ** -10
    g = torch.Generator(device=dev).manual_seed(5)
    # distinct grid points 64 s apart (|x| < 4, multiples of 2^-20: every coordinate and offset exact in float32)
    cell = torch.randperm(100 ** 3, device=dev, generator=g)[:2000]
    base = (torch.stack([cell // 10_000, cell // 100 % 100, cell % 100], 1) - 50).float() * (64 * s)
    base[:, 0] += torch.randint(-32, 32, (2000,), device=dev, generator=g).float() * s ** 2
    x = torch.cat([base, base + torch.tensor([3 * s, 4 * s, 0.0], device=dev)])
    x = torch.cat([x, x[:200]])                       # some pairs carry a duplicate
    prune, c = check(x, 1, 5 * s)
    assert int(c[200:2000].max()) == 1               # only the point itself
    up = float(np.nextafter(5 * s, 1.0))
    prune, c = check(x, 1, up)
    assert int(c[200:2000].min()) == 2 and not bool(prune[:4000].any())
    assert torch.equal(radius_outlier_mask(x, 1, up), prune)


def test_cell_faces_at_negative_coordinates(dev):
    """Points within r of each other on both sides of cell faces at negative coordinates, where floor and truncation
    toward zero disagree."""
    g = torch.Generator(device=dev).manual_seed(6)
    h = R * (1 + 2.0 ** -20)
    face = -torch.randint(1, 200, (4000, 1), device=dev, generator=g).double() * h
    off = (torch.rand((4000, 3), device=dev, generator=g, dtype=torch.float64) * 2 - 1) * R * 0.9
    off[:, 1:] *= 0.3
    x = torch.cat([face + off[:, :1], off[:, 1:] - 0.5], 1).float()
    x = torch.cat([x, x[:, [1, 0, 2]], x[:, [2, 1, 0]]])         # the same on the y and z axes
    for nb in (0, 3, 10):
        check(x, nb, R)


def test_non_finite_rows(dev):
    x = _shell(20_000, dev, seed=7)
    nan, inf = float("nan"), float("inf")
    bad = torch.tensor([[nan, 1.0, 1.0], [inf, 0.0, 1.0], [-inf, 0.0, 1.0], [0.0, inf, -inf], [nan, nan, nan],
                        [0.0, 0.0, inf]], device=dev)
    x[:6] = bad
    x[6:12] = bad
    prune, c = check(x, NB, R)
    assert bool(prune[:12].all()) and int(c[:12].abs().sum()) == 0
    prune0, c0 = check(x, 0, R)
    assert bool(prune0[:12].all()) and not bool(prune0[12:].any())


@pytest.mark.parametrize("P", [0, 1, 2])
def test_tiny_inputs(P, dev):
    from vidu4d_b200.knn import radius_outlier_mask
    x = torch.tensor([[0.1, 0.2, 0.3], [0.1, 0.2, 0.301]], device=dev)[:P]
    for nb in (0, 1, 2):
        prune, c = check(x, nb, R)
        assert prune.shape == (P,)
    if P == 2:
        assert radius_outlier_mask(x, 1, R).tolist() == [False, False]
        assert radius_outlier_mask(x, 1, 5e-4).tolist() == [True, True]


def test_radius_covers_everything(dev):
    g = torch.Generator(device=dev).manual_seed(8)
    x = torch.rand((3000, 3), device=dev, generator=g)
    for nb in (0, 5, 2999, 3000):
        prune, c = check(x, nb, 1e3)
    assert not bool(check(x, 2999, 1e3)[0].any()) and bool(check(x, 3000, 1e3)[0].all())


def test_tiny_radius_counts_only_duplicates(dev):
    g = torch.Generator(device=dev).manual_seed(9)
    x = torch.rand((5000, 3), device=dev, generator=g)
    x = torch.cat([x, x[:1000], x[:300]])
    prune, c = check(x, 1, 1e-30)
    assert int((~prune).sum()) == 2 * 1000 + 300


def test_bit_identical_and_permutation_equivariant(dev):
    from vidu4d_b200.knn import radius_outlier_mask
    x = _shell(300_000, dev, seed=10)
    x = torch.cat([x, x[:30_000]])
    a, ca = radius_outlier_mask(x, NB, R, return_counts=True)
    b, cb = radius_outlier_mask(x, NB, R, return_counts=True)
    assert torch.equal(a, b) and torch.equal(ca, cb)
    perm = torch.randperm(x.shape[0], device=dev, generator=torch.Generator(device=dev).manual_seed(10))
    p, cp = radius_outlier_mask(x[perm], NB, R, return_counts=True)
    assert torch.equal(p, a[perm]) and torch.equal(cp, ca[perm])
    # a non-contiguous float64 view is converted, not misread
    wide = torch.zeros((x.shape[0], 5), dtype=torch.float64, device=dev)
    wide[:, 1:4] = x.double()
    assert torch.equal(radius_outlier_mask(wide[:, 1:4], NB, R), a)


def test_graph_capture_and_replay(dev):
    from vidu4d_b200.knn import radius_outlier_mask
    P = 100_000
    static = _shell(P, dev, seed=11)
    s = torch.cuda.Stream(device=dev)
    s.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(s):
        radius_outlier_mask(static, NB, R, return_counts=True)          # warm-up outside the capture
    torch.cuda.current_stream(dev).wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        prune_g, counts_g = radius_outlier_mask(static, NB, R, return_counts=True)
    for seed in (12, 13):
        static.copy_(_shell(P, dev, seed=seed))
        graph.replay()
        prune_e, counts_e = radius_outlier_mask(static, NB, R, return_counts=True)
        assert torch.equal(prune_g, prune_e) and torch.equal(counts_g, counts_e)
    c = oracle_counts(static, R)
    assert torch.equal(prune_g, ~(c > NB))


def test_scratch_bound(dev):
    from vidu4d_b200 import _capi
    from vidu4d_b200.knn import radius_outlier_mask
    lib = _capi.load()
    for P in (1, 1000, 300_000, 1_000_000):
        assert lib.sr_radius_outlier_scratch_bytes(P) <= 48 * P + (2 << 20)
    # the call allocates nothing beyond its outputs and that scratch
    x = _shell(1_000_000, dev, seed=14)
    torch.cuda.synchronize(dev)
    torch.cuda.reset_peak_memory_stats(dev)
    base = torch.cuda.memory_allocated(dev)
    radius_outlier_mask(x, NB, R, return_counts=True)
    torch.cuda.synchronize(dev)
    extra = torch.cuda.max_memory_allocated(dev) - base
    assert extra <= lib.sr_radius_outlier_scratch_bytes(1_000_000) + 1_000_000 * (1 + 4 + 1) + (4 << 20), extra


def test_flat_model_remove_radius_outliers_equals_prune_points(dev):
    from vidu4d_b200.surfel_store import FlatSurfelModel
    P = 60_000
    xyz = _shell(P, dev, seed=15)
    g = torch.Generator(device=dev).manual_seed(15)
    r = lambda *shape: torch.randn(shape, device=dev, generator=g)   # noqa: E731
    inputs = (xyz, r(P, 1, 3), r(P, 15, 3), r(P, 1), r(P, 2) - 5.0, r(P, 4))
    feat = r(P, 16)
    models = [FlatSurfelModel(*inputs, regist_feat=feat) for _ in range(2)]
    grads = [r(P, k) for k in (3, 3, 45, 1, 2, 4, 16)]
    vs, vis, radii = r(P, 3) * 1e-3, torch.rand(P, device=dev, generator=g) > 0.3, torch.randint(0, 9, (P,), device=dev, generator=g)
    for m in models:
        for _ in range(2):
            for p, gr in zip(m.flat_params(), grads):
                p.grad.copy_(gr.view(p.shape))
            m.adam_step()
        m.add_densification_stats(vs, vis, radii)
    want_mask = ~(oracle_counts(models[1]._xyz.detach(), R) > NB)
    n = models[0].remove_radius_outliers(NB, R)
    models[1].prune_points(want_mask)
    assert n == int(want_mask.sum()) > 0 and models[0].P == models[1].P == P - n
    a, b = models
    assert torch.equal(a.flat, b.flat) and torch.equal(a.exp_avg, b.exp_avg) and torch.equal(a.exp_avg_sq, b.exp_avg_sq)
    assert torch.equal(a._regist_feat, b._regist_feat)
    for k in ("xyz_gradient_accum", "denom", "max_radii2D"):
        assert torch.equal(getattr(a, k), getattr(b, k)), k
    # nothing left to prune: the model (and its buffer addresses) stay as they are
    ptr = a.flat.data_ptr()
    assert a.remove_radius_outliers(0, R) == 0 and a.flat.data_ptr() == ptr
