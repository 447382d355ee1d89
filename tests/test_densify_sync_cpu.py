"""CPU: the pieces that keep every rank's surfels identical through densification -- sync_densification_stats,
shared_generator and check_replicas on a two-rank gloo group with CPU tensors; FlatSurfelModel without the CUDA library
(the packed statistics, the one-frame torch path, the batched form's argument errors); sr_densify_stats' own messages."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from .conftest import ROOT

P = 37


def _model(P=P, seed=0):
    from vidu4d_b200.surfel_store import FlatSurfelModel
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(s, generator=g)  # noqa: E731
    return FlatSurfelModel(r(P, 3), r(P, 1, 3), r(P, 15, 3), r(P, 1), r(P, 2) - 3.0, r(P, 4))


def _worker(rank, world, port, out):
    sys.path.insert(0, ROOT)
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    from vidu4d_b200 import distributed as D
    D.init_distributed("gloo")
    res = {}
    m = _model()
    # each rank's own statistics: rank r sees the surfels i with i % (r + 2) == 0
    g = torch.Generator().manual_seed(100 + rank)
    vis = torch.arange(P) % (rank + 2) == 0
    m.add_densification_stats(torch.randn((P, 3), generator=g), vis, torch.randint(1, 50, (P,), generator=g), grad_scale=0.5)
    res["local"] = torch.cat([m.densify_stats.reshape(-1), m.max_radii2D]).numpy()
    m.sync_densification_stats()
    res["synced"] = torch.cat([m.densify_stats.reshape(-1), m.max_radii2D]).numpy()
    # the parameters are identical on both ranks: check_replicas passes, also on the (still per-rank-equal) statistics
    D.check_replicas({"P": m.P, "flat": m.flat, "device_step": m.device_step, "densify_stats": m.densify_stats})
    # shared_generator: rank 0's seed wins, whatever the others pass; seed=None draws one on rank 0
    res["gen"] = torch.randn(8, generator=D.shared_generator("cpu", seed=7 + rank)).numpy()
    res["gen_none"] = torch.randn(8, generator=D.shared_generator("cpu")).numpy()
    # one element differs on rank 1
    if rank == 1:
        m.flat[5 * P + 3] += 1.0
    try:
        D.check_replicas({"P": m.P, "flat": m.flat, "exp_avg": m.exp_avg})
        res["flip"] = ""
    except RuntimeError as e:
        res["flip"] = str(e)
    if rank == 1:
        m.flat[5 * P + 3] -= 1.0
    # the same words in another order
    x = torch.arange(10, dtype=torch.float32)
    try:
        D.check_replicas({"x": x if rank == 0 else x.flip(0)})
        res["swap"] = ""
    except RuntimeError as e:
        res["swap"] = str(e)
    # another P
    try:
        D.check_replicas({"P": P + rank, "flat": m.flat})
        res["size"] = ""
    except RuntimeError as e:
        res["size"] = str(e)
    # allreduce_grads_ over the current (re-bound) buffer
    m.grad_flat.fill_(rank + 1.0)
    m.allreduce_grads_(average_over=4)
    res["grads"] = m.grad_flat[:5].numpy()
    np.savez(out + f".{rank}.npz", **res)
    dist.destroy_process_group()


@pytest.fixture(scope="module")
def two_ranks(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("sync") / "r")
    port = 29900 + (os.getpid() % 97)
    mp.start_processes(_worker, args=(2, port, out), nprocs=2, join=True, start_method="spawn")
    return [dict(np.load(out + f".{r}.npz")) for r in range(2)]


def test_sync_densification_stats_sums_and_maxes(two_ranks):
    loc = [r["local"] for r in two_ranks]
    want = np.concatenate([(loc[0][:2 * P] + loc[1][:2 * P]), np.maximum(loc[0][2 * P:], loc[1][2 * P:])])
    for r in two_ranks:
        assert np.array_equal(r["synced"], want)
    assert not np.array_equal(loc[0], loc[1])


def test_shared_generator_takes_rank_zeros_seed(two_ranks):
    a, b = two_ranks
    assert np.array_equal(a["gen"], b["gen"]) and np.array_equal(a["gen_none"], b["gen_none"])
    assert np.array_equal(a["gen"], torch.randn(8, generator=torch.Generator().manual_seed(7)).numpy())


def test_check_replicas_names_the_differing_tensor(two_ranks):
    for r in two_ranks:
        flip, swap, size = (str(r[k]) for k in ("flip", "swap", "size"))
        assert "'flat'" in flip and "bits" in flip and "[1]" in flip, flip
        assert "'x'" in swap, swap
        assert "'P'" in size, size


def test_allreduce_grads_sums_then_averages(two_ranks):
    for r in two_ranks:
        assert np.array_equal(r["grads"], np.full(5, 0.75, np.float32))


def test_one_rank_is_a_no_op():
    from vidu4d_b200 import distributed as D
    assert not dist.is_initialized()
    m = _model()
    m.densify_stats.fill_(2.0)
    m.sync_densification_stats()
    D.check_replicas({"flat": m.flat})
    m.grad_flat.fill_(3.0)
    m.allreduce_grads_(average_over=2)
    assert float(m.densify_stats.sum()) == 4.0 * P and float(m.grad_flat.max()) == 1.5
    a = torch.rand(4, generator=D.shared_generator("cpu", seed=3))
    assert torch.equal(a, torch.rand(4, generator=torch.Generator().manual_seed(3)))


def test_checksum_sees_every_word():
    from vidu4d_b200.distributed import _checksum
    x = torch.randn(1001)
    c = int(_checksum(x))
    for i in (0, 500, 1000):
        for bit in (0, 22, 31):
            y = x.clone()
            y.view(torch.int32)[i] ^= 1 << bit
            assert int(_checksum(y)) != c
    assert int(_checksum(torch.zeros(3, dtype=torch.uint8))) != int(_checksum(torch.ones(3, dtype=torch.uint8)))
    assert 0 <= c < 1 << 63


def test_statistics_are_views_of_one_packed_buffer():
    """FlatSurfelModel builds on CPU tensors without the CUDA library; accum and denom keep their (P,1) shapes and
    names as rows of densify_stats, also through assignment."""
    m = _model()
    assert m.densify_stats.shape == (2, P) and m.xyz_gradient_accum.shape == (P, 1) and m.denom.shape == (P, 1)
    m.xyz_gradient_accum += 1.0
    m.denom = torch.full((P, 1), 3.0)
    assert torch.equal(m.densify_stats, torch.stack([torch.ones(P), torch.full((P,), 3.0)]))
    g = torch.Generator().manual_seed(1)
    grad, vis, radii = torch.randn((P, 3), generator=g), torch.arange(P) % 3 != 0, torch.randint(0, 9, (P,), generator=g)
    m.add_densification_stats(grad, vis, radii, grad_scale=0.25)
    want = 1.0 + torch.norm(grad * 0.25, dim=-1) * vis.float()
    assert torch.equal(m.xyz_gradient_accum[:, 0], want)
    assert m.densify_stats.data_ptr() == m.xyz_gradient_accum.data_ptr()
    assert m.denom.data_ptr() == m.densify_stats[1].data_ptr()
    with pytest.raises(RuntimeError):
        m.xyz_gradient_accum = torch.zeros((P + 1, 1))


def test_batched_form_checks_shapes_and_devices_before_launching():
    m = _model()
    M = 3
    grad, radii = torch.zeros((M, P, 3)), torch.ones((M, P), dtype=torch.int32)
    cases = [((torch.zeros((M, P + 1, 3)), None, radii), "viewspace_grad must be (M,P,3)"),
             ((torch.zeros((M, P, 2)), None, radii), "viewspace_grad must be (M,P,3)"),
             ((grad, None, None), "needs radii (M,P)"),
             ((grad, None, radii[:2]), "needs radii (M,P)"),
             ((grad, radii[:, :3] > 0, radii), "update_filter must be (M,P)"),
             ((grad.double(), None, radii), "must be float32"),
             ((grad, None, radii.long()), "radii must be int32"),
             ((grad, radii > 0, radii), "must be a CUDA tensor")]
    for (g, f, r), msg in cases:
        with pytest.raises(RuntimeError, match=msg.replace("(", r"\(").replace(")", r"\)")):
            m.add_densification_stats(g, f, r)
    assert float(m.densify_stats.abs().sum()) == 0.0


def test_densify_stats_bad_arguments_set_their_own_message(built):
    from vidu4d_b200 import _capi
    lib = _capi.load()
    D = 1 << 20
    good = [4, 100, D, D, 1.0, D, D, D, None]
    cases = [({0: -1}, b"M and P must be >= 0"), ({1: -5}, b"M and P must be >= 0"), ({2: None}, b"must not be NULL"),
             ({7: None}, b"must not be NULL"), ({3: D + 2}, b"4-byte aligned")]
    for change, want in cases:
        args = list(good)
        for k, v in change.items():
            args[k] = v
        assert lib.sr_debug_view(0, 0, 0, 0, None) == -1
        sentinel = lib.sr_last_error()
        assert lib.sr_densify_stats(*args) == -1
        msg = lib.sr_last_error()
        assert msg != sentinel and b"sr_densify_stats" in msg and want in msg, msg
    # nothing to do: no launch, no device needed
    assert lib.sr_densify_stats(0, 100, None, None, 1.0, None, None, None, None) == 0
    assert lib.sr_densify_stats(3, 0, None, None, 1.0, None, None, None, None) == 0
