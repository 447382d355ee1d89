"""Every output and gradient element of the global match (csrc/match.cu: sr_global_match_forward, match_bwd and
match_scatter in sr_global_match_backward) against the float64 restatement of its kernels (tests/match_bounds.py,
pinned to tests/reproj_model.py by tests/test_match_bounds_cpu.py), under the a-priori rounding-error bound
|gpu - value| <= K u B + FLOOR, with K = 2.

The entry points are driven through _capi.call, so g_cand (C, 19) is compared before the scatter: a failure says
whether match_bwd or match_scatter went wrong.  The top-K lists are checked as data (outside knife pixels equal to the
float64 lists, in order); every value is then evaluated on the kernel's own lists, and the backward on the forward's
own prob and score buffers.  Every output buffer starts as NaN (or -7 for top_idx), so an element the op fails to
write fails the comparison.  Each case prints its knife count and the largest err / tol per tensor.

Cases, each asserting its edge from the GPU's buffers: C = 1, K, 255, 256, 257 (the forward's 256-row staging ring),
2048, the backward's shared-memory cap, cap + 1 and 2 cap + 5 (the global-atomic backward); every K from 1 to 8; N at
the forward's 256-thread and the backward's 1024-thread block edges; invalid candidate indices at positions 255, 256 and
C - 1, so many that fewer than K candidates are valid, and none valid at all; duplicated surfels (exact ties); a
temperature at which the tail probabilities underflow to 0 and one at which they are flat; most pixels masked (zero
upstream), whose candidates must get exactly nothing; feature scales 0.1, 1 and 30; and an odd-P FlatSurfelModel
_regist_feat view (rows only 8-byte aligned).  The CUDA-event profile of each backward names the instantiation that ran ("match_bwd" in shared
memory, "match_bwd_global" past the cap), and each case asserts the one its C calls for.
"""
import numpy as np
import pytest
import torch

from . import match_bounds as mb

pytestmark = pytest.mark.gpu

STATIC_SMEM = 128          # match_bwd_kernel's static shared memory: red[1024 / 32] floats (the profile confirms the path)
N1025 = (1, 25, 41)
CASES = {
    "C_1": dict(shape=N1025, P=800, C=1, K=1, hot=(0,)),
    "C_8": dict(shape=N1025, P=800, C=8, K=8, hot=(7,)),
    "C_255": dict(shape=N1025, P=800, C=255, K=8, hot=(254,)),
    "C_256": dict(shape=N1025, P=800, C=256, K=8, hot=(255,)),
    "C_257": dict(shape=N1025, P=800, C=257, K=8, hot=(256,)),
    "C_2048": dict(shape=N1025, P=4000, C=2048, K=8, hot=(0, 255, 256, 2047)),
    "C_cap": dict(shape=N1025, P=8000, C="cap", K=8, hot=(0, -1)),
    "C_cap1": dict(shape=N1025, P=8000, C="cap1", K=8, hot=(0, -1)),
    "C_2cap5": dict(shape=N1025, P=8000, C="2cap5", K=8, hot=(0, -1)),
    **{f"K_{k}": dict(shape=(1, 1, 257), P=500, C=300, K=k, hot=(299,)) for k in range(1, 9)},
    **{f"N_{n}": dict(shape=sh, P=700, C=513, K=8, hot=(512,), masked=0.0)
       for n, sh in ((1, (1, 1, 1)), (255, (1, 15, 17)), (257, (1, 1, 257)), (1023, (3, 11, 31)), (1025, N1025))},
    "invalid_edges": dict(shape=(3, 11, 31), P=400, C=600, K=8, hot=(254, 257),
                          invalid=(255, 256, 599) + tuple(range(3, 590, 7))),
    "invalid_few": dict(shape=(1, 15, 17), P=10, C=10, K=8, invalid=(0, 4, 9), hot=(5,)),
    "invalid_all": dict(shape=(1, 15, 17), P=10, C=5, K=3, invalid=(0, 1, 2, 3, 4)),
    "duplicates": dict(shape=(2, 16, 32), P=600, C=900, K=8, dup=40),
    "logsigma_underflow": dict(shape=N1025, P=800, C=700, K=8, logsigma=np.log(1000.0)),
    "logsigma_flat": dict(shape=N1025, P=800, C=700, K=8, logsigma=np.log(1e-6)),
    "masked": dict(shape=N1025, P=800, C=700, K=8, masked=0.95, hot=(3,)),
    "scale_0.1": dict(shape=N1025, P=4000, C=2048, K=8, scale=0.1),
    "scale_1": dict(shape=N1025, P=4000, C=2048, K=8, scale=1.0),
    "scale_30": dict(shape=N1025, P=4000, C=2048, K=8, scale=30.0),
    "flat_view_P5003": dict(shape=(1, 31, 33), P=5003, C=2048, K=8, flat=True, hot=(2047,)),
}


@pytest.fixture(scope="module")
def dev(built):
    from vidu4d_b200 import _capi
    _capi.load()
    return torch.device("cuda:0")


def smem_cap(dev):
    """The largest C whose (C, 19) rows fit the backward's shared memory beside its static shared memory."""
    optin = torch.cuda.get_device_properties(dev).shared_memory_per_block_optin
    return (optin - STATIC_SMEM) // (mb.ROW * 4)


def _c(spec, dev):
    cap = smem_cap(dev)
    return {"cap": cap, "cap1": cap + 1, "2cap5": 2 * cap + 5}.get(spec, spec)


def make(name, dev, seed=0):
    c = dict(CASES[name])
    M, H, W = c.pop("shape")
    C = _c(c.pop("C"), dev)
    c.pop("flat", None)
    c["hot"] = tuple(C + h if h < 0 else h for h in c.get("hot", ()))
    return mb.scene(seed + sum(map(ord, name)), M, H, W, c.pop("P"), C, c.pop("K"), **c)


def _flat_regist_feat(rf, dev):
    """rf copied into the _regist_feat view of a FlatSurfelModel with P surfels."""
    from vidu4d_b200.surfel_store import FlatSurfelModel
    P = rf.shape[0]
    z = lambda *s: torch.zeros(s, device=dev)  # noqa: E731
    m = FlatSurfelModel(z(P, 3), z(P, 1, 3), z(P, 15, 3), z(P, 1), z(P, 2), z(P, 4), regist_feat=z(P, 16))
    v = m._regist_feat.detach()
    v.copy_(torch.from_numpy(rf).to(dev))
    return m, v


def gpu(s, dev, flat=False):
    """sr_global_match_forward, then sr_global_match_backward on its own buffers.  Returns numpy outputs."""
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    M, H, W, P, C, Kn = (s[k] for k in ("M", "H", "W", "P", "C", "K"))
    N = M * H * W
    feat, xyz, cand, ls, g = T(s["feat"]), T(s["xyz"]), T(s["cand"]), T(s["logsigma"]), T(s["g"])
    keep = None
    if flat:
        keep, rf = _flat_regist_feat(s["rf"], dev)
        assert rf.data_ptr() % 16 != 0 and rf.is_contiguous(), "the odd-P view must be only 8-byte aligned"
    else:
        rf = T(s["rf"])
    nan = lambda *sh: torch.full(sh, float("nan"), device=dev)  # noqa: E731
    xm, prob, score = nan(N, 3), nan(N, Kn), nan(N, Kn)
    idx = torch.full((N, Kn), -7, dtype=torch.int32, device=dev)
    from vidu4d_b200 import _capi
    _capi.call("sr_global_match_forward", dev, M, H, W, P, C, Kn, feat, rf, xyz, cand, ls, xm, idx, prob, score)
    gc, grf, gx, gl = nan(C, mb.ROW), nan(P, mb.FEAT), nan(P, 3), nan(1)
    _capi.get_profile()
    _capi.set_profiling(True)
    try:
        _capi.call("sr_global_match_backward", dev, M, H, W, P, C, Kn, feat, xyz, cand, ls, idx, prob, score, g, gc, grf, gx,
                   gl)
        torch.cuda.synchronize(dev)
        prof = _capi.get_profile()
    finally:
        _capi.set_profiling(False)
    del keep
    n = lambda t: t.cpu().numpy()  # noqa: E731
    return dict(xyz_matched=n(xm), top_idx=n(idx).astype(np.int64), top_prob=n(prob), top_score=n(score), g_cand=n(gc),
                g_regist_feat=n(grf), g_xyz=n(gx), g_logsigma=n(gl).reshape(()), bwd_kernels=sorted(prof))


def _cmp(name, what, mine, e, report, where=None):
    mine = np.asarray(mine, np.float64)
    tol = mb.K * mb.U * e.b + mb.FLOOR
    ratio = np.abs(mine - e.v) / tol
    ratio = np.where(np.isnan(mine), np.inf, ratio)
    if where is not None:
        ratio = np.where(where, ratio, 0.0)
    i = int(np.argmax(ratio))
    report[what] = max(report.get(what, 0.0), float(ratio.flat[i]))
    assert ratio.flat[i] <= 1.0, (name, what, "element", np.unravel_index(i, np.shape(mine)), "gpu", mine.flat[i],
                                  "value", e.v.flat[i], "bound", tol.flat[i])


def run(name, s, dev, flat=False):
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    g = gpu(s, dev, flat)
    path = "match_bwd" if s["C"] <= smem_cap(dev) else "match_bwd_global"
    assert g["bwd_kernels"] == sorted([path, "match_scatter"]), (name, "backward path", g["bwd_kernels"])
    m = mb.model(s, sms, g["top_idx"], g["top_prob"], g["top_score"])
    idx = g["top_idx"]
    ok = idx >= 0
    assert (g["top_prob"][~ok] == 0).all() and (g["top_score"][~ok] == 0).all(), (name, "empty slots: prob and score 0")
    report = {}
    fw, bw = m["fwd"], m["bwd"]
    _cmp(name, "top_score", g["top_score"], fw["score"], report, ok)
    _cmp(name, "top_prob", g["top_prob"], fw["prob"], report)
    for a in range(3):
        _cmp(name, "xyz_matched", g["xyz_matched"][:, a], fw["xyz_matched"][a], report)
    _cmp(name, "g_cand", g["g_cand"], bw["g_cand"], report)
    _cmp(name, "g_logsigma", g["g_logsigma"], bw["g_logsigma"], report)
    # rows no live pixel chose (masked pixels, invalid or unchosen positions) get exactly nothing
    assert (g["g_cand"][bw["users"] == 0] == 0).all(), (name, "a row without live users is not exactly 0")
    grf, gx = mb.scatter(mb._leaf(g["g_cand"]), s["cand"], s["M"] * s["P"], s["P"])
    _cmp(name, "g_regist_feat", g["g_regist_feat"], grf, report)
    _cmp(name, "g_xyz", g["g_xyz"], gx, report)
    nk = int(m["knife"].sum())
    N = idx.shape[0]
    print(f"\n[{name}] N={N} C={s['C']} K={s['K']}: knife {nk}; " + ", ".join(f"{k} {v:.3g}" for k, v in report.items()))
    assert nk <= 4 + N // 256, (name, "knife pixels", nk)
    return m, g


@pytest.mark.parametrize("name", list(CASES))
def test_global_match_every_element_within_bound(name, dev):
    s = make(name, dev)
    m, g = run(name, s, dev, flat=CASES[name].get("flat", False))
    idx, prob, live = g["top_idx"], g["top_prob"], m["bwd"]["live"]
    C = s["C"]
    for h in CASES[name].get("hot", ()):
        pos = C + h if h < 0 else h
        assert (idx == pos).any(), (name, "hot position never chosen", pos)
        assert (g["g_cand"][pos] != 0).any(), (name, "hot position got no gradient", pos)
    if name.startswith("C_") and C > 1:
        assert idx.max() == C - 1 and (idx[:, 0] >= 256).any() == (C > 256)
    if name == "C_2cap5":
        assert C > 2 * smem_cap(dev)
    if name == "invalid_edges":
        assert not np.isin(idx, (255, 256, C - 1)).any() and (idx == 254).any() and (idx == 257).any()
    if name == "invalid_few":
        assert (idx[:, -1] == -1).all() and (idx[:, :-1] >= 0).all()
    if name == "duplicates":
        a, b = s["dup_at"]
        both = (idx == a).any(1) & (idx == b).any(1)
        assert both.any(), "no pixel chose both copies of a duplicated surfel"
        sc = g["top_score"]
        ka, kb = np.argmax(idx == a, 1), np.argmax(idx == b, 1)
        r = np.nonzero(both)[0]
        first, second = (ka, kb) if a < b else (kb, ka)          # equal scores: the lower position first
        assert (sc[r, ka[r]] == sc[r, kb[r]]).all() and (first[r] + 1 == second[r]).all()
    if name == "logsigma_underflow":
        assert ((prob == 0) & (idx >= 0)).any(), "no tail probability underflowed to 0"
    if name == "logsigma_flat":
        assert np.abs(prob * s["K"] - 1.0).max() < 1e-3
    if name == "masked":
        assert (~live).sum() > 0.9 * len(live)
        assert ((m["bwd"]["users"] == 0) & np.isin(np.arange(C), idx)).any(), "no candidate chosen by masked pixels only"
    if name == "invalid_all":
        assert (idx == -1).all() and (prob == 0).all() and (g["top_score"] == 0).all() and (g["xyz_matched"] == 0).all()
        assert (g["g_cand"] == 0).all() and g["g_logsigma"] == 0 and (g["g_regist_feat"] == 0).all()
    if name.startswith("K_"):
        assert idx.shape[1] == s["K"] and (idx >= 0).all()


def test_autograd_backward_beyond_shared_memory_matches_float64_model(dev):
    """global_match -> .sum() -> backward at C = cap + 1 (the global-atomic backward), against tests/reproj_model.py
    evaluated on the kernel's own top-K lists."""
    from vidu4d_b200.registration import global_match
    from .reproj_model import global_match as ref_match
    C = smem_cap(dev) + 1
    s = mb.scene(11, 2, 24, 20, 2000, C, 8)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    rf, xyz, ls = (T(s[k]).requires_grad_(True) for k in ("rf", "xyz", "logsigma"))
    feat = T(s["feat"]).reshape(2, 24, 20, 16)
    xm, idx, _ = global_match(feat, rf, xyz, T(s["cand"]), ls, num_grad=8, return_topk=True)
    xm.sum().backward()
    d = lambda t: t.detach().double().cpu().requires_grad_(True)  # noqa: E731
    rf64, xyz64, ls64 = d(rf), d(xyz), d(ls)
    xm64, _, _, _ = ref_match(feat.double().cpu(), rf64, xyz64, torch.from_numpy(s["cand"]), ls64, 8,
                              order=idx.reshape(-1, 8).long().cpu())
    xm64.sum().backward()
    for a, b in ((xm, xm64), (rf.grad, rf64.grad), (xyz.grad, xyz64.grad), (ls.grad, ls64.grad)):
        a = a.detach().double().cpu()
        assert float((a - b).abs().max()) <= 1e-5 * float(b.abs().max()) + 1e-30
    assert float(rf.grad.abs().max()) > 0
