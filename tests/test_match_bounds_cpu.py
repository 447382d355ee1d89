"""The restated global match and its bound (tests/match_bounds.py), on the CPU: its float64 top-K lists, forward values and
hand-written backward equal the float64 autograd of tests/reproj_model.py's global_match on the same fp32 inputs, on the
committed reproj_*.npz fixtures and on seeded scenes; and its fp32 shadow lies within K u B + FLOOR of its value for
every output and gradient (the backward and scatter fed the forward's own values)."""
import os

import numpy as np
import pytest
import torch

from . import match_bounds as mb
from .conftest import GOLDEN_DIR

FIXTURES = ("reproj_ragged_48x40", "reproj_dup_nodelta_24x20", "reproj_undetected_k4_20x16", "reproj_empty_mask_20x16")
SEEDED = {
    "dup_k8": dict(seed=1, M=2, H=7, W=9, P=300, C=400, Kn=8, dup=3, hot=(0, 255, 399)),
    "k1_scale30": dict(seed=2, M=1, H=5, W=13, P=500, C=257, Kn=1, scale=30.0),
    "k5_scale0.1": dict(seed=3, M=3, H=4, W=6, P=90, C=270, Kn=5, scale=0.1, masked=0.5),
    "underflow": dict(seed=4, M=1, H=9, W=9, P=400, C=300, Kn=8, logsigma=np.log(1000.0)),
}
SMS = 132


def fixture_scene(name):
    g = dict(np.load(os.path.join(GOLDEN_DIR, name + ".npz")))
    M, H, W = g["in_feat_px"].shape[:3]
    rng = np.random.default_rng(0)
    up = rng.normal(size=(M * H * W, 3)).astype(np.float32)
    up[g["in_mask"].reshape(-1) == 0] = 0.0
    return dict(M=M, H=H, W=W, P=g["in_regist_feat"].shape[0], C=g["in_cand"].shape[0], K=int(g["in_meta"][0]),
                feat=g["in_feat_px"].reshape(-1, 16), rf=g["in_regist_feat"], xyz=g["in_xyz"], cand=g["in_cand"],
                logsigma=g["in_logsigma"], g=up)


def _scenes():
    out = {n: (lambda n=n: fixture_scene(n)) for n in FIXTURES}
    for n, kw in SEEDED.items():
        out[n] = lambda kw=kw: seeded(**kw)
    return out


def seeded(seed, M, H, W, P, C, Kn, **kw):
    return mb.scene(seed, M, H, W, P, C, Kn, **kw)


SCENES = _scenes()


def autograd(s, order):
    """reproj_model.global_match in float64 on the scene's inputs and the given lists, backward from s["g"]."""
    from .reproj_model import global_match
    f = lambda a: torch.tensor(np.asarray(a, np.float64), requires_grad=True)  # noqa: E731
    rf, xyz, ls = f(s["rf"]), f(s["xyz"]), f(s["logsigma"])
    feat = torch.tensor(s["feat"], dtype=torch.float64).reshape(s["M"], s["H"], s["W"], 16)
    xm, order, prob, score = global_match(feat, rf, xyz, torch.from_numpy(s["cand"]), ls, s["K"],
                                          order=torch.from_numpy(order))
    (xm.reshape(-1, 3) * torch.tensor(s["g"], dtype=torch.float64)).sum().backward()
    n = lambda t: t.detach().numpy()  # noqa: E731
    return dict(xyz_matched=n(xm).reshape(-1, 3), prob=n(prob), score=n(score), g_regist_feat=n(rf.grad),
                g_xyz=n(xyz.grad), g_logsigma=float(ls.grad))


def _close(a, b, what, rel=1e-12):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert np.abs(a - b).max() <= rel * max(np.abs(b).max(), 1e-300), what


@pytest.mark.parametrize("name", list(SCENES))
def test_model_equals_float64_autograd(name):
    s = SCENES[name]()
    m = mb.model(s, SMS)
    ref = autograd(s, m["idx"])
    from .reproj_model import all_scores
    want = torch.sort(-all_scores(torch.tensor(s["feat"], dtype=torch.float64), torch.tensor(s["rf"], dtype=torch.float64),
                                  torch.from_numpy(s["cand"])), dim=1, stable=True).indices[:, :s["K"]].numpy()
    assert np.array_equal(m["idx"], want), "float64 top-K lists differ from the model's sort"
    fw, bw = m["fwd"], m["bwd"]
    _close(np.take_along_axis(ref["score"], m["idx"], 1), fw["score"].v, "score")
    _close(ref["prob"], fw["prob"].v, "prob")
    _close(ref["xyz_matched"], np.stack([e.v for e in fw["xyz_matched"]], -1), "xyz_matched")
    grf, gx = mb.scatter(bw["g_cand"], s["cand"], s["M"] * s["P"], s["P"])
    _close(ref["g_regist_feat"], grf.v, "g_regist_feat")
    _close(ref["g_xyz"], gx.v, "g_xyz")
    _close(ref["g_logsigma"], bw["g_logsigma"].v, "g_logsigma")


def _within(e, what):
    assert e.f is not None, what
    tol = mb.K * mb.U * e.b + mb.FLOOR
    err = np.abs(e.f.astype(np.float64) - e.v)
    assert (err <= tol).all(), (what, float((err / tol).max()))


@pytest.mark.parametrize("name", list(SCENES))
def test_fp32_shadow_within_its_bound(name):
    s = SCENES[name]()
    m = mb.model(s, SMS)
    # the shadow rounds each product of the score chain (no FMA): still one valid evaluation of the charged chain
    _within(m["scores"], "scores")
    fw, bw = m["fwd"], m["bwd"]
    _within(fw["score"], "top_score")
    _within(fw["prob"], "prob")
    for e in fw["xyz_matched"]:
        _within(e, "xyz_matched")
    _within(bw["g_cand"], "g_cand")
    _within(bw["g_logsigma"], "g_logsigma")
    grf, gx = mb.scatter(bw["g_cand"], s["cand"], s["M"] * s["P"], s["P"])
    _within(grf, "g_regist_feat")
    _within(gx, "g_xyz")


def test_knife_rule_flags_a_near_tie_and_not_an_exact_duplicate():
    """Two copies of one surfel tie exactly (not a knife); nudging one copy's score by one ulp makes the pixel a knife."""
    s = mb.scene(5, 2, 1, 3, 50, 60, 2, dup=1)
    a, b = s["dup_at"]
    sc = mb.scores(s["feat"], s["rf"], s["cand"], 100)
    assert np.array_equal(sc.v[:, a], sc.v[:, b])
    for col in range(sc.v.shape[1]):
        if col not in (a, b):
            sc.v[:, col] = -1e3
    _, knife, _ = mb.topk(sc, s["cand"], 100, 2)
    assert not knife.any()
    sc.v[:, b] = np.nextafter(sc.v[:, a], np.inf)
    _, knife, _ = mb.topk(sc, s["cand"], 100, 2)
    assert knife.all()


def test_no_valid_candidate_gives_empty_slots_and_zero_gradients():
    """Every candidate index outside [0, M P): the lists are all -1, prob, xyz and every gradient exactly 0."""
    s = mb.scene(6, 1, 3, 5, 20, 5, 3, invalid=(0, 1, 2, 3, 4))
    m = mb.model(s, SMS)
    assert (m["idx"] == -1).all() and not m["knife"].any()
    fw, bw = m["fwd"], m["bwd"]
    assert (fw["prob"].v == 0).all() and (fw["prob"].f == 0).all()
    assert all((e.v == 0).all() and (e.f == 0).all() for e in fw["xyz_matched"])
    assert (bw["g_cand"].v == 0).all() and bw["g_logsigma"].v == 0
    knife, _ = mb.check_topk(m["scores"], s["cand"], 20, 3, m["idx"])
    assert not knife.any()
