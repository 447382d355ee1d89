"""The restated skinning chain and its bound (tests/skin_bounds.py), on the CPU: its values and hand-written VJP equal
the float64 autograd of the oracle's expressions (oracle/warp_oracle.py) evaluated on the same fp32 tables; its fp32
shadow lies within K u B + FLOOR of its value for every output and gradient outside the knife mask; and on a wide-bone
scene the bound is not vacuous."""
import numpy as np
import pytest
import torch

from . import skin_bounds as sb
from .skin_bounds import warp_scene as scene


def oracle(s):
    """oracle/warp_oracle.py's bob_warp expressions on the kernel's own tables, float64, with autograd; the upstream of
    the model's knife points is zeroed as the test zeroes it.  Returns (outputs, gradients)."""
    from oracle import warp_oracle as wo
    T = {k: torch.tensor(v, dtype=torch.float64, requires_grad=True) for k, v in s["tab"].items()}
    X = torch.tensor(s["xyz"], dtype=torch.float64, requires_grad=True)
    R = torch.tensor(s["rot"], dtype=torch.float64, requires_grad=True)
    D = None if s["delta"] is None else torch.tensor(s["delta"], dtype=torch.float64, requires_grad=True)
    P, B, M = X.shape[0], T["oq"].shape[0], T["sr"].shape[0]
    xb = wo.qapply(T["oq"][None].expand(P, -1, -1), X[:, None, :].expand(-1, B, -1)) + T["ot"][None]
    d2 = ((xb * T["ig"][None]) ** 2).sum(-1)
    logits = -(d2 + D) if D is not None else -d2
    w = torch.softmax(logits, -1)
    qa = T["sr"][:, w.argmax(-1)]
    sign = ((qa[:, :, None, :] * T["sr"][:, None]).sum(-1) > 0).to(X.dtype) * 2 - 1
    ws = w[None] * sign
    QR, QD = torch.einsum("mpb,mbl->mpl", ws, T["sr"]), torch.einsum("mpb,mbl->mpl", ws, T["sd"])
    inv = 1.0 / QR.norm(dim=-1, keepdim=True)
    q, t = wo.dq_to_qt(QR * inv, QD * inv)
    rt = wo.qmul(q, R[None].expand(M, -1, -1))
    xc = wo.qapply(T["cq"][:, None], wo.qapply(q, X[None].expand(M, -1, -1)) + t) + T["ct"][:, None]
    rc = wo.qmul(T["cq"][:, None].expand_as(rt), rt)
    ent = wo.skin_entropy(logits)
    f = lambda a: torch.tensor(a, dtype=torch.float64)  # noqa: E731
    ((xc * f(s["gx"])).sum() + (rc * f(s["gr"])).sum() + (ent * f(s["ge"])).sum()).backward()
    outs = dict(xyz_cam=xc, rot_cam=rc, entropy=ent)
    grads = dict(g_xyz=X.grad, g_rot=R.grad, **{"g_" + k: v.grad for k, v in T.items()})
    if D is not None:
        grads["g_delta"] = D.grad
    return ({k: v.detach().numpy() for k, v in outs.items()}, {k: v.numpy() for k, v in grads.items()})


def _model(s):
    m = sb.warp_model(s["xyz"], s["rot"], s["tab"], s["delta"], s["gx"], s["gr"], s["ge"])
    kn = m["knife"]
    s["gx"][:, kn] = 0.0
    s["gr"][:, kn] = 0.0
    s["ge"][kn] = 0.0
    return m, kn


GRID = [(B, M, delta, wide) for B in (1, 2, 3, 4, 5, 31, 32, 33, 34, 63, 64) for M, delta, wide in
        [((1, 2)[B % 2], ("small", None)[B % 3 == 0], B % 4 == 1)]]


def _check(m, kn, outs, grads):
    """Outside the knife rows: the restatement equals the oracle to 1e-12 of each tensor's max, and its fp32 shadow lies
    within K u B + FLOOR of it."""
    for k, ref in list(outs.items()) + list(grads.items()):
        e = m[k]
        rows = (slice(None), ~kn) if k in ("xyz_cam", "rot_cam") else (~kn if k in ("entropy", "g_xyz", "g_rot", "g_delta")
                                                                           else slice(None))
        v, b, f, ref = e.v[rows], e.b[rows], e.f[rows], ref[rows]
        scale = np.abs(ref).max() + 1e-300
        assert np.abs(v - ref).max() <= 1e-12 * scale, (k, np.abs(v - ref).max() / scale)
        ratio = np.abs(f.astype(np.float64) - v) / (sb.K * sb.U * b + sb.FLOOR)
        assert ratio.max() <= 1.0, (k, float(ratio.max()), np.unravel_index(int(np.argmax(ratio)), ratio.shape))


@pytest.mark.parametrize("B,M,delta,wide", GRID)
def test_restatement_equals_oracle_and_shadow_meets_bound(B, M, delta, wide):
    s = scene(seed=40 + B, P=300, B=B, M=M, delta=delta, wide=wide)
    m, kn = _model(s)
    assert kn.sum() <= 3, int(kn.sum())
    _check(m, kn, *oracle(s))


def test_table_oracle_equals_warp_oracle():
    """oracle() on float64 tables from vidu4d_b200.warp.warp_tables is oracle/warp_oracle.py's bob_warp itself, so the
    pinning follows that oracle's arg-max and sign rules."""
    from oracle import warp_oracle as wo
    from tests.golden.make_warp_golden import make_inputs
    from vidu4d_b200.warp import warp_tables
    from .reproj_model import q2dq
    inp = {k: v.double() for k, v in make_inputs(3, 400, 9, 3, True).items()}
    rest, art = q2dq(inp["rest_q"], inp["rest_t"]), q2dq(inp["art_q"], inp["art_t"])
    with torch.no_grad():
        oq, ot, ig, sr, sd = warp_tables(rest, art, inp["log_gauss"])
        rest_m = (rest[0][None].expand(3, -1, -1), rest[1][None].expand(3, -1, -1))
        ref = wo.bob_warp(inp["xyz"], inp["rot"], rest, torch.exp(-inp["log_gauss"]), wo.dq_mul(art, wo.dq_inverse(rest_m)),
                          (inp["cam_q"], inp["cam_t"]), inp["delta"])
    z = lambda *sh: np.zeros(sh)  # noqa: E731
    s = dict(xyz=inp["xyz"].numpy(), rot=inp["rot"].numpy(), delta=inp["delta"].numpy(), gx=z(3, 400, 3), gr=z(3, 400, 4),
             ge=z(400), tab={k: v.numpy() for k, v in dict(oq=oq, ot=ot, ig=ig, sr=sr, sd=sd, cq=inp["cam_q"],
                                                            ct=inp["cam_t"]).items()})
    outs, _ = oracle(s)
    for k, r in zip(("xyz_cam", "rot_cam", "entropy"), ref):
        assert np.abs(outs[k] - r.numpy()).max() <= 1e-12 * np.abs(r.numpy()).max(), k


def test_bound_is_not_vacuous_on_wide_bones():
    """On the cycle fixtures' wide bones (median surfel: at least 4 bones above 1e-3) the median of u B / |value| stays
    under a stated ceiling: 1e-4 (a few hundred u) for the outputs and the per-point gradients of rotation; 3e-3 for
    dL/dxyz and dL/ddelta, whose softmax VJP cancels (sum_b dL/dlogit_b = 0); 1e-2 for the table gradients, sums over
    points of terms of either sign whose total is far below the sum of their magnitudes that the reduction charges."""
    s = scene(seed=7, P=512, B=25, M=2, delta="small", wide=True)
    m, kn = _model(s)
    w = sb.skin(sb._pts(s["xyz"]), sb._bones(s["tab"]["oq"], s["tab"]["ot"], s["tab"]["ig"]), sb._E.leaf(s["delta"]))["w"].v
    assert np.median((w > 1e-3).sum(-1)) >= 4
    for k in ("xyz_cam", "rot_cam", "entropy", "g_xyz", "g_rot", "g_delta", "g_oq", "g_ot", "g_ig", "g_sr", "g_sd",
              "g_cq", "g_ct"):
        e = m[k]
        nz = e.v != 0
        med = float(np.median(sb.U * e.b[nz] / np.abs(e.v[nz])))
        ceil = 1e-2 if k in sb.TABLE_GRADS else 3e-3 if k in ("g_xyz", "g_delta") else 1e-4
        assert med < ceil, (k, med)


def test_exact_decisions():
    """An exact logit tie takes the lower bone; an exactly orthogonal rotation takes sign -1 -- in the restatement, as
    torch.argmax and `qdot > 0` do, and neither is a knife."""
    s = scene(seed=5, P=256, B=4, M=1, delta=None, wide=True)
    tab = s["tab"]
    for k in ("oq", "ot", "ig"):
        tab[k][2] = tab[k][1]
    tab["sr"][0, 0] = (1.0, 0.0, 0.0, 0.0)
    tab["sr"][0, 3] = (0.0, 1.0, 0.0, 0.0)
    x = sb._pts(s["xyz"])
    sk = sb.skin(x, sb._bones(tab["oq"], tab["ot"], tab["ig"]), None)
    assert not (sk["anchor"] == 2).any() and (sk["anchor"] == 1).any()
    assert not sk["knife"].any()
    bl = sb.blend(sk, tab["sr"][0], tab["sd"][0])
    a0 = sk["anchor"] == 0
    assert a0.any() and (bl[2][a0, 3] == -1.0).all() and not bl[4][a0].any()
    m, kn = _model(s)
    assert not kn.any()
    _check(m, kn, *oracle(s))


# ------------------------------------------------------------------------------------------------ reproj and cycle
def _t_chain(oq, ot, ig, sr, sd, X, D):
    """The skinning chain of oracle/warp_oracle.py on one frame's tables (float64 torch): (q, t, logits)."""
    from oracle import warp_oracle as wo
    P, B = X.shape[0], oq.shape[0]
    xb = wo.qapply(oq[None].expand(P, -1, -1), X[:, None, :].expand(-1, B, -1)) + ot[None]
    d2 = ((xb * ig[None]) ** 2).sum(-1)
    logits = -(d2 + D) if D is not None else -d2
    w = torch.softmax(logits, -1)
    qa = sr[w.argmax(-1)]
    sign = ((qa[:, None, :] * sr[None]).sum(-1) > 0).to(X.dtype) * 2 - 1
    ws = w * sign
    QR, QD = ws @ sr, ws @ sd
    inv = 1.0 / QR.norm(dim=-1, keepdim=True)
    q, t = wo.dq_to_qt(QR * inv, QD * inv)
    return q, t, logits


def _leaves(d):
    return {k: (None if v is None else torch.tensor(np.asarray(v), dtype=torch.float64, requires_grad=True)) for k, v in d.items()}


def reproj_oracle(s):
    """tests/reproj_model.py's projection and reproj_loss on the kernel's tables, float64, with autograd."""
    from oracle import warp_oracle as wo
    from .reproj_model import reproj_loss
    T = _leaves(s["tab"])
    X, D = _leaves(dict(x=s["xyz_m"], d=s["delta"])).values()
    M = X.shape[0]
    xy = []
    for m in range(M):
        q, t, _ = _t_chain(T["oq"], T["ot"], T["ig"], T["sr"][m], T["sd"][m], X[m], None if D is None else D[m])
        xc = wo.qapply(T["cq"][m][None], wo.qapply(q, X[m]) + t) + T["ct"][m][None]
        h = xc @ torch.tensor(s["Kmat"][m], dtype=torch.float64).T
        xy.append(h[:, :2] / (h[:, 2:] + 1e-6))
    xy = torch.stack(xy)
    f = lambda k: torch.tensor(s[k], dtype=torch.float64)  # noqa: E731
    # (M,HW) pixels as (M,H=HW,W=1) images
    loss, terms, counts = reproj_loss(xy[:, :, None], f("hxy")[:, :, None], f("mask")[:, :, None], f("det"), float(s["weight"]),
                                      float(s["train_res"]))
    (loss * float(s["g_loss"])).backward()
    grads = dict(g_xyz=X.grad, **{"g_" + k: v.grad for k, v in T.items()})
    if D is not None:
        grads["g_delta"] = D.grad
    return dict(xy=xy.detach(), loss=loss.detach(), terms=terms.detach(), counts=counts), grads


def cycle_oracle(s):
    """tests/cycle_model.py's values and positive_mean_terms on the kernel's tables, float64, with autograd."""
    from oracle import warp_oracle as wo
    from .cycle_model import positive_mean_terms
    T = _leaves(s["tab"])
    X, XC, D = _leaves(dict(x=s["xyz"], xc=s["xyz_cam"], d=s["delta"])).values()
    M = XC.shape[0]
    vals = [[], [], []]
    for m in range(M):
        qi = wo.qconj(T["cq"][m])
        xt = wo.qapply(qi[None], XC[m]) + wo.qapply(qi, -T["ct"][m])[None]
        q, t, logits = _t_chain(T["oq"][m], T["ot"][m], T["ig"], T["sr"][m], T["sd"][m], xt, None if D is None else D[m])
        vals[0].append((wo.qapply(q, xt) + t - X).norm(dim=-1))
        vals[1].append((D[m] ** 2).mean(-1) if D is not None else torch.zeros_like(vals[0][-1]))
        vals[2].append(wo.skin_entropy(logits))
    loss, terms, counts = positive_mean_terms([torch.stack(v) for v in vals], [float(w) for w in s["weights"]])
    (loss * float(s["g_loss"])).backward()
    grads = dict(g_xyz=X.grad, g_xyz_cam=XC.grad, **{"g_" + k: v.grad for k, v in T.items()})
    if D is not None:
        grads["g_delta"] = D.grad
    return dict(loss=loss.detach(), terms=terms.detach(), counts=counts), grads


def _pin(m, outs, grads, skip=()):
    for k, ref in list(outs.items()) + list(grads.items()):
        if k == "counts":
            assert np.array_equal(m[k], ref.numpy()), (k, m[k], ref)
            continue
        e, ref = m[k], ref.numpy()
        scale = np.abs(ref).max() + 1e-300
        assert np.abs(e.v - ref).max() <= 1e-12 * scale, (k, np.abs(e.v - ref).max() / scale)
        ratio = np.abs(e.f.astype(np.float64) - e.v) / (sb.K * sb.U * e.b + sb.FLOOR)
        assert ratio.max() <= 1.0, (k, float(ratio.max()))


def run_reproj_model(s):
    kn = sb.reproj_knife(s["xyz_m"], s["delta"], s["tab"], s["Kmat"], s["hxy"])
    s["mask"][kn] = 0.0
    m = sb.reproj_model(s["xyz_m"], s["delta"], s["tab"], s["Kmat"], s["hxy"], s["mask"], s["det"], s["weight"],
                        s["train_res"], s["g_loss"])
    return m, kn


def run_cycle_model(s):
    """The model on the surfels with no knife value in any frame (dropped from the inputs, as on the GPU side)."""
    m = sb.cycle_model(s["xyz"], s["xyz_cam"], s["tab"], s["delta"], s["weights"], s["g_loss"])
    kn = m["knife"]
    if kn.any():
        s.update(xyz=s["xyz"][~kn], xyz_cam=s["xyz_cam"][:, ~kn], delta=None if s["delta"] is None else s["delta"][:, ~kn])
        m = sb.cycle_model(s["xyz"], s["xyz_cam"], s["tab"], s["delta"], s["weights"], s["g_loss"])
        assert not m["knife"].any()
    return m, kn


@pytest.mark.parametrize("B,M,HW,delta", [(1, 2, 129, True), (5, 1, 300, False), (34, 3, 127, True), (64, 2, 200, True)])
def test_reproj_restatement(B, M, HW, delta):
    s = sb.reproj_scene(seed=60 + B, M=M, HW=HW, B=B, delta=delta)
    m, kn = run_reproj_model(s)
    assert kn.sum() <= 3
    outs, grads = reproj_oracle(s)
    _pin(m, outs, grads)


@pytest.mark.parametrize("B,M,P,delta", [(1, 2, 129, True), (4, 1, 300, False), (33, 3, 127, True), (64, 2, 200, True)])
def test_cycle_restatement(B, M, P, delta):
    s = sb.cycle_scene(seed=70 + B, P=P, B=B, M=M, delta=delta)
    m, kn = run_cycle_model(s)
    assert kn.sum() <= 3, int(kn.sum())
    outs, grads = cycle_oracle(s)
    _pin(m, outs, grads)
