"""CPU pinning of the Adam element restatement and its rounding-error bound (tests/optim_model.py adam()): with torch's
scalars kept in double its float64 value is torch.optim.Adam run in float64; its fp32 shadow, with and without FMA,
lies inside the bound; and eight kernel mistakes planted in the shadow -- among them the kernel as it was before its
scalars were formed as torch forms them -- fall outside it on a clear share of some tensor's elements."""
import numpy as np
import pytest
import torch

from . import optim_model as om

# seven groups of the flat surfel store (xyz, f_dc, f_rest, opacity, scaling, rotation, regist_feat) at P = 13, with
# the reference's rates; one more group at rate 0
WIDTHS = (3, 3, 45, 1, 2, 4, 16, 5)
LRS = (1.6e-4, 2.5e-3, 2.5e-3 / 20.0, 5e-2, 5e-3, 1e-3, 2.5e-3, 0.0)
P = 13


def _layout():
    sizes = [P * w for w in WIDTHS]
    lr = np.concatenate([np.full(n, r) for n, r in zip(sizes, LRS)])
    return sizes, lr


def _inputs(seed):
    """One of every om.CASES element set, back to back over the eight groups (each case fills a slice)."""
    sizes, lr = _layout()
    n = sum(sizes)
    parts = [om.case_inputs(c, n, seed) for c in om.CASES]
    cut = np.linspace(0, n, len(parts) + 1).astype(int)
    out = [np.concatenate([p[k][a:b] for p, a, b in zip(parts, cut, cut[1:])]) for k in range(4)]
    return out, lr


def test_value_is_torch_adam_in_float64():
    """50 steps with 8 groups, clipping, grad_scale and every om.CASES edge: from each step's fp32 state, the model's
    float64 value with double scalars equals torch.optim.Adam(foreach=False) in float64 on the CPU to 1e-14 of the
    bound's scale, NaN and Inf where torch has them."""
    (p, g0, _, _), lr = _inputs(1)
    m, v = np.zeros_like(p), np.zeros_like(p)          # torch starts from zero moments
    sizes, _ = _layout()
    params = [torch.zeros(n, dtype=torch.float64, requires_grad=True) for n in sizes]
    opt = torch.optim.Adam([{"params": [q], "lr": r} for q, r in zip(params, LRS)], lr=0.0, eps=1e-15, foreach=False)
    cuts = np.cumsum([0] + list(sizes))
    rng = np.random.default_rng(5)
    gs = np.float32(0.3)
    for t in range(1, 51):
        g = (g0 * np.float32(10.0 ** rng.uniform(-1, 1))).astype(np.float32)
        coef = np.float32(rng.uniform(0.2, 1.0)) if t % 2 else np.float32(1.0)
        e = om.adam(p, g, m, v, lr, step=t, grad_scale=gs, coef=coef, f32=False)
        gr = (g.astype(np.float64) * float(gs)) * float(coef)          # gs, coef: fp32 values
        for i, q in enumerate(params):
            a, b = cuts[i], cuts[i + 1]
            with torch.no_grad():
                q.copy_(torch.from_numpy(p[a:b].astype(np.float64)))
            q.grad = torch.from_numpy(gr[a:b].copy())
            st = opt.state[q]
            if st:
                st["exp_avg"].copy_(torch.from_numpy(m[a:b].astype(np.float64)))
                st["exp_avg_sq"].copy_(torch.from_numpy(v[a:b].astype(np.float64)))
        opt.step()
        got = {"param": torch.cat([q.detach() for q in params]).numpy(),
               "exp_avg": torch.cat([opt.state[q]["exp_avg"] for q in params]).numpy(),
               "exp_avg_sq": torch.cat([opt.state[q]["exp_avg_sq"] for q in params]).numpy()}
        for name, x in e.items():
            want = got[name]
            fin = np.isfinite(want)
            assert np.array_equal(np.isnan(x.v), np.isnan(want)), (t, name)
            assert np.array_equal(x.v[~fin & ~np.isnan(want)], want[~fin & ~np.isnan(want)]), (t, name)
            err = np.abs(x.v[fin] - want[fin])
            assert (err <= 1e-14 * x.b[fin] + 1e-300).all(), (t, name, float(err.max()))
        # the next step starts from the fp32 rounding of this one's value (so that errors never compound)
        with np.errstate(all="ignore"):
            p, m, v = (e[k].v.astype(np.float32) for k in ("param", "exp_avg", "exp_avg_sq"))
        p = np.where(np.isfinite(p), p, np.float32(0.5))
        m = np.where(np.isfinite(m), m, np.float32(0.0))
        v = np.where(np.isfinite(v), v, np.float32(0.0))


CONFIGS = [(t, dev_lr, beta1) for t in (1, 2, 10, 1000, 100000) for dev_lr in (False, True) for beta1 in (0.9,)] + \
          [(3, False, 0.3), (3, True, 0.3)]


@pytest.mark.parametrize("fma", [True, False])
@pytest.mark.parametrize("t,device_lr,beta1", CONFIGS)
def test_shadow_inside_bound(t, device_lr, beta1, fma):
    """The fp32 shadow of every element lies inside K u B + FLOOR, fused or not, at every step count, with the rate as
    torch holds it and as the device holds it, and on the other lerp branch (beta1 = 0.3).  Every case's elements are
    checked (the non-finite ones are the GPU tests' to compare with torch)."""
    (p, g, m, v), lr = _inputs(t)
    for coef in (1.0, 0.37):
        e = om.adam(p, g, m, v, lr, beta1=beta1, step=t, grad_scale=0.3, coef=coef, device_lr=device_lr, fma=fma)
        sp = om.special(e)
        assert (~sp).sum() > 0.6 * sp.size
        for name, x in e.items():
            r = om.ratio(x.f, x, sp)
            assert r.max() <= 1.0, (name, float(r.max()), int(np.argmax(r)))


def _outside(e):
    """Per tensor: the number of finite elements whose shadow lies outside the bound."""
    sp = om.special(e)
    return {n: int((om.ratio(x.f, x, sp) > 1.0).sum()) for n, x in e.items()}


MUTANTS = {
    # name: (case, step, keyword arguments of om.adam, the tensor that must fail, why); fresh: zero moments, as at the
    # start of training (a moment carried over from earlier steps dilutes this step's increment)
    "today": ("realistic", 1, {"fresh": True}, "exp_avg_sq", "1 - beta2 formed in fp32: every increment 1.29e-5 (216 u) small"),
    "c2_f32": ("realistic", 1000, {"fresh": True}, "exp_avg_sq", "1 - beta2 formed in fp32"),
    "bc_f32": ("zero_param", 1, {}, "param", "sqrt(1 - 0.999f) is 6.4e-6 off sqrt(1 - 0.999)"),
    "eps_in_sqrt": ("eps_decides", 10, {}, "param", "sqrt(v + eps) swamps sqrt(v) ~ 1e-15"),
    "eps_before_div": ("eps_decides", 2, {}, "param", "eps scaled by 1 / sqrt(1 - beta2^2) = 22"),
    "no_coef": ("zero_param", 10, {"coef": 0.37}, "exp_avg_sq", "the clip coefficient never applied"),
    "gs_twice": ("zero_param", 10, {"grad_scale": 0.3}, "exp_avg", "the averaging applied twice"),
    "neighbour_rate": ("zero_param", 10, {}, "param", "each group stepped at the next group's rate"),
}


@pytest.mark.parametrize("name", list(MUTANTS))
def test_mutants_fall_outside(name):
    """Each planted mistake puts at least a quarter of the named tensor's elements outside the bound; the counts per
    tensor are printed.  "today" is the kernel as it was: fp32 1 - beta, fp32-beta bias corrections, an fp32 lr / bc1."""
    case, t, kw, tensor, why = MUTANTS[name]
    sizes, lr = _layout()
    n = sum(sizes)
    p, g, m, v = om.case_inputs(case, n, seed=3)
    kw = dict(kw, step=t)
    if kw.pop("fresh", False):
        m, v = np.zeros_like(m), np.zeros_like(v)
    if name == "neighbour_rate":
        shift = np.concatenate([np.full(s, r) for s, r in zip(sizes, LRS[1:] + LRS[:1])])
        e = om.adam(p, g, m, v, lr, shadow_lr=shift, **kw)
    else:
        e = om.adam(p, g, m, v, lr, mutant=name, **kw)
    clean = om.adam(p, g, m, v, lr, **kw)
    assert all(c == 0 for c in _outside(clean).values())
    out = _outside(e)
    print(f"{name}: outside the bound {out} of {n} ({why})")
    assert out[tensor] >= 0.25 * n, (name, out)
