"""GPU: every element of both Adam entry points (sr_adam_flat, sr_adam_flat_state; csrc/optim.cu) against torch's Adam.

Each call runs from fp32 inputs set by the test (so errors never compound) and every element of param, exp_avg and
exp_avg_sq must lie inside tests/optim_model.py's bound, |gpu - value| <= K u B + FLOOR, whose value is torch's foreach
Adam in float64.  Where the model's value or fp32 shadow is not finite (NaN / Inf gradients or coefficient, grad * grad
past FLT_MAX) the kernel must give torch.optim.Adam's own bits on the same GPU; with rates that are fp32 values it must
give them everywhere.  A 2 000-step run of clip_grad_norm_ + step() next to torch's clip_grad_norm_ + Adam compares the
moments bit for bit and the update element by element.  Each case prints the largest err / (K u B) per tensor."""
import ctypes as C

import numpy as np
import pytest
import torch

from . import optim_model as om

pytestmark = pytest.mark.gpu

SURFEL_WIDTHS = (3, 3, 45, 1, 2, 4, 16)
STAGE3_LRS = (1.6e-4, 2.5e-3, 2.5e-3 / 20.0, 5e-2, 5e-3, 1e-3, 2.5e-3)
MULTI_PASS = 132 * 16 * 1024          # elements one grid-stride pass of the capped grid covers


@pytest.fixture(scope="module")
def dev(built):
    from vidu4d_b200 import _capi
    _capi.load()
    return torch.device("cuda:0")


def _layout(name):
    """(group sizes, torch's rates): the seven surfel groups at P = 1 / 5003 / 30000, empty groups, all 8 groups with
    their own rates and one at 0."""
    if name in ("p1", "p5003", "multi_pass"):
        P = {"p1": 1, "p5003": 5003, "multi_pass": 30000}[name]
        return [P * w for w in SURFEL_WIDTHS], list(STAGE3_LRS)
    if name == "empty_groups":
        return [0, 37, 0, 1, 5, 0, 1023, 6], [1e-3, 2e-3, 3e-3, 4e-3, 5e-3, 6e-3, 7e-3, 8e-3]
    if name == "maxg_lr0":
        return [13, 7, 29, 1, 3, 22, 9, 17], [1.6e-4, 2.5e-3, 1.25e-4, 5e-2, 0.0, 1e-3, 2.5e-3, 3.3e-2]
    raise KeyError(name)


def _fill(sizes, seed):
    """Every om.CASES element set over one slice of the buffer (so every case meets several groups)."""
    n = sum(sizes)
    parts = [om.case_inputs(c, n, seed) for c in om.CASES]
    cut = np.linspace(0, n, len(parts) + 1).astype(int)
    return [np.concatenate([p[k][a:b] for p, a, b in zip(parts, cut, cut[1:])]) for k in range(4)], cut


def _kernel(entry, sizes, lrs, p, g, m, v, t, grad_scale, coef, dev):
    """One call of the entry point on copies of the fp32 inputs; returns (param, exp_avg, exp_avg_sq) as numpy."""
    from vidu4d_b200 import _capi
    T = [torch.from_numpy(x.copy()).to(dev) for x in (p, g, m, v)]
    begin = (C.c_int64 * (len(sizes) + 1))(*np.concatenate([[0], np.cumsum(sizes)]).tolist())
    if entry == "flat":
        assert coef == 1.0
        lr = (C.c_float * len(sizes))(*lrs)
        _capi.call("sr_adam_flat", dev, len(sizes), begin, lr, 0.9, 0.999, 1e-15, t, float(grad_scale), *T)
    else:
        lr = torch.tensor(lrs, dtype=torch.float32, device=dev)
        step = torch.tensor(t - 1, dtype=torch.int64, device=dev)
        cf = torch.tensor(coef, dtype=torch.float32, device=dev)
        _capi.call("sr_adam_flat_state", dev, len(sizes), begin, lr, 0.9, 0.999, 1e-15, step, float(grad_scale), cf, *T)
        assert int(step) == t
    torch.cuda.synchronize()
    return [x.cpu().numpy() for x in (T[0], T[2], T[3])]


def _torch(sizes, lrs, p, g, m, v, t, grad_scale, coef, dev, fused=False):
    """torch.optim.Adam (foreach, or fused) on the same GPU from the same state at step t, one tensor per group, on the
    gradient (g * grad_scale) * coef rounded as the kernel rounds it."""
    cuts = np.concatenate([[0], np.cumsum(sizes)])
    gr = torch.from_numpy(g).to(dev) * np.float32(grad_scale) * torch.tensor(coef, dtype=torch.float32, device=dev)
    ps = [torch.nn.Parameter(torch.from_numpy(p[a:b].copy()).to(dev)) for a, b in zip(cuts, cuts[1:])]
    opt = torch.optim.Adam([{"params": [q], "lr": r} for q, r in zip(ps, lrs)], lr=0.0, eps=1e-15,
                           foreach=not fused, fused=fused)
    for q, a, b in zip(ps, cuts, cuts[1:]):
        q.grad = gr[a:b].clone()
        opt.state[q] = {"step": torch.tensor(float(t - 1)) if not fused else torch.tensor(float(t - 1), device=dev),
                        "exp_avg": torch.from_numpy(m[a:b].copy()).to(dev),
                        "exp_avg_sq": torch.from_numpy(v[a:b].copy()).to(dev)}
    opt.step()
    cat = lambda xs: torch.cat([x.detach().flatten() for x in xs]).cpu().numpy()  # noqa: E731
    return [cat(ps), cat([opt.state[q]["exp_avg"] for q in ps]), cat([opt.state[q]["exp_avg_sq"] for q in ps])]


def _same_bits(a, b):
    return (a.view(np.int32) == b.view(np.int32)) | (np.isnan(a) & np.isnan(b))


NAMES = ("param", "exp_avg", "exp_avg_sq")


def _check(entry, layout, rates, t, coef, dev, grad_scale=0.3, seed=0):
    """One call against the model and torch; returns the largest err / (K u B) per tensor and the edges reached."""
    sizes, lrs = _layout(layout)
    if rates == "fp32":
        lrs = [float(np.float32(r)) for r in lrs]
    (p, g, m, v), cut = _fill(sizes, seed + t)
    lr_el = np.concatenate([np.full(n, r) for n, r in zip(sizes, lrs)])
    got = _kernel(entry, sizes, lrs, p, g, m, v, t, grad_scale, coef, dev)
    want = _torch(sizes, lrs, p, g, m, v, t, grad_scale, coef, dev)
    e = om.adam(p, g, m, v, lr_el, step=t, grad_scale=grad_scale, coef=coef, device_lr=rates != "fp32")
    worst = {}
    sp = om.special(e)
    for name, x, gk, wt in zip(NAMES, (e[k] for k in NAMES), got, want):
        r = om.ratio(gk, x, sp)
        bad = np.flatnonzero(r > 1.0)
        assert bad.size == 0, (entry, layout, t, coef, name, bad[:5], gk[bad[:5]], x.v[bad[:5]], x.b[bad[:5]])
        # outside the bound's reach, and everywhere when the kernel has torch's exact scalars: torch's own bits
        same = _same_bits(gk, wt)
        assert same[sp].all(), (entry, layout, t, coef, name, gk[sp][~same[sp]][:5], wt[sp][~same[sp]][:5])
        if rates == "fp32" or name != "param":
            assert same.all(), (entry, layout, t, coef, name, int((~same).sum()), gk[~same][:5], wt[~same][:5])
        else:
            assert om.rate_rounding_ok(gk, wt, p).all(), (entry, layout, t, name)
        worst[name] = float(r.max())
    # the edges: every case's slice reaches what it stands for
    sl = {c: slice(a, b) for c, a, b in zip(om.CASES, cut, cut[1:])}
    pk, mk, vk = got
    fin = np.isfinite(vk)
    edges = {
        "zero": np.array_equal(pk[sl["zero"]].view(np.int32), p[sl["zero"]].view(np.int32))
                and not mk[sl["zero"]].any() and not vk[sl["zero"]].any(),
        "zero_param": bool((pk[sl["zero_param"]] != 0).mean() > 0.5),
        "subnormal": bool(((vk[sl["subnormal"]] > 0) & (vk[sl["subnormal"]] < np.finfo(np.float32).tiny)).any()),
        "eps_decides": bool((np.abs(np.log10(np.sqrt(vk[sl["eps_decides"]].astype(np.float64) / (1 - 0.999 ** t)) / 1e-15))
                             <= 1).any()),
        "overflow": bool((~fin[sl["overflow"]]).any() and fin[sl["overflow"]].any()) or coef != 1.0 or grad_scale != 1.0,
        "nonfinite": bool(np.isnan(pk[sl["nonfinite"]]).any()),
    }
    if coef == coef and coef != 0.0:
        assert all(edges.values()), edges
    return worst, edges


LAYOUTS = ["p1", "p5003", "empty_groups", "maxg_lr0", "multi_pass"]


@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("entry", ["flat", "state"])
def test_every_element_inside_bound(entry, layout, dev):
    """t = 1, 2, 10, 1000, 100 000 at realistic rates and at fp32 rates; for the device-state entry point also the clip
    coefficients 0.37, 0, and NaN.  Groups start inside a float4 (P = 1, 5003, the empty and 8-group layouts), the
    multi-pass layout makes the capped grid stride more than once, one group has rate 0."""
    sizes, _ = _layout(layout)
    if layout == "multi_pass":
        assert sum(sizes) > MULTI_PASS
    else:
        assert any(b % 4 for b in np.cumsum(sizes)[:-1])
    report = {}
    for t in (1, 2, 10, 1000, 100000):
        for rates in ("stage3", "fp32"):
            gs = 1.0 if t in (1, 1000) else 0.3
            coefs = (1.0,) if entry == "flat" else (1.0, 0.37, 0.0, float("nan"))
            for coef in coefs:
                worst, _ = _check(entry, layout, rates, t, coef, dev, grad_scale=gs)
                for k, w in worst.items():
                    report[k] = max(report.get(k, 0.0), w)
    print(f"{entry} {layout}: largest err / (K u B) {report}")


def _surfel_model(P, dev, lrs, seed=4):
    from vidu4d_b200.surfel_store import FlatSurfelModel
    g = torch.Generator(device=dev).manual_seed(seed)
    mk = lambda k: torch.randn((P, k), device=dev, generator=g)  # noqa: E731
    names = ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation", "regist_feat")
    return FlatSurfelModel(mk(3), mk(3).view(P, 1, 3), mk(45).view(P, 15, 3), mk(1), mk(2), mk(4), regist_feat=mk(16) * 0.1,
                           lrs=dict(zip(names, lrs)))


@pytest.mark.parametrize("rates", ["stage3", "fp32"])
def test_2000_steps_against_torch_clip_and_adam(rates, dev):
    """2 000 steps of clip_grad_norm_(5, extras) + step() next to torch.nn.utils.clip_grad_norm_ + torch.optim.Adam
    (foreach, eps 1e-15) over the seven groups plus extras, clipping on most steps.  Each step starts both from torch's
    state.  exp_avg and exp_avg_sq equal torch's bit for bit; the parameters too with fp32 rates, and within the rate's
    rounding otherwise.  Prints the largest update difference relative to the update, and fused=True's for
    information."""
    lrs = [float(np.float32(r)) for r in STAGE3_LRS] if rates == "fp32" else list(STAGE3_LRS)
    P = 5003
    m = _surfel_model(P, dev, lrs)
    gen = torch.Generator(device=dev).manual_seed(2)
    extras = [torch.nn.Parameter(torch.rand(3, device=dev, generator=gen)),
              torch.nn.Parameter(torch.randn((64, 32), device=dev, generator=gen))]
    ref = [p.detach().clone().requires_grad_(True) for p in m.flat_params()]
    fus = [p.detach().clone().requires_grad_(True) for p in m.flat_params()]
    ref_x = [p.detach().clone().requires_grad_(True) for p in extras]
    opt_ref = torch.optim.Adam([{"params": [p], "lr": r} for p, r in zip(ref, lrs)] + [{"params": ref_x, "lr": 1e-3}],
                               lr=0.0, eps=1e-15, foreach=True)
    opt_fus = torch.optim.Adam([{"params": [p], "lr": r} for p, r in zip(fus, lrs)], lr=0.0, eps=1e-15, fused=True)
    worst, worst_fused, clipped, coef_differs = 0.0, 0.0, 0, 0
    for step in range(1, 2001):
        m.zero_grad_flat()
        m.grad_flat.copy_(torch.randn(m.grad_flat.shape, device=dev, generator=gen) * (3e-2 if step % 5 else 1e-4))
        for p, r, f in zip(m.flat_params(), ref, fus):
            r.grad, f.grad = p.grad.detach().clone(), p.grad.detach().clone()
        for p, r in zip(extras, ref_x):
            gx = torch.randn(p.shape, device=dev, generator=gen) * 1e-2
            p.grad, r.grad = gx.clone(), gx.clone()
        raw = [r.grad.clone() for r in ref]
        # both start from torch's state
        with torch.no_grad():
            for p, r in zip(m.flat_params(), ref):
                p.copy_(r)
            if step > 1:
                m.exp_avg.copy_(torch.cat([opt_ref.state[r]["exp_avg"].flatten() for r in ref]))
                m.exp_avg_sq.copy_(torch.cat([opt_ref.state[r]["exp_avg_sq"].flatten() for r in ref]))
        before = torch.cat([r.detach().flatten() for r in ref])
        total = m.clip_grad_norm_(5.0, extras)
        total_t = torch.nn.utils.clip_grad_norm_(ref + ref_x, 5.0)
        assert abs(float(total) - float(total_t)) <= 4 * float(np.spacing(np.float32(float(total_t)))), step
        # the moments compare bit for bit from the same gradient: where the two totals differ in their last bits, so
        # that torch's coefficient is not the kernel's, torch's Adam gets the kernel's coefficient
        if not bool(torch.clamp(5.0 / (total_t + 1e-6), max=1.0) == m.clip_coef):
            coef_differs += 1
            for r, g0 in zip(ref, raw):
                r.grad = g0 * m.clip_coef
        for f, r in zip(fus, ref):
            f.grad = r.grad.clone()
        clipped += float(m.clip_coef) < 1.0
        m.step()
        opt_ref.step()
        opt_fus.step()
        assert int(m.device_step) == step
        got_m, got_v = m.exp_avg, m.exp_avg_sq
        want_m = torch.cat([opt_ref.state[r]["exp_avg"].flatten() for r in ref])
        want_v = torch.cat([opt_ref.state[r]["exp_avg_sq"].flatten() for r in ref])
        assert torch.equal(got_m, want_m) and torch.equal(got_v, want_v), (step, int((got_m != want_m).sum()),
                                                                           int((got_v != want_v).sum()))
        pk, pt = m.flat.detach(), torch.cat([r.detach().flatten() for r in ref])
        uk, ut = (pk - before).double(), (pt - before).double()
        if rates == "fp32":
            assert torch.equal(pk, pt), (step, int((pk != pt).sum()))
        else:
            assert om.rate_rounding_ok(pk.cpu().numpy(), pt.cpu().numpy(), before.cpu().numpy()).all(), step
        nz = ut != 0
        worst = max(worst, float(((uk - ut).abs()[nz] / ut.abs()[nz]).max()) if bool(nz.any()) else 0.0)
        pf = torch.cat([f.detach().flatten() for f in fus]).double()
        uf = pf - before.double()
        worst_fused = max(worst_fused, float(((uf - ut).abs()[nz] / ut.abs()[nz]).max()) if bool(nz.any()) else 0.0)
        with torch.no_grad():
            for f, r in zip(fus, ref):
                f.copy_(r)
            for f, r in zip(fus, ref):
                opt_fus.state[f]["exp_avg"].copy_(opt_ref.state[r]["exp_avg"])
                opt_fus.state[f]["exp_avg_sq"].copy_(opt_ref.state[r]["exp_avg_sq"])
    assert clipped > 1000
    print(f"{rates} rates, 2000 steps: exp_avg and exp_avg_sq equal torch's bit for bit; largest |update - torch's| / "
          f"|torch's update| {worst:.3g} (fused=True against foreach: {worst_fused:.3g}); clip coefficients that differ "
          f"from torch's: {coef_differs}")
