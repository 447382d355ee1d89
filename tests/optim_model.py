"""Models of the device-state optimizer step (csrc/optim.cu, include/surfel_optim.h), shared by the CPU and GPU tests.

clip() and bias_corrections() restate sr_grad_norm_flat's coefficient and the Adam pass's scalars.  adam() restates one
element of adam_flat_kernel operation by operation on tests/error_bound.py's _E: a float64 value, a first-order bound B
(in units of u = 2^-24) on the error of an fp32 evaluation of the same operations, and that fp32 evaluation (the shadow).
The value is torch.optim.Adam's foreach step (torch/optim/adam.py _multi_tensor_adam, the default on CUDA) in float64:

    grad     = (g * grad_scale) * coef                       the averaging, then clip_grad_norm_'s in-place multiply
    exp_avg  = lerp(exp_avg, grad, 1 - beta1)                ATen Lerp.h: m + w (grad - m) for |w| < 0.5,
                                                             grad - (grad - m)(1 - w) otherwise
    exp_avg_sq = exp_avg_sq * beta2 + (1 - beta2) (grad grad)   _foreach_mul_, then _foreach_addcmul_ (one fma)
    denom    = sqrt(exp_avg_sq) / sqrt(1 - beta2^t) + eps
    param    = param + (-lr / (1 - beta1^t)) (exp_avg / denom)   _foreach_addcdiv_ (one fma)

with torch's scalars: 1 - beta, beta^t and lr / (1 - beta1^t) in double, each rounded once to the fp32 the foreach ops
compute with (constants(f32=True)); constants(f32=False) keeps them in double, which is torch run in float64.  Every
multiply-add is charged two roundings, so the bound holds whether or not it is fused.  A kernel that reads an fp32 rate
lr_f from the device (sr_adam_flat_state) forms fl(lr_f / bc1) instead of torch's fl(lr / bc1): that step size is
charged 3u of its size (one rounding of lr, one of the quotient, one of torch's own quotient).

check: |gpu - value| <= K u B + FLOOR element by element, K = 2 as in the other bound files, FLOOR = 2^-149 (one
subnormal spacing: _rnd already charges each underflowing rounding its 2^-150, and a larger floor would hide the
subnormal moments).  Elements whose float64 value or fp32 shadow is not finite (NaN / Inf gradients, a NaN coefficient,
grad * grad past FLT_MAX) are outside the bound's reach: the GPU tests compare them with torch's own result instead.
"""
import math

import numpy as np

from .error_bound import _E, _c

U = 2.0 ** -24
K = 2.0
FLOOR = 2.0 ** -149
DEVICE_LR_CHARGE = 3.0


def clip(group_sumsq, extra_norms, max_norm):
    """(total, coef) as sr_grad_norm_flat forms them from the float64 group sums of squares and the fp32 norms of the
    other gradients: total = fp32(sqrt(sum)), coef = min(fp32(fp32(1 / fp32(total + 1e-6)) * max_norm), 1), NaN kept."""
    t = 0.0
    for s in group_sumsq:
        t += float(s)
    for n in extra_norms:
        n = float(np.float32(n))
        t += n * n
    total = np.float32(math.sqrt(t) if t == t and t >= 0 else t)
    with np.errstate(over="ignore", divide="ignore", invalid="ignore"):
        rcp = np.float32(1.0) / (total + np.float32(1e-6))
        c = rcp * np.float32(max_norm)
    return total, (np.float32(1.0) if c > 1.0 else c)


def bias_corrections(beta1, beta2, step):
    """The Adam pass's bias corrections from torch's double betas: (1 - beta1^t in double, fp32(sqrt(1 - beta2^t)))."""
    return 1.0 - float(beta1) ** step, np.float32(math.sqrt(1.0 - float(beta2) ** step))


def constants(lr, beta1=0.9, beta2=0.999, eps=1e-15, step=1, f32=True):
    """torch's Adam scalars for step t: c1 = 1 - beta1, b2 = beta2, c2 = 1 - beta2, bc2s = sqrt(1 - beta2^t),
    step = lr / (1 - beta1^t) (lr: a number or a per-element float64 array), eps; each rounded to fp32 when f32."""
    bc1, _ = bias_corrections(beta1, beta2, step)
    c = {"c1": 1.0 - beta1, "b2": beta2, "c2": 1.0 - beta2, "bc2s": math.sqrt(1.0 - beta2 ** step),
         "step": np.asarray(lr, np.float64) / bc1, "eps": eps}
    if f32:
        c = {k: np.asarray(v, np.float32).astype(np.float64) for k, v in c.items()}
    return c


def kernel_constants(lr, beta1=0.9, beta2=0.999, eps=1e-15, step=1, device_lr=False, mutant=None):
    """The fp32 scalars adam_flat_kernel computes with.  device_lr: the rate is read back as fp32 first.  mutant: the
    scalars of a wrong kernel -- "c2_f32" (1 - beta2 in fp32 from the fp32 beta2), "bc_f32" (bias corrections from the
    fp32 betas), "today" (both, 1 - beta1 in fp32 as well, and lr / bc1 as an fp32 quotient of fp32 values)."""
    f = np.float32
    lr = np.asarray(lr, np.float64)
    if device_lr:
        lr = lr.astype(np.float32).astype(np.float64)
    c = {k: np.asarray(v, np.float32) for k, v in constants(lr, beta1, beta2, eps, step).items()}
    if mutant in ("c2_f32", "today"):
        c["c2"] = f(1.0) - f(beta2)
    if mutant in ("bc_f32", "today"):
        b1, b2 = float(f(beta1)), float(f(beta2))
        c["bc2s"] = f(math.sqrt(1.0 - b2 ** step))
        c["step"] = (lr / (1.0 - b1 ** step)).astype(np.float32)
    if mutant == "today":
        c["c1"] = f(1.0) - f(beta1)
        c["step"] = lr.astype(np.float32) / f(1.0 - float(f(beta1)) ** step)
    return c


def _fma(a, b, c, fused):
    """a * b + c charged as two roundings; the shadow rounds once when fused (nvcc's contraction, or __fmaf_rn)."""
    r = a * b + c
    if fused and r.f is not None:
        with np.errstate(all="ignore"):
            r.f = (np.asarray(a.f, np.longdouble) * np.asarray(b.f, np.longdouble) + np.asarray(c.f, np.longdouble)).astype(np.float32)
    return r


def adam(p, g, m, v, lr, beta1=0.9, beta2=0.999, eps=1e-15, step=1, grad_scale=1.0, coef=1.0, device_lr=False, fma=True,
         f32=True, mutant=None, shadow_lr=None):
    """One Adam step of every element: {"param", "exp_avg", "exp_avg_sq"} as _E (value, bound, fp32 shadow).

    p, g, m, v: fp32 arrays of one shape; lr: each element's rate (torch's double rate), a number or an array.
    grad_scale, coef: fp32 numbers.  device_lr: the kernel reads the rate as fp32 (sr_adam_flat_state), charged as the
    module docstring says.  f32=False: torch's scalars kept in double (the value is then torch's Adam in float64).
    The shadow uses kernel_constants(mutant) and, for the mutants that change an operation, that operation:
    "eps_in_sqrt" sqrt(v + eps) / bc2s, "eps_before_div" (sqrt(v) + eps) / bc2s, "no_coef", "gs_twice";
    shadow_lr: the rate the shadow uses instead of lr (a wrong group lookup)."""
    tc = constants(lr, beta1, beta2, eps, step, f32)
    kc = kernel_constants(lr if shadow_lr is None else shadow_lr, beta1, beta2, eps, step, device_lr, mutant)
    charge = {"step": DEVICE_LR_CHARGE * np.abs(tc["step"]) if device_lr else None}
    k = {n: _E(tc[n], charge.get(n), kc[n]) for n in tc}
    P, G, M, V = (_E.leaf(x) for x in (p, g, m, v))
    gs, cf = (_E.leaf(np.float32(x)) for x in (grad_scale, coef))        # both reach the kernel as fp32 values
    gr = (G * gs) * cf
    if mutant == "no_coef":
        gr.f = (G * gs).f
    elif mutant == "gs_twice":
        gr.f = ((G * gs) * gs * cf).f
    d = gr - M
    w = float(tc["c1"])
    if abs(w) < 0.5:
        M1 = _fma(k["c1"], d, M, fma)
    else:
        M1 = _fma(-d, _c(1.0) - k["c1"], gr, fma)
    V1 = _fma(k["c2"], gr * gr, V * k["b2"], fma)
    s = V1.sqrt()
    den = s / k["bc2s"] + k["eps"]
    if mutant == "eps_in_sqrt":
        den.f = ((V1 + k["eps"]).sqrt() / k["bc2s"]).f
    elif mutant == "eps_before_div":
        den.f = ((s + k["eps"]) / k["bc2s"]).f
    P1 = _fma(-k["step"], M1 / den, P, fma)
    return {"param": P1, "exp_avg": M1, "exp_avg_sq": V1}


def special(e):
    """Elements outside the bound's reach, given adam()'s dict: a non-finite float64 value or fp32 shadow in any of the
    three tensors (an exp_avg_sq that overflows to Inf leaves a finite but different parameter)."""
    bad = np.zeros(np.shape(e["param"].v), bool)
    for x in e.values():
        bad |= ~np.isfinite(x.v)
        if x.f is not None:
            bad |= ~np.isfinite(x.f)
    return bad


def ratio(x, e, skip=None):
    """err / (K u B + FLOOR) element by element (NaN infinite), 0 where skip."""
    x = np.asarray(x, np.float64)
    with np.errstate(invalid="ignore"):
        r = np.abs(x - e.v) / (K * U * e.b + FLOOR)
    r = np.where(np.isnan(r), np.inf, r)
    return np.where(skip, 0.0, r) if skip is not None else r


# ---- seeded element sets shared by the CPU and GPU tests: name -> what edge it reaches ----------------------------------
CASES = {
    "realistic": "O(1) parameters, gradients over six decades, moments of their size",
    "zero_param": "parameters 0, so that the new parameter is minus the update, exactly",
    "eps_decides": "sqrt(v / bc2) within a factor of 10 of eps = 1e-15",
    "subnormal": "grad * grad and the new second moment subnormal",
    "zero": "zero gradient and zero moments: everything stays 0, the parameter unchanged",
    "overflow": "|g| from 0.5 to 3.2 sqrt(FLT_MAX) = 1.8447e19: grad * grad overflows in fp32 on one side",
    "nonfinite": "NaN and +-Inf gradients next to finite ones",
}


def case_inputs(name, n, seed=0):
    """(p, g, m, v) fp32 arrays of n elements for a CASES entry."""
    rng = np.random.default_rng(seed)
    f = np.float32
    sc = 10.0 ** rng.uniform(-4, 2, n)
    p = rng.standard_normal(n)
    g = rng.standard_normal(n) * sc
    m = rng.standard_normal(n) * sc * 0.3
    v = (rng.standard_normal(n) * sc) ** 2
    if name == "zero_param":
        p = np.zeros(n)
    elif name == "eps_decides":
        sc = 1e-15 * 10.0 ** rng.uniform(-1, 1, n)
        p, g, m, v = np.zeros(n), rng.standard_normal(n) * sc, rng.standard_normal(n) * sc * 0.3, (rng.standard_normal(n) * sc) ** 2
    elif name == "subnormal":
        sc = 10.0 ** rng.uniform(-23, -20, n)
        p, g, m, v = np.zeros(n), rng.standard_normal(n) * sc, rng.standard_normal(n) * sc * 0.3, (rng.standard_normal(n) * sc) ** 2
    elif name == "zero":
        g, m, v = np.zeros(n), np.zeros(n), np.zeros(n)
    elif name == "overflow":
        g = np.sign(rng.standard_normal(n)) * 1.8446744e19 * 10.0 ** rng.uniform(-0.3, 0.5, n)
        m, v = np.zeros(n), np.zeros(n)
    elif name == "nonfinite":
        g[0::5] = np.nan
        g[1::5] = np.inf
        g[2::5] = -np.inf
    return tuple(np.asarray(x, np.float64).astype(f) for x in (p, g, m, v))


def rate_rounding_ok(p_new, p_want, p_old):
    """A kernel step whose only difference from torch's is the fp32 rate (step size within DEVICE_LR_CHARGE u of
    torch's): per element, |p_new - p_want| <= DEVICE_LR_CHARGE u |update| + u (|p_new| + |p_want|) -- the step-size
    charge on the update plus the final rounding of each parameter."""
    p_new, p_want, p_old = (np.asarray(x, np.float64) for x in (p_new, p_want, p_old))
    lim = DEVICE_LR_CHARGE * U * np.abs(p_want - p_old) + U * (np.abs(p_new) + np.abs(p_want))
    return (np.abs(p_new - p_want) <= lim) | (np.isnan(p_new) & np.isnan(p_want)) | (p_new == p_want)
