"""TEST INFRASTRUCTURE -- a first-order running error bound of an fp32 expression, evaluated in float64.

_E holds a float64 value v, a bound b (in units of u = 2^-24) on the absolute error of the fp32 evaluation of the same
expression on the same fp32 inputs, and optionally f, that fp32 evaluation itself (the "shadow": float32 NumPy, the same
operations in the same order).  Each operation adds |a| err(b) + |b| err(a) for a product, err(a) / |b| + |a/b| err(b) / |b|
for a quotient, and so on, plus one rounding of its result unless that result is exact in fp32 (a product with an exact 0
is); a rounding is charged u |v| plus 2^-150, the most a result that underflows to a subnormal can lose.  The shadow is carried
only where every operand has one (leaves made with _E.leaf); _c gives plain numbers one.

The library functions are charged their CUDA accuracy without --use_fast_math: expf <= 2 ulp, logf <= 1 ulp,
rsqrtf <= 2 ulp, counting 1 ulp as <= 2u|v| for a normal result; sqrtf and / are correctly rounded.  nvcc contracts
a*b + c into one FMA, which rounds once: the two roundings charged for it still bound it.
"""
import numpy as np


TINY_U = 2.0 ** -126       # half the subnormal spacing 2^-149, in units of u: a result that underflows errs by up to 2^-150


def _rnd(v, exact):
    """The rounding of one fp32 operation whose exact result is v: none where the operands are exact and v is a float;
    otherwise u |v| for a normal result, and at most 2^-150 more where it is subnormal."""
    r = np.abs(v)
    return np.where(exact & (v.astype(np.float32).astype(np.float64) == v), 0.0, r + TINY_U)


def _sh(fn, *xs):
    """The shadow of an operation: fn of the operands' fp32 shadows, or None when one of them has none."""
    if any(x.f is None for x in xs):
        return None
    with np.errstate(all="ignore"):
        return np.asarray(fn(*(x.f for x in xs)), np.float32)


class _E:
    """A float64 value and a bound (in units of u) on the absolute error of its fp32 evaluation, to first order."""
    __slots__ = ("v", "b", "f")

    def __init__(self, v, b=None, f=None):
        self.v = np.asarray(v, np.float64)
        self.b = np.zeros_like(self.v) if b is None else np.asarray(b, np.float64)
        self.f = None if f is None else np.asarray(f, np.float32)

    @staticmethod
    def const(c):
        """The exact value c of a constant the kernel rounds to fp32 (1.0f / 3.0f, 1e12f, 1e-12f): one rounding."""
        return _E(c, _rnd(np.asarray(c, np.float64), True), np.float32(c))

    @staticmethod
    def leaf(x):
        """An fp32 input: exact, and its own shadow."""
        x = np.asarray(x, np.float32)
        return _E(x.astype(np.float64), None, x)

    def __add__(s, o):
        o = _c(o)
        v = s.v + o.v
        return _E(v, s.b + o.b + _rnd(v, (s.b == 0) & (o.b == 0)), _sh(np.add, s, o))

    def __sub__(s, o):
        return s + (-_c(o))

    def __neg__(s):
        return _E(-s.v, s.b, None if s.f is None else -s.f)

    def __mul__(s, o):
        o = _c(o)
        v = s.v * o.v
        ex = ((s.b == 0) & (o.b == 0)) | ((s.v == 0) & (s.b == 0)) | ((o.v == 0) & (o.b == 0))     # x * exact 0 = 0
        return _E(v, np.abs(s.v) * o.b + np.abs(o.v) * s.b + _rnd(v, ex), _sh(np.multiply, s, o))

    def __truediv__(s, o):
        o = _c(o)
        with np.errstate(divide="ignore", invalid="ignore"):
            v = s.v / o.v
            b = s.b / np.abs(o.v) + np.abs(v) * o.b / np.abs(o.v)
        return _E(v, b + _rnd(v, ((s.b == 0) & (o.b == 0)) | ((s.v == 0) & (s.b == 0))), _sh(np.divide, s, o))

    def __getitem__(s, i):
        return _E(s.v[i], s.b[i], None if s.f is None else s.f[i])

    def abs(s):
        return _E(np.abs(s.v), s.b, None if s.f is None else np.abs(s.f))

    def sqrt(s):
        v = np.sqrt(s.v)
        with np.errstate(divide="ignore", invalid="ignore"):
            b = np.where(s.b > 0, s.b / (2.0 * v), 0.0)
        return _E(v, b + _rnd(v, s.b == 0), _sh(np.sqrt, s))

    # ---- the operations of the skinning kernels (csrc/warp_common.cuh)
    def scale(s, c):
        """Multiplication by an exact power of two (or its negative): exact in fp32, no rounding."""
        return _E(s.v * c, s.b * abs(c), None if s.f is None else s.f * np.float32(c))

    def exp(s):
        """expf: <= 2 ulp; exp(0) = 1 exactly."""
        v = np.exp(s.v)
        exact = (s.b == 0) & (s.v == 0)
        return _E(v, v * s.b + np.where(exact, 0.0, 4.0 * v), _sh(np.exp, s))

    def log(s):
        """logf: <= 1 ulp; log(1) = 0 exactly."""
        v = np.log(s.v)
        exact = (s.b == 0) & (s.v == 1)
        return _E(v, s.b / s.v + np.where(exact, 0.0, 2.0 * np.abs(v)), _sh(np.log, s))

    def rsqrt(s):
        """rsqrtf: <= 2 ulp, charged always."""
        v = 1.0 / np.sqrt(s.v)
        return _E(v, 0.5 * v * s.b / s.v + 4.0 * v, _sh(lambda x: np.float32(1.0) / np.sqrt(x), s))


def _c(x):
    return x if isinstance(x, _E) else _E(x, None, np.float32(x) if np.ndim(x) == 0 else np.asarray(x, np.float32))


def _where(c, a, b):
    a, b = _c(a), _c(b)
    f = None if a.f is None or b.f is None else np.where(c, a.f, b.f)
    return _E(np.where(c, a.v, b.v), np.where(c, a.b, b.b), f)


def _max(xs):
    """fmaxf over a sequence, in order: the value and bound of the float64 maximum, and the first arg-max as data (what
    torch.argmax and the kernels' `w[b] == mx` scan pick).  Returns (max, argmax index array)."""
    v = np.stack([x.v for x in xs], -1)
    i = np.argmax(v, -1)
    return _take(xs, i), i


def _take(xs, i):
    """Per element, xs[i] of a sequence of _E (a gather by data)."""
    pick = lambda a: np.take_along_axis(np.stack(a, -1), np.asarray(i)[..., None], -1)[..., 0]  # noqa: E731
    f = None if any(x.f is None for x in xs) else pick([x.f for x in xs])
    return _E(pick([x.v for x in xs]), pick([x.b for x in xs]), f)


def _seqsum(t, axis=-1, init=None):
    """A sum in one thread, term after term along `axis` (optionally onto init): each partial sum is one rounding.
    Adding a term to an exact 0.f start is exact."""
    v = np.cumsum(np.moveaxis(t.v, axis, -1), -1)
    b = np.moveaxis(t.b, axis, -1).sum(-1)
    rnd = np.abs(v[..., 1:]).sum(-1)
    f = None if t.f is None else np.add.accumulate(np.moveaxis(t.f, axis, -1), -1)[..., -1]
    out = _E(v[..., -1], b + rnd, f)
    if init is not None:
        init = _c(init)
        out_v = init.v + out.v
        # init + t0 + t1 + ... : the partials of the whole chain
        rnd_all = np.abs(init.v[..., None] + v).sum(-1)
        f = None if (t.f is None or init.f is None) else np.add.accumulate(
            np.concatenate([np.asarray(init.f)[..., None] * np.ones_like(np.moveaxis(t.f, axis, -1)[..., :1]),
                            np.moveaxis(t.f, axis, -1)], -1), -1)[..., -1]
        out = _E(out_v, init.b + b + rnd_all, f)
    return out
