"""TEST INFRASTRUCTURE -- a pairwise covering array over the batched rasterizer's options, and the oracle reference and
rounding-error tolerance of one frame's gradients under any combination of them (tests/test_gpu_batch_bounds.py).

The batched entry points take about ten independent options; holding each to the oracle bound one at a time leaves
their interactions unchecked (a stride, a frame index or a summed-versus-per-frame output chosen from the wrong flag).
Every combination is far too many to run, so CASES is a covering array: every level of every factor, and every pair
of levels of any two factors, appears in at least one case, except the pairs no valid call can hold:

  * the feature options (how the feature planes' gradient is passed, the background's length) without features;
  * an SH degree with colors_precomp (the "sh" factor is None exactly when the colour source is precomputed).

The array is built greedily from a fixed seed (each row the best of many seeded candidates by the number of pairs it
newly covers), so it is the same on every machine; tests/test_batch_options_cpu.py asserts that and the coverage.

Imports no GPU code: the tolerance half needs the CPU oracle only.
"""
import itertools
import random

import numpy as np

FACTORS = {
    "M": (1, 2, 5),
    "means3D": ("shared", "per_frame"),
    "rotations": ("shared", "per_frame"),
    "scales": ("shared", "per_frame"),
    "opacities": ("shared", "per_frame"),              # per frame as (M,P,1)
    "colour": ("sh_shared", "sh_per_frame", "precomp_shared", "precomp_per_frame"),
    "sh": ((3, 16), (1, 16), (0, 1), None),            # (degree, coefficients); None with colors_precomp
    "features": (0, 7, 22, -32),                       # F shared; -32: F = 32 per frame
    "planes": ("tail", "separate", None),              # dL_dout_color's tail or dL_dout_features; None without features
    "background": (3, "3+F", None),                    # None without features (then 3 values)
    "camera": ("scalar", "table", "table_offsets"),
    "sum_shared": (False, True),
    "backward": ("default", "deterministic"),
    "grad_scale": (None, -1.7, 0.0),                   # the same device scalar as grad_scale and features_grad_scale
    "want_transmat": (False, True),
    "outs": (False, True),
}
NAMES = tuple(FACTORS)
SEED = 20261018
CANDIDATES = 400


def valid(case):
    """Whether a partial or complete assignment {factor: level} can be completed to a valid call."""
    c = case.get
    if "colour" in case and "sh" in case and (c("colour").startswith("precomp") != (c("sh") is None)):
        return False
    for k in ("planes", "background"):
        if "features" in case and k in case and ((c("features") == 0) != (c(k) is None)):
            return False
    if "planes" in case and "background" in case and ((c("planes") is None) != (c("background") is None)):
        return False
    return True


def all_pairs():
    """Every pair ((factor, level), (factor, level)) of two factors that a valid call can hold."""
    out = set()
    for a, b in itertools.combinations(NAMES, 2):
        for la in FACTORS[a]:
            for lb in FACTORS[b]:
                if valid({a: la, b: lb}):
                    out.add(((a, la), (b, lb)))
    return out


def pairs_of(case):
    return {((a, case[a]), (b, case[b])) for a, b in itertools.combinations(NAMES, 2)}


def _random_case(rng, want):
    """A valid complete case holding the pair `want`, the rest drawn at random."""
    (a, la), (b, lb) = want
    case = {}
    order = [a, b] + [n for n in NAMES if n not in (a, b)]
    for n in order:
        levels = [la] if n == a else [lb] if n == b else list(FACTORS[n])
        rng.shuffle(levels)
        for lv in levels:
            if valid(dict(case, **{n: lv})):
                case[n] = lv
                break
    return {n: case[n] for n in NAMES}


def covering_array(seed=SEED):
    rng = random.Random(seed)
    todo = all_pairs()
    rows = []
    while todo:
        first = min(todo, key=repr)          # a deterministic uncovered pair seeds every candidate
        best = max((_random_case(rng, first) for _ in range(CANDIDATES)), key=lambda c: len(pairs_of(c) & todo))
        todo -= pairs_of(best)
        rows.append(best)
    return rows


CASES = covering_array()


def case_id(c):
    F = c["features"]
    parts = [f"M{c['M']}"]
    parts += [k[:3] for k in ("means3D", "rotations", "scales", "opacities") if c[k] == "per_frame"]
    parts.append(c["colour"] + ("" if c["sh"] is None else f"_d{c['sh'][0]}k{c['sh'][1]}"))
    if F:
        parts.append(f"F{abs(F)}{'pf' if F < 0 else ''}_{c['planes']}_bg{c['background']}")
    parts += [c["camera"], "sum" if c["sum_shared"] else "nosum", c["backward"][:3], f"gs{c['grad_scale']}"]
    parts += (["tm"] if c["want_transmat"] else []) + (["outs"] if c["outs"] else [])
    return "-".join(parts)


# ------------------------------------------------------------------------------------------------ oracle tolerance
U = 2.0 ** -24
K = 2.0
C3 = slice(15, 18)       # oracle.surfel_oracle.ACC_COLOR .. + 3


def frame_reference(st, og_c, og_g, adds, off=None):
    """One frame's oracle gradients and their tolerances K u B' (see tests/test_gpu_grad_bounds.py).

    og_c is the colour run's so.backward (bounds=True), og_g the feature groups' (tests/test_gpu_feature_bounds.py:
    each group's colour slots are dL/dfeatures, its other slots add to the geometry's accumulator), adds (P,) the
    roundings per unit of the accumulator's absolute sum that the caller's path adds (reductions, chain, ...).
    off = (cx_off, cy_off) of a camera-table row: tests/camera_model.py's offset chain and bound sums on the combined
    accumulator.  Without features this is the off-centre test's composition, with zero offsets the feature test's."""
    from oracle import surfel_oracle as so
    from . import camera_model as cm
    acc, bnd, asm = (np.array(og_c[k], np.float64, copy=True) for k in ("acc", "bound", "asum"))
    for og in og_g:
        for dst, k in ((acc, "acc"), (bnd, "bound"), (asm, "asum")):
            a = np.array(og[k], np.float64, copy=True)
            a[:, C3] = 0.0
            dst += a
    B = bnd +np.asarray(adds, np.float64)[:, None] * asm
    if off is not None and (off[0] != 0.0 or off[1] != 0.0):
        tm = so.chain(st, acc)["dL_dtransMat"]
        B = cm.offset_bound_sums(st, B, acc, tm, off[0], off[1])
        ref = cm.offset_chain(st, acc, tm, off[0], off[1])
    else:
        ref = so.chain(st, acc)
    return ref, {k: K * U * v for k, v in so.chain_bound(st, B).items()}
