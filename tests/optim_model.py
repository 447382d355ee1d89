"""Models of the device-state optimizer step (csrc/optim.cu, include/surfel_optim.h), shared by the CPU and GPU tests."""
import math

import numpy as np


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
    """sr_adam_flat's host formula: (float)(1 - pow(beta1, t)), (float)sqrt(1 - pow(beta2, t)), beta* fp32 widened."""
    b1, b2 = float(np.float32(beta1)), float(np.float32(beta2))
    return np.float32(1.0 - math.pow(b1, step)), np.float32(math.sqrt(1.0 - math.pow(b2, step)))
