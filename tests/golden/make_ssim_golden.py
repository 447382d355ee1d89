"""Generate tests/golden/ssim_*.npz from the REFERENCE's own SSIM code, run on the CPU.

At run time this reads gs/utils/loss_utils.py from the reference checkout, extracts the source text of gaussian,
create_window, ssim and _ssim with `ast`, and exec()s it on seeded images in float32 (the reference's own precision) and
in float64, with torch autograd giving dL/dimg1 for a seeded upstream.  Only the data is stored; no reference source
enters the tree.  The fixtures pin tests/ssim_model.py (tests/test_ssim_cpu.py) and the CUDA op (tests/test_gpu_ssim.py).

    python tests/golden/make_ssim_golden.py [reference checkout]     # writes tests/golden/ssim_*.npz
"""
import ast
import math
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
REF = sys.argv[1] if len(sys.argv) > 1 else "/root/reference"


def reference_ssim():
    path = os.path.join(REF, "gs/utils/loss_utils.py")
    src = open(path).read()
    names = {"gaussian", "create_window", "ssim", "_ssim"}
    code = "\n\n".join(ast.get_source_segment(src, n) for n in ast.parse(src).body
                       if isinstance(n, ast.FunctionDef) and n.name in names)
    ns = {"torch": torch, "F": F, "Variable": torch.autograd.Variable, "exp": math.exp}
    exec(compile(code, path, "exec"), ns)
    return ns["ssim"]


def make_case(seed, shape, kind):
    rng = np.random.default_rng(seed)
    x = rng.uniform(0.0, 1.0, size=shape)
    if kind == "near_constant":                 # sigma^2 close to its own rounding error
        x = 0.5 + 1e-4 * rng.normal(size=shape)
        y = 0.5 + 1e-4 * rng.normal(size=shape)
    elif kind == "identical":
        y = x.copy()
    elif kind == "hdr":                         # rendered colours can leave [0, 1]
        x = rng.uniform(-0.5, 1.8, size=shape)
        y = rng.uniform(-0.3, 1.5, size=shape)
    else:                                       # a target that resembles the image: blur-free noise on top of it
        y = np.clip(x + 0.15 * rng.normal(size=shape), 0.0, 1.0)
    x, y = x.astype(np.float32), y.astype(np.float32)
    batched = len(shape) == 4
    g = rng.normal(size=shape[0] if batched else ()).astype(np.float32)     # the seeded upstream
    ssim = reference_ssim()
    res = {"in_img1": x, "in_img2": y, "in_gup": np.asarray(g, np.float32)}
    for tag, dt in (("32", torch.float32), ("64", torch.float64)):
        a = torch.from_numpy(x).to(dt).requires_grad_(True)
        b = torch.from_numpy(y).to(dt)
        mean = ssim(a, b)
        res["ref" + tag + "_mean"] = np.asarray(mean.detach().numpy(), np.float64)
        if batched:                             # the reference's size_average=False only works on (N,C,H,W)
            per = ssim(a, b, size_average=False)
            res["ref" + tag + "_per_image"] = per.detach().numpy().astype(np.float64)
            (per * torch.from_numpy(g).to(dt)).sum().backward()
        else:
            (mean * float(g)).backward()
        res["ref" + tag + "_grad"] = a.grad.numpy().astype(np.float64)
    return res


CASES = {"ssim_3x37x29": dict(seed=1, shape=(3, 37, 29), kind="random"),
         "ssim_batch_4x3x40x33": dict(seed=2, shape=(4, 3, 40, 33), kind="random"),
         "ssim_small_3x7x5": dict(seed=3, shape=(3, 7, 5), kind="random"),
         "ssim_1x1x1": dict(seed=4, shape=(1, 1, 1), kind="random"),
         "ssim_c1_2x1x24x19": dict(seed=5, shape=(2, 1, 24, 19), kind="random"),
         "ssim_near_constant_2x3x16x20": dict(seed=6, shape=(2, 3, 16, 20), kind="near_constant"),
         "ssim_identical_3x21x26": dict(seed=7, shape=(3, 21, 26), kind="identical"),
         "ssim_hdr_2x3x18x23": dict(seed=8, shape=(2, 3, 18, 23), kind="hdr")}

if __name__ == "__main__":
    for name, kw in CASES.items():
        r = make_case(**kw)
        np.savez_compressed(os.path.join(ROOT, "tests", "golden", name + ".npz"), **r)
        print(name, float(r["ref64_mean"]), float(np.abs(r["ref32_mean"] - r["ref64_mean"])))
