"""Build vidu4d_b200/lib/libsurfel_raster.so (the C-ABI CUDA library) in-tree with nvcc for sm_90a (H100).

nvcc cross-compiles without a GPU.  The .so is a build product (git-ignored); build() recompiles whatever is stale.
Usage: python -m vidu4d_b200.build [--force] [--verbose]
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIBDIR, "libsurfel_raster.so")
SOURCES = ["api.cu", "preprocess.cu", "sort.cu", "composite_fwd.cu", "composite_tile.cu", "composite_feat.cu", "surfel_bwd.cu",
           "postprocess.cu", "loss.cu", "warp.cu", "match.cu", "cycle.cu", "feature_rows.cu", "optim.cu", "knn.cu", "outlier.cu", "ssim.cu",
           "skin_mlp.cu", "mask_loss.cu"]
HEADERS = [os.path.join(CSRC, "common.cuh"), os.path.join(CSRC, "composite_common.cuh"), os.path.join(CSRC, "post_common.cuh"),
           os.path.join(CSRC, "warp_common.cuh"),
           os.path.join(HERE, "..", "include", "surfel_raster.h"), os.path.join(HERE, "..", "include", "surfel_ssim.h"),
           os.path.join(HERE, "..", "include", "surfel_optim.h"), os.path.join(HERE, "..", "include", "surfel_skin_mlp.h"),
           os.path.join(HERE, "..", "include", "surfel_mask_loss.h")]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden",
    # no --use_fast_math: expf / div / sqrt must be the same IEEE / libdevice variants the reference build uses
]


def _nvcc() -> str:
    p = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(p):
        raise RuntimeError("nvcc not found; cannot build libsurfel_raster.so")
    return p


def _stale(target: str, deps) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(LIBDIR, exist_ok=True)
    objdir = os.path.join(LIBDIR, "obj")
    os.makedirs(objdir, exist_ok=True)
    nvcc = _nvcc()
    env = dict(os.environ)
    # nvcc's host compiler is the system g++ even where CC/CXX point at another toolchain
    ccbin = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else None
    # objects compiled with other flags (another target architecture) are stale whatever their mtime
    stamp = os.path.join(objdir, "flags")
    flags = " ".join(NVCC_FLAGS)
    if not os.path.exists(stamp) or open(stamp).read() != flags:
        force = True

    def compile_one(src):
        s = os.path.join(CSRC, src)
        o = os.path.join(objdir, src.replace(".cu", ".o"))
        if force or _stale(o, [s] + HEADERS):
            cmd = [nvcc] + NVCC_FLAGS + (["-ccbin", ccbin] if ccbin else []) + (["-Xptxas", "-v"] if verbose else []) + ["-c", s, "-o", o]
            r = subprocess.run(cmd, capture_output=True, text=True, env=env)
            if r.returncode != 0:
                raise RuntimeError(f"nvcc failed on {src}:\n{r.stdout}\n{r.stderr}")
            if verbose:
                sys.stderr.write(r.stderr)
        return o

    with ThreadPoolExecutor(max_workers=len(SOURCES)) as ex:
        objs = list(ex.map(compile_one, SOURCES))
    if force or _stale(LIB, objs):
        cmd = [nvcc, "-shared", "-o", LIB] + objs + (["-ccbin", ccbin] if ccbin else []) + ["-Xcompiler", "-fPIC", "-lcudart"]
        r = subprocess.run(cmd, capture_output=True, text=True, env=env)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    with open(stamp, "w") as f:
        f.write(flags)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
