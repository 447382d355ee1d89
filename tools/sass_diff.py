"""Check that kernels compile to the same SASS as at another commit.

A change that shares device code between kernels, or adds code next to them, can leave a kernel's instructions as they
were; this script shows whether it did.  It compiles SOURCES for sm_90a, from the working tree and from BASE, with the
library's own nvcc flags, and compares the disassembly of every kernel in KERNELS that BASE has, after removing
addresses, encodings and the kernel's mangled name (a template parameter changes the name, not the code).

BASE defaults to HEAD, which checks uncommitted work against the last commit; HEAD^ checks the last commit.

Usage: python tools/sass_diff.py [--base REV]      exit status 0 = identical, 1 = a kernel differs or is missing
"""
from __future__ import annotations

import argparse
import os
import re
import subprocess
import sys
import tarfile
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from vidu4d_b200.build import NVCC_FLAGS, _nvcc  # noqa: E402

SOURCES = ["composite_tile.cu", "composite_feat.cu", "composite_det.cu", "surfel_bwd.cu", "preprocess.cu", "composite_fwd.cu",
           "postprocess.cu"]
_STATS = r"\((?:bool|<unnamed>::Stats)\)"      # composite_fwd_kernel's fourth template argument, either spelling
_LW = r"(, \(int\)0)?"                          # its fifth, the lift's channel width, absent before the lift
_FWD_ONLY = [(1, 0)] + [(v, nf) for nf in (8, 16, 24, 32) for v in (4, 2, 1)]
# (demangled-name pattern in the base build, pattern of the same kernel in the working tree)
KERNELS = [
    (r"composite_tile_bwd_kernel(<\(bool\)0>)?\(", r"composite_tile_bwd_kernel(<\(bool\)0>)?\("),
    (r"composite_tile_fwd_kernel\(", r"composite_tile_fwd_kernel\("),       # shares the chunk wait with the backward
    (r"det_zero_kernel\(", r"det_zero_kernel\("),
    (r"det_gather_kernel\(", r"det_gather_kernel\("),
    (r"feature_bwd_kernel<\(int\)4>\(", r"feature_bwd_kernel<\(int\)4>\("),
    (r"feature_bwd_kernel<\(int\)2>\(", r"feature_bwd_kernel<\(int\)2>\("),
    (r"feature_bwd_kernel<\(int\)1>\(", r"feature_bwd_kernel<\(int\)1>\("),
    (r"surfel_bwd_kernel\(", r"surfel_bwd_kernel\("),
    (r"preprocess_fwd_kernel\(", r"preprocess_fwd_kernel\("),
    (r"emit_keys_kernel\(", r"emit_keys_kernel\("),
    (r"scan_block_sums_kernel\(", r"scan_block_sums_kernel\("),
    (r"mark_visible_kernel\(", r"mark_visible_kernel\("),
    # the training instantiation of the composite forward (the forward-only ones are <(bool)0, ...>).  A fourth template
    # parameter names what the forward-only walk gathers: (bool)0 / (bool)1 before the silhouette statistics, then the
    # Stats enum's OFF = 0, WEIGHTS = 1 (the contribution statistics), MASKED = 2 (their background share) and LIFT = 3
    # (the lifted maps, new); a fifth, the lift's channel width, is (int)0 in every other instantiation
    (rf"composite_fwd_kernel(<\(bool\)1, \(int\)1, \(int\)0(, {_STATS}0{_LW})?>)?\(",
     rf"composite_fwd_kernel(<\(bool\)1, \(int\)1, \(int\)0(, {_STATS}0{_LW})?>)?\("),
    # the forward-only instantiations without and with the contribution statistics and with their background share:
    # (V, NF) = (1, 0), and V in {4, 2, 1} for NF in {8, 16, 24, 32}
] + [
    (rf"composite_fwd_kernel<\(bool\)0, \(int\){v}, \(int\){nf}(, {_STATS}0{_LW})?>\(",
     rf"composite_fwd_kernel<\(bool\)0, \(int\){v}, \(int\){nf}(, {_STATS}0{_LW})?>\(")
    for v, nf in _FWD_ONLY
] + [
    (rf"composite_fwd_kernel<\(bool\)0, \(int\){v}, \(int\){nf}, {_STATS}{st}{_LW}>\(",
     rf"composite_fwd_kernel<\(bool\)0, \(int\){v}, \(int\){nf}, {_STATS}{st}{_LW}>\(")
    for st in (1, 2) for v, nf in _FWD_ONLY
] + [
    # the lifts, colour-only walks of LW = 8, 16, 24 and 32 channels; the anchors (Stats 4) are new
    (rf"composite_fwd_kernel<\(bool\)0, \(int\)1, \(int\)0, {_STATS}3, \(int\){lw}>\(",
     rf"composite_fwd_kernel<\(bool\)0, \(int\)1, \(int\)0, {_STATS}3, \(int\){lw}>\(")
    for lw in (8, 16, 24, 32)
] + [
    (r"feature_fwd_kernel<\(int\)4>\(", r"feature_fwd_kernel<\(int\)4>\("),
    (r"feature_fwd_kernel<\(int\)2>\(", r"feature_fwd_kernel<\(int\)2>\("),
    (r"feature_fwd_kernel<\(int\)1>\(", r"feature_fwd_kernel<\(int\)1>\("),
    # sr_post_forward's kernels (sr_post_forward_frames' are <(bool)1, ...>)
    (r"post_fwd_kernel(<\(bool\)0, \(bool\)0>)?\(", r"post_fwd_kernel(<\(bool\)0, \(bool\)0>)?\("),
    (r"post_normal_kernel(<\(bool\)0, \(bool\)0>)?\(", r"post_normal_kernel(<\(bool\)0, \(bool\)0>)?\("),
    (r"post_bwd_kernel\(", r"post_bwd_kernel\("),
]


def _sass(tree: str, src: str, out: str) -> dict:
    """{demangled kernel name: normalised instruction list} of one translation unit."""
    obj = os.path.join(out, src.replace(".cu", ".o"))
    subprocess.run([_nvcc()] + NVCC_FLAGS + ["-c", os.path.join(tree, "vidu4d_b200", "csrc", src), "-o", obj], check=True)
    text = subprocess.run(["cuobjdump", "-sass", obj], check=True, capture_output=True, text=True).stdout
    names = subprocess.run(["cu++filt"], input="\n".join(re.findall(r"Function : (\S+)", text)), capture_output=True,
                           text=True).stdout.split("\n")
    kernels, cur, i = {}, None, 0
    for line in text.split("\n"):
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = names[i] if i < len(names) and names[i] else m.group(1)
            i += 1
            kernels[cur] = []
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(.*?)\s*;", line)
        if cur and m:
            ins = re.sub(r"\b_Z\w+", "<sym>", m.group(1))              # branch targets / calls carry the mangled name
            kernels[cur].append(ins)
    return kernels


def _find(kernels: dict, pattern: str):
    hits = [k for k in kernels if re.search(pattern, k)]
    return hits[0] if len(hits) == 1 else None


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--base", default="HEAD", help="commit to compare with (default: HEAD)")
    args = ap.parse_args()
    with tempfile.TemporaryDirectory() as tmp:
        base = os.path.join(tmp, "base")
        os.makedirs(base)
        tarpath = os.path.join(tmp, "base.tar")
        subprocess.run(["git", "-C", ROOT, "archive", "-o", tarpath, args.base, "vidu4d_b200/csrc", "include"], check=True)
        with tarfile.open(tarpath) as t:
            t.extractall(base)
        ok = True
        for src in SOURCES:
            old = _sass(base, src, os.path.join(tmp, "base"))
            os.makedirs(os.path.join(tmp, "new"), exist_ok=True)
            new = _sass(ROOT, src, os.path.join(tmp, "new"))
            for pat_old, pat_new in KERNELS:
                ko = _find(old, pat_old)
                if ko is None:
                    continue                                        # not in this translation unit
                kn = _find(new, pat_new)
                if kn is None:
                    print(f"MISSING  {ko}: no kernel matching {pat_new!r} in the working tree")
                    ok = False
                elif old[ko] != new[kn]:
                    diff = sum(a != b for a, b in zip(old[ko], new[kn])) + abs(len(old[ko]) - len(new[kn]))
                    print(f"DIFFERS  {ko} -> {kn}: {len(old[ko])} vs {len(new[kn])} instructions, {diff} differ")
                    ok = False
                else:
                    print(f"same     {kn}: {len(new[kn])} instructions")
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
