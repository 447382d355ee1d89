"""Record what the unmodified reference extension computes on the two large parity workloads, so that the comparison with
it runs where the reference is not installed.

The workloads are too large to store whole (300 K surfels at 512x512: ~90 MB of gradients per view), and their inputs are
regenerated from seeds, so a record keeps, per case:
  * num_rendered;
  * SHA-256 digests of every buffer the tests require bit-exact: radii, sorted (tile|depth) keys, sorted surfel ids, tile
    ranges, contributor counts;
  * for every float tensor (colour, each allmap plane, the eight gradients): max |value| and the values at a fixed set of
    flat indices -- the 64 largest magnitudes plus 192 drawn with a fixed seed.

Run on a GPU with oracle/_ref/_C.so built (oracle/build_ref.sh):
    python tests/golden/make_reference_records.py OUTDIR      # writes OUTDIR/ref_*.npz; copy them to tests/golden/
It also prints how far this build of the rasterizer is from the reference on each tensor.
"""
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GRADS = ("dL_dmeans2D", "dL_dcolors", "dL_dopacity", "dL_dmeans3D", "dL_dtransMat", "dL_dsh", "dL_dscales", "dL_drotations")
# bit-exact buffers and the dtype each is digested in (the reference's own)
EXACT = {"radii": np.int32, "keys": np.int64, "point_list": np.int32, "ranges": np.int32, "n_contrib0": np.int64,
         "n_contrib1": np.int64}
NTOP, NRAND = 64, 192
# name: (test module input builder, arguments)
CASES = {
    "ref_headline_identity": ("headline", None),
    "ref_headline_orbit0": ("headline", 0),
    "ref_headline_orbit17": ("headline", 17),
    "ref_c2_100k": ("c2", None),
}


def case_inputs(name):
    kind, arg = CASES[name]
    if kind == "headline":
        from tests.test_gpu_headline import bench_inputs
        return bench_inputs(arg)
    from tests.golden.make_golden import build_case
    return build_case(100_000, 512, 512, 31, rigid=True)          # BASELINE config C2


def digest(a) -> np.ndarray:
    a = np.ascontiguousarray(a)
    return np.frombuffer(hashlib.sha256(str(a.dtype).encode() + str(a.shape).encode() + a.tobytes()).digest(), np.uint8)


def n_contrib_planes(n_contrib, ranges, W, H):
    """Plane 0 everywhere; plane 1 only in tiles with a non-empty instance list (see test_gpu_parity._assert_n_contrib)."""
    nc = np.asarray(n_contrib).astype(np.int64) & 0xFFFFFFFF
    ys, xs = np.mgrid[0:H, 0:W]
    t = (ys // 16) * ((W + 15) // 16) + xs // 16
    rg = np.asarray(ranges).astype(np.int64)
    nonempty = (rg[:, 1] - rg[:, 0])[t] > 0
    return nc[0], nc[1][nonempty]


def float_tensors(color, allmap, grads):
    out = {"color": np.asarray(color, np.float32)}
    for ch in range(8):
        out[f"allmap{ch}"] = np.asarray(allmap[ch], np.float32)
    for k in GRADS:
        out[k] = np.asarray(grads[k], np.float32)
    return out


def sample_index(ref: np.ndarray) -> np.ndarray:
    flat = ref.reshape(-1)
    rnd = np.random.default_rng(0).choice(flat.size, size=min(NRAND, flat.size), replace=False)
    top = np.argsort(-np.abs(flat), kind="stable")[:NTOP]
    return np.union1d(rnd, top).astype(np.int64)


def exact_digests(radii, keys, point_list, ranges, n_contrib, W, H):
    n0, n1 = n_contrib_planes(n_contrib, ranges, W, H)
    arrays = {"radii": radii, "keys": keys, "point_list": point_list, "ranges": ranges, "n_contrib0": n0, "n_contrib1": n1}
    return {k: digest(np.asarray(arrays[k]).astype(dt)) for k, dt in EXACT.items()}


def make_record(ref, W, H):
    rec = {"num_rendered": np.asarray(ref["num_rendered"], np.int64)}
    for k, d in exact_digests(ref["radii"], ref["bin_keys"], ref["bin_point_list"], ref["img_ranges"], ref["img_n_contrib"],
                              W, H).items():
        rec["sha_" + k] = d
    for k, v in float_tensors(ref["color"], ref["allmap"], {g: ref["grad_" + g] for g in GRADS}).items():
        idx = sample_index(v)
        rec["max_" + k] = np.array([np.abs(v).max() if v.size else 0.0], np.float64)
        rec["idx_" + k] = idx.astype(np.int32)
        rec["val_" + k] = v.reshape(-1)[idx]
    return rec


def main(outdir):
    import torch
    from tests.golden.make_golden import run_reference
    from tests.test_gpu_parity import _np, _run_ours
    dev = torch.device("cuda:0")
    os.makedirs(outdir, exist_ok=True)
    for name in CASES:
        inp = case_inputs(name)
        P, W, H = [int(v) for v in inp["meta"][:3]]
        ref = run_reference(inp, dev)
        rec = make_record(ref, W, H)
        np.savez_compressed(os.path.join(outdir, name + ".npz"), **rec)
        r = _run_ours(inp, dev)
        print(name, "R =", int(rec["num_rendered"][0]), "ours R =", int(r["num_rendered"]))
        mine = float_tensors(_np(r["color"]), _np(r["allmap"]), {g: _np(r["grads"][g]).reshape(ref["grad_" + g].shape) for g in GRADS})
        for k, v in float_tensors(ref["color"], ref["allmap"], {g: ref["grad_" + g] for g in GRADS}).items():
            d = np.abs(mine[k].astype(np.float64) - v)
            print(f"  {k:14s} max|ref| {np.abs(v).max():.4e}  max diff {d.max():.3e}  rel {d.max() / (np.abs(v).max() + 1e-30):.3e}  "
                  f"differing {int((d > 0).sum())} of {v.size}  identical {bool(np.array_equal(mine[k], v))}")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden"))
