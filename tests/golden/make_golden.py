"""Generate the golden fixtures that pin the CPU oracle (and the CUDA path) to the REFERENCE ITSELF.

The reference (yikaiw/Vidu4D, gs/submodules/diff-surfel-rasterization) has no tests or golden vectors for
this path (SURVEY.md section 4), and it has no CPU implementation, so its outputs can only be produced on a
GPU.  This script runs the UNMODIFIED reference extension (oracle/_ref/_C.so, built by oracle/build_ref.sh) on seeded
scenes and stores inputs + every output / intermediate buffer:

    python tests/golden/make_golden.py OUTDIR   # writes OUTDIR/*.npz; copy them to tests/golden/ to replace the fixtures

The committed fixtures come from the reference compiled for sm_100a, whose FMA contraction the kernels follow bit for
bit; the reference compiled for sm_90a differs from them in the last bits of its float buffers.

Fixtures are small (<= ~1.5K surfels, <= 96x64 px).  tests/test_oracle_golden.py (CPU) checks the oracle
against them; tests/test_gpu_parity.py (GPU) checks the CUDA library against them and against the live
reference.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import ref_ext  # noqa: E402
from vidu4d_b200.synthetic import object_scene, projection_matrix, random_rotation, rigid_view  # noqa: E402

CASES = {
    # name: (P, W, H, seed, options)
    "id_deg3_64": dict(P=1000, W=64, H=64, seed=11),
    "rigid_bg_96x64": dict(P=1200, W=96, H=64, seed=12, rigid=True, bg=(0.2, 0.5, 0.7)),
    "ragged_80x48_deg1": dict(P=900, W=80, H=48, seed=13, sh_degree=1, rigid=True),
    "precomp_init_70x50": dict(P=800, W=70, H=50, seed=14, colors_precomp=True, opacity="init"),
    "big_surfels_64": dict(P=300, W=64, H=64, seed=15, scale_mul=6.0, sh_degree=2),
    "near_cull_64": dict(P=600, W=64, H=64, seed=16, center=(0.0, 0.0, 0.45), sh_degree=0),
    "single_32": dict(P=1, W=32, H=32, seed=17),
}


def build_case(P, W, H, seed, rigid=False, bg=(0.0, 0.0, 0.0), sh_degree=3, colors_precomp=False, opacity="trained",
               scale_mul=1.0, center=(0.0, 0.0, 1.0)):
    sc = object_scene(P, seed=seed, opacity=opacity, sh_degree=sh_degree, center=center)
    sc.scales = (sc.scales * scale_mul).astype(np.float32)
    vm = np.eye(4, dtype=np.float32)
    campos = np.zeros(3, np.float32)
    if rigid:
        rng = np.random.default_rng(seed + 100)
        sc, vm, campos = rigid_view(sc, random_rotation(rng), np.array([0.3, -0.2, 0.5]))
    tan = 0.5
    pm = (vm.astype(np.float64) @ projection_matrix(tan, tan).astype(np.float64)).astype(np.float32)
    rng = np.random.default_rng(seed + 7)
    inp = dict(
        means3D=sc.means3D, scales=sc.scales, rotations=sc.rotations, opacities=sc.opacities,
        shs=sc.shs if not colors_precomp else np.zeros((0,), np.float32),
        colors_precomp=rng.uniform(0, 1, size=(P, 3)).astype(np.float32) if colors_precomp else np.zeros((0,), np.float32),
        viewmatrix=vm, projmatrix=pm, campos=campos, bg=np.asarray(bg, np.float32),
        dL_dcolor=rng.normal(size=(3, H, W)).astype(np.float32),
        dL_dallmap=rng.normal(size=(8, H, W)).astype(np.float32),
        meta=np.array([P, W, H, sh_degree, int(colors_precomp)], np.int64),
        tanfov=np.array([tan, tan], np.float32),
    )
    return inp


def run_reference(inp, dev):
    P, W, H, deg, pre = [int(v) for v in inp["meta"]]
    t = {k: torch.from_numpy(np.ascontiguousarray(v)).to(dev) for k, v in inp.items() if k not in ("meta",)}
    shs = None if pre else t["shs"]
    col = t["colors_precomp"] if pre else None
    kw = dict(sh_degree=deg, tanfovx=float(inp["tanfov"][0]), tanfovy=float(inp["tanfov"][1]), bg=t["bg"],
              viewmatrix=t["viewmatrix"], projmatrix=t["projmatrix"], campos=t["campos"])
    fw = ref_ext.forward(t["means3D"], t["opacities"], t["scales"], t["rotations"], shs=shs, colors_precomp=col,
                         W=W, H=H, **kw)
    gb = ref_ext.backward(fw, t["means3D"], t["scales"], t["rotations"], shs=shs, colors_precomp=col,
                          dL_dcolor=t["dL_dcolor"], dL_dallmap=t["dL_dallmap"], **kw)
    R = int(fw["num_rendered"])
    out = dict(num_rendered=np.array([R], np.int64), color=ref_ext.to_np(fw["color"]), allmap=ref_ext.to_np(fw["allmap"]),
               radii=ref_ext.to_np(fw["radii"]))
    for k, v in ref_ext.decode_geom(fw["geomBuffer"], P).items():
        out["geom_" + k] = ref_ext.to_np(v)
    for k, v in ref_ext.decode_binning(fw["binningBuffer"], R).items():
        out["bin_" + k] = ref_ext.to_np(v)
    for k, v in ref_ext.decode_image(fw["imgBuffer"], W, H).items():
        out["img_" + k] = ref_ext.to_np(v)
    for k, v in gb.items():
        out["grad_" + k] = ref_ext.to_np(v)
    return out


def main(outdir):
    dev = torch.device("cuda:0")
    os.makedirs(outdir, exist_ok=True)
    for name, kw in CASES.items():
        inp = build_case(**kw)
        out = run_reference(inp, dev)
        np.savez_compressed(os.path.join(outdir, name + ".npz"), **{"in_" + k: v for k, v in inp.items()},
                            **{"ref_" + k: v for k, v in out.items()})
        print(name, "R =", int(out["num_rendered"][0]), "visible =", int((out["radii"] > 0).sum()))


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit("usage: python tests/golden/make_golden.py OUTDIR")
    main(sys.argv[1])
