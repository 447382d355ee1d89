"""Generate tests/golden/frows_*.npz from the REFERENCE's own code, run on the CPU in this container.

Nothing is copied: like make_cycle_golden.py (whose _grab it uses), it starts from make_warp_golden.py's loader, inputs and
forward warp, and exec()s the source text of DeformableGaussian.compute_gauss_density, compute_flow and flip_pair
(lab4d/nnutils/deformable_gaussian.py), SkinningWarp.get_gauss_density (lab4d/nnutils/warping.py), get_xyz_bone_distance
(lab4d/utils/transforms.py) and Kmatinv with mat2K / K2inv (lab4d/utils/geom_utils.py); quaternion_apply comes with the
loaded quat_transform.py.  They are chained as query_field (deformable_gaussian.py:1106-1182) chains them, starting from
the reference forward warp's xyz_cam / rot_cam so that the gradients include the path through the warp.

The reference runs on CUDA, where quaternion_mul flattens both operands to rows (quat_transform.py:106-112): the normal's
`quaternion_apply(rotation_t (M,P,4), axis.repeat -> (M,1,P,3))` pairs row (m,p) with axis p.  The loader's CPU
dispatcher broadcasts instead ((M,M,P,.)), so quaternion_apply is given a row-by-row product while the normal is built.

The chain runs twice: in float32 (outputs and autograd gradients, the yardstick of the kernel) and on the same inputs
recast to float64 with float64 as torch's default dtype (mat2K / K2inv allocate with the default), to pin
tests/feature_rows_model.py.  The scalar loss is sum(rows * w_rows) + s * w_s + sum(gauss_density * w_dens) with seeded
weights that are stored too.

    python tests/golden/make_feature_rows_golden.py        # needs /root/reference
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_cycle_golden import _grab  # noqa: E402
from make_warp_golden import ROOT, _load_reference, make_inputs, run_reference  # noqa: E402

CF = 16
INIT_BETA = 0.01                                             # SkinningWarp(init_beta=0.01), warping.py:348,375-376


def load():
    ns = _load_reference()
    _grab(ns, "lab4d/utils/transforms.py", "get_xyz_bone_distance")
    for name in ("mat2K", "K2inv", "Kmatinv"):
        _grab(ns, "lab4d/utils/geom_utils.py", name)
    warp_ns, model_ns = {}, {}
    _grab(warp_ns, "lab4d/nnutils/warping.py", "get_gauss_density", in_class="SkinningWarp")
    for name in ("compute_gauss_density", "compute_flow", "flip_pair"):
        _grab(model_ns, "lab4d/nnutils/deformable_gaussian.py", name, in_class="DeformableGaussian")
    for f in list(warp_ns.values()) + list(model_ns.values()):
        if callable(f):
            f.__globals__.update(ns)          # exec'd into their own dicts: give them the reference helpers
    # stand-ins for the two classes, carrying only the exec'd methods the chain calls
    SkinningWarp = type("SkinningWarp", (), {"get_gauss_density": warp_ns["get_gauss_density"]})
    DeformableGaussian = type("DeformableGaussian", (), {"flip_pair": staticmethod(model_ns["flip_pair"]),
                                                         "compute_flow": model_ns["compute_flow"],
                                                         "compute_gauss_density": model_ns["compute_gauss_density"]})
    for g in (warp_ns, model_ns):
        g.update(SkinningWarp=SkinningWarp, DeformableGaussian=DeformableGaussian)
    ns.update(SkinningWarp=SkinningWarp, DeformableGaussian=DeformableGaussian)
    return ns


def _rowwise_qmul(dispatch):
    """quaternion_mul as the CUDA helper calls it: both operands flattened to rows (quat_transform.py:106-112)."""
    def qmul(a, b):
        return dispatch(a.reshape(-1, a.shape[-1]), b.reshape(-1, b.shape[-1])).view(tuple(a.shape[:-1]) + (4,))
    return qmul


def run_rows(ns, inp):
    """forward warp (make_warp_golden.run_reference), then query_field's feature rows; returns the leaves, rows (M,P,Cf+6),
    s, gauss_density (P,1), Kmat and the warp outputs (with their .grad retained)."""
    t, xc, rc, _, _ = run_reference(ns, {k: v for k, v in inp.items() if k in ("xyz", "rot", "rest_q", "rest_t", "log_gauss",
                                                                                "art_q", "art_t", "cam_q", "cam_t", "delta")})
    for k in ("regist", "logibeta"):
        t[k] = inp[k].clone().requires_grad_(True)
    xc.retain_grad(); rc.retain_grad()
    M, P = xc.shape[:2]
    q2dq = ns["quaternion_translation_to_dual_quaternion"]
    rest = q2dq(t["rest_q"], t["rest_t"])
    rest_m = (rest[0][None].expand(M, -1, -1), rest[1][None].expand(M, -1, -1))
    warp = ns["SkinningWarp"]()
    warp.logibeta = t["logibeta"]
    model = ns["DeformableGaussian"]()
    model.warp = warp
    samples_dict = {"rest_articulation": rest_m}
    # compute_gauss_density(self._xyz, samples_dict)  (:1106-1108)
    gauss_density = model.compute_gauss_density(t["xyz"], samples_dict)["gauss_density"]          # (P,1)
    # the normal (:1127-1148)
    scaling = inp["scaling"]
    values, shortest_axis = torch.min(scaling, dim=1)
    axis = torch.zeros_like(t["xyz"])
    axis[torch.arange(axis.size(0)), shortest_axis] = 1
    axis = axis[None, ...].repeat(M, 1, 1, 1)
    qa = ns["quaternion_apply"]
    dispatch = qa.__globals__["quaternion_mul"]
    qa.__globals__["quaternion_mul"] = _rowwise_qmul(dispatch)
    try:
        normal = qa(rc, axis)
        q = t["cam_q"][:, None].repeat(1, P, 1)
        normal = qa(q, normal)
    finally:
        qa.__globals__["quaternion_mul"] = dispatch
    # the flow (:1152-1161) and its scale (:1178-1179)
    field2cam = (t["cam_q"], t["cam_t"])
    frame_id = torch.arange(M)
    flow = model.compute_flow(xc[:, :, None, :], frame_id, frame_id * 0, field2cam, inp["Kinv"], {})       # (M,P,1,2)
    flow_scale = torch.max(flow.max(), torch.abs(flow.min())) + 1e-6
    flow_scaled = flow / flow_scale
    rows = torch.stack([torch.cat([t["regist"], flow_scaled[i, :, 0, :], normal[i], gauss_density], dim=-1) for i in range(M)])
    Kmat = ns["Kmatinv"](inp["Kinv"])
    return t, rows, flow_scale, gauss_density, flow[:, :, 0], Kmat, xc, rc


def make_case(seed, P, B, M, dup=False, eq_scales=False):
    """make_warp_golden.make_inputs, with three quarters of the surfels within ~0.01 of a rest bone's centre (elsewhere the
    density underflows to 0: 0.01 is the Gaussian bones' radius), a (P,16) registration feature, two tangent scales,
    per-frame intrinsics and logibeta.  dup: every surfel twice (clone densification's bit-identical copies), so the
    flow's max and min are tied.  eq_scales: half of the surfels with equal tangent scales (the arg-min tie)."""
    P0 = P // 2 if dup else P
    inp = make_inputs(seed, P0, B, M, True)
    rng = np.random.default_rng(seed + 30)
    near = rng.random(P0) < 0.75
    b = rng.integers(0, B, P0)
    xyz = inp["xyz"].numpy().astype(np.float64)
    xyz[near] = inp["rest_t"].numpy()[b[near]] + 0.012 * rng.normal(size=(int(near.sum()), 3))
    inp["xyz"] = torch.tensor(xyz, dtype=torch.float32)
    inp["regist"] = torch.tensor(rng.normal(size=(P0, CF)), dtype=torch.float32)
    sc = np.exp(-4.0 + 0.5 * rng.normal(size=(P0, 2)))
    if eq_scales:
        sc[::2, 1] = sc[::2, 0]
    inp["scaling"] = torch.tensor(sc, dtype=torch.float32)
    if dup:
        idx = torch.from_numpy(rng.permutation(np.concatenate([np.arange(P0), np.arange(P0)])))
        for k in ("xyz", "rot", "delta", "regist", "scaling"):
            inp[k] = inp[k][idx].contiguous()
    K = np.zeros((M, 3, 3))
    K[:, 0, 0] = 280.0 + 40.0 * rng.random(M); K[:, 1, 1] = 280.0 + 40.0 * rng.random(M)
    K[:, 0, 2] = 128.0 + 4.0 * rng.normal(size=M); K[:, 1, 2] = 128.0 + 4.0 * rng.normal(size=M); K[:, 2, 2] = 1.0
    inp["Kinv"] = torch.tensor(np.linalg.inv(K), dtype=torch.float32)
    inp["logibeta"] = torch.tensor([-np.log(INIT_BETA) + 0.1 * rng.normal()], dtype=torch.float32)
    return inp


CASES = {"frows_b25_m2": dict(seed=21, P=400, B=25, M=2),
         "frows_b7_m4_dup": dict(seed=22, P=300, B=7, M=4, dup=True),
         "frows_b7_m2_eqscale": dict(seed=23, P=200, B=7, M=2, eq_scales=True),
         "frows_b7_m1": dict(seed=24, P=200, B=7, M=1)}

if __name__ == "__main__":
    ns = load()
    for name, kw in CASES.items():
        inp = make_case(**kw)
        out = {"in_" + k: v.numpy() for k, v in inp.items() if v is not None}
        M, P = kw["M"], kw["P"]
        rng = np.random.default_rng(kw["seed"] + 50)
        w = {"w_rows": rng.normal(size=(M, P, CF + 6)), "w_s": rng.normal(size=(1,)), "w_dens": rng.normal(size=(P, 1))}
        out.update(w)
        for tag, dtype in (("ref", torch.float32), ("ref64", torch.float64)):
            torch.set_default_dtype(dtype)
            try:
                t, rows, s, dens, flow, Kmat, xc, rc = run_rows(ns, {k: (v.to(dtype) if v is not None else None) for k, v in inp.items()})
                wt = {k: torch.tensor(v, dtype=dtype) for k, v in w.items()}
                ((rows * wt["w_rows"]).sum() + s * wt["w_s"][0] + (dens * wt["w_dens"]).sum()).backward()
            finally:
                torch.set_default_dtype(torch.float32)
            out.update({f"{tag}_rows": rows.detach().numpy(), f"{tag}_flow_scale": np.array([float(s)]),
                        f"{tag}_gauss_density": dens.detach().numpy(), f"{tag}_flow": flow.detach().numpy(),
                        f"{tag}_Kmat": Kmat.numpy(), f"{tag}_xyz_cam": xc.detach().numpy(), f"{tag}_rot_cam": rc.detach().numpy(),
                        f"{tag}_grad_xyz_cam": xc.grad.numpy(), f"{tag}_grad_rot_cam": rc.grad.numpy()})
            for k, v in t.items():
                if v is not None and v.grad is not None:
                    out[f"{tag}_grad_{k}"] = v.grad.numpy()
            fl = flow.detach()
            ties = (int((fl == fl.max()).sum()), int((fl == fl.min()).sum()))
            print(name, tag, "s", float(s), "ties(max,min)", ties, "density>0", int((dens > 0).sum()), "of", P)
        np.savez_compressed(os.path.join(ROOT, "tests", "golden", name + ".npz"), **out)
