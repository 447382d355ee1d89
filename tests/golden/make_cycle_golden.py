"""Generate tests/golden/cycle_*.npz from the REFERENCE's own code, run on the CPU in this container.

Nothing is copied: like make_warp_golden.py (whose _load_reference / make_inputs / run_reference this script imports), it
loads lab4d/utils/quat_transform.py from /root/reference by path and exec()s the source text of
DeformableGaussian.cam_to_field (lab4d/nnutils/deformable_gaussian.py), apply_se3mat (lab4d/utils/geom_utils.py) and
dvr_model.apply_loss_weights (lab4d/engine/model.py) next to the helpers make_warp_golden.py already loads
(get_bone_coords, dual_quaternion_skinning, cross_entropy_skin_loss, apply_qt_to_gaussian).  It chains them as
DeformableGaussian.cycle_loss (deformable_gaussian.py:1517-1574) and SkinningWarp.forward(backward=True)
(lab4d/nnutils/warping.py:378-444) do, starting from the reference forward warp's xyz_cam, so that the gradients include
the path through the forward warp; the three terms are reduced as model.py:850-853 and apply_loss_weights do.

The chain runs twice: in float32 (outputs and autograd gradients, the yardstick of the kernel) and on the same inputs
recast to float64 (values, counts and gradients that pin tests/cycle_model.py's cycle_loss).

    python tests/golden/make_cycle_golden.py        # needs /root/reference
"""
import ast
import os
import sys
import textwrap

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_warp_golden import REF, ROOT, _load_reference, make_inputs, run_reference  # noqa: E402

WEIGHTS = {"reg_deform_cyc_wt": 0.01, "reg_delta_skin_wt": 5e-3, "reg_skin_entropy_wt": 5e-4}   # lab4d/config.py:91-95
TERMS = ("reg_deform_cyc", "reg_delta_skin", "reg_skin_entropy")


def _grab(ns, path, name, in_class=None):
    src = open(os.path.join(REF, path)).read()
    tree = ast.parse(src)
    body = tree.body
    if in_class:
        body = next(n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == in_class).body
    node = next(n for n in body if isinstance(n, ast.FunctionDef) and n.name == name)
    node.decorator_list = []
    exec(textwrap.dedent(ast.get_source_segment(src, node)), ns)


def load():
    ns = _load_reference()
    _grab(ns, "lab4d/utils/geom_utils.py", "apply_se3mat")
    _grab(ns, "lab4d/nnutils/deformable_gaussian.py", "cam_to_field", in_class="DeformableGaussian")
    _grab(ns, "lab4d/engine/model.py", "apply_loss_weights", in_class="dvr_model")
    return ns


def run_cycle(ns, inp):
    """forward warp (make_warp_golden.run_reference), then cycle_loss with the backward warp; returns the leaves, the
    per-element values (M,P) and the weighted loss."""
    t, xc, _, _, _ = run_reference(ns, {k: v for k, v in inp.items() if k != "cdelta"})
    cdelta = inp.get("cdelta")
    if cdelta is not None:
        t["cdelta"] = cdelta.clone().requires_grad_(True)
    M, B = t["art_q"].shape[:2]
    P = t["xyz"].shape[0]
    q2dq = ns["quaternion_translation_to_dual_quaternion"]
    rest = q2dq(t["rest_q"], t["rest_t"])
    art = q2dq(t["art_q"], t["art_t"])
    rest_m = (rest[0][None].expand(M, -1, -1), rest[1][None].expand(M, -1, -1))
    xyz_cam = xc.reshape(M, P, 1, 3)
    xyz_t = ns["cam_to_field"](xyz_cam, field2cam=(t["cam_q"], t["cam_t"]))                 # (M,P,1,3)
    # SkinningWarp.forward(backward=True): se3 = rest o t^-1, skinning on t_articulation (warping.py:407-411)
    se3 = ns["dual_quaternion_mul"](rest_m, ns["dual_quaternion_inverse"](art))
    articulation = (art[0][:, None, None].expand(xyz_t.shape[:3] + (-1, -1)),
                    art[1][:, None, None].expand(xyz_t.shape[:3] + (-1, -1)))
    xyz_bone = ns["get_bone_coords"](xyz_t, articulation) / t["log_gauss"].exp().view(1, 1, 1, B, 3)   # skinning.py:126-142
    dist2 = xyz_bone.pow(2).sum(-1)
    if cdelta is not None:
        skin = -(dist2 + t["cdelta"][:, :, None, :])
        delta_skin = t["cdelta"][:, :, None, :].pow(2).mean(-1, keepdims=True)
    else:
        skin = -dist2
        delta_skin = torch.zeros_like(xyz_cam[..., :1])                      # cycle_loss's initial value (:1534-1536)
    q, tr = ns["dual_quaternion_skinning"](se3, xyz_t, skin.softmax(-1), return_qt=True)
    entropy = ns["cross_entropy_skin_loss"](skin)[..., None]
    xyz_cycled, _ = ns["apply_qt_to_gaussian"](xyz_t, None, q, tr, M)
    xyz_reshape = t["xyz"].reshape(1, P, 1, 3).expand(M, -1, -1, -1)
    cyc_dist = (xyz_cycled - xyz_reshape).norm(2, -1, keepdim=True)
    vals = {"reg_deform_cyc": cyc_dist, "reg_delta_skin": delta_skin, "reg_skin_entropy": entropy}
    loss_dict = dict(vals)
    ns["apply_loss_weights"](loss_dict, dict(WEIGHTS))
    loss = sum(loss_dict[k] for k in TERMS)
    return t, {k: v.reshape(M, P) for k, v in vals.items()}, loss


def make_case(seed, P, B, M, with_delta):
    """make_inputs with wider Gaussian bones (scale ~0.2 instead of 0.03): every surfel blends several bones, so every
    cycle distance lies far above fp32 rounding (a knife-edge-free fixture: its counts and gradient directions are exact
    yardsticks) and every skinning entropy far above fp32's log(1 + eps) = 0 threshold.  cdelta (M,P,B) is the backward
    warp's frame-conditioned delta; the forward warp keeps make_inputs' (P,B) delta."""
    inp = make_inputs(seed, P, B, M, with_delta)
    rng = np.random.default_rng(seed + 90)
    inp["log_gauss"] = torch.tensor(np.log(0.2) + 0.3 * rng.normal(size=(B, 3)), dtype=torch.float32)
    if with_delta:
        rng = np.random.default_rng(seed + 70)
        inp["cdelta"] = torch.tensor(np.maximum(rng.normal(size=(M, P, B)), 0.0) * 0.1, dtype=torch.float32)
    return inp


CASES = {"cycle_b25_m3": dict(seed=11, P=400, B=25, M=3, with_delta=True),
         "cycle_b7_m2_nodelta": dict(seed=12, P=300, B=7, M=2, with_delta=False)}

if __name__ == "__main__":
    ns = load()
    for name, kw in CASES.items():
        inp = make_case(**kw)
        out = {"in_" + k: v.numpy() for k, v in inp.items() if v is not None}
        for tag, dtype in (("ref", torch.float32), ("ref64", torch.float64)):
            t, vals, loss = run_cycle(ns, {k: (v.to(dtype) if v is not None else None) for k, v in inp.items()})
            loss.backward()
            out[tag + "_loss"] = np.array([float(loss.detach())])
            for k, v in vals.items():
                out[f"{tag}_{k}"] = v.detach().numpy()
            out[tag + "_counts"] = np.stack([(vals[k] > 0).sum(-1).numpy() for k in TERMS], -1).astype(np.int32)
            for k, v in t.items():
                if v is not None and v.grad is not None:
                    out[f"{tag}_grad_{k}"] = v.grad.numpy()
        np.savez_compressed(os.path.join(ROOT, "tests", "golden", name + ".npz"), **out)
        print(name, float(out["ref_loss"][0]), float(out["ref64_loss"][0]), out["ref_counts"].tolist(), out["ref64_counts"].tolist())
