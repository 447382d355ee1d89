"""Generate tests/golden/featloss_*.npz from the REFERENCE's own loss code, run on the CPU with torch autograd.

This script does not copy the reference: at run time it reads lab4d/engine/model.py from the reference checkout, takes
the source TEXT of (i) the two statements of compute_recon_loss that build loss_dict["feature"] (:665-667) and
loss_dict["reg_gauss_mask"] (:743-745), (ii) mask_losses (:895-977) and (iii) apply_loss_weights (:980-1012), and
exec()s them on seeded float32 CPU tensors with the reference's configuration defaults (field_type "fg", no_loss_mask,
maskloss_no_vis2d and vis2d_dilate off).  The terms, the counts of positive elements and the gradients with respect to
the feature planes are stored with the inputs; they pin tests/feature_loss_model.py (tests/test_feature_loss_cpu.py).

The flow loss of compute_recon_loss (:697-704) is not included: for Gaussian fields `rendered` is the field's feat_dict
(:517-518), which has no "depth" key (lab4d/nnutils/deformable_gaussian.py:1252-1267), so :699 raises inside the try
and :701 never runs.

    python tests/golden/make_feature_loss_golden.py [REFERENCE_DIR]      # writes tests/golden/featloss_*.npz
"""
import ast
import os
import sys
import textwrap
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _reference_code(ref):
    src = open(os.path.join(ref, "lab4d/engine/model.py")).read()
    tree = ast.parse(src)
    funcs, stmts = {}, {}
    for node in ast.walk(tree):
        if isinstance(node, ast.FunctionDef) and node.name in ("mask_losses", "apply_loss_weights"):
            funcs[node.name] = textwrap.dedent(ast.get_source_segment(src, node, padded=True))
        if isinstance(node, ast.FunctionDef) and node.name == "compute_recon_loss":
            for st in ast.walk(node):
                if (isinstance(st, ast.Assign) and isinstance(st.targets[0], ast.Subscript)
                        and isinstance(st.targets[0].slice, ast.Constant)
                        and st.targets[0].slice.value in ("feature", "reg_gauss_mask")):
                    stmts[st.targets[0].slice.value] = textwrap.dedent(ast.get_source_segment(src, st, padded=True))
    assert set(funcs) == {"mask_losses", "apply_loss_weights"} and set(stmts) == {"feature", "reg_gauss_mask"}
    ns = {"torch": torch}
    for code in funcs.values():
        exec(code, ns)
    return ns["mask_losses"], ns["apply_loss_weights"], stmts


def make_case(ref, seed, M, W, H, F, Cf, gm, is_detected, empty_frame=None, weights=(1e-2, 6e-3)):
    mask_losses, apply_loss_weights, stmts = _reference_code(ref)
    rng = np.random.default_rng(seed)
    feat = rng.normal(size=(M, F, H, W)).astype(np.float32)
    target = rng.normal(size=(M, Cf, H, W)).astype(np.float32)
    # a few pixels where the rendered feature equals the target (||d|| = 0: not counted, zero gradient)
    same = rng.random((M, H, W)) < 0.05
    for c in range(Cf):
        feat[:, c][same] = target[:, c][same]
    mask = (rng.random((M, H, W)) < 0.6).astype(np.float32) * rng.uniform(0.5, 1.0, size=(M, H, W)).astype(np.float32)
    if empty_frame is not None:
        mask[empty_frame] = 0.0
    alpha = rng.uniform(0.0, 1.0, size=(M, H, W)).astype(np.float32)
    alpha[rng.random((M, H, W)) < 0.2] = 0.0
    if gm >= 0:
        feat[:, gm] = rng.uniform(0.0, 1.0, size=(M, H, W))
        eq = rng.random((M, H, W)) < 0.05                     # gauss mask == acc: v = 0, not counted
        feat[:, gm][eq] = alpha[eq]
    det = np.asarray(is_detected, np.float32)

    planes = torch.from_numpy(feat).requires_grad_(True)
    nhwc = planes.permute(0, 2, 3, 1)                          # the reference's (M,H,W,C) layout
    aux_dict = {"fg": {"feature": nhwc[..., :Cf]}}
    batch = {"feature": torch.from_numpy(target).permute(0, 2, 3, 1), "mask": torch.from_numpy(mask)[..., None],
             "vis2d": torch.ones((M, H, W, 1)), "is_detected": torch.from_numpy(det)}
    loss_dict = {}
    loc = {"loss_dict": loss_dict, "aux_dict": aux_dict, "batch": batch, "torch": torch}
    exec(stmts["feature"], loc)
    if gm >= 0:
        aux_dict["fg"]["gauss_mask"] = nhwc[..., gm:gm + 1]
        loc["rendered_fg_mask"] = torch.from_numpy(alpha)[..., None]
        exec(stmts["reg_gauss_mask"], loc)
    cfg = {"vis2d_dilate": False, "no_loss_mask": False, "maskloss_no_vis2d": False}
    mask_losses(types.SimpleNamespace(config=cfg), loss_dict, batch, {"field_type": "fg"})
    counts = {k: int((v > 0).sum()) for k, v in loss_dict.items()}
    apply_loss_weights(loss_dict, {"feature_wt": weights[0], "reg_gauss_mask_wt": weights[1], "train_res": 256})
    names = ("feature", "reg_gauss_mask")
    terms = np.array([float(loss_dict[k].detach()) if k in loss_dict else 0.0 for k in names], np.float64)
    sum(loss_dict.values()).backward()
    return {"in_features": feat, "in_target": target, "in_mask": mask, "in_is_detected": det, "in_alpha": alpha,
            "in_gauss_mask_channel": np.array([gm], np.int32), "in_weights": np.array(weights, np.float32),
            "ref_terms": terms, "ref_counts": np.array([counts.get(k, 0) for k in names], np.int64),
            "ref_grad_features": planes.grad.numpy()}


CASES = {"featloss_ragged_48x40": dict(seed=11, M=2, W=48, H=40, F=22, Cf=16, gm=21, is_detected=[1, 1]),
         "featloss_undetected_36x20": dict(seed=12, M=2, W=36, H=20, F=22, Cf=16, gm=21, is_detected=[0, 1]),
         "featloss_empty_mask_36x20": dict(seed=13, M=2, W=36, H=20, F=22, Cf=16, gm=21, is_detected=[1, 1], empty_frame=1),
         "featloss_no_gauss_36x20": dict(seed=14, M=2, W=36, H=20, F=22, Cf=16, gm=-1, is_detected=[1, 1])}

if __name__ == "__main__":
    ref = sys.argv[1] if len(sys.argv) > 1 else os.environ.get("VIDU4D_REFERENCE", "../reference")
    for name, kw in CASES.items():
        r = make_case(ref, **kw)
        np.savez_compressed(os.path.join(ROOT, "tests", "golden", name + ".npz"), **r)
        print(name, r["ref_terms"], r["ref_counts"])
