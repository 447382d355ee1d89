"""Generate tests/golden/maskloss_*.npz from the REFERENCE's own loss code, run on the CPU with torch autograd.

This script does not copy the reference: at run time it reads lab4d/engine/model.py from the reference checkout, takes
the source TEXT of (i) get_mask_balance_wt (:587-611), (ii) the field_type "fg" branch of compute_recon_loss's mask
statement (:648-650), (iii) mask_losses (:895-977) and (iv) apply_loss_weights (:980-1012), and exec()s them on seeded
float32 CPU tensors in the reference's (M,H,W,1) layout with its configuration defaults (field_type "fg", no_loss_mask,
maskloss_no_vis2d and vis2d_dilate off).  pos_wt and neg_wt are read from get_mask_balance_wt's own frame as it returns.
The balance weights, the loss, the counts of positive values and dL/dacc are stored with the inputs; they pin
tests/mask_loss_model.py (tests/test_mask_loss_cpu.py) and the kernels (tests/test_gpu_mask_loss.py).

    python tests/golden/make_mask_loss_golden.py [REFERENCE_DIR]      # writes tests/golden/maskloss_*.npz
"""
import ast
import os
import sys
import textwrap
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _is_fg_test(test):
    return (isinstance(test, ast.Compare) and isinstance(test.comparators[0], ast.Constant)
            and test.comparators[0].value == "fg" and isinstance(test.left, ast.Subscript)
            and isinstance(test.left.slice, ast.Constant) and test.left.slice.value == "field_type")


def _assigns_mask(st):
    t = st.targets[0] if isinstance(st, ast.Assign) else st.target if isinstance(st, ast.AugAssign) else None
    return isinstance(t, ast.Subscript) and isinstance(t.slice, ast.Constant) and t.slice.value == "mask"


def _reference_code(ref):
    src = open(os.path.join(ref, "lab4d/engine/model.py")).read()
    tree = ast.parse(src)
    funcs, fg = {}, None
    for node in ast.walk(tree):
        if isinstance(node, ast.FunctionDef) and node.name in ("get_mask_balance_wt", "mask_losses", "apply_loss_weights"):
            funcs[node.name] = textwrap.dedent(ast.get_source_segment(src, node, padded=True))
        if isinstance(node, ast.FunctionDef) and node.name == "compute_recon_loss":
            for st in ast.walk(node):         # the if/elif chain on field_type whose "fg" branch builds loss_dict["mask"]
                if isinstance(st, ast.If) and _is_fg_test(st.test) and st.body and all(_assigns_mask(b) for b in st.body):
                    fg = "\n".join(textwrap.dedent(ast.get_source_segment(src, b, padded=True)) for b in st.body)
    assert set(funcs) == {"get_mask_balance_wt", "mask_losses", "apply_loss_weights"} and fg is not None
    ns = {"torch": torch}
    for code in funcs.values():
        exec(code, ns)
    return ns["get_mask_balance_wt"], ns["mask_losses"], ns["apply_loss_weights"], fg


def _balance_with_locals(fn, *args):
    """fn(*args) and the local variables of its frame as it returns (pos_wt / neg_wt when the branch runs)."""
    seen = {}

    def prof(frame, event, arg):
        if event == "return" and frame.f_code is fn.__code__:
            seen.update(frame.f_locals)
    old = sys.getprofile()
    sys.setprofile(prof)
    try:
        out = fn(*args)
    finally:
        sys.setprofile(old)
    return out, seen


def make_case(ref, seed, M, W, H, is_detected, kind="binary", weight=0.1):
    get_mask_balance_wt, mask_losses, apply_loss_weights, fg = _reference_code(ref)
    rng = np.random.default_rng(seed)
    vis = (rng.random((M, H, W)) < 0.85).astype(np.float32)
    if kind == "fractional":
        mask = np.where(rng.random((M, H, W)) < 0.5, rng.uniform(0.0, 1.0, (M, H, W)), 0.0).astype(np.float32)
    else:
        mask = (rng.random((M, H, W)) < 0.4).astype(np.float32)
    if kind == "all_zero":
        mask[:] = 0.0
    if kind == "all_one":
        mask[:] = 1.0
    if kind == "outside_vis":                                  # every mask pixel lies where vis2d = 0
        mask = ((vis == 0) & (rng.random((M, H, W)) < 0.7)).astype(np.float32)
    alpha = rng.uniform(0.0, 1.0, (M, H, W)).astype(np.float32)
    alpha[rng.random((M, H, W)) < 0.1] = 0.0
    same = rng.random((M, H, W)) < 0.05                        # acc == gt: v = 0, not counted
    alpha[same] = mask[same]
    if kind == "acc_eq_gt":
        alpha = mask.copy()
    det = np.asarray(is_detected, np.float32)

    acc = torch.from_numpy(alpha).requires_grad_(True)
    batch = {"mask": torch.from_numpy(mask)[..., None], "vis2d": torch.from_numpy(vis)[..., None],
             "is_detected": torch.from_numpy(det)}
    bw, frame = _balance_with_locals(get_mask_balance_wt, batch["mask"], batch["vis2d"], batch["is_detected"])
    on = "pos_wt" in frame
    loss_dict = {}
    exec(fg, {"loss_dict": loss_dict, "rendered_fg_mask": acc[..., None], "batch": batch, "mask_balance_wt": bw,
              "torch": torch})
    cfg = {"vis2d_dilate": False, "no_loss_mask": False, "maskloss_no_vis2d": False}
    mask_losses(types.SimpleNamespace(config=cfg), loss_dict, batch, {"field_type": "fg"})
    v = loss_dict["mask"].detach()[..., 0]
    counts = (v > 0).reshape(M, -1).sum(1).numpy().astype(np.int64)
    apply_loss_weights(loss_dict, {"mask_wt": weight, "train_res": 256})
    loss = loss_dict["mask"]
    loss.backward()
    bw_map = (bw * torch.ones((M, H, W, 1)))[..., 0] if torch.is_tensor(bw) else torch.full((M, H, W), float(bw))
    nan = np.float32(np.nan)
    return {"in_alpha": alpha, "in_mask": mask, "in_vis2d": vis, "in_is_detected": det,
            "in_weight": np.array([weight], np.float32),
            "ref_branch": np.array([on], np.int32),
            "ref_pos_wt": np.array([float(frame["pos_wt"]) if on else nan], np.float32),
            "ref_neg_wt": np.array([float(frame["neg_wt"]) if on else nan], np.float32),
            "ref_balance_wt": bw_map.detach().numpy().astype(np.float32), "ref_v": v.numpy(),
            "ref_loss": np.array([float(loss.detach())], np.float32), "ref_counts": counts,
            "ref_grad_alpha": acc.grad.numpy()}


CASES = {"maskloss_binary_48x40": dict(seed=21, M=2, W=48, H=40, is_detected=[1, 1]),
         "maskloss_fractional_48x40": dict(seed=22, M=2, W=48, H=40, is_detected=[1, 1], kind="fractional"),
         "maskloss_undetected_48x40": dict(seed=23, M=2, W=48, H=40, is_detected=[0, 1]),
         "maskloss_none_detected_48x40": dict(seed=24, M=2, W=48, H=40, is_detected=[0, 0]),
         "maskloss_all_zero_48x40": dict(seed=25, M=2, W=48, H=40, is_detected=[1, 1], kind="all_zero"),
         "maskloss_all_one_48x40": dict(seed=26, M=2, W=48, H=40, is_detected=[1, 1], kind="all_one"),
         "maskloss_outside_vis_48x40": dict(seed=27, M=2, W=48, H=40, is_detected=[1, 1], kind="outside_vis"),
         "maskloss_acc_eq_gt_48x40": dict(seed=28, M=2, W=48, H=40, is_detected=[1, 1], kind="acc_eq_gt"),
         "maskloss_m8_37x23": dict(seed=29, M=8, W=37, H=23, is_detected=[1, 1, 0, 1, 1, 1, 0, 1])}

if __name__ == "__main__":
    ref = sys.argv[1] if len(sys.argv) > 1 else os.environ.get("VIDU4D_REFERENCE", "../reference")
    for name, kw in CASES.items():
        r = make_case(ref, **kw)
        np.savez_compressed(os.path.join(ROOT, "tests", "golden", name + ".npz"), **r)
        print(name, r["ref_branch"], r["ref_pos_wt"], r["ref_neg_wt"], r["ref_loss"], r["ref_counts"])
