"""Generate tests/golden/reproj_*.npz from the REFERENCE's own code for Stage 3's feat_reproj loss, run on the CPU.

Nothing is copied: at run time this script reads the reference checkout and exec()s the source TEXT of
  - DeformableGaussian.global_match (lab4d/nnutils/deformable_gaussian.py:1436-1486), on a stand-in `self` holding
    logsigma, with torch.randperm seeded and the drawn indices recorded;
  - the forward_warp chain of make_warp_golden.py (get_bone_coords, dual_quaternion_skinning, apply_qt_to_gaussian, as
    SkinningWarp.forward chains them) on the matched points, shaped (M,N,1,3) with rotation None, as forward_project
    (:1488-1513) calls it;
  - Kmatinv / mat2K / K2inv / K2mat and pinhole_projection (lab4d/utils/geom_utils.py);
  - the feat_reproj statement of compute_recon_loss (lab4d/engine/model.py:669-672), mask_losses and apply_loss_weights
    with the reference's configuration defaults (field_type "fg", feat_reproj_wt, train_res).
Inputs, outputs, the drawn candidate indices and the autograd gradient of the loss with respect to every input are
stored; they pin tests/reproj_model.py (tests/test_reproj_cpu.py).

    python tests/golden/make_reproj_golden.py [REFERENCE_DIR]      # writes tests/golden/reproj_*.npz
"""
import ast
import importlib.util
import os
import sys
import textwrap
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _grab(ref, path, names, ns, in_class=None):
    src = open(os.path.join(ref, path)).read()
    tree = ast.parse(src)
    body = tree.body
    if in_class:
        body = next(n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == in_class).body
    for name in names:
        node = next(n for n in body if isinstance(n, ast.FunctionDef) and n.name == name)
        node.decorator_list = []
        exec(textwrap.dedent(ast.get_source_segment(src, node)), ns)


def _reference_code(ref):
    spec = importlib.util.spec_from_file_location("make_warp_golden", os.path.join(ROOT, "tests", "golden", "make_warp_golden.py"))
    mwg = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mwg)
    mwg.REF = ref
    ns = mwg._load_reference()                       # quaternion helpers, get_bone_coords, dual_quaternion_skinning, ...
    _grab(ref, "lab4d/nnutils/deformable_gaussian.py", ["global_match"], ns, in_class="DeformableGaussian")
    _grab(ref, "lab4d/utils/geom_utils.py", ["pinhole_projection", "K2mat", "mat2K", "K2inv", "Kmatinv"], ns)
    src = open(os.path.join(ref, "lab4d/engine/model.py")).read()
    tree = ast.parse(src)
    loss_ns = {"torch": torch}
    stmt = None
    for node in ast.walk(tree):
        if isinstance(node, ast.FunctionDef) and node.name in ("mask_losses", "apply_loss_weights"):
            exec(textwrap.dedent(ast.get_source_segment(src, node, padded=True)), loss_ns)
        if isinstance(node, ast.FunctionDef) and node.name == "compute_recon_loss":
            for st in ast.walk(node):
                if (isinstance(st, ast.Assign) and isinstance(st.targets[0], ast.Subscript)
                        and isinstance(st.targets[0].slice, ast.Constant) and st.targets[0].slice.value == "feat_reproj"):
                    stmt = textwrap.dedent(ast.get_source_segment(src, st, padded=True))
    assert stmt is not None
    return mwg, ns, loss_ns["mask_losses"], loss_ns["apply_loss_weights"], stmt


def make_case(ref, seed, M, H, W, P, B, num_grad, with_delta=True, is_detected=None, empty_frame=None, num_candidates=2048,
              weight=5e-2, train_res=256):
    mwg, ns, mask_losses, apply_loss_weights, stmt = _reference_code(ref)
    rng = np.random.default_rng(seed)
    warp_in = mwg.make_inputs(seed, P, B, M, False)                  # bones, articulations, field2cam as the warp fixtures
    # features: distinct scores (continuous values), unit-ish scale so the top-8 sets are unambiguous
    feat_px = rng.normal(size=(M, H, W, 16)).astype(np.float32)
    regist = rng.normal(size=(P, 16)).astype(np.float32)
    logsigma = np.array([np.log(2.0)], np.float32)
    f = np.array([[300.0, 0, W / 2], [0, 310.0, H / 2], [0, 0, 1]], np.float32)
    Kmat = np.stack([f + np.array([[0, 0, 0.5 * m], [0, 0, -0.3 * m], [0, 0, 0]], np.float32) for m in range(M)])
    ys, xs = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    hxy = np.stack([np.broadcast_to(xs, (M, H, W)), np.broadcast_to(ys, (M, H, W)), np.ones((M, H, W))], -1).astype(np.float32)
    hxy[..., :2] += rng.normal(size=(M, H, W, 2)).astype(np.float32)
    mask = (rng.random((M, H, W)) < 0.7).astype(np.float32)
    if empty_frame is not None:
        mask[empty_frame] = 0.0
    det = np.asarray(is_detected if is_detected is not None else [1.0] * M, np.float32)
    delta = (np.maximum(rng.normal(size=(M, H, W, B)), 0.0) * 0.1).astype(np.float32) if with_delta else None

    leaf = lambda a: torch.from_numpy(np.ascontiguousarray(a)).requires_grad_(True)  # noqa: E731
    t = {"feat_px": torch.from_numpy(feat_px), "regist_feat": leaf(regist), "xyz": warp_in["xyz"].clone().requires_grad_(True),
         "logsigma": leaf(logsigma), "rest_q": warp_in["rest_q"].clone().requires_grad_(True),
         "rest_t": warp_in["rest_t"].clone().requires_grad_(True), "log_gauss": warp_in["log_gauss"].clone().requires_grad_(True),
         "art_q": warp_in["art_q"].clone().requires_grad_(True), "art_t": warp_in["art_t"].clone().requires_grad_(True),
         "cam_q": warp_in["cam_q"].clone().requires_grad_(True), "cam_t": warp_in["cam_t"].clone().requires_grad_(True)}
    if delta is not None:
        t["delta"] = leaf(delta)

    # ---- global_match, with the candidate draw recorded
    drawn = []
    randperm = torch.randperm

    def recording_randperm(n, *a, **k):
        idx = randperm(n, *a, **k)
        drawn.append(idx[:min(num_candidates, n)].clone())
        return idx
    ns["torch"] = types.SimpleNamespace(**{k: getattr(torch, k) for k in dir(torch) if not k.startswith("__")})
    ns["torch"].randperm = recording_randperm
    torch.manual_seed(seed)
    regist_reshape = t["regist_feat"].reshape(1, P, 1, 16).expand(M, -1, -1, -1).contiguous()
    xyz_reshape = t["xyz"].reshape(1, P, 1, 3).expand(M, -1, -1, -1).contiguous()
    self_ = types.SimpleNamespace(logsigma=t["logsigma"])
    xyz_m = ns["global_match"](self_, t["feat_px"], regist_reshape, xyz_reshape, num_candidates=num_candidates,
                               num_grad=num_grad)                    # (M,H,W,3)
    ns["torch"] = torch

    # ---- forward_project: forward_warp (no rotation) + Kmatinv + pinhole_projection
    q2dq = ns["quaternion_translation_to_dual_quaternion"]
    rest = q2dq(t["rest_q"], t["rest_t"])
    art = q2dq(t["art_q"], t["art_t"])
    rest_m = (rest[0][None].expand(M, -1, -1), rest[1][None].expand(M, -1, -1))
    se3 = ns["dual_quaternion_mul"](art, ns["dual_quaternion_inverse"](rest_m))
    xyz4 = xyz_m.reshape(M, -1, 1, 3)
    articulation = (rest_m[0][:, None, None].expand(xyz4.shape[:3] + (-1, -1)),
                    rest_m[1][:, None, None].expand(xyz4.shape[:3] + (-1, -1)))
    xyz_bone = ns["get_bone_coords"](xyz4, articulation) / t["log_gauss"].exp().view(1, 1, 1, B, 3)
    dist2 = xyz_bone.pow(2).sum(-1)
    skin = -(dist2 + t["delta"].reshape(M, -1, 1, B)) if delta is not None else -dist2
    q, tr = ns["dual_quaternion_skinning"](se3, xyz4, skin.softmax(-1), return_qt=True)
    xyz_t, _ = ns["apply_qt_to_gaussian"](xyz4, None, q, tr, M)
    qc = t["cam_q"][:, None].repeat(1, xyz_t.shape[1], 1)
    tc = t["cam_t"][:, None].repeat(1, xyz_t.shape[1], 1)
    xyz_cam, _ = ns["apply_qt_to_gaussian"](xyz_t, None, qc, tc, M)
    xyz_cam = xyz_cam[:, :, 0]
    Kinv = torch.linalg.inv(torch.from_numpy(Kmat).double()).float()
    Kref = ns["Kmatinv"](Kinv)
    xy_reproj = ns["pinhole_projection"](Kref, xyz_cam)[..., :2].reshape(M, H, W, 2)

    # ---- the loss: compute_recon_loss's statement, mask_losses, apply_loss_weights
    loss_dict = {}
    batch = {"hxy": torch.from_numpy(hxy), "mask": torch.from_numpy(mask)[..., None], "vis2d": torch.ones((M, H, W, 1)),
             "is_detected": torch.from_numpy(det)}
    exec(stmt, {"loss_dict": loss_dict, "aux_dict": {"fg": {"xy_reproj": xy_reproj}}, "batch": batch, "torch": torch})
    cfg = {"vis2d_dilate": False, "no_loss_mask": False, "maskloss_no_vis2d": False}
    mask_losses(types.SimpleNamespace(config=cfg), loss_dict, batch, {"field_type": "fg"})
    v = loss_dict["feat_reproj"].detach()
    counts = (v > 0).reshape(M, -1).sum(1).numpy().astype(np.int64)
    apply_loss_weights(loss_dict, {"feat_reproj_wt": weight, "train_res": train_res})
    loss = loss_dict["feat_reproj"]
    loss.backward()
    out = {"in_feat_px": feat_px, "in_regist_feat": regist, "in_logsigma": logsigma, "in_Kmat": Kref.detach().numpy(),
           "in_hxy": hxy, "in_mask": mask, "in_is_detected": det, "in_cand": drawn[0].numpy().astype(np.int32),
           "in_meta": np.array([num_grad, train_res], np.int32), "in_weight": np.array([weight], np.float32),
           "ref_xyz_matched": xyz_m.detach().numpy(), "ref_xy_reproj": xy_reproj.detach().numpy(),
           "ref_loss": np.array([float(loss.detach())], np.float64), "ref_counts": counts}
    for k in ("xyz", "rest_q", "rest_t", "log_gauss", "art_q", "art_t", "cam_q", "cam_t"):
        out["in_" + k] = warp_in[k].numpy()
    if delta is not None:
        out["in_delta"] = delta
    for k, v_ in t.items():
        if v_.grad is not None:
            out["ref_grad_" + k] = v_.grad.numpy()
    return out


CASES = {
    # ragged frame, C = M*P < 2048: every surfel copy is a candidate
    "reproj_ragged_48x40": dict(seed=21, M=2, H=40, W=48, P=500, B=7, num_grad=8),
    # M*P > 2048: C = 2048, and both copies of some surfels are drawn (duplicates sum into one row); no delta
    "reproj_dup_nodelta_24x20": dict(seed=22, M=2, H=20, W=24, P=1500, B=5, num_grad=8, with_delta=False),
    # a frame that is not detected, K < 8
    "reproj_undetected_k4_20x16": dict(seed=23, M=2, H=16, W=20, P=300, B=4, num_grad=4, is_detected=[0.0, 1.0]),
    # a frame with an empty mask
    "reproj_empty_mask_20x16": dict(seed=24, M=2, H=16, W=20, P=300, B=4, num_grad=8, empty_frame=1),
}

if __name__ == "__main__":
    ref = sys.argv[1] if len(sys.argv) > 1 else os.environ.get("VIDU4D_REFERENCE", "../reference")
    for name, kw in CASES.items():
        r = make_case(ref, **kw)
        np.savez_compressed(os.path.join(ROOT, "tests", "golden", name + ".npz"), **r)
        print(name, float(r["ref_loss"][0]), r["ref_counts"], os.path.getsize(os.path.join(ROOT, "tests", "golden", name + ".npz")))
