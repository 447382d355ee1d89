"""Generate tests/golden/dskin_*.npz from the REFERENCE's own delta-skinning code, run on the CPU in this container.

Nothing is copied: like make_cycle_golden.py (whose loader this script reuses) it loads lab4d/utils/quat_transform.py from
/root/reference by path and exec()s the source text of get_bone_coords (lab4d/utils/transforms.py), of the classes BaseMLP
and CondMLP (lab4d/nnutils/base.py), InstEmbedding and PosEmbedding (lab4d/nnutils/embedding.py), and of
SkinningField.forward / get_gauss_bone_coords / get_gauss (lab4d/nnutils/skinning.py:89-153), which run as the methods of
a holder object whose attributes are the reference's own modules: pos_embedding = PosEmbedding(3B, 0), delta_field =
CondMLP(num_inst, D=2, W=64, in_channels=3B+128, inst_channels=32, out_channels=B) as skinning.py:68-85 builds them.  The
time embedding is the caller's and is an input here: a stand-in returns the given (128,) mean code or the given per-frame
codes.  The instance code comes from the reference's InstEmbedding (the mean code for inst_id None, the frame's otherwise).

Each case runs in float32 (delta and its autograd gradients for the upstream gradient w_delta) and on the same inputs in
float64.  `in_cond` is cat(t_embed, inst_code) as CondMLP.forward concatenates them; `*_grad_cond` its gradient.

    python tests/golden/make_delta_skin_golden.py        # needs /root/reference
"""
import ast
import os
import sys
import textwrap

import numpy as np
import torch
from torch import nn

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_cycle_golden import _grab  # noqa: E402
from make_warp_golden import REF, ROOT, _load_reference, rand_unit_quat  # noqa: E402

T_CHANNELS, INST_CHANNELS = 128, 32


def _grab_class(ns, path, name):
    src = open(os.path.join(REF, path)).read()
    node = next(n for n in ast.parse(src).body if isinstance(n, ast.ClassDef) and n.name == name)
    exec(textwrap.dedent(ast.get_source_segment(src, node)), ns)


def load():
    ns = _load_reference()
    ns.update(nn=nn, np=np)
    for name in ("PosEmbedding", "InstEmbedding"):
        _grab_class(ns, "lab4d/nnutils/embedding.py", name)
    for name in ("BaseMLP", "CondMLP"):
        _grab_class(ns, "lab4d/nnutils/base.py", name)
    for name in ("forward", "get_gauss_bone_coords", "get_gauss"):
        _grab(ns, "lab4d/nnutils/skinning.py", name, in_class="SkinningField")
        ns["skin_" + name] = ns.pop(name)
    return ns


class _TimeCodes:
    """Stand-in for the caller's TimeEmbedding: the codes are inputs."""
    out_channels = T_CHANNELS

    def __init__(self, mean, frames):
        self.mean, self.frames = mean, frames

    def get_mean_embedding(self, device):
        return self.mean[None]

    def __call__(self, frame_id):
        return self.frames[frame_id]


def make_field(ns, B, num_inst, seed):
    """A holder with the attributes SkinningField.__init__ creates and the reference's three methods."""
    torch.manual_seed(seed)

    class Field(nn.Module):
        forward = ns["skin_forward"]
        get_gauss_bone_coords = ns["skin_get_gauss_bone_coords"]
        get_gauss = ns["skin_get_gauss"]
    f = Field()
    f.symm_idx = None
    f.pos_embedding = ns["PosEmbedding"](3 * B, 0)
    f.delta_field = ns["CondMLP"](num_inst=num_inst, D=2, W=64, in_channels=f.pos_embedding.out_channels + T_CHANNELS,
                                  inst_channels=INST_CHANNELS, out_channels=B, skips=[4], activation=nn.ReLU(True), final_act=False)
    return f


def make_case(ns, seed, B, shape, per_frame=False, b3=None, on_bones=False):
    """shape: the points' shape without the trailing 3.  per_frame: bones and cond per frame (shape[0] frames).  b3: every output bias
    (so negative that every output is clipped).  on_bones: the first B points sit on the bone centres."""
    rng = np.random.default_rng(seed)
    M = shape[0] if len(shape) > 1 else 1
    Mb = M if per_frame else 1
    centres = rng.normal(size=(Mb, B, 3)) * 0.15
    q = rand_unit_quat(rng, Mb, B)
    pts = rng.normal(size=tuple(shape) + (3,)) * 0.15
    if on_bones:
        flat = pts.reshape(-1, 3)
        flat[:B] = centres[0].astype(np.float32)
    f32 = lambda a: torch.tensor(np.asarray(a), dtype=torch.float32)  # noqa: E731
    art_r, art_d = ns["quaternion_translation_to_dual_quaternion"](f32(q if per_frame else q[0]),
                                                                   f32(centres if per_frame else centres[0]))
    inp = dict(points=f32(pts), art_r=art_r, art_d=art_d,
               log_gauss=f32(np.log(0.03) + 0.3 * rng.normal(size=(B, 3))),
               t_mean=f32(rng.normal(size=(T_CHANNELS,)) * 0.5), t_frames=f32(rng.normal(size=(M, T_CHANNELS)) * 0.5),
               w_delta=f32(rng.normal(size=tuple(shape) + (B,))))
    return inp, dict(B=B, M=M, per_frame=per_frame, b3=b3, seed=seed)


def run_reference(ns, inp, meta, dtype):
    B, M, per_frame = meta["B"], meta["M"], meta["per_frame"]
    # one instance when the code is shared: its mean code is then that instance's code exactly, in either precision
    field = make_field(ns, B, num_inst=M if per_frame else 1, seed=meta["seed"]).to(dtype)
    if meta["b3"] is not None:
        with torch.no_grad():
            field.delta_field.linear_final.bias.fill_(meta["b3"])
    t = {k: v.to(dtype).clone().requires_grad_(k != "w_delta") for k, v in inp.items()}
    field.log_gauss = t["log_gauss"]
    field.time_embedding = _TimeCodes(t["t_mean"], t["t_frames"])
    art = (t["art_r"], t["art_d"])
    xyz = t["points"]
    while xyz.dim() < 4:                                                    # (M,N,D,3) as SkinningField.forward documents
        xyz = xyz[None] if xyz.dim() == 2 else xyz[:, :, None]
    lead = xyz.shape[:3]
    bone2obj = tuple((h[:, None, None] if per_frame else h[None, None, None]).expand(lead + (B, 4)) for h in art)
    ids = torch.arange(M) if per_frame else None
    _, delta = field(xyz, bone2obj, ids, ids)
    delta = delta.reshape(t["w_delta"].shape)
    (delta * t["w_delta"]).sum().backward()
    emb = field.delta_field.inst_embedding.mapping.weight
    if per_frame:
        cond = torch.cat((t["t_frames"], emb[:M]), -1)
        g_cond = torch.cat((t["t_frames"].grad, emb.grad[:M]), -1)
    else:
        cond = torch.cat((t["t_mean"], emb.mean(0)), -1)
        g_cond = torch.cat((t["t_mean"].grad, emb.grad.sum(0)), -1)
    mlp = field.delta_field
    params = dict(W1=mlp.linear_1[0].weight, b1=mlp.linear_1[0].bias, W2=mlp.linear_2[0].weight, b2=mlp.linear_2[0].bias,
                  W3=mlp.linear_final.weight, b3=mlp.linear_final.bias)
    vals = dict(points=t["points"], art_r=art[0], art_d=art[1], log_gauss=t["log_gauss"], **params)
    out = {"delta": delta.detach().numpy(), "grad_cond": g_cond.detach().numpy()}
    out.update({"grad_" + k: v.grad.numpy() for k, v in vals.items()})
    ins = {k: v.detach().numpy() for k, v in vals.items()}
    ins.update(cond=cond.detach().numpy(), w_delta=t["w_delta"].numpy())
    return ins, out


CASES = {"dskin_b25_shared": dict(seed=21, B=25, shape=(333,)),
         "dskin_b25_m2_frames": dict(seed=22, B=25, shape=(2, 201), per_frame=True),
         "dskin_b25_grid": dict(seed=23, B=25, shape=(2, 9, 11)),
         "dskin_b7": dict(seed=24, B=7, shape=(150,)),
         "dskin_b25_n1": dict(seed=25, B=25, shape=(1,)),
         "dskin_b25_clipped": dict(seed=26, B=25, shape=(140,), b3=-1e3),
         "dskin_b25_on_bones": dict(seed=27, B=25, shape=(90,), on_bones=True),
         "dskin_b64_m3_frames": dict(seed=28, B=64, shape=(3, 130), per_frame=True)}

if __name__ == "__main__":
    ns = load()
    for name, kw in CASES.items():
        inp, meta = make_case(ns, **kw)
        ins, ref = run_reference(ns, inp, meta, torch.float32)
        ins64, ref64 = run_reference(ns, inp, meta, torch.float64)
        for k, v in ins.items():                        # the float64 run starts from the float32 run's inputs
            assert np.array_equal(v.astype(np.float64), ins64[k]), (name, k)
        out = {"in_" + k: v for k, v in ins.items()}
        out.update({"ref_" + k: v for k, v in ref.items()})
        out.update({"ref64_" + k: v for k, v in ref64.items()})
        np.savez_compressed(os.path.join(ROOT, "tests", "golden", name + ".npz"), **out)
        print(name, ins["points"].shape, "delta > 0:", float((ref["delta"] > 0).mean()), "max", float(ref["delta"].max()))
