"""CPU: FlatSurfelModel checkpoints, the reference's load_checkpoint sequence on a store, torch.optim.Adam state import
and export, and 2DGS's vertex PLY (vidu4d_b200/ply.py).  No kernel runs: the store is built on CPU tensors."""
import io

import numpy as np
import pytest
import torch

from vidu4d_b200 import ply
from vidu4d_b200.surfel_store import STORE_KEYS, FlatSurfelModel

ATTRS = ("_xyz", "_features_dc", "_features_rest", "_opacity", "_scaling", "_rotation", "_regist_feat")
NAMES = ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation", "regist_feat")
TAILS = ((3,), (1, 3), (15, 3), (1,), (2,), (4,), (16,))


def _store(P, regist=True, seed=0, state=True):
    """A store of P random surfels; with `state`, random moments, statistics, step counts, rates and constants."""
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g)  # noqa: E731
    m = FlatSurfelModel(r(P, 3), r(P, 1, 3), r(P, 15, 3), r(P, 1), r(P, 2), r(P, 4), sh_degree=1,
                        regist_feat=r(P, 16) if regist else None)
    if state:
        m.exp_avg.copy_(r(m.flat.numel()))
        m.exp_avg_sq.copy_(r(m.flat.numel()).abs())
        m.densify_stats.copy_(r(2, P).abs())
        m.max_radii2D.copy_(r(P).abs() * 9)
        m.device_step.fill_(37 + seed)
        m.step_count = 11 + seed
        for i, (n, _) in enumerate(m.groups):
            m.set_lr(n, 1e-3 * (i + 1) + seed * 1e-5)
        m.active_sh_degree = 2
        m.betas, m.eps, m.percent_dense = (0.8, 0.99), 1e-12, 0.02
    return m


def _bits(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(a.reshape(-1).view(torch.uint8),
                                                                      b.reshape(-1).view(torch.uint8))


def _same_store(a, b):
    assert a.P == b.P and a.groups == b.groups
    for name in ("flat", "exp_avg", "exp_avg_sq", "device_step", "device_lr", "densify_stats", "max_radii2D"):
        assert _bits(getattr(a, name), getattr(b, name)), name
    assert (a.step_count, a.active_sh_degree, a.betas, a.eps, a.percent_dense, a.lrs) == \
           (b.step_count, b.active_sh_degree, b.betas, b.eps, b.percent_dense, b.lrs)


def _views_of_flat(m):
    off, total = m._offsets(m.P)
    for p, o, (n, k) in zip(m.flat_params(), off, m.groups):
        assert p.data_ptr() == m.flat.data_ptr() + 4 * o or m.P == 0, n
        assert p.grad is not None and (p.grad.data_ptr() == m.grad_flat.data_ptr() + 4 * o or m.P == 0), n
        assert tuple(p.shape) == (m.P,) + TAILS[NAMES.index(n)]
    assert m.flat.numel() == m.grad_flat.numel() == m.exp_avg.numel() == total


def _saved(m):
    buf = io.BytesIO()
    torch.save(m.state_dict(), buf)
    buf.seek(0)
    return torch.load(buf, weights_only=True)


# ---- state dict ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("P", [0, 1, 7, 64, 1001])
@pytest.mark.parametrize("regist", [False, True])
def test_state_dict_round_trip_bit_for_bit(P, regist):
    src = _store(P, regist, seed=1)
    sd = _saved(src)
    n = len(NAMES) - (not regist)
    assert list(sd)[:n] == list(ATTRS[:n]) and set(STORE_KEYS) <= set(sd)
    for a, tail in zip(ATTRS[:n], TAILS):
        assert tuple(sd[a].shape) == (P,) + tail
    for P0 in (P, P + 5):                              # same P (in place) and another P (fresh buffers)
        dst = _store(P0, regist, seed=2)
        dst.load_state_dict(sd)
        _same_store(dst, src)
        _views_of_flat(dst)


def test_same_p_load_keeps_every_address():
    src, dst = _store(13, seed=1), _store(13, seed=2)
    ptrs = lambda m: [t.data_ptr() for t in (m.flat, m.grad_flat, m.exp_avg, m.exp_avg_sq, m.device_step,  # noqa: E731
                                              m.device_lr, m.densify_stats, m.max_radii2D)]
    before, params = ptrs(dst), dst.flat_params()
    dst.grad_flat.fill_(3.0)
    dst.load_state_dict(src.state_dict())
    assert ptrs(dst) == before and all(a is b for a, b in zip(params, dst.flat_params()))
    _same_store(dst, src)
    assert not dst.grad_flat.any()


def test_other_p_load_rebinds_views_and_gradients():
    src, dst = _store(21, seed=1), _store(8, seed=2)
    dst.load_state_dict(src.state_dict())
    _views_of_flat(dst)
    dst.grad_flat.copy_(torch.arange(dst.grad_flat.numel(), dtype=torch.float32))
    off, _ = dst._offsets(dst.P)
    assert float(dst._opacity.grad[5, 0]) == off[3] + 5
    assert dst.xyz_gradient_accum.shape == (21, 1)


def test_group_lists_cannot_be_confused():
    with pytest.raises(RuntimeError, match="surfel groups"):
        _store(5, regist=False).load_state_dict(_store(5, regist=True).state_dict())
    with pytest.raises(RuntimeError, match="surfel groups"):
        _store(5, regist=True).load_state_dict(_store(5, regist=False).state_dict())


# ---- the reference's load_checkpoint (lab4d/engine/trainer.py:386-396) on a store ----------------------------------------
class _Fields(torch.nn.Module):
    def __init__(self, fg):
        super().__init__()
        self.fg = fg


def _reference_load(model_states, fg, upto=None):
    """trainer.py:386-396 verbatim on `model.fields.field_params.fg`, stopping after `upto` surfel-group assignments if
    given."""
    model = torch.nn.Module()
    model.fields = torch.nn.Module()
    model.fields.field_params = _Fields(fg)
    steps = [
        lambda: setattr(model.fields.field_params.fg, "_xyz", torch.nn.Parameter(new_xyz)),
        lambda: setattr(model.fields.field_params.fg, "_xyz", torch.nn.Parameter(model.fields.field_params.fg._xyz[:num_pts].clone().detach())),
        lambda: setattr(model.fields.field_params.fg, "_features_dc", torch.nn.Parameter(model.fields.field_params.fg._features_dc[:num_pts].clone().detach())),
        lambda: setattr(model.fields.field_params.fg, "_features_rest", torch.nn.Parameter(model.fields.field_params.fg._features_rest[:num_pts].clone().detach())),
        lambda: setattr(model.fields.field_params.fg, "_opacity", torch.nn.Parameter(model.fields.field_params.fg._opacity[:num_pts].clone().detach())),
        lambda: setattr(model.fields.field_params.fg, "_scaling", torch.nn.Parameter(model.fields.field_params.fg._scaling[:num_pts].clone().detach())),
        lambda: setattr(model.fields.field_params.fg, "_rotation", torch.nn.Parameter(model.fields.field_params.fg._rotation[:num_pts].clone().detach())),
        lambda: setattr(model.fields.field_params.fg, "_regist_feat", torch.nn.Parameter(model.fields.field_params.fg._regist_feat[:num_pts].clone().detach())),
    ]
    scale = torch.tensor([1])  # scale of the field
    model.fields.field_params.fg.logscale = torch.nn.Parameter(scale.log())
    num_pts = model_states["fields.field_params.fg._xyz"].shape[0]
    new_xyz = model.fields.field_params.fg._xyz[:num_pts].clone().detach()
    for s in steps[:upto]:
        s()
    if upto is None:
        model.load_state_dict(model_states, strict=False)
    return model


def _states(m):
    return {"fields.field_params.fg." + k: v for k, v in _saved(m).items()}


@pytest.mark.parametrize("P_live,P_ckpt", [(40, 17), (17, 17), (17, 40), (9, 0)])
@pytest.mark.parametrize("store_ckpt", [True, False])
def test_reference_sequence_keeps_the_store_whole(P_live, P_ckpt, store_ckpt):
    src = _store(P_ckpt, seed=1)
    states = _states(src)
    if not store_ckpt:
        states = {k: v for k, v in states.items() if k.split(".")[-1] in ATTRS}
    fg = _store(P_live, seed=2)
    _reference_load(states, fg)
    assert fg.P == P_ckpt and not fg._foreign
    _views_of_flat(fg)
    assert _bits(fg.flat, src.flat)
    if store_ckpt:
        _same_store(fg, src)
    else:
        # the reference's resume: parameters only, Adam from zero and step 0
        assert not fg.exp_avg.any() and not fg.exp_avg_sq.any() and int(fg.device_step) == 0 and fg.step_count == 0
        assert not fg.densify_stats.any() and not fg.max_radii2D.any()


@pytest.mark.parametrize("P_live,P_ckpt", [(40, 17), (17, 17)])
def test_reference_sequence_loads_the_other_parameters(P_live, P_ckpt):
    """trainer.py:387-388 resets fg.logscale before load_state_dict: the checkpoint's value must come back."""
    src = _store(P_ckpt, seed=1)
    src.logscale = torch.nn.Parameter(torch.tensor([0.7]))
    fg = _store(P_live, seed=2)
    _reference_load(_states(src), fg)
    assert float(fg.logscale.detach()) == np.float32(0.7)
    _same_store(fg, src)


class _Fg(FlatSurfelModel):
    """A store with fields of its own beside the surfel groups."""

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.logscale = torch.nn.Parameter(torch.zeros(1))
        self.register_buffer("near_far", torch.zeros(2))


def _fg(P, seed):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g)  # noqa: E731
    return _Fg(r(P, 3), r(P, 1, 3), r(P, 15, 3), r(P, 1), r(P, 2), r(P, 4), regist_feat=r(P, 16))


@pytest.mark.parametrize("P0", [11, 30])
def test_other_parameters_and_buffers_load_strictly(P0):
    src, dst = _fg(11, seed=1), _fg(P0, seed=2)
    with torch.no_grad():
        src.logscale.fill_(0.25)
        src.near_far.copy_(torch.tensor([0.5, 9.0]))
    res = dst.load_state_dict(_saved(src))             # strict: every key of the store's own state dict is known
    assert not res.missing_keys and not res.unexpected_keys
    assert float(dst.logscale.detach()) == 0.25 and dst.near_far.tolist() == [0.5, 9.0] and _bits(dst.flat, src.flat)
    sd = _saved(src)
    sd["stray"] = torch.zeros(1)
    with pytest.raises(RuntimeError, match="Unexpected key.*stray"):
        dst.load_state_dict(sd)
    del sd["stray"], sd["logscale"]
    with pytest.raises(RuntimeError, match="Missing key.*logscale"):
        dst.load_state_dict(sd)
    assert not dst.load_state_dict(sd, strict=False).unexpected_keys


def test_missing_group_cannot_take_a_held_tensor_of_another_count():
    m = _store(12, seed=3)
    m._opacity = torch.nn.Parameter(torch.ones(1, 1))
    sd = {k: v for k, v in _store(12, seed=4).state_dict().items() if k != "_opacity"}
    with pytest.raises(RuntimeError, match="_opacity is missing from the checkpoint"):
        m.load_state_dict(sd, strict=False)
    with pytest.raises(RuntimeError, match="disagree on the surfel count"):
        m.flat_params()


def test_assigning_a_group_the_store_lacks_raises():
    m = _store(5, regist=False)
    with pytest.raises(AttributeError, match="no regist_feat group"):
        m._regist_feat = torch.nn.Parameter(torch.zeros(5, 16))
    assert "_regist_feat" not in dict(m.named_parameters())


@pytest.mark.parametrize("upto", [1, 3, 7])
def test_half_finished_sequence_raises_on_use(upto):
    fg = _store(40, seed=2)
    _reference_load(_states(_store(17, seed=1)), fg, upto=upto)
    uses = [lambda: fg.get_xyz, lambda: fg.get_features, lambda: fg.get_opacity, lambda: fg.get_scaling,
            lambda: fg.get_rotation, fg.flat_params, fg.step, fg.adam_step, lambda: fg.clip_grad_norm_(1.0),
            lambda: fg.densify_and_prune(1e-4, 0.005, 1.0, None), lambda: fg.prune_points(torch.zeros(40, dtype=torch.bool)),
            lambda: fg.add_densification_stats(torch.zeros(40, 3), torch.ones(40, dtype=torch.bool)), fg.reset_opacity,
            fg.state_dict, fg.allreduce_grads_, fg.replica_state]
    for use in uses:
        with pytest.raises(RuntimeError, match="disagree on the surfel count"):
            use()
    # finishing with load_state_dict makes it whole
    src = _store(17, seed=1)
    fg.load_state_dict(src.state_dict(), strict=False)   # as the reference loads
    _same_store(fg, src)
    _views_of_flat(fg)


def test_same_p_assignment_is_in_place():
    m = _store(12, seed=3)
    ptr, moments = m.flat.data_ptr(), m.exp_avg.clone()
    new = torch.randn(12, 15, 3)
    m._features_rest = torch.nn.Parameter(new)
    assert m.flat.data_ptr() == ptr and torch.equal(m._features_rest, new) and torch.equal(m.exp_avg, moments)
    assert m._features_rest.data_ptr() != new.data_ptr()
    _views_of_flat(m)
    with pytest.raises(ValueError, match=r"\(P,15,3\)"):
        m._features_rest = torch.zeros(12, 45)


# ---- cross-loading with the reference's GaussianModel --------------------------------------------------------------------
class _GaussianModel(torch.nn.Module):
    """The attributes the reference's GaussianModel / DeformableGaussian keeps as parameters (gaussian_model.py)."""

    def __init__(self, P, seed=0):
        super().__init__()
        g = torch.Generator().manual_seed(seed)
        for a, tail in zip(ATTRS, TAILS):
            setattr(self, a, torch.nn.Parameter(torch.randn((P,) + tail, generator=g)))
        self.active_sh_degree, self.percent_dense = 3, 0.01


def test_store_checkpoint_loads_into_the_reference_model():
    src = _store(23, seed=4)
    gm = _GaussianModel(23)
    res = gm.load_state_dict(_saved(src), strict=False)
    assert set(res.unexpected_keys) == set(STORE_KEYS) and not res.missing_keys
    for a, p in zip(ATTRS, src.flat_params()):
        assert _bits(getattr(gm, a).detach(), p.detach())


def test_reference_state_dict_loads_into_the_store():
    gm = _GaussianModel(31, seed=5)
    m = _store(10, seed=6)
    m.load_state_dict(gm.state_dict())                 # strict: the reference's keys are all the store needs
    assert m.P == 31 and int(m.device_step) == 0 and not m.exp_avg.any()
    for a, p in zip(ATTRS, m.flat_params()):
        assert _bits(getattr(gm, a).detach(), p.detach())


# ---- torch.optim.Adam interop (trainer.py:243-253) -------------------------------------------------------------------------
def _torch_adam(gm, steps=3, seed=0, skip=()):
    lrs = (1.6e-4, 2.5e-3, 1.25e-4, 5e-2, 5e-3, 1e-3, 2.5e-3)
    bg = torch.nn.Parameter(torch.rand(3))
    groups = [{"params": [getattr(gm, a)], "lr": lr, "name": n} for a, n, lr in zip(ATTRS, NAMES, lrs)]
    opt = torch.optim.Adam(groups + [{"params": [bg], "lr": 1e-3, "name": "bg_rgb"}], lr=1e-3, eps=1e-15)
    g = torch.Generator().manual_seed(seed)
    for _ in range(steps):
        for a in ATTRS:
            p = getattr(gm, a)
            p.grad = None if a in skip else torch.randn(p.shape, generator=g)
        bg.grad = torch.randn(3, generator=g)
        opt.step()
    return opt


def test_adam_import_export_round_trip_bit_for_bit():
    gm = _GaussianModel(19, seed=7)
    opt = _torch_adam(gm)
    want = opt.state_dict()
    m = FlatSurfelModel.from_gaussian_model(gm, opt)
    assert int(m.device_step) == m.step_count == 3 and m.eps == 1e-15 and m.betas == (0.9, 0.999)
    assert m.lrs["f_rest"] == 1.25e-4
    for a, p in zip(ATTRS, m.flat_params()):
        assert _bits(getattr(gm, a).detach(), p.detach())
    got = m.adam_state_dict(opt)
    assert [g["name"] for g in got["param_groups"]] == list(NAMES) + ["bg_rgb"]
    for i in want["state"]:
        for k in ("step", "exp_avg", "exp_avg_sq"):
            assert _bits(got["state"][i][k], want["state"][i][k]), (i, k)
    # into a fresh optimizer over a fresh model, and back into a store
    gm2 = _GaussianModel(19, seed=8)
    opt2 = _torch_adam(gm2, steps=0)
    opt2.load_state_dict(got)
    back = FlatSurfelModel.from_gaussian_model(gm2, opt2)
    for name in ("exp_avg", "exp_avg_sq", "device_step"):
        assert _bits(getattr(back, name), getattr(m, name)), name


def test_adam_export_without_an_optimizer_loads_into_torch():
    src = _store(9, seed=9)
    gm = _GaussianModel(9)
    opt = _torch_adam(gm, steps=0)
    groups = [{"params": [getattr(gm, a)], "lr": 0.0, "name": n} for a, n in zip(ATTRS, NAMES)]
    opt = torch.optim.Adam(groups, eps=1e-15)
    opt.load_state_dict(src.adam_state_dict())
    back = FlatSurfelModel.from_gaussian_model(gm, opt)
    assert _bits(back.exp_avg, src.exp_avg) and _bits(back.exp_avg_sq, src.exp_avg_sq)
    assert int(back.device_step) == int(src.device_step) and back.lrs == src.lrs


def test_adam_import_refuses_different_steps():
    gm = _GaussianModel(6)
    opt = _torch_adam(gm, steps=2)
    gm._opacity.grad = torch.ones(6, 1)
    for a in ATTRS:
        if a != "_opacity":
            getattr(gm, a).grad = None
    opt.step()
    with pytest.raises(ValueError, match="steps differ"):
        FlatSurfelModel.from_gaussian_model(gm, opt)


# ---- PLY ---------------------------------------------------------------------------------------------------------------------
def _reference_bytes(m):
    """What gaussian_model.py save_ply writes, built as it builds it: a numpy structured array of the attribute list."""
    xyz = m._xyz.detach().numpy()
    f_dc = m._features_dc.detach().transpose(1, 2).flatten(start_dim=1).contiguous().numpy()
    f_rest = m._features_rest.detach().transpose(1, 2).flatten(start_dim=1).contiguous().numpy()
    attributes = np.concatenate((xyz, np.zeros_like(xyz), f_dc, f_rest, m._opacity.detach().numpy(),
                                 m._scaling.detach().numpy(), m._rotation.detach().numpy()), axis=1)
    names = ["x", "y", "z", "nx", "ny", "nz"] + [f"f_dc_{i}" for i in range(3)] + [f"f_rest_{i}" for i in range(45)] + \
        ["opacity", "scale_0", "scale_1", "rot_0", "rot_1", "rot_2", "rot_3"]
    elements = np.empty(xyz.shape[0], dtype=[(n, "<f4") for n in names])
    elements[:] = list(map(tuple, attributes))
    return names, elements.tobytes()


@pytest.mark.parametrize("P", [0, 1, 37])
def test_save_ply_bytes_are_2dgs_layout(P, tmp_path):
    m = _store(P, seed=10)
    path = tmp_path / "s.ply"
    m.save_ply(path, regist_feat=False)
    data = path.read_bytes()
    names, body = _reference_bytes(m)
    head, sep, rest = data.partition(b"end_header\n")
    lines = head.decode("ascii").split("\n")
    assert lines[0] == "ply" and lines[1] == "format binary_little_endian 1.0" and lines[2] == f"element vertex {P}"
    assert lines[3:-1] == [f"property float {n}" for n in names] and lines[-1] == ""
    assert sep and rest == body


def test_regist_feat_is_extra_properties_after_the_2dgs_ones(tmp_path):
    m = _store(11, seed=11)
    path = tmp_path / "s.ply"
    m.save_ply(path)
    v = ply.read_vertices(path)
    assert list(v.dtype.names) == ply.attribute_names(True)
    names, body = _reference_bytes(m)
    assert _bits(torch.from_numpy(np.stack([v[n] for n in names], 1).copy()),
                 torch.from_numpy(np.frombuffer(body, "<f4").reshape(11, -1).copy()))
    assert np.array_equal(np.stack([v[f"regist_feat_{i}"] for i in range(16)], 1), m._regist_feat.detach().numpy())


@pytest.mark.parametrize("regist", [False, True])
def test_ply_round_trip_bit_for_bit(regist, tmp_path):
    src = _store(29, regist, seed=12)
    path = tmp_path / "s.ply"
    src.save_ply(path)
    dst = _store(4, regist, seed=13)
    dst.load_ply(path)
    assert dst.P == 29 and dst.active_sh_degree == dst.max_sh_degree == 3 and _bits(dst.flat, src.flat)
    assert not dst.exp_avg.any() and int(dst.device_step) == 0
    _views_of_flat(dst)
    same = _store(29, regist, seed=14)
    ptr = same.flat.data_ptr()
    same.load_ply(path)
    assert same.flat.data_ptr() == ptr and _bits(same.flat, src.flat)


def test_reader_takes_permuted_properties_and_other_types(tmp_path):
    m = _store(17, regist=False, seed=15)
    names = ply.attribute_names()
    vals = {n: c for n, c in zip(names, np.frombuffer(_reference_bytes(m)[1], "<f4").reshape(17, -1).T)}
    perm = list(np.random.default_rng(0).permutation(names)) + ["red"]
    dtype = [(n, "<f4") for n in perm[:-1]] + [("red", "u1")]
    el = np.empty(17, dtype=dtype)
    for n in perm[:-1]:
        el[n] = vals[n]
    el["red"] = 200
    head = ["ply", "format binary_little_endian 1.0", "comment written elsewhere", "element vertex 17"]
    head += [f"property float {n}" for n in perm[:-1]] + ["property uchar red", "end_header"]
    path = tmp_path / "p.ply"
    path.write_bytes(("\n".join(head) + "\n").encode() + el.tobytes())
    got = ply.read_surfels(path)
    for n, p in zip(NAMES, m.flat_params()):
        assert _bits(got[n], p.detach()), n
    assert "regist_feat" not in got


def test_reader_reads_vertices_before_a_face_element(tmp_path):
    m = _store(6, regist=False, seed=16)
    path = tmp_path / "f.ply"
    m.save_ply(path)
    data = path.read_bytes().replace(b"end_header\n", b"element face 1\nproperty list uchar int vertex_indices\n"
                                                       b"end_header\n")
    path.write_bytes(data + bytes([3]) + np.array([0, 1, 2], "<i4").tobytes())
    got = ply.read_surfels(path)
    for n, p in zip(NAMES, m.flat_params()):
        assert _bits(got[n], p.detach()), n
    head = ply.header(ply.attribute_names(), 0).replace(b"end_header", b"property list uchar int idx\nend_header")
    path.write_bytes(head)
    with pytest.raises(ValueError, match="vertex element has list properties"):
        ply.read_vertices(path)


@pytest.mark.parametrize("fmt", ["ascii", "binary_big_endian"])
def test_reader_rejects_other_formats(fmt, tmp_path):
    path = tmp_path / "b.ply"
    path.write_bytes(f"ply\nformat {fmt} 1.0\nelement vertex 0\nproperty float x\nend_header\n".encode())
    with pytest.raises(ValueError, match="only binary_little_endian"):
        ply.read_vertices(path)


def test_reader_checks_the_sh_count(tmp_path):
    names = [n for n in ply.attribute_names() if n != "f_rest_44"]
    path = tmp_path / "c.ply"
    path.write_bytes(ply.header(names, 2) + np.zeros((2, len(names)), "<f4").tobytes())
    with pytest.raises(ValueError, match="44 f_rest properties"):
        ply.read_surfels(path)
    path.write_bytes(ply.header(ply.attribute_names(), 3) + np.zeros((2, 62), "<f4").tobytes())
    with pytest.raises(ValueError, match="truncated"):
        ply.read_surfels(path)
