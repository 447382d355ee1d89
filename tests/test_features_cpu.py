"""CPU tests of the feature-channel path: argument validation through the C ABI and the Python binding (no device
needed -- every bad call is rejected before any CUDA work), and the float64 model of the feature planes and their backward
(tests/feature_model.py) against the C oracle's colour planes and against finite differences."""
import ctypes as C

import numpy as np
import pytest
import torch


def _frame(P=10, W=64, H=64):
    from vidu4d_b200 import _capi
    return _capi.SrFrame(P, 0, 0, W, H, 0.5, 0.5, 1.0, 0, 0, 0)


def _fwd_args(F, bg_channels, features=True):
    """sr_forward arguments with dummy (never dereferenced) pointers."""
    from vidu4d_b200 import _capi
    fr, bt = _frame(), _capi.SrBatch(1, 0, 0, 0, 0, 0, 0, 0)
    d = 4096
    return [C.byref(fr), C.byref(bt), d, bg_channels, d, None, d, d, d, d, d if features else None, F, 0, d, d, d,
            d, 0, d, 0, d, d, d, d, d, 1024, d, None, None]


def _bwd_args(F, bg_channels, features=True):
    from vidu4d_b200 import _capi
    fr, bt = _frame(), _capi.SrBatch(1, 0, 0, 0, 0, 0, 0, 0)
    d = 4096
    return [C.byref(fr), C.byref(bt), d, bg_channels, d, None, d, d, d, d if features else None, F, 0, d, d, d, d,
            d, 0, d, 0, d, None, None, d, d, d, 1024] + [d] * 9 + [None]


@pytest.mark.parametrize("entry", ["forward", "backward"])
def test_sr_forward_backward_reject_bad_feature_arguments(built, entry):
    from vidu4d_b200 import _capi
    lib = _capi.load()
    fn, mk = (lib.sr_forward, _fwd_args) if entry == "forward" else (lib.sr_backward, _bwd_args)
    assert fn(*mk(33, 36)) == -1 and b"F must be in [1, 32]" in lib.sr_last_error()
    assert fn(*mk(-1, 3)) == -1 and b"F must be in [1, 32]" in lib.sr_last_error()
    assert fn(*mk(0, 3)) == -1 and b"got 0" in lib.sr_last_error()           # F = 0 with a features pointer
    assert fn(*mk(0, 25, features=False)) == -1 and b"3 channels" in lib.sr_last_error()
    assert fn(*mk(4, 5)) == -1 and b"3 or 3+F = 7" in lib.sr_last_error()
    assert fn(*mk(4, 7, features=False)) == -1 and b"features pointer is NULL" in lib.sr_last_error()


def test_python_rejects_bad_features():
    from vidu4d_b200.rasterizer import _check_features
    bg3, bg = torch.zeros(3), torch.zeros(25)
    with pytest.raises(RuntimeError, match="1..32 channels"):
        _check_features(torch.zeros((10, 0)), 10, bg3)
    with pytest.raises(RuntimeError, match="1..32 channels"):
        _check_features(torch.zeros((10, 33)), 10, bg3)
    with pytest.raises(RuntimeError, match="dimensions"):
        _check_features(torch.zeros((11, 22)), 10, bg)
    with pytest.raises(RuntimeError, match="dimensions"):
        _check_features(torch.zeros((2, 10, 22)), 10, bg)              # per-frame features only in the batched entry
    with pytest.raises(RuntimeError, match="3 or 3\\+F = 25"):
        _check_features(torch.zeros((10, 22)), 10, torch.zeros(4))
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        _check_features(torch.zeros((10, 22)), 10, bg)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        _check_features(torch.zeros((2, 10, 22)), 10, bg3, batched=True)
    with pytest.raises(RuntimeError, match="must be a tensor"):
        _check_features(np.zeros((10, 22)), 10, bg3)


def test_python_entry_points_validate_before_the_device(built):
    from vidu4d_b200 import rasterizer as RZ
    x = torch.zeros((10, 3))
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        RZ._C.rasterize_gaussians_features(torch.zeros(3), x, torch.empty(0), torch.zeros((10, 1)), torch.zeros((10, 2)),
                                           torch.zeros((10, 4)), 1.0, torch.empty(0), torch.eye(4), torch.eye(4), 0.5, 0.5,
                                           64, 64, torch.zeros((10, 1, 3)), 0, torch.zeros(3), False, False,
                                           torch.zeros((10, 22)))
    rs = RZ.GaussianRasterizationSettings(64, 64, 0.5, 0.5, torch.zeros(3), 1.0, torch.eye(4), torch.eye(4), 0, torch.zeros(3),
                                          False, False)
    with pytest.raises(RuntimeError, match="1..32 channels"):
        RZ.GaussianRasterizer(rs).forward_features(x, x, torch.zeros((10, 1)), torch.zeros((10, 33)),
                                                   shs=torch.zeros((10, 1, 3)), scales=torch.zeros((10, 2)),
                                                   rotations=torch.zeros((10, 4)))


# ------------------------------------------------------------------------------------- float64 model (tests/feature_model.py)
@pytest.mark.parametrize("name", ["id_deg3_64", "precomp_init_70x50", "rigid_bg_96x64"])
def test_model_features_equal_to_colour_reproduce_colour_planes(built, name):
    """The model's feature walk over an oracle forward state reproduces the oracle's colour planes (to 1e-4 of their
    max: the oracle is fp32) when the features are the colours, with the background's 3 values (3+F background) or a
    black one (3-value background)."""
    from oracle import surfel_oracle as so
    from .conftest import load_golden, oracle_forward_from_golden
    from .feature_model import planes
    g = load_golden(name)
    st = oracle_forward_from_golden(g)
    pre = int(g["in_meta"][4])
    cols = g["in_colors_precomp"].reshape(-1, 3) if pre else st.rgb
    bg = g["in_bg"].reshape(3)
    m = planes(st, cols, np.concatenate([bg, bg]))
    assert np.abs(m - st.color).max() <= 1e-4 * np.abs(st.color).max()
    st0 = so.forward(g["in_means3D"], g["in_opacities"], g["in_scales"], g["in_rotations"],
                     shs=None if pre else g["in_shs"], colors_precomp=g["in_colors_precomp"] if pre else None,
                     sh_degree=int(g["in_meta"][3]), W=st.W, H=st.H, tanfovx=float(g["in_tanfov"][0]),
                     tanfovy=float(g["in_tanfov"][1]), bg=(0, 0, 0), viewmatrix=g["in_viewmatrix"],
                     projmatrix=g["in_projmatrix"], campos=g["in_campos"])
    m0 = planes(st, cols, bg)
    assert np.abs(m0 - st0.color).max() <= 1e-4 * np.abs(st0.color).max()


def scene_1k():
    """1 K surfels, 64x64, one camera in front of an object-centric cloud: (scene, oracle forward state)."""
    from oracle import surfel_oracle as so
    from vidu4d_b200.synthetic import object_scene, projection_matrix
    sc = object_scene(1000, seed=21)
    vm = np.eye(4, dtype=np.float32)
    st = so.forward(sc.means3D, sc.opacities, sc.scales, sc.rotations, shs=sc.shs, sh_degree=3, W=64, H=64, tanfovx=0.5,
                    tanfovy=0.5, bg=(0.1, 0.2, 0.3), viewmatrix=vm,
                    projmatrix=(vm.astype(np.float64) @ projection_matrix(0.5, 0.5)).astype(np.float32), campos=(0, 0, 0))
    return sc, st


def test_model_feature_backward_matches_float64_finite_differences(built):
    from .feature_model import backward, planes
    sc, st = scene_1k()
    P, F, H, W = 1000, 5, 64, 64
    rng = np.random.default_rng(22)
    feat = rng.standard_normal((P, F))
    bg = np.concatenate([[0.1, 0.2, 0.3], rng.random(F)])
    G = rng.standard_normal((F, H, W))
    dfeat, dop = backward(st, feat, bg, G)
    opac = st.normal_opacity[:, 3].astype(np.float64)
    loss = lambda fe, op: float((G * planes(st, fe, bg, op)).sum())  # noqa: E731
    vis = np.nonzero(st.radii > 0)[0]
    assert np.abs(dfeat).max() > 0 and np.abs(dop).max() > 0
    # dL/dfeatures: the planes are linear in the features
    for sid in rng.choice(vis, 4, replace=False):
        for c in (0, F - 1):
            e = np.zeros((P, F)); e[sid, c] = 1.0
            fd = loss(feat + e, opac) - loss(feat, opac)
            assert abs(dfeat[sid, c] - fd) <= 1e-9 * np.abs(dfeat).max(), (sid, c)
    # the alpha term, through the opacities (surfels whose alpha never reaches the 0.99 clamp)
    cand = [i for i in vis if opac[i] < 0.9]
    for sid in sorted(cand, key=lambda i: -abs(dop[i]))[:6]:
        h = 1e-6
        op_p, op_m = opac.copy(), opac.copy()
        op_p[sid] += h; op_m[sid] -= h
        fd = (loss(feat, op_p) - loss(feat, op_m)) / (2 * h)
        assert abs(dop[sid] - fd) <= 1e-6 * np.abs(dop).max(), (sid, dop[sid], fd)
