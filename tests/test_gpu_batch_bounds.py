"""The batched rasterizer backward under the oracle's rounding-error bound, for every case of the pairwise covering array
of tests/batch_options.py: per-frame or shared positions, rotations, scales and (M,P,1) opacities; SH shared or per
frame at three degrees, or colors_precomp shared or per frame; no features, F = 7 or 22 shared, F = 32 per frame, their
planes' gradient as dL_dout_color's tail or a separate dL_dout_features, a 3 or 3+F background; scalar tangents or a
camera table with zero or non-zero principal-point offsets; sum_shared; the default or the deterministic backward; a
device grad_scale (also the features_grad_scale) of none, -1.7 or 0; want_transmat; outs= in place.

Each case runs P = 6,000 surfels of vidu4d_b200.synthetic.object_scene on a 104 x 72 image (7 x 5 tiles, the last row
and column partial).  Frame 0 takes the shared values; frame f of a per-frame input is perturbed by f times a fixed
noise.  Per frame the forward is decoded and the oracle composited from its records (test_gpu_grad_bounds._oracle_frame,
which holds the records to the preprocess model for that frame's own inputs and camera row; with features,
test_gpu_feature_bounds._oracle_fwd and one oracle per group of 3 channels), and the forward planes are held to their
bound.  Upstream gradients are zeroed on knife-edge pixels, then every returned tensor is held element by element to
|gpu - oracle| <= K u B' + FLOOR, B' composed by batch_options.frame_reference from:

  * the reductions into the accumulator: default backward, one add per tile touched and per pair past the pair buffer
    (test_gpu_grad_bounds._fallback_pairs); deterministic backward, one per tile touched (test_gpu_deterministic);
  * the chain's roundings, CHAIN;
  * features: the feature pass's adds, n_chunks m_feat and SLACK = 8 (default) or m_feat and SLACK = F (deterministic),
    as test_gpu_feature_bounds / test_gpu_deterministic derive them;
  * grad_scale: the kernels multiply every upstream value by the device scalar, and the oracle is fed fl32(dout * gs).
    nvcc may contract that product into a later FMA, which skips its rounding, so each upstream value may differ from
    the oracle's by u |dout * gs|: every term of every accumulator is linear in one upstream value, so this adds one u
    times the accumulator's absolute sum (GS = 1 in the adds).  gs = 0 must give exact zeros in every tensor; the case
    then runs again without a scale so its other options still meet the oracle;
  * offsets: camera_model's offset chain and bound sums on the combined colour and feature accumulator;
  * summed gradients (sum_shared with M > 1, inputs whose frame stride is 0): the sum of the frames' oracles, plus
    M u sum_f |oracle_f| for the per-surfel kernel's sequential frame sum.  Per-frame inputs keep their leading M.

Each case asserts from the GPU's own buffers that it reached its combination: every per-frame input changes frame
M-1's records (held to the preprocess model with that one input taken from frame 0, they fail), the deterministic or
default kernels ran (profiler names), each plane that receives an upstream gradient has a non-zero one, and with
offsets the last frame's object is cut by the right image edge.  Each case prints its knife pixels and per tensor the
largest err / tolerance, and keeps its knife mask within 4 n + 8 of the count measured on an H100 (KNIFE_MEASURED).
"""
import numpy as np
import pytest
import torch

from . import batch_options as BO
from .test_gpu_grad_bounds import CHAIN, FLOOR, GRADS, K, U, _check_forward, _check_grad, _fallback_pairs, _np, _oracle_frame

pytestmark = pytest.mark.gpu

P, W, H = 6000, 104, 72
FC = 8                   # SR_FEAT_CHUNK
ALL = GRADS + ("dL_dfeatures",)
ACC_LEVEL = ("dL_dcolors", "dL_dopacity")
# the input each gradient belongs to, and its per-surfel shape
INPUT = {"dL_dmeans3D": ("means3D", (3,)), "dL_dcolors": ("colors", (3,)), "dL_dopacity": ("opacities", (1,)),
         "dL_dsh": ("sh", None), "dL_dscales": ("scales", (2,)), "dL_drotations": ("rotations", (4,)),
         "dL_dfeatures": ("features", None)}
OUTS = ("dL_dmeans3D", "dL_dsh", "dL_dopacity", "dL_dscales", "dL_drotations", "dL_dcolors")
DEFAULT_KERNELS = {"composite_bwd", "surfel_bwd"}
DET_KERNELS = {"det_zero", "composite_bwd_det", "det_gather", "surfel_bwd"}

# Masked (knife-edge) pixels per case over all its frames, measured on an H100; a case may mask at most 4 n + 8.
KNIFE_MEASURED = {
    "M1-mea-sca-sh_per_frame_d3k16-F7_separate_bg3+F-table-sum-det-gs-1.7-outs": 0,
    "M1-rot-opa-precomp_shared-F32pf_tail_bg3-table_offsets-nosum-def-gs0.0-tm": 0,
    "M1-sh_shared_d1k16-scalar-nosum-def-gsNone-outs": 1,
    "M1-mea-rot-sca-opa-precomp_per_frame-F22_separate_bg3+F-table-nosum-det-gsNone-tm": 0,
    "M1-mea-rot-sca-opa-sh_per_frame_d0k1-table_offsets-sum-det-gs0.0-tm": 0,
    "M2-rot-sh_shared_d0k1-F22_tail_bg3+F-scalar-sum-det-gs-1.7-tm-outs": 0,
    "M2-mea-sca-opa-sh_shared_d3k16-F32pf_tail_bg3-scalar-sum-def-gs0.0-outs": 1,
    "M2-mea-precomp_shared-table-sum-def-gs-1.7": 0,
    "M2-rot-sca-opa-sh_per_frame_d1k16-F7_separate_bg3-table_offsets-nosum-def-gsNone-outs": 1,
    "M2-precomp_per_frame-F7_separate_bg3+F-scalar-sum-def-gs0.0-tm": 2,
    "M5-mea-sca-opa-sh_shared_d1k16-F32pf_separate_bg3+F-table_offsets-sum-det-gs-1.7-tm-outs": 3,
    "M5-rot-sh_per_frame_d0k1-F22_tail_bg3-table-nosum-det-gs-1.7-outs": 3,
    "M5-rot-sh_shared_d3k16-table-nosum-def-gs0.0-tm": 1,
    "M5-rot-precomp_shared-F32pf_separate_bg3+F-scalar-sum-det-gsNone-tm-outs": 3,
    "M5-mea-sca-precomp_per_frame-F22_tail_bg3+F-table_offsets-sum-def-gs0.0-outs": 1,
    "M5-mea-opa-sh_shared_d0k1-F7_tail_bg3+F-table-nosum-def-gsNone-tm": 3,
    "M2-mea-opa-precomp_per_frame-F32pf_tail_bg3-table-sum-def-gs-1.7-outs": 1,
    "M1-opa-precomp_per_frame-table-sum-det-gsNone-tm-outs": 0,
    "M5-sca-precomp_shared-F22_separate_bg3-scalar-sum-det-gs-1.7-tm-outs": 4,
    "M1-rot-opa-precomp_shared-F7_tail_bg3-table-nosum-det-gs-1.7": 0,
    "M5-mea-rot-sca-sh_per_frame_d1k16-F22_tail_bg3-scalar-nosum-det-gs0.0-tm": 2,
    "M1-rot-sca-opa-sh_per_frame_d0k1-F32pf_separate_bg3+F-table_offsets-nosum-det-gsNone-tm-outs": 0,
    "M1-sca-opa-sh_per_frame_d1k16-F7_separate_bg3+F-table-sum-det-gsNone-tm": 0,
    "M5-mea-sca-opa-sh_shared_d3k16-F22_tail_bg3-table_offsets-nosum-def-gsNone-tm": 2,
    "M3-mea-rot-sh_shared_d3k16-F22_separate_bg3-table_offsets-sum-def-gs1.7": 0,
    "M8-mea-rot-sh_shared_d3k16-F22_separate_bg3-table_offsets-sum-def-gs1.7": 3,
    "M3-mea-rot-sh_shared_d3k16-F22_separate_bg3-table_offsets-sum-det-gs1.7": 0,
    "M8-mea-rot-sh_shared_d3k16-F22_separate_bg3-table_offsets-sum-det-gs1.7": 3,
}


@pytest.fixture(scope="module")
def dev(built):
    from vidu4d_b200 import _capi
    _capi.load()
    return torch.device("cuda:0")


def _rows(M, offsets):
    """Camera-table rows (tan_x, tan_y, cx_off, cy_off): both tangents differ between frames; with offsets, non-integer
    ones of either sign, and the last frame's principal point pushed 0.45 W right, so its object crosses the edge."""
    rows = []
    for f in range(M):
        s = -1.0 if f % 2 else 1.0
        off = (s * (0.08 * W + 0.375), -s * (0.08 * H + 0.3125)) if offsets else (0.0, 0.0)
        if offsets and f == M - 1:
            off = (0.45 * W + 0.25, -0.1 * H - 0.125)
        rows.append((0.5 + 0.02 * f, 0.45 - 0.015 * f) + off)
    return np.array(rows, np.float32)


def _inputs(c, seed):
    """numpy inputs of a case: each per-surfel input (P,...) shared or (M,P,...) per frame."""
    from vidu4d_b200.synthetic import object_scene
    M = c["M"]
    sc = object_scene(P, seed=seed, center=(0.0, 0.0, 0.0))
    rng = np.random.default_rng(seed)
    f32 = lambda a: np.ascontiguousarray(a, np.float32)  # noqa: E731

    def per(base, step, fix=lambda a: a):
        noise = rng.standard_normal(base.shape)
        return f32(np.stack([fix(base + step * f * noise) for f in range(M)]))

    def pick(name, base, step, fix=lambda a: a):
        return per(base, step, fix) if c[name] == "per_frame" else f32(base)

    def unit(q):
        return q / np.linalg.norm(q, axis=-1, keepdims=True)
    inp = dict(means3D=pick("means3D", sc.means3D, 0.002), rotations=pick("rotations", sc.rotations, 0.02, unit),
               scales=pick("scales", sc.scales, 0.05 * sc.scales, np.abs),
               opacities=pick("opacities", sc.opacities.reshape(P, 1), 0.05, lambda a: np.clip(a, 0.02, 0.98)))
    src, pf = c["colour"].split("_", 1)
    if src == "sh":
        deg, ncoef = c["sh"]
        base = sc.shs[:, :ncoef]
        inp["sh"] = per(base, 0.05) if pf == "per_frame" else f32(base)
        inp["deg"], inp["colors"] = deg, None
    else:
        base = rng.uniform(0.0, 1.0, (P, 3))
        inp["colors"] = per(base, 0.05) if pf == "per_frame" else f32(base)
        inp["deg"], inp["sh"] = 0, None
    F = abs(c["features"])
    inp["F"] = F
    inp["features"] = None
    bg = [0.2, 0.1, 0.4]
    if F:
        base = rng.standard_normal((P, F))
        inp["features"] = per(base, 0.1) if c["features"] < 0 else f32(base)
        if c["background"] == "3+F":
            bg += list(rng.uniform(0.2, 1.0, F))
    inp["bg"] = f32(bg)
    return inp


def _frame_of(inp, name, f):
    a = inp[name]
    if a is None:
        return None
    shared_ndim = 3 if name == "sh" else 2
    return a[f] if a.ndim == shared_ndim + 1 else a


def _kernels(fn):
    from vidu4d_b200 import _capi
    _capi.set_profiling(True)
    try:
        _capi.get_profile()
        out = fn()
        return out, set(_capi.get_profile())
    finally:
        _capi.set_profiling(False)


def _summed(c, key, M, sum_shared):
    """Whether the backward returns key summed over the frames: sum_shared, M > 1 and the input's frame stride 0."""
    if key in ("dL_dmeans2D", "dL_dtransMat") or not sum_shared or M == 1:
        return False
    name = INPUT[key][0]
    if name == "colors":
        return c["colour"] != "precomp_per_frame"             # SH or shared colours: no per-frame colour input
    if name == "sh":
        return c["colour"] != "sh_per_frame"
    if name == "features":
        return c["features"] > 0
    return c[name] == "shared"


def _shape(c, key, M, P, ncoef, F, sum_shared):
    tail = {"dL_dmeans2D": (3,), "dL_dtransMat": (9,), "dL_dsh": (ncoef, 3), "dL_dfeatures": (F,)}.get(key)
    tail = tail if tail is not None else INPUT[key][1]
    return ((P,) if _summed(c, key, M, sum_shared) else (M, P)) + tail


def _records_depend_on(c, inp, frame, dec, name):
    """Frame M-1's records, held to the preprocess model with one per-frame input taken from frame 0, must fail."""
    from . import preprocess_bounds as pb
    M = c["M"]
    src = "sh" if inp["sh"] is not None else "precomp"
    for k in ("means3D", "rotations", "scales", "opacities", "sh", "colors"):
        a = inp[k]
        if a is None or a.ndim != (4 if k == "sh" else 3):
            continue
        assert not np.array_equal(a[0], a[M - 1]), (name, k)
        wrong = {n: _frame_of(inp, n, M - 1) for n in ("means3D", "rotations", "scales", "opacities", "sh", "colors")}
        wrong[k] = a[0]
        x = dict(means3D=wrong["means3D"], rotations=wrong["rotations"], scales=wrong["scales"],
                 opacities=wrong["opacities"], shs=wrong["sh"], colors_precomp=wrong["colors"], deg=inp["deg"])
        with pytest.raises(AssertionError):
            pb.check_records(dec, x, frame["cam"], src, f"{name} frame {M - 1} with frame 0's {k}")


# ------------------------------------------------------------------------------------------------ the oracle side
def _forward_frames(name, c, inp, out, cams, rows, W_, H_):
    """Per frame: decode, the oracle composited from the records (records checked against that frame's inputs and
    camera row), the forward planes under their bound."""
    from vidu4d_b200 import debug as dbg
    from . import preprocess_bounds as pb
    from . import test_gpu_feature_bounds as FB
    M, F, P = c["M"], inp["F"], inp["means3D"].shape[-2]
    nr, color, allmap, radii, gb, bb, ib = out[:7]
    planes = None if not F else (color[:, 3:] if c["planes"] == "tail" else out[7])
    vms, pms, cps = (_np(x) for x in cams)
    frames = []
    for f in range(M):
        dec = dbg.decode(gb.view(M, -1)[f], bb.view(M, -1)[f], ib.view(M, -1)[f], P, W_, H_, nr[f])
        dec["radii"] = _np(radii[f])
        dec["num_rendered"] = nr[f]
        tan = (float(rows[f][0]), float(rows[f][1]))
        off = None if c["camera"] != "table_offsets" else (float(rows[f][2]), float(rows[f][3]))
        fi = {k: _frame_of(inp, k, f) for k in ("means3D", "rotations", "scales", "opacities", "sh", "colors", "features")}
        tag = f"{name} frame {f}"
        fr = dict(dec=dec, off=off, F=F, fi=fi, cam=pb.camera(vms[f], cps[f], W_, H_, tan, off))
        if F:
            meta = np.array([P, W_, H_, inp["deg"], int(fi["colors"] is not None)])
            finp = dict(meta=meta, tanfov=np.float32(tan), opacities=fi["opacities"], scales=fi["scales"],
                        rotations=fi["rotations"], shs=fi["sh"], colors_precomp=fi["colors"], bg=inp["bg"][:3],
                        viewmatrix=vms[f], projmatrix=pms[f], campos=cps[f])
            c3f = torch.cat([color[f, :3], planes[f]], 0)
            o = FB._oracle_fwd(tag, dec, finp, fi["means3D"], fi["features"], inp["bg"][3:] if inp["bg"].size > 3 else None,
                               c3f, allmap[f], off=off)
            fr.update(st=o["st"], ext=o["ext"], groups=o["groups"], fwd=o["fwd"])
        else:
            st, ext = _oracle_frame(dec, P, W_, H_, fi["means3D"], fi["opacities"], fi["scales"], fi["rotations"], fi["sh"],
                                    fi["colors"], inp["deg"], inp["bg"][:3], vms[f], pms[f], cps[f], tan, off=off, name=tag)
            fr.update(st=st, ext=ext, groups=[], fwd=_check_forward(tag, st, ext, _np(color[f]), _np(allmap[f]), dec, W_, H_))
        frames.append(fr)
    return frames


def _oracle_backward(frames, dLc, dLo, dLf, gs, fgs, det):
    """Each frame's oracle reference and tolerance for upstream gradients already masked; gs / fgs: the scales the
    kernels apply to the colour and allmap planes / to the feature planes (None = 1)."""
    from oracle import surfel_oracle as so
    from . import test_gpu_feature_bounds as FB

    def scaled(a, s):
        return a if s is None else (a.astype(np.float64) * np.float64(np.float32(s))).astype(np.float32)
    for f, fr in enumerate(frames):
        st, dec, F = fr["st"], fr["dec"], fr["F"]
        adds = _np(dec["tiles_touched"]).astype(np.float64) + CHAIN + (0 if gs is None and fgs is None else 1)
        if not det:
            adds = adds + _fallback_pairs(dec, st.P)
        if F:
            FB._oracle_bwd(fr, scaled(dLc[f], gs), scaled(dLo[f], gs), scaled(dLf[f], fgs))
            m = FB._pair_counts(dec, st.P)
            fr["m"] = m + (0 if fgs is None else 1)         # the features_grad_scale term, see the docstring
            adds = adds + (m + F if det else FB._chunks(F)[0] * m + FC)
        else:
            fr["og_c"] = so.backward(st, scaled(dLc[f], gs), scaled(dLo[f], gs), bounds=True)
            fr["og_g"] = []
        fr["ref"], fr["tol"] = BO.frame_reference(st, fr["og_c"], fr["og_g"], adds, fr["off"])


def _check_grads(name, c, frames, gr, sum_shared, report):
    """Every returned tensor against the oracle: per frame (accumulator level first, then dL/dSH from the GPU's own
    dL/dcolors, then the rest), or summed over the frames."""
    from oracle import surfel_oracle as so
    from . import test_gpu_feature_bounds as FB
    M = len(frames)
    keys = [k for k in GRADS if gr.get(k) is not None]
    ordered = [k for k in ACC_LEVEL if k in keys] + [k for k in keys if k not in ACC_LEVEL]
    for f, fr in enumerate(frames):
        st = fr["st"]
        for k in ordered:
            if _summed(c, k, M, sum_shared):
                continue
            _check_grad(f"{name} frame {f}", k, gr[k][f], fr["ref"][k], fr["tol"][k], report)
            if k == "dL_dcolors" and fr["ref"]["dL_dsh"].size and not _summed(c, "dL_dsh", M, sum_shared):
                acc = np.zeros((st.P, so.NACC), np.float32)
                acc[:, so.ACC_COLOR:so.ACC_COLOR + 3] = _np(gr["dL_dcolors"][f]).reshape(st.P, 3)
                ctol = K * U * CHAIN * so.chain_bound(st, np.abs(acc.astype(np.float64)))["dL_dsh"]
                _check_grad(f"{name} frame {f} [per-surfel backward, GPU accumulators]", "dL_dsh", gr["dL_dsh"][f],
                            so.chain(st, acc)["dL_dsh"], ctol, {})
    for k in ordered:
        if _summed(c, k, M, sum_shared):
            ref = sum(fr["ref"][k].astype(np.float64) for fr in frames)
            tol = sum(fr["tol"][k] for fr in frames) + M * U * sum(np.abs(fr["ref"][k].astype(np.float64)) for fr in frames)
            _check_grad(f"{name} summed", k, gr[k], ref, tol, report)
    if frames[0]["F"]:
        if _summed(c, "dL_dfeatures", M, sum_shared):
            ref, tol = FB._dfeat_ref(frames, sum(fr["m"] for fr in frames))
            _check_grad(f"{name} summed [feature backward]", "dL_dfeatures", gr["dL_dfeatures"], ref, tol, report)
        else:
            for f, fr in enumerate(frames):
                ref, tol = FB._dfeat_ref([fr], fr["m"])
                _check_grad(f"{name} frame {f} [feature backward]", "dL_dfeatures", gr["dL_dfeatures"][f], ref, tol, report)


def _autograd_backward(c, ti, bg, cams, tan, table, deg, out, dcol, dlo):
    """The same forward through rasterize_gaussians_batch with leaf tensors (its planes, radii and allmap bit for bit the
    _C forward's), then autograd's backward from (dcol, dlo): every input's p.grad, in the input's own shape, under the
    names of the _C backward's tensors and viewed as that backward returns them; and the kernels the backward ran."""
    from vidu4d_b200.rasterizer import BatchRasterizationSettings, rasterize_gaussians_batch
    M, F = c["M"], abs(c["features"])
    names = {"means3D": "dL_dmeans3D", "sh": "dL_dsh", "colors": "dL_dcolors", "opacities": "dL_dopacity",
             "scales": "dL_dscales", "rotations": "dL_drotations", "features": "dL_dfeatures"}
    leaf = {k: ti[k].clone().requires_grad_(True) for k in names if ti[k] is not None}
    m2d = torch.zeros((M, P, 3), device=bg.device, requires_grad=True)
    rs = BatchRasterizationSettings(H, W, tan[0], tan[1], bg, 1.0, cams[0], cams[1], deg, cams[2], intrinsics=table)
    color, radii, allmap = rasterize_gaussians_batch(leaf["means3D"], m2d, leaf.get("sh"), leaf.get("colors"),
                                                     leaf["opacities"], leaf["scales"], leaf["rotations"], rs,
                                                     features=leaf.get("features"))
    assert torch.equal(color, out[1]) and torch.equal(radii, out[3]) and torch.equal(allmap, out[2])
    _, ran = _kernels(lambda: torch.autograd.backward([color, allmap], [dcol, dlo]))
    gr = {"dL_dmeans2D": m2d.grad, "dL_dtransMat": None}
    ncoef = 0 if ti["sh"] is None else ti["sh"].shape[-2]
    for k, g in names.items():
        if k not in leaf:
            continue
        x = leaf[k]
        assert x.grad is not None and x.grad.shape == x.shape, (k, None if x.grad is None else tuple(x.grad.shape))
        gr[g] = x.grad.view(_shape(c, g, M, P, ncoef, F, True))
    return gr, ran


# ------------------------------------------------------------------------------------------------ the cases
def _run_case(c, seed, dev, mode="direct"):
    """mode: "direct", the _C backward with grad_scale as the features_grad_scale too; "prescaled", as Stage 3 calls it
    (renderer._RasterLossBatch.backward): grad_scale for the colour and allmap planes, the feature planes scaled
    beforehand in fp32 and no features_grad_scale; "autograd", rasterize_gaussians_batch's backward into p.grad."""
    from vidu4d_b200 import rasterizer as R
    from .test_gpu_batch import _cams
    name = BO.case_id(c)
    M, F = c["M"], abs(c["features"])
    inp = _inputs(c, seed)
    T = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    e = torch.empty((0,), device=dev)
    cams = _cams(M, dev)
    rows = _rows(M, c["camera"] == "table_offsets")
    if c["camera"] == "scalar":
        rows[:] = (0.5, 0.5, 0.0, 0.0)
    table = None if c["camera"] == "scalar" else T(rows)
    tan = (0.5, 0.5) if table is None else (float("nan"), float("nan"))
    ti = {k: T(inp[k]) for k in ("means3D", "rotations", "scales", "opacities", "sh", "colors", "features")}
    bg = T(inp["bg"])
    kw = {} if not F else dict(features=ti["features"], concat=c["planes"] == "tail")
    out = R._C.rasterize_gaussians_batch(bg, ti["means3D"], e if ti["colors"] is None else ti["colors"], ti["opacities"],
                                         ti["scales"], ti["rotations"], 1.0, *cams[:2], tan[0], tan[1], H, W,
                                         e if ti["sh"] is None else ti["sh"], inp["deg"], cams[2], intrinsics=table, **kw)
    nr, color, allmap, radii = out[:4]
    assert min(nr) > 0, (name, nr)
    frames = _forward_frames(name, c, inp, out, cams, rows, W, H)
    if c["camera"] == "table_offsets":
        assert float(allmap[M - 1, 1, :, -1].max()) > 0.5, (name, "the last frame's object does not cross the right edge")
    if M > 1:
        _records_depend_on(c, inp, frames[M - 1], frames[M - 1]["dec"], name)

    # upstream gradients, zero on every frame's knife-edge pixels
    rng = np.random.default_rng(seed + 1)
    keep = np.stack([(~fr["ext"]["knife"]).astype(np.float32) for fr in frames])[:, None]
    dLc = rng.standard_normal((M, 3, H, W)).astype(np.float32) * keep
    dLo = (0.1 * rng.standard_normal((M, 8, H, W))).astype(np.float32) * keep
    dLf = rng.standard_normal((M, F, H, W)).astype(np.float32) * keep
    for what, a in (("colour", dLc), ("allmap", dLo), ("feature", dLf))[:3 if F else 2]:
        live = (a != 0).reshape(M, a.shape[1], -1).any(2).any(0)
        assert live.all(), (name, what, "planes without a non-zero upstream value", np.nonzero(~live)[0].tolist())
    dLf_in, fgs_of = dLf, (lambda gs: gs)
    if mode == "prescaled":
        assert F and c["grad_scale"] not in (None, 0.0)
        dLf_in = (dLf.astype(np.float64) * np.float64(np.float32(c["grad_scale"]))).astype(np.float32)
        fgs_of = lambda gs: None  # noqa: E731
    dcol = T(np.concatenate([dLc, dLf_in], 1) if F and c["planes"] == "tail" else dLc)
    ncoef = 0 if inp["sh"] is None else inp["sh"].shape[-2]
    sum_shared = c["sum_shared"]

    def backward(gs):
        outs = None
        if c["outs"]:
            outs = {k: torch.full(_shape(c, k, M, P, ncoef, F, sum_shared), float("nan"), device=dev) for k in OUTS
                    if not (k == "dL_dsh" and ncoef == 0)}
        g = None if gs is None else torch.tensor(gs, device=dev)
        bkw = dict(grad_scale=g, sum_shared=sum_shared, opacity_shared=c["opacities"] == "shared",
                   want_transmat=c["want_transmat"], outs=outs, intrinsics=table)
        if F:
            fg = fgs_of(gs)
            bkw.update(features=ti["features"], features_grad_scale=None if fg is None else torch.tensor(fg, device=dev),
                       dL_dout_features=None if c["planes"] == "tail" else T(dLf_in))
        R.set_deterministic(c["backward"] == "deterministic")
        try:
            if mode == "autograd":
                gr, ran = _autograd_backward(c, ti, bg, cams, tan, table, inp["deg"], out, dcol, T(dLo))
            else:
                gr, ran = _kernels(lambda: R._C.rasterize_gaussians_backward_batch(
                    bg, ti["means3D"], radii, e if ti["colors"] is None else ti["colors"], ti["scales"], ti["rotations"],
                    1.0, *cams[:2], tan[0], tan[1], dcol, T(dLo), e if ti["sh"] is None else ti["sh"], inp["deg"],
                    cams[2], *out[4:7], **bkw))
        finally:
            R.set_deterministic(False)
        want = (DET_KERNELS | ({"feature_bwd_det"} if F else set()) if c["backward"] == "deterministic"
                else DEFAULT_KERNELS | ({"feature_bwd"} if F else set()))
        assert ran == want, (name, sorted(ran))
        if mode == "autograd":
            return gr
        gr = dict(zip(ALL, gr))
        for k in ALL:
            if k == "dL_dfeatures" and not F:
                assert k not in gr, name
                continue
            if k == "dL_dtransMat" and not c["want_transmat"] and not (M == 1 and not sum_shared):
                assert gr[k] is None, name
                continue
            assert tuple(gr[k].shape) == _shape(c, k, M, P, ncoef, F, sum_shared), (name, k, tuple(gr[k].shape))
            if outs is not None and k in outs:
                assert gr[k].data_ptr() == outs[k].data_ptr(), (name, k, "not written in place")
        if sum_shared:
            # autograd's _reduce_like maps every gradient back to its input's shape
            for k in OUTS + (("dL_dfeatures",) if F else ()):
                x = ti[INPUT[k][0]]
                if x is not None:
                    assert tuple(R._reduce_like(gr[k], x).shape) == tuple(x.shape), (name, k)
        return gr

    gs = c["grad_scale"]
    if gs == 0.0:
        gr = backward(0.0)
        for k, v in gr.items():
            if v is not None:
                assert int(torch.count_nonzero(v)) == 0, (name, k, "grad_scale = 0 leaves non-zero elements")
        gs = None
    gr = backward(gs)
    _oracle_backward(frames, dLc, dLo, dLf_in, gs, fgs_of(gs), c["backward"] == "deterministic")
    report = {}
    _check_grads(name, c, frames, gr, sum_shared, report)
    knife = sum(int(fr["ext"]["knife"].sum()) for fr in frames)
    print(f"\n[{name}] knife pixels {knife}; forward err/bound {max(fr['fwd'] for fr in frames):.3g}; "
          + ", ".join(f"{k} {v:.3g}" for k, v in report.items()))
    assert knife <= 4 * KNIFE_MEASURED.get(name, 0) + 8, (name, "knife pixels", knife)
    return report


@pytest.mark.parametrize("i", range(len(BO.CASES)), ids=[BO.case_id(c) for c in BO.CASES])
def test_batch_option_case(i, dev):
    _run_case(BO.CASES[i], 7000 + i, dev)


# the options of Stage 3's backward call (renderer._RasterLossBatch.backward): per-frame positions and orientations, a
# camera table with offsets, F = 22 shared features with their planes' gradient separate and scaled beforehand (no
# features_grad_scale), sum_shared, the upstream scalar as grad_scale, shared opacities, no transMat
STAGE3 = dict(means3D="per_frame", rotations="per_frame", scales="shared", opacities="shared", colour="sh_shared",
              sh=(3, 16), features=22, planes="separate", background=3, camera="table_offsets", sum_shared=True,
              grad_scale=1.7, want_transmat=False, outs=False)


@pytest.mark.parametrize("M", [3, 8])
@pytest.mark.parametrize("backward", ["default", "deterministic"])
def test_stage3_options(M, backward, dev):
    c = dict(STAGE3, M=M, backward=backward)
    assert BO.valid(c) and set(c) == set(BO.NAMES)
    _run_case({n: c[n] for n in BO.NAMES}, 7100 + M, dev, mode="prescaled")


# per-frame (M,P,1) opacities and per-frame scales through rasterize_gaussians_batch into p.grad
AUTOGRAD = dict(M=3, means3D="per_frame", rotations="shared", scales="per_frame", opacities="per_frame",
                colour="sh_shared", sh=(3, 16), features=7, planes="tail", background="3+F", camera="table_offsets",
                sum_shared=True, grad_scale=None, want_transmat=False, outs=False)


@pytest.mark.parametrize("backward", ["default", "deterministic"])
def test_autograd_per_frame_opacities_and_scales(backward, dev):
    c = dict(AUTOGRAD, backward=backward)
    assert BO.valid(c) and set(c) == set(BO.NAMES)
    _run_case({n: c[n] for n in BO.NAMES}, 7200, dev, mode="autograd")



# ------------------------------------------------------------------------------------------------ Stage 3's own call
@pytest.mark.parametrize("backward", ["default", "deterministic"])
@pytest.mark.parametrize("case", ["65x33_m3"])
def test_stage3_loss_pass_call(case, backward, dev, monkeypatch):
    """render_loss_batch as Stage 3 calls it (test_gpu_loss_pass_bounds.py's cases, with per-frame positions and
    orientations): the spy on the rasterizer backward composites the oracle from the forward's own buffers and zeroes
    the captured planes on knife-edge pixels before the real backward runs; every gradient that backward returns is then
    held to the oracle fed those planes and the captured upstream scalar (grad_scale on colour and allmap; the feature
    planes arrive scaled, with no features_grad_scale).  Through autograd, viewspace_points.grad, the features' and the SH
    rows' .grad are that backward's tensors bit for bit, _xyz.grad their sum over the frames under the summed bound, and
    _opacity.grad / _scaling.grad the sigmoid / exp derivative times the oracle, three more roundings."""
    from vidu4d_b200 import debug as dbg, rasterizer as R
    from . import test_gpu_loss_pass_bounds as LP
    W_, H_, M, with_bk, with_vis = LP.CASES[case]
    det = backward == "deterministic"
    c = dict(STAGE3, M=M, backward=backward, grad_scale=float(LP.UP))
    c = {n: c[n] for n in BO.NAMES}
    name = f"stage3 {case} {backward}"
    st = {}

    def hook(a, k, out, pc):
        n_ = lambda t: t.detach().cpu().numpy()  # noqa: E731
        assert k.get("features_grad_scale") is None and k["sum_shared"] and k["opacity_shared"] and not k["want_transmat"]
        gb, bb, ib = a[16:19]
        nr = [int(dbg.decode(gb.view(M, -1)[f], bb.view(M, -1)[f], ib.view(M, -1)[f], P_, W_, H_, 0)["point_offsets"][-1])
              for f in range(M)]
        inp = dict(means3D=n_(a[1]), rotations=n_(a[5]), scales=n_(a[4]), opacities=n_(pc.get_opacity), sh=n_(a[13]),
                   colors=None, features=n_(k["features"]), deg=int(a[14]), F=F_, bg=n_(a[0]))
        rows = n_(k["intrinsics"])
        fwd = (nr, out["render"], out["allmap"], a[2], gb, bb, ib, out["features"])
        frames = _forward_frames(name, c, inp, fwd, (a[7], a[8], a[15]), rows, W_, H_)
        keep = torch.from_numpy(np.stack([(~fr["ext"]["knife"]).astype(np.float32) for fr in frames])).to(dev)[:, None]
        for t in (a[11], a[12], k["dL_dout_features"]):
            t.mul_(keep)
        st.update(frames=frames, planes=[n_(t) for t in (a[11], a[12], k["dL_dout_features"])],
                  gs=float(k["grad_scale"]), inp=inp)

    P_ = 20000 if M < 8 else 60000
    F_ = LP.F
    R.set_deterministic(det)
    try:
        out, _, spied = LP._run(case, W_, H_, M, with_bk, with_vis, dev, monkeypatch, hook=hook, per_frame=True)
    finally:
        R.set_deterministic(False)
    frames, (dLc, dLo, dLf), gs = st["frames"], st["planes"], st["gs"]
    assert gs == float(LP.UP)
    for what, x in (("colour", dLc), ("allmap", dLo[:, [1, 2, 3, 4, 6]]), ("feature", dLf[:, :21])):
        live = (x != 0).reshape(M, x.shape[1], -1).any(2).any(0)
        assert live.all(), (name, what, np.nonzero(~live)[0].tolist())
    gr = dict(zip(ALL, spied["grads"]))
    assert gr["dL_dtransMat"] is None
    _oracle_backward(frames, dLc, dLo, dLf, gs, None, det)
    report = {}
    _check_grads(name, c, frames, gr, True, report)

    # autograd: the parameters' .grad
    cloud_grads_exact = [(out["viewspace_points"].grad, gr["dL_dmeans2D"]), (spied["feat"].grad, gr["dL_dfeatures"])]
    sh_grad = gr["dL_dsh"]
    for got, want in cloud_grads_exact:
        assert got is not None and torch.equal(got, want.view(got.shape)), name
    cloud = spied["pc"]
    assert torch.equal(cloud._features_dc.grad, sh_grad[:, :1]) and torch.equal(cloud._features_rest.grad, sh_grad[:, 1:])
    ref_m3d = sum(fr["ref"]["dL_dmeans3D"].astype(np.float64) for fr in frames)
    tol_m3d = (sum(fr["tol"]["dL_dmeans3D"] for fr in frames)
               + M * U * sum(np.abs(fr["ref"]["dL_dmeans3D"].astype(np.float64)) for fr in frames))
    _check_grad(f"{name} _xyz.grad", "_xyz.grad", cloud._xyz.grad, ref_m3d, tol_m3d, report)
    for leaf, key, deriv in ((cloud._opacity, "dL_dopacity", lambda y: y * (1.0 - y)),
                             (cloud._scaling, "dL_dscales", lambda y: y)):
        y = (torch.sigmoid(leaf) if key == "dL_dopacity" else torch.exp(leaf)).detach().double().cpu().numpy()
        d = deriv(y).reshape(-1, y.shape[-1])
        ref = sum(fr["ref"][key].astype(np.float64) for fr in frames).reshape(d.shape)
        tol = (sum(fr["tol"][key] for fr in frames) + M * U * sum(np.abs(fr["ref"][key].astype(np.float64)) for fr in frames))
        tol = tol.reshape(d.shape) * np.abs(d) + 3 * U * np.abs(ref * d)
        _check_grad(f"{name} {key} leaf", key + " leaf", leaf.grad, ref * d, tol, report)
    knife = sum(int(fr["ext"]["knife"].sum()) for fr in frames)
    print(f"\n[{name}] knife pixels {knife}; forward err/bound {max(fr['fwd'] for fr in frames):.3g}; "
          + ", ".join(f"{k} {v:.3g}" for k, v in report.items()))
    assert knife <= 4 * KNIFE_MEASURED.get(name, 0) + 8, (name, "knife pixels", knife)
