"""TEST INFRASTRUCTURE -- sr_post_forward_frames (csrc/postprocess.cu) under the rounding-error bound: the forward maps of
test_gpu_loss_bounds' post model with each frame's own camera, the check of a frame's maps against them, and the camera
mistakes a kernel could plausibly make (the negative controls).

The model is test_gpu_loss_bounds._post_model's forward half, its camera built by _cam from the frame's camera-table row
(tan_x, tan_y, cx_off, cy_off) instead of the shared tangents.  Each map element is held to  |gpu - ref| <= K u B + FLOOR
outside the stencil knife mask (test_gpu_loss_bounds._stencil_knife), with ref the float64 oracle
(oracle/post_oracle.post_forward through camera_model's offset rays) and B the model's bound; the model's value must
agree with the oracle far inside that bound, so the bound is evaluated on the expression that is compared.
"""
import numpy as np

from .error_bound import _E
from .test_gpu_loss_bounds import (FLOOR, K, POST_CH, POST_KEYS, U, _cam, _dot3, _full, _stencil_knife, _stencils,
                                   _surf_depth, _where)
from .test_gpu_loss_pass_bounds import _table

MODEL_REL = 1.0 / 64        # the model's value agrees with the oracle's within this share of the bound

# sr_post_forward_frames' cases (W, H, M, camera path, depth ratio, learnable background): every combination of path,
# ratio and background once, on test_gpu_loss_bounds' 32 x 8 block edges (1 x 1, no interior stencil, 1-column and
# partial last blocks, odd sizes), at M = 1 and 3; and 257 frames of small images for blockIdx.z and the frame offsets.
SHAPES = ((1, 1), (2, 3), (3, 3), (1, 8), (3, 2), (31, 9), (32, 2), (33, 17), (63, 7), (65, 9), (97, 17), (33, 8))
GRID = [(W, H, 3 if (i // 2) % 2 == 0 else 1, path, r, bk)
        for i, ((W, H), (path, r, bk)) in enumerate(zip(SHAPES, [(p, r, b) for p in ("table", "scalar")
                                                                 for r in (0.0, 0.37, 1.0) for b in (False, True)]))]
GRID += [(33, 9, 257, "table", 0.37, True), (17, 3, 257, "scalar", 1.0, False)]


def frame_rows(M, W, H):
    """(M,4) fp32 camera-table rows: test_gpu_loss_pass_bounds._table's for the first three frames (both tangents differ
    per frame, non-integer offsets of either sign); its tangents would fall through zero past frame 33, so from frame 3 on
    they wind through [0.3, 0.7) x [0.3, 0.7) H / W along two Weyl sequences and stay distinct."""
    rows = _table(M, W, H)
    f = np.arange(3, M, dtype=np.float64)
    rows[3:, 0] = 0.3 + 0.4 * ((0.6180339887 * f) % 1.0)
    rows[3:, 1] = (0.3 + 0.4 * ((0.7548776662 * f + 0.37) % 1.0)) * H / W
    return rows


def cam(wvt, W, H, row, swap=False):
    """_cam for one camera-table row (tan_x, tan_y, cx_off, cy_off); swap: fx and fy exchanged (a negative control)."""
    c = _cam(wvt, W, H, *(float(x) for x in row))
    if swap:
        c["fx"], c["fy"] = c["fy"], c["fx"]
    return c


def forward_model(am, c, r):
    """post_fwd_kernel / post_normal_kernel for one frame with camera c: {map: [_E per channel]} and the stencil knife
    mask."""
    _, H, W = am.shape
    r = _E(float(np.float32(r)))
    a = _E(am[1])
    sd, ex, med, _, _ = _surf_depth(am, r)
    R = c["R"]
    n = [_E(am[2 + k]) for k in range(3)]
    fw = {"acc": [a], "rend_normal": [_dot3(R, (3 * k, 3 * k + 1, 3 * k + 2), n) for k in range(3)],
          "rend_dist": [_E(am[6])], "render_depth_median": [med], "render_depth_expected": [ex], "surf_depth": [sd]}
    fw["surf_normal"] = [_E(np.zeros((H, W)))] * 3
    own = np.zeros((H, W), bool)
    if H >= 3 and W >= 3:
        st = _stencils(c, sd, H, W)
        inv = _E(1.0) / _where(st["ln"].v > 1e-12, st["ln"], _E.const(1e-12))
        fw["surf_normal"] = [_full((st["n"][k] * inv) * a[1:-1, 1:-1], H, W) for k in range(3)]
        own, _ = _stencil_knife(st, H, W)
    return fw, own


def oracle(am, wvt, W, H, row, r):
    """post_oracle.post_forward with the row's tangents and camera_model's offset rays."""
    from oracle import post_oracle as po
    from . import camera_model as cm
    return cm._with_rays(float(row[2]), float(row[3]), po.post_forward, am, wvt, float(row[0]), float(row[1]),
                         float(np.float32(r)))


def ratios(got, fw, own, ref=None):
    """{map: |got - ref| / (K u B + FLOOR) per channel element, 0 on the knife mask (surf_normal only)}; ref defaults to
    the model's value.  A NaN from the GPU counts as out of bound."""
    out = {}
    for k in POST_KEYS:
        rs = []
        for ch in range(len(fw[k])):
            e = fw[k][ch]
            want = e.v if ref is None else np.asarray(ref[k][ch], np.float64)
            g = np.asarray(got[k][ch], np.float64)
            with np.errstate(invalid="ignore"):
                x = np.abs(g - want) / (K * U * e.b + FLOOR)
            x = np.where(np.isnan(g) & ~np.isnan(want), np.inf, np.nan_to_num(x, nan=0.0))
            rs.append(np.where(own, 0.0, x) if k == "surf_normal" else x)
        out[k] = np.stack(rs)
    return out


def check_frame(name, got, am, wvt, row, r, report, ref=None):
    """One frame's seven maps (got: {map: (channels, H, W)}) under the bound, against the oracle; the model's value agrees
    with the oracle within MODEL_REL of the bound.  Records per map the largest ratio under report[map]; returns the
    number of knife pixels."""
    _, H, W = am.shape
    fw, own = forward_model(am, cam(wvt, W, H, row), r)
    ref = oracle(am, wvt, W, H, row, r) if ref is None else ref
    for k in POST_KEYS:
        assert got[k].shape == (len(fw[k]), H, W), (name, k, got[k].shape)
    dm = ratios({k: [e.v for e in fw[k]] for k in POST_KEYS}, fw, own, ref)
    for k, x in dm.items():
        assert x.max() <= MODEL_REL, (name, k, "model != oracle", float(x.max()), np.argwhere(x > MODEL_REL)[:4].tolist())
    for k, x in ratios(got, fw, own, ref).items():
        i = int(np.argmax(x))
        report[k] = max(report.get(k, 0.0), float(x.flat[i]))
        c, y, xx = np.unravel_index(i, x.shape)
        assert x.flat[i] <= 1.0, (name, k, "element", (c, y, xx), "gpu", float(got[k][c, y, xx]), "oracle",
                                  float(ref[k][c][y, xx]), "bound", K * U * fw[k][c].b[y, xx] + FLOOR)
    return int(own.sum())


# ------------------------------------------------------------------------------------------------ negative controls
# name: the camera mistake.  Held to the model evaluated with the mistake, a kernel's correct maps must leave the bound
# (surf_normal or surf_depth) on at least CONTROL_SHARE of the pixels whose surf_normal is non-zero, over the frames the
# mistake changes.
CONTROLS = {
    "row0_tangents": "frame f reads row 0's tangents",
    "fx_fy_swapped": "fx and fy swapped",
    "cx_half_pixel": "cx off by half a pixel",
    "oy_sign": "the y offset with the wrong sign",
    "one_minus_ratio": "the depth ratio applied as 1 - r",
}
CONTROL_SHARE = 0.25


def mutated(control, rows, f, r):
    """The frame's (row, swap, depth ratio) under the control's mistake."""
    row = np.array(rows[f], np.float32)
    swap = False
    if control == "row0_tangents":
        row[:2] = rows[0][:2]
    elif control == "fx_fy_swapped":
        swap = True
    elif control == "cx_half_pixel":
        row[2] = row[2] + np.float32(0.5)
    elif control == "oy_sign":
        row[3] = -row[3]
    elif control == "one_minus_ratio":
        r = float(np.float32(1.0) - np.float32(r))
    return row, swap, r


def control_failures(control, got, am, wvt, rows, r):
    """(covered pixels out of the bound, covered pixels) over the frames the control changes, a covered pixel being one
    with a non-zero surf_normal: got is the list of each frame's maps, evaluated against the model with the mistake."""
    M, _, H, W = am.shape
    bad = live = 0
    for f in range(M):
        if control == "row0_tangents" and f == 0:
            continue
        row, swap, rr = mutated(control, rows, f, r)
        fw, own = forward_model(am[f], cam(wvt[f], W, H, row, swap), rr)
        x = ratios(got[f], fw, own)
        out = np.zeros((H, W), bool)
        for k in ("surf_normal", "surf_depth"):
            out |= (x[k] > 1.0).any(0)
        covered = (np.asarray(got[f]["surf_normal"]) != 0).any(0)
        bad += int((out & covered).sum())
        live += int(covered.sum())
    return bad, live


def maps_of(tensors, f):
    """{map: (channels, H, W) float32 numpy} of frame f from {map: (M, c, H, W)} tensors or arrays (broadcast depth maps:
    their first channel)."""
    out = {}
    for k, c in zip(POST_KEYS, POST_CH):
        t = tensors[k][f][:c]
        out[k] = t.cpu().numpy() if hasattr(t, "cpu") else np.asarray(t)
    return out
