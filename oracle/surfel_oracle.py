"""ctypes wrapper around oracle/libsurfel_oracle.so (the CPU restatement).

TEST INFRASTRUCTURE ONLY -- see the header of surfel_oracle.c.  Only tests/,
__graft_entry__.smoke() and bench.py (cpu_baseline / reference legs) import this.
Nothing in vidu4d_b200/ does.

API (numpy in, numpy out):
    st = forward(means3D, opacities, scales, rotations, shs=None, colors_precomp=None, *,
                 sh_degree, W, H, tanfovx, tanfovy, bg, viewmatrix, projmatrix, campos)
        -> OracleState with .color (3,H,W) .allmap (8,H,W) .radii (P,) .num_rendered
           and every intermediate buffer of the reference (keys, point_list, ranges, ...)
    grads = backward(st, dL_dcolor, dL_dallmap) -> dict of gradient arrays, reference order

Rounding-error bounds (see the error analysis in surfel_oracle.c):
    st, ext = from_records(inputs, transMat=, means2D=, normal_opacity=, rgb=, radii=, clamped=, point_list=, ranges=)
        composite only, from given per-surfel records (e.g. the GPU's); ext = composite_ext(st)
    ext = composite_ext(st) -> dict(knife (H,W) bool, walk_S (H,W), fbound (14,H,W), nblend (H,W)); also refreshes
        st's planes
    grads = backward(st, dL_dcolor, dL_dallmap, bounds=True) -> adds "acc", "bound", "asum" (P,18), SO_A_* order
    chain(st, acc) -> the gradient dict from given (P,18) accumulators
    chain_bound(st, B) -> per output element sum_j |d out / d acc_j| B_j
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from dataclasses import dataclass, field

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libsurfel_oracle.so")
_lib = None

f32p = C.POINTER(C.c_float)
f64p = C.POINTER(C.c_double)
# accumulator order of so_chain / backward(bounds=True): dL/dT 9, dL/dmean2D 2 (low-pass branch), dL/dnormal 3,
# dL/dopacity 1, dL/dcolour 3
ACC_T, ACC_M2D, ACC_NORMAL, ACC_OPAC, ACC_COLOR, NACC = 0, 9, 11, 14, 15, 18


class _Params(C.Structure):
    _fields_ = [
        ("P", C.c_int), ("D", C.c_int), ("M", C.c_int), ("W", C.c_int), ("H", C.c_int),
        ("tanfovx", C.c_float), ("tanfovy", C.c_float),
        ("bg", f32p), ("means3D", f32p), ("shs", f32p), ("colors_precomp", f32p),
        ("opacities", f32p), ("scales", f32p), ("rotations", f32p),
        ("viewmatrix", f32p), ("projmatrix", f32p), ("campos", f32p),
    ]


class _State(C.Structure):
    _fields_ = [
        ("P", C.c_int), ("W", C.c_int), ("H", C.c_int), ("tiles_x", C.c_int), ("tiles_y", C.c_int),
        ("R", C.c_int), ("bit", C.c_int),
        ("depths", f32p), ("clamped", C.POINTER(C.c_uint8)), ("radii", C.POINTER(C.c_int)),
        ("means2D", f32p), ("transMat", f32p), ("normal_opacity", f32p), ("rgb", f32p),
        ("tiles_touched", C.POINTER(C.c_uint32)), ("point_offsets", C.POINTER(C.c_uint32)),
        ("keys_unsorted", C.POINTER(C.c_uint64)), ("values_unsorted", C.POINTER(C.c_uint32)),
        ("keys", C.POINTER(C.c_uint64)), ("point_list", C.POINTER(C.c_uint32)),
        ("ranges", C.POINTER(C.c_uint32)), ("final_T", f32p), ("n_contrib", C.POINTER(C.c_uint32)),
        ("out_color", f32p), ("out_others", f32p),
    ]


def build(force: bool = False) -> str:
    """Compile the C restatement (gcc, a second or two)."""
    src = os.path.join(_HERE, "surfel_oracle.c")
    if force or not os.path.exists(_LIB_PATH) or os.path.getmtime(src) > os.path.getmtime(_LIB_PATH):
        subprocess.check_call(["make", "-C", _HERE, "libsurfel_oracle.so"], stdout=subprocess.DEVNULL)
    return _LIB_PATH


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = C.CDLL(_LIB_PATH)
        _lib.so_forward.restype = C.POINTER(_State)
        _lib.so_forward.argtypes = [C.POINTER(_Params)]
        _lib.so_free.argtypes = [C.POINTER(_State)]
        _lib.so_backward.argtypes = [C.POINTER(_Params), C.POINTER(_State)] + [f32p] * 11
        _lib.so_backward_ex.argtypes = [C.POINTER(_Params), C.POINTER(_State)] + [f32p] * 11 + [f64p] * 4
        _lib.so_composite.argtypes = [C.POINTER(_State), f32p, f32p, C.POINTER(C.c_uint8), f64p, f64p,
                                      C.POINTER(C.c_uint32)]
        _lib.so_chain.argtypes = [C.POINTER(_Params), C.POINTER(_State), f32p] + [f32p] * 9
        _lib.so_chain_bound.argtypes = [C.POINTER(_Params), C.POINTER(_State), f64p] + [f64p] * 9
        _lib.so_mark_visible.argtypes = [C.c_int, f32p, f32p, C.POINTER(C.c_uint8)]
        _lib.so_num_threads.restype = C.c_int
    return _lib


def num_threads() -> int:
    return int(lib().so_num_threads())


def _f(a, shape=None):
    if a is None:
        return None
    a = np.ascontiguousarray(np.asarray(a, dtype=np.float32))
    if shape is not None:
        a = a.reshape(shape)
    return a


def _ptr(a):
    return a.ctypes.data_as(f32p) if a is not None and a.size > 0 else None


def _copy(ptr, n, dtype):
    if n == 0:
        return np.zeros((0,), dtype=dtype)
    return np.ctypeslib.as_array(ptr, shape=(n,)).astype(dtype, copy=True)


@dataclass
class OracleState:
    P: int
    W: int
    H: int
    num_rendered: int
    bit: int
    color: np.ndarray
    allmap: np.ndarray
    radii: np.ndarray
    depths: np.ndarray
    clamped: np.ndarray
    means2D: np.ndarray
    transMat: np.ndarray
    normal_opacity: np.ndarray
    rgb: np.ndarray
    tiles_touched: np.ndarray
    point_offsets: np.ndarray
    keys_unsorted: np.ndarray
    values_unsorted: np.ndarray
    keys: np.ndarray
    point_list: np.ndarray
    ranges: np.ndarray
    final_T: np.ndarray
    n_contrib: np.ndarray
    _inputs: dict = field(default_factory=dict, repr=False)
    walk_S: np.ndarray = None


def _make_params(inp):
    p = _Params()
    p.P, p.D, p.M, p.W, p.H = inp["P"], inp["D"], inp["M"], inp["W"], inp["H"]
    p.tanfovx, p.tanfovy = inp["tanfovx"], inp["tanfovy"]
    for k in ("bg", "means3D", "shs", "colors_precomp", "opacities", "scales", "rotations",
              "viewmatrix", "projmatrix", "campos"):
        setattr(p, k, _ptr(inp[k]))
    return p


def forward(means3D, opacities, scales, rotations, shs=None, colors_precomp=None, *, sh_degree=0,
            W, H, tanfovx, tanfovy, bg=(0, 0, 0), viewmatrix=None, projmatrix=None, campos=(0, 0, 0)):
    means3D = _f(means3D, (-1, 3))
    P = means3D.shape[0]
    if (shs is None) == (colors_precomp is None):
        raise Exception('Please provide excatly one of either SHs or precomputed colors!')
    shs_a = _f(shs)
    M = 0
    if shs_a is not None:
        shs_a = shs_a.reshape(P, -1, 3)
        M = shs_a.shape[1]
    inp = dict(
        P=P, D=int(sh_degree), M=M, W=int(W), H=int(H), tanfovx=float(tanfovx), tanfovy=float(tanfovy),
        bg=_f(bg, (3,)), means3D=means3D, shs=shs_a, colors_precomp=_f(colors_precomp),
        opacities=_f(opacities, (-1,)), scales=_f(scales, (-1, 2)), rotations=_f(rotations, (-1, 4)),
        viewmatrix=_f(np.eye(4) if viewmatrix is None else viewmatrix, (16,)),
        projmatrix=_f(np.eye(4) if projmatrix is None else projmatrix, (16,)),
        campos=_f(campos, (3,)),
    )
    prm = _make_params(inp)
    sp = lib().so_forward(C.byref(prm))
    s = sp.contents
    N, R, tiles = W * H, s.R, s.tiles_x * s.tiles_y
    st = OracleState(
        P=P, W=W, H=H, num_rendered=R, bit=s.bit,
        color=_copy(s.out_color, 3 * N, np.float32).reshape(3, H, W),
        allmap=_copy(s.out_others, 8 * N, np.float32).reshape(8, H, W),
        radii=_copy(s.radii, P, np.int32),
        depths=_copy(s.depths, P, np.float32),
        clamped=_copy(s.clamped, 3 * P, np.uint8).reshape(P, 3),
        means2D=_copy(s.means2D, 2 * P, np.float32).reshape(P, 2),
        transMat=_copy(s.transMat, 9 * P, np.float32).reshape(P, 9),
        normal_opacity=_copy(s.normal_opacity, 4 * P, np.float32).reshape(P, 4),
        rgb=_copy(s.rgb, 3 * P, np.float32).reshape(P, 3),
        tiles_touched=_copy(s.tiles_touched, P, np.uint32),
        point_offsets=_copy(s.point_offsets, P, np.uint32),
        keys_unsorted=_copy(s.keys_unsorted, R, np.uint64),
        values_unsorted=_copy(s.values_unsorted, R, np.uint32),
        keys=_copy(s.keys, R, np.uint64),
        point_list=_copy(s.point_list, R, np.uint32),
        ranges=_copy(s.ranges, 2 * tiles, np.uint32).reshape(tiles, 2),
        final_T=_copy(s.final_T, 3 * N, np.float32).reshape(3, H, W),
        n_contrib=_copy(s.n_contrib, 2 * N, np.uint32).reshape(2, H, W),
        _inputs=inp,
    )
    lib().so_free(sp)
    return st


def _cstate(st: OracleState, keep: list):
    """A C state that points at st's numpy arrays (kept alive through `keep`)."""
    s = _State()
    s.P, s.W, s.H = st.P, st.W, st.H
    s.tiles_x, s.tiles_y = (st.W + 15) // 16, (st.H + 15) // 16
    s.R, s.bit = st.num_rendered, st.bit

    def setp(name, arr, ctype):
        arr = np.ascontiguousarray(arr)
        keep.append(arr)
        setattr(s, name, arr.ctypes.data_as(C.POINTER(ctype)))

    setp("depths", st.depths, C.c_float); setp("clamped", st.clamped, C.c_uint8)
    setp("radii", st.radii, C.c_int); setp("means2D", st.means2D, C.c_float)
    setp("transMat", st.transMat, C.c_float); setp("normal_opacity", st.normal_opacity, C.c_float)
    setp("rgb", st.rgb, C.c_float); setp("point_list", st.point_list, C.c_uint32)
    setp("ranges", st.ranges, C.c_uint32); setp("final_T", st.final_T, C.c_float)
    setp("n_contrib", st.n_contrib, C.c_uint32)
    return s


def _grad_arrays(P, M, dtype=np.float32):
    return dict(
        dL_dmeans2D=np.zeros((P, 3), dtype), dL_dcolors=np.zeros((P, 3), dtype),
        dL_dopacity=np.zeros((P, 1), dtype), dL_dmeans3D=np.zeros((P, 3), dtype),
        dL_dtransMat=np.zeros((P, 9), dtype), dL_dsh=np.zeros((P, M, 3), dtype),
        dL_dscales=np.zeros((P, 2), dtype), dL_drotations=np.zeros((P, 4), dtype),
        dL_dnormal=np.zeros((P, 3), dtype),
    )


def backward(st: OracleState, dL_dcolor, dL_dallmap, bounds=False):
    """Returns the reference's 8 gradient tensors (+ dL_dnormal) for a forward state.  bounds=True (needs st.walk_S, set
    by composite_ext) adds the (P,18) double accumulators "acc" and their bound sums "bound" and "asum"."""
    inp = st._inputs
    P, M, W, H = st.P, inp["M"], st.W, st.H
    prm = _make_params(inp)
    keep = []
    s = _cstate(st, keep)
    dc = _f(dL_dcolor, (3, H, W)); do = _f(dL_dallmap, (8, H, W))
    out = _grad_arrays(P, M)
    extra = {}
    if bounds:
        if st.walk_S is None:
            raise ValueError("bounds=True needs the composite's walk_S: run composite_ext(st) first")
        extra = {k: np.zeros((P, NACC), np.float64) for k in ("acc", "bound", "asum")}
    if P > 0:
        ws = np.ascontiguousarray(st.walk_S, np.float64) if bounds else None
        dp = lambda a: a.ctypes.data_as(f64p) if a is not None else None  # noqa: E731
        lib().so_backward_ex(C.byref(prm), C.byref(s), _ptr(dc), _ptr(do),
                             *[o.ctypes.data_as(f32p) for o in out.values()],
                             dp(ws), dp(extra.get("acc")), dp(extra.get("bound")), dp(extra.get("asum")))
    out.update(extra)
    return out


def composite_ext(st: OracleState):
    """Re-runs the composite on st's records (in place: color, allmap, final_T, n_contrib) and returns its optional
    outputs: knife (H,W) bool, walk_S (H,W), fbound (14,H,W) -- per plane (colour 3, allmap 8, final_T 3) the sum
    over terms of (weight in units of 2^-24) * |term| -- and nblend (H,W), the pairs blended into each pixel (the
    composite evaluates every pair of the tile's list: it does not cull).  Also stores walk_S on st for
    backward(bounds=True)."""
    W, H, N = st.W, st.H, st.W * st.H
    keep = []
    st.final_T = np.zeros((3, H, W), np.float32)
    st.n_contrib = np.zeros((2, H, W), np.uint32)
    s = _cstate(st, keep)
    color = np.zeros(3 * N, np.float32); others = np.zeros(8 * N, np.float32)
    s.out_color = color.ctypes.data_as(f32p); s.out_others = others.ctypes.data_as(f32p)
    knife = np.zeros(N, np.uint8); walk_S = np.zeros(N, np.float64); fbound = np.zeros(14 * N, np.float64)
    nblend = np.zeros(N, np.uint32)
    inp = st._inputs
    feat = inp["colors_precomp"] if inp["colors_precomp"] is not None else np.ascontiguousarray(st.rgb, np.float32)
    keep.append(feat)
    lib().so_composite(C.byref(s), _ptr(feat), _ptr(inp["bg"]), knife.ctypes.data_as(C.POINTER(C.c_uint8)),
                       walk_S.ctypes.data_as(f64p), fbound.ctypes.data_as(f64p),
                       nblend.ctypes.data_as(C.POINTER(C.c_uint32)))
    st.color = color.reshape(3, H, W); st.allmap = others.reshape(8, H, W)
    st.walk_S = walk_S.reshape(H, W)
    return dict(knife=knife.reshape(H, W).astype(bool), walk_S=st.walk_S, fbound=fbound.reshape(14, H, W),
                nblend=nblend.reshape(H, W))


def from_records(means3D, opacities, scales, rotations, shs=None, colors_precomp=None, *, sh_degree=0, W, H, tanfovx,
                 tanfovy, bg=(0, 0, 0), viewmatrix=None, projmatrix=None, campos=(0, 0, 0), transMat, means2D,
                 normal_opacity, rgb, radii, clamped, point_list, ranges):
    """An OracleState whose per-surfel records, sorted list and tile ranges are given (e.g. decoded from the GPU's
    buffers) and whose image planes come from the composite alone; returns (state, composite_ext(state)).
    clamped: (P,3) bools.  The inputs the per-surfel backward reads (positions, scales, rotations, SH, camera) as in
    forward()."""
    means3D = _f(means3D, (-1, 3))
    P = means3D.shape[0]
    shs_a = _f(shs)
    M = 0
    if shs_a is not None:
        shs_a = shs_a.reshape(P, -1, 3)
        M = shs_a.shape[1]
    inp = dict(
        P=P, D=int(sh_degree), M=M, W=int(W), H=int(H), tanfovx=float(tanfovx), tanfovy=float(tanfovy),
        bg=_f(bg, (3,)), means3D=means3D, shs=shs_a, colors_precomp=_f(colors_precomp),
        opacities=_f(opacities, (-1,)), scales=_f(scales, (-1, 2)), rotations=_f(rotations, (-1, 4)),
        viewmatrix=_f(np.eye(4) if viewmatrix is None else viewmatrix, (16,)),
        projmatrix=_f(np.eye(4) if projmatrix is None else projmatrix, (16,)),
        campos=_f(campos, (3,)),
    )
    tiles = ((W + 15) // 16) * ((H + 15) // 16)
    pl = np.ascontiguousarray(point_list, np.uint32).reshape(-1)
    st = OracleState(
        P=P, W=W, H=H, num_rendered=int(pl.size), bit=0, color=None, allmap=None,
        radii=np.ascontiguousarray(radii, np.int32).reshape(P), depths=np.zeros(P, np.float32),
        clamped=np.ascontiguousarray(clamped, np.uint8).reshape(P, 3), means2D=_f(means2D, (P, 2)),
        transMat=_f(transMat, (P, 9)), normal_opacity=_f(normal_opacity, (P, 4)), rgb=_f(rgb, (P, 3)),
        tiles_touched=np.zeros(P, np.uint32), point_offsets=np.zeros(P, np.uint32),
        keys_unsorted=np.zeros(0, np.uint64), values_unsorted=np.zeros(0, np.uint32), keys=np.zeros(0, np.uint64),
        point_list=pl, ranges=np.ascontiguousarray(ranges, np.uint32).reshape(tiles, 2), final_T=None, n_contrib=None,
        _inputs=inp,
    )
    return st, composite_ext(st)


def chain(st: OracleState, acc):
    """backward()'s per-surfel part on given accumulators acc (P,18), ACC_* order."""
    inp = st._inputs
    P, M = st.P, inp["M"]
    out = _grad_arrays(P, M)
    if P > 0:
        keep = []
        s = _cstate(st, keep)
        a = _f(acc, (P, NACC))
        lib().so_chain(C.byref(_make_params(inp)), C.byref(s), _ptr(a), *[o.ctypes.data_as(f32p) for o in out.values()])
    return out


def chain_bound(st: OracleState, B):
    """Per output element of backward(), sum over the 18 accumulators j of |d out / d acc_j| * B[:, j] (float64)."""
    inp = st._inputs
    P, M = st.P, inp["M"]
    out = _grad_arrays(P, M, np.float64)
    if P > 0:
        keep = []
        s = _cstate(st, keep)
        b = np.ascontiguousarray(B, np.float64).reshape(P, NACC)
        lib().so_chain_bound(C.byref(_make_params(inp)), C.byref(s), b.ctypes.data_as(f64p),
                             *[o.ctypes.data_as(f64p) for o in out.values()])
    return out


def mark_visible(means3D, viewmatrix):
    means3D = _f(means3D, (-1, 3))
    P = means3D.shape[0]
    out = np.zeros((P,), np.uint8)
    if P:
        lib().so_mark_visible(P, _ptr(means3D), _ptr(_f(viewmatrix, (16,))), out.ctypes.data_as(C.POINTER(C.c_uint8)))
    return out.astype(bool)
