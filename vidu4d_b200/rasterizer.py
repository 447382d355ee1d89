"""Python host side of the surfel rasterizer: the reference's operator interface, re-implemented over
the C ABI of libsurfel_raster.so.

Mirrors, name for name, RAST/diff_surfel_rasterization/__init__.py (RAST = gs/submodules/
diff-surfel-rasterization of yikaiw/Vidu4D):

    GaussianRasterizationSettings   __init__.py:158-170
    GaussianRasterizer              __init__.py:172-222   (forward, markVisible)
    rasterize_gaussians             __init__.py:21-42
    _RasterizeGaussians             __init__.py:44-156    (autograd.Function)
    _C.rasterize_gaussians / _C.rasterize_gaussians_backward / _C.mark_visible
                                    RAST/rasterize_points.h:18-68, RAST/ext.cpp:15-19

so `gs/gaussian_renderer/__init__.py:14` (`from diff_surfel_rasterization import ...`) works unchanged
when the repo root is on sys.path (see the top-level `diff_surfel_rasterization/` shim).

PyTorch is plumbing here: it owns device memory and streams; every kernel is in the CUDA library.
"""
from __future__ import annotations

import ctypes as C
from typing import NamedTuple, Optional

import torch
import torch.nn as nn

from . import _capi

# --------------------------------------------------------------------------------------------
# capacity policy for the instance ("binning") buffer
# --------------------------------------------------------------------------------------------
_CAP_ALIGN = 256           # capacities are multiples of this so that bytes -> capacity is invertible
_cap_hint: dict = {}       # (device index, W, H) -> last seen num_rendered
_sync_mode = True          # True: read num_rendered back after every forward (like the reference)
_deterministic = False     # set_deterministic
_pending: list = []        # nosync mode: (pinned host words (frames,2), key, capacity, stream) awaiting check_overflow()
_MAX_PENDING = 4096        # nosync forwards that may accumulate before check_overflow() is forced
_host_pool: list = []      # pinned (64,2) int32 status blocks, pre-allocated so that a forward never allocates pinned memory
_host_next = 0             #   (cudaHostAlloc is illegal during CUDA-graph capture)
# The module state above belongs to the (single) thread that issues forwards; autograd's backward thread only calls
# rasterize_gaussians_backward, which touches none of it.


def set_sync_mode(flag: bool):
    """sync=True (default): each forward reads `num_rendered` back (one stream sync, as the reference does at
    rasterizer_impl.cu:282) and transparently re-runs with a larger buffer on overflow.
    sync=False: no host<->device synchronisation at all; call check_overflow() once per step."""
    global _sync_mode
    _sync_mode = bool(flag)


def set_deterministic(flag: bool):
    """flag=True: every rasterizer backward runs the deterministic kernels (include/surfel_deterministic.h): no float
    atomic touches a gradient and every sum has an order fixed by the data, so the same inputs give the same gradient
    bits on every call, and each frame of a batch the bits of a one-frame call.  It costs one scratch of
    sr_backward_det_bytes(capacity, F) per frame (from torch's allocator) and some time (BASELINE.md).  The mode is also
    on while torch.are_deterministic_algorithms_enabled().  Process-wide, like set_sync_mode; the forward is unaffected."""
    global _deterministic
    _deterministic = bool(flag)


def deterministic() -> bool:
    """Whether the rasterizer backward runs deterministically: set_deterministic(True) or
    torch.use_deterministic_algorithms(True)."""
    return _deterministic or torch.are_deterministic_algorithms_enabled()


def _round_cap(n: int) -> int:
    n = max(int(n), _CAP_ALIGN)
    return (n + _CAP_ALIGN - 1) // _CAP_ALIGN * _CAP_ALIGN


def _pick_capacity(key, P: int) -> int:
    r = _cap_hint.get(key)
    if r is None:
        return _round_cap(max(4 * P, 4096))
    return _round_cap(int(r * 1.5) + 4096)     # headroom for frame-to-frame growth in nosync mode (136 B / instance)


_bytes_to_cap: dict = {}


def _capacity_from_bytes(nbytes: int, W: int, H: int) -> int:
    """Inverse of sr_binning_bytes(., W, H) for capacities that are multiples of _CAP_ALIGN."""
    key = (nbytes, W, H)
    if key in _bytes_to_cap:
        return _bytes_to_cap[key]
    lib = _capi.load()
    lo, hi = 1, 1 << 22   # in units of _CAP_ALIGN
    while lo < hi:
        mid = (lo + hi) // 2
        if lib.sr_binning_bytes(mid * _CAP_ALIGN, W, H) < nbytes:
            lo = mid + 1
        else:
            hi = mid
    cap = lo * _CAP_ALIGN
    if lib.sr_binning_bytes(cap, W, H) != nbytes:
        raise _capi.SurfelRasterError("binningBuffer was not produced by this library's forward")
    _bytes_to_cap[key] = cap
    return cap


_HOST_SLOT_FRAMES = 64      # frames one pinned status block can hold


def reserve_host_slots(n: int):
    """Pre-allocate pinned status words for the next `n` nosync forwards (needed before CUDA-graph capture)."""
    while len(_host_pool) - _host_next < n:
        _host_pool.append(torch.zeros((_HOST_SLOT_FRAMES, 2), dtype=torch.int32).pin_memory())


def _host_slot(frames: int = 1):
    """Pinned {num_rendered, status} words for one (batched) forward: (frames, 2) int32."""
    global _host_next
    if frames > _HOST_SLOT_FRAMES:
        return torch.zeros((frames, 2), dtype=torch.int32).pin_memory()
    if _host_next >= len(_host_pool):
        _host_pool.append(torch.zeros((_HOST_SLOT_FRAMES, 2), dtype=torch.int32).pin_memory())
    h = _host_pool[_host_next]
    _host_next += 1
    return h[:frames]


def check_overflow(keep: bool = False, sync: bool = True):
    """nosync mode: synchronise once, verify that no forward since the last call overflowed its instance
    buffer, and refresh the capacity hints.  Raises SurfelRasterError if a frame was dropped.
    keep=True leaves the watch list in place (a captured CUDA graph rewrites the same status words on every
    replay: call check_overflow(keep=True) after each replay).  sync=False: the caller has already waited for the
    forwards in question (e.g. on an event recorded behind them) -- used to check step k-1 while step k is in flight."""
    global _host_next
    bad, prefilter = None, False
    # Every device a pending forward ran on is synchronised (not just the current one): the asynchronous D2H copies of the
    # status words have landed.  Device-wide rather than per stream, because a forward recorded into a CUDA graph replays
    # on whatever stream the graph is launched on, not on the stream it was captured on.
    devices, bare = set(), []
    for _, _, _, stream in _pending:
        d = getattr(stream, "device", None)
        if d is not None:
            devices.add(d)
        elif stream not in bare:
            bare.append(stream)
    if sync:
        for d in devices:
            torch.cuda.synchronize(d)
        for stream in bare:
            stream.synchronize()
    for host, key, cap, stream in _pending:
        for r, status in host.tolist():
            _cap_hint[key] = max(_cap_hint.get(key, 0), r)
            if status & _capi.SR_STATUS_OVERFLOW:
                bad = (r, cap)
            if status & _capi.SR_STATUS_PREFILTER:
                prefilter = True
    if not keep:
        _pending.clear()
        _host_next = 0
    if prefilter:
        raise RuntimeError("Point is filtered although prefiltered is set. This shouldn't happen!")
    if bad:
        raise _capi.SurfelRasterError(
            f"instance buffer overflow in nosync mode: num_rendered={bad[0]}, "
            f"capacity={bad[1]}; the frame was not rendered. Hints updated -- re-run the step.")


def _ptr(t):
    """Device pointer of a tensor, or None for the 'not provided' empty tensor (the reference's kernels test
    for a null data pointer the same way, forward.cu:215,247)."""
    if t is None or t.numel() == 0:
        return None
    return t.data_ptr()


def _f32c(t, name):
    if t is None:
        return None
    if not t.is_cuda:
        raise RuntimeError(f"{name} must be a CUDA tensor")   # CHECK_INPUT, rasterize_points.cu:27-28
    if t.dtype != torch.float32:
        t = t.float()
    t = t.contiguous()
    if t.data_ptr() % 16 != 0 and t.numel() != 0:
        # the kernels use 128-bit loads (rotations, SH rows) and 64-bit loads (scales); a contiguous view at an odd
        # storage offset (e.g. `rot[1:]`, a slice of a flat parameter buffer) is re-homed; the reference's scalar glm
        # loads accept such tensors, so must we
        t = t.clone()
    return t


def _batch_inputs(M: int, **named):
    """Normalise the per-surfel inputs of a batched call.  Each value is (tensor, trailing shape or None); a tensor is
    either shared by the M frames (its single-frame shape) or per frame (leading M).  Returns (contiguous float32
    tensors, per-frame strides in floats: 0 = shared)."""
    out, strides = {}, {}
    for name, (t, tail) in named.items():
        if t is None or t.numel() == 0:
            out[name], strides[name] = None, 0
            continue
        t = _f32c(t, name)
        base_ndim = 3 if name == "sh" else 2
        if t.ndim == base_ndim + 1:
            if t.shape[0] != M:
                raise RuntimeError(f"{name}: leading dimension {t.shape[0]} != number of frames {M}")
            strides[name] = int(t[0].numel()) if M > 1 else 0
        elif t.ndim == base_ndim:
            strides[name] = 0
        else:
            raise RuntimeError(f"{name} must have {base_ndim} (shared) or {base_ndim + 1} (per frame) dimensions")
        if tail is not None and tuple(t.shape[-len(tail):]) != tail:
            raise RuntimeError(f"{name} must have trailing dimensions {tail}")
        out[name] = t
    return out, strides


def _check_features(features, P: int, background, batched: bool = False) -> int:
    """Validate per-surfel feature channels: float (P,F) -- or, batched, (M,P,F) -- with 1 <= F <= 32, on the GPU, and a
    background of 3 or 3+F values.  Returns F."""
    if not torch.is_tensor(features):
        raise RuntimeError("features must be a tensor")
    if features.ndim not in ((2, 3) if batched else (2,)) or int(features.shape[-2]) != P:
        want = "(P,F) or (M,P,F)" if batched else "(P,F)"
        raise RuntimeError(f"features must have dimensions {want} with P = {P}, got {tuple(features.shape)}")
    F = int(features.shape[-1])
    if not 1 <= F <= _capi.FEATURES_MAX:
        raise RuntimeError(f"features must have 1..{_capi.FEATURES_MAX} channels, got {F}")
    nbg = int(background.numel())
    if nbg not in (3, 3 + F):
        raise RuntimeError(f"background must have 3 or 3+F = {3 + F} values with {F} feature channels, got {nbg}")
    if not features.is_cuda:
        raise RuntimeError("features must be a CUDA tensor")
    return F


def _as_float(x) -> float:
    # the reference passes CUDA 0-d tensors to pybind `float` params (gaussian_renderer/__init__.py:36-43)
    return float(x.item()) if torch.is_tensor(x) else float(x)


_STRIDED = ("means3D", "sh", "colors", "opacity", "scales", "rotations")     # sr_batch's per-surfel strides, in its order


def _check_intrinsics(intrinsics, M: int, ref):
    """The (M,4) per-frame camera table (tan_fovx, tan_fovy, cx_off, cy_off) of include/surfel_camera.h: float32, contiguous,
    on ref's device.  Only its shape is checked -- its values stay on the device."""
    if intrinsics is None:
        return None
    if not torch.is_tensor(intrinsics) or intrinsics.dtype != torch.float32 or tuple(intrinsics.shape) != (M, 4):
        raise RuntimeError(f"intrinsics must be a float32 (M,4) = {(M, 4)} tensor of (tan_fovx, tan_fovy, cx_off, cy_off)")
    if not intrinsics.is_cuda or intrinsics.device != ref.device:
        raise RuntimeError(f"intrinsics must be a CUDA tensor on {ref.device}")
    return intrinsics.contiguous()


def _frame(P, degree, Msh, W, H, tan_fovx, tan_fovy, scale_modifier, prefiltered, debug, intrinsics):
    """sr_frame, or with a camera table sr_frame_cameras (whose tangents are not read, so nothing is read back from the
    device).  Returns (the struct to keep alive, the sr_frame pointer to pass)."""
    if intrinsics is None:
        fr = _capi.SrFrame(P, int(degree), Msh, W, H, _as_float(tan_fovx), _as_float(tan_fovy), float(scale_modifier),
                           int(bool(prefiltered)), int(bool(debug)), 0)
        return fr, C.byref(fr)
    fc = _capi.SrFrameCameras(_capi.SrFrame(P, int(degree), Msh, W, H, 0.0, 0.0, float(scale_modifier), int(bool(prefiltered)),
                                            int(bool(debug)), _capi.SR_FRAME_CAMERAS), intrinsics.data_ptr())
    return fc, C.byref(fc.frame)


class _RenderOut:
    """Where a forward-only _forward writes: preallocated, packed views of the caller's (T,...) outputs for this call's
    frames (color (M,3,H,W), features (M,F,H,W) or None, others (M,8,H,W), radii (M,P)), and the arena that the calls of
    one render share (include/surfel_render.h), grown only when a call needs more.  contrib: an _capi.SrContrib the call
    adds its contribution statistics into (sr_render_forward_contrib), or None.  With it, a call of M > 1 frames that
    overflows is not re-run -- its other frames have added already -- and `overflowed` lists the frames to re-run alone.
    mask: with contrib, an _capi.SrContribMask whose `mask` points at this call's first frame's foreground mask: the call
    also adds the background share of the statistics (sr_render_forward_contrib_masked); or None.  lift: with contrib,
    an _capi.SrLift whose `values` points at this call's first frame's values: the call also adds its lifted values
    (sr_render_forward_lift); or None.  anchors: without contrib, an _capi.SrAnchors whose arrays point at this call's
    first frame's slots: the call also writes each pixel's heaviest pairs (sr_render_forward_anchors), overwriting them,
    so an overflowed call re-runs whole as the plain render does; or None."""
    __slots__ = ("color", "features", "others", "radii", "arena", "contrib", "overflowed", "mask", "lift", "anchors")

    def __init__(self, color, features, others, radii, arena=None, contrib=None, mask=None, lift=None, anchors=None):
        self.color, self.features, self.others, self.radii, self.arena = color, features, others, radii, arena
        self.contrib, self.overflowed, self.mask, self.lift, self.anchors = contrib, [], mask, lift, anchors


def _forward(M, frame_dim, strides, background, means3D, sh, colors, opacity, scales, rotations, features, viewmatrix,
             projmatrix, campos, H, W, degree, tan_fovx, tan_fovy, scale_modifier, prefiltered, debug, concat=True,
             intrinsics=None, render=None):
    """The one sr_forward call behind every _C forward: M frames, F = 0 without features.  The caller has validated the
    inputs and made them contiguous float32 CUDA tensors; `strides` gives the floats between consecutive frames of each
    per-surfel input (absent = shared).  intrinsics: the checked (M,4) camera table, which replaces tan_fovx / tan_fovy,
    or None.  The outputs get a leading frame dimension iff frame_dim.  In sync mode an
    overflowed call is re-run with a larger instance buffer; in nosync mode the status words join _pending.
    Returns (num_rendered (list of M ints, or -1 in nosync mode), out_color, out_others, radii, geom, binning, img,
    out_feat): with concat, out_color holds 3+F planes per frame and out_feat is the view of the last F; None when F = 0.
    render: a _RenderOut -- forward-only (sr_render_forward): the outputs are its views, the scratch is its arena, nothing
    is kept for a backward (geom, binning and img are None), and the instance counts are read back in either sync mode."""
    lib = _capi.load()
    dev = means3D.device
    P, N = int(means3D.shape[-2]), H * W
    Msh = int(sh.shape[-2]) if sh is not None and sh.numel() != 0 else 0
    F = int(features.shape[-1]) if features is not None else 0
    lead = (M,) if frame_dim else ()
    fr, frp = _frame(P, degree, Msh, W, H, tan_fovx, tan_fovy, scale_modifier, prefiltered, debug, intrinsics)
    bt = _capi.SrBatch(M, 0, *(strides.get(k, 0) for k in _STRIDED))
    with torch.cuda.device(dev):
        if render is not None:
            out_color, out_feat, out_others, radii = render.color, render.features, render.others, render.radii
            cstride, fstride = 3 * N, F * N
        elif F and concat:
            out_color = torch.empty(lead + (3 + F, H, W), dtype=torch.float32, device=dev)
            out_feat = out_color[..., 3:, :, :]
            cstride = fstride = (3 + F) * N
        else:
            out_color = torch.empty(lead + (3, H, W), dtype=torch.float32, device=dev)
            out_feat = torch.empty(lead + (F, H, W), dtype=torch.float32, device=dev) if F else None
            cstride, fstride = 3 * N, F * N
        geom = binning = img = None
        if render is None:
            out_others = torch.empty(lead + (8, H, W), dtype=torch.float32, device=dev)
            radii = torch.empty(lead + (P,), dtype=torch.int32, device=dev)
            geom = torch.empty((M * lib.sr_geom_bytes(P),), dtype=torch.uint8, device=dev)
            img = torch.empty((M * lib.sr_image_bytes(W, H),), dtype=torch.uint8, device=dev)
        nr_dev = torch.empty((M, 2), dtype=torch.int32, device=dev)
        stream = torch.cuda.current_stream(dev)
        key = (dev.index, W, H)
        cap = _pick_capacity(key, P)
        while True:
            nosync = render is None and (not _sync_mode) and key in _cap_hint
            host = _host_slot(M) if nosync else torch.empty((M, 2), dtype=torch.int32, pin_memory=True)
            args = (dev, frp, C.byref(bt), _ptr(background), int(background.numel()), _ptr(means3D), _ptr(sh), _ptr(colors),
                    _ptr(opacity), _ptr(scales), _ptr(rotations), _ptr(features), F, strides.get("features", 0),
                    _ptr(viewmatrix), _ptr(projmatrix), _ptr(campos), out_color, cstride, _ptr(out_feat), fstride, out_others,
                    _ptr(radii))
            # an overflow re-run below re-runs the feature pass too
            if render is None:
                binning = torch.empty((M * lib.sr_binning_bytes(cap, W, H),), dtype=torch.uint8, device=dev)
                _capi.call("sr_forward", *args, geom, binning, img, cap, nr_dev, host)
            else:
                need = M * int(lib.sr_render_bytes(P, cap, W, H))
                if render.arena is None or render.arena.numel() < need:
                    render.arena = None                  # release the smaller arena before allocating its successor
                    render.arena = torch.empty((need,), dtype=torch.uint8, device=dev)
                if render.anchors is not None:
                    _capi.call("sr_render_forward_anchors", *args, render.arena, cap, nr_dev, host, C.byref(render.anchors))
                elif render.contrib is None:
                    _capi.call("sr_render_forward", *args, render.arena, cap, nr_dev, host)
                elif render.lift is not None:
                    _capi.call("sr_render_forward_lift", *args, render.arena, cap, nr_dev, host, C.byref(render.contrib),
                               C.byref(render.lift))
                elif render.mask is not None:
                    _capi.call("sr_render_forward_contrib_masked", *args, render.arena, cap, nr_dev, host,
                               C.byref(render.contrib), C.byref(render.mask))
                else:
                    _capi.call("sr_render_forward_contrib", *args, render.arena, cap, nr_dev, host, C.byref(render.contrib))
            if nosync:
                _pending.append((host, key, cap, stream))
                if len(_pending) > _MAX_PENDING:
                    check_overflow()      # an unchecked backlog must not grow without bound (nor hide dropped frames)
                num_rendered = -1
                break
            stream.synchronize()
            words = host.tolist()
            num_rendered = [r for r, _ in words]
            status = 0
            for _, s in words:
                status |= s
            _cap_hint[key] = max(_cap_hint.get(key, 0), max(num_rendered)) if not _sync_mode else max(num_rendered)
            if status & _capi.SR_STATUS_PREFILTER:
                raise RuntimeError("Point is filtered although prefiltered is set. This shouldn't happen!")
            if status & _capi.SR_STATUS_OVERFLOW:
                if render is not None and render.contrib is not None and M > 1:
                    render.overflowed = [m for m, (_, st) in enumerate(words) if st & _capi.SR_STATUS_OVERFLOW]
                    break
                cap = _round_cap(int(max(num_rendered) * 1.1) + 4096)
                continue
            break
    return num_rendered, out_color, out_others, radii, geom, binning, img, out_feat


def _backward(M, frame_dim, strides, background, means3D, sh, colors, scales, rotations, features, viewmatrix, projmatrix,
              campos, radii, dL_dout_color, dL_dout_features, dL_dout_others, geomBuffer, binningBuffer, imageBuffer, degree,
              tan_fovx, tan_fovy, scale_modifier, debug, grad_scale=None, features_grad_scale=None, sum_shared=False,
              want_transmat=True, outs=None, intrinsics=None):
    """The one sr_backward call behind every _C backward; none when P = 0, whose gradients are zero-filled.  Inputs as
    for _forward; strides["opacity"] is the forward's opacity stride.  The feature planes' gradient is dL_dout_features,
    or the tail of dL_dout_color when that is None.  Each gradient is (M,P,.), or (P,.) without frame_dim and, under
    sum_shared, for an input the frames share.  Returns (dL_dmeans2D, dL_dcolors, dL_dopacity, dL_dmeans3D,
    dL_dtransMat, dL_dsh, dL_dscales, dL_drotations), and dL_dfeatures ninth when there are features."""
    dev = means3D.device
    P, H, W = int(means3D.shape[-2]), int(dL_dout_color.shape[-2]), int(dL_dout_color.shape[-1])
    N = H * W
    Msh = int(sh.shape[-2]) if sh is not None and sh.numel() != 0 else 0
    F = int(features.shape[-1]) if features is not None else 0
    cstride, fstride, dfeat_ptr = 3 * N, F * N, _ptr(dL_dout_features) if F else None
    if F and dL_dout_features is None:
        cstride = fstride = (3 + F) * N
        dfeat_ptr = dL_dout_color.data_ptr() + 3 * N * 4
    lead = (M,) if frame_dim else ()
    with torch.cuda.device(dev):
        alloc = torch.empty if P > 0 else torch.zeros

        def mk(name, *tail):   # (P,.) when the input is shared and the kernel sums over frames
            shape = ((P,) if (sum_shared and M > 1 and strides.get(name, 0) == 0) else lead + (P,)) + tail
            o = outs.get("dL_d" + name) if outs else None
            if o is not None:
                if (o.numel() != int(torch.Size(shape).numel()) or not o.is_contiguous() or o.dtype != torch.float32
                        or o.data_ptr() % 16 != 0):
                    raise RuntimeError(f"outs['dL_d{name}'] must be a contiguous, 16-byte aligned float32 tensor of {shape}")
                return o.view(shape)
            return alloc(shape, dtype=torch.float32, device=dev)
        dL_dmeans2D = alloc(lead + (P, 3), dtype=torch.float32, device=dev)
        dL_dmeans3D, dL_dcolors, dL_dopacity = mk("means3D", 3), mk("colors", 3), mk("opacity", 1)
        dL_dtransMat = alloc(lead + (P, 9), dtype=torch.float32, device=dev) \
            if (want_transmat or (M == 1 and not sum_shared)) else None
        dL_dsh, dL_dscales, dL_drotations = mk("sh", Msh, 3), mk("scales", 2), mk("rotations", 4)
        dL_dfeatures = mk("features", F) if F else None
        if P > 0:
            cap = _capacity_from_bytes(int(binningBuffer.numel()) // M, W, H)
            fr, frp = _frame(P, degree, Msh, W, H, tan_fovx, tan_fovy, scale_modifier, False, debug, intrinsics)
            flags = _capi.SR_BATCH_SUM_SHARED if sum_shared else 0
            if deterministic():
                nbytes = M * int(_capi.load().sr_backward_det_bytes(cap, F))
                scratch = torch.empty((nbytes,), dtype=torch.uint8, device=dev)
                bd = _capi.SrBatchDet(_capi.SrBatch(M, flags | _capi.SR_BATCH_DETERMINISTIC, *(strides.get(k, 0) for k in _STRIDED)),
                                      scratch.data_ptr(), nbytes)
                bt = bd.batch
            else:
                bt = _capi.SrBatch(M, flags, *(strides.get(k, 0) for k in _STRIDED))
            gs = fgs = None
            if grad_scale is not None:
                gs = grad_scale.to(device=dev, dtype=torch.float32).reshape(()).contiguous()
            if F and features_grad_scale is not None:
                fgs = features_grad_scale.to(device=dev, dtype=torch.float32).reshape(()).contiguous()
            _capi.call("sr_backward", dev, frp, C.byref(bt), _ptr(background), int(background.numel()), _ptr(means3D),
                       _ptr(sh), _ptr(colors), _ptr(scales), _ptr(rotations), _ptr(features), F, strides.get("features", 0),
                       _ptr(viewmatrix), _ptr(projmatrix), _ptr(campos), _ptr(radii), _ptr(dL_dout_color), cstride, dfeat_ptr,
                       fstride, _ptr(dL_dout_others), _ptr(gs), _ptr(fgs), geomBuffer, binningBuffer, imageBuffer, cap,
                       dL_dmeans2D, dL_dcolors, dL_dopacity, dL_dmeans3D, _ptr(dL_dtransMat), _ptr(dL_dsh), dL_dscales,
                       dL_drotations, _ptr(dL_dfeatures))
    grads = (dL_dmeans2D, dL_dcolors, dL_dopacity, dL_dmeans3D, dL_dtransMat, dL_dsh, dL_dscales, dL_drotations)
    return grads + (dL_dfeatures,) if F else grads


class _CNamespace:
    """Stand-in for the reference's pybind module `_C` with the same three entry points, plus the feature and batched
    variants.  Each checks its arguments' shapes and hands _forward / _backward normalised inputs."""

    @staticmethod
    def rasterize_gaussians(background, means3D, colors, opacity, scales, rotations, scale_modifier,
                            transMat_precomp, viewmatrix, projmatrix, tan_fovx, tan_fovy, image_height,
                            image_width, sh, degree, campos, prefiltered, debug):
        return _CNamespace.rasterize_gaussians_features(
            background, means3D, colors, opacity, scales, rotations, scale_modifier, transMat_precomp, viewmatrix,
            projmatrix, tan_fovx, tan_fovy, image_height, image_width, sh, degree, campos, prefiltered, debug, None)

    @staticmethod
    def rasterize_gaussians_features(background, means3D, colors, opacity, scales, rotations, scale_modifier,
                                     transMat_precomp, viewmatrix, projmatrix, tan_fovx, tan_fovy, image_height,
                                     image_width, sh, degree, campos, prefiltered, debug, features):
        """rasterize_gaussians plus per-surfel features (P,F), 1 <= F <= 32 (not in the reference): out_color is
        (3+F,H,W) -- the colour planes, then F feature planes composited with the colour's weights over a background of
        background[3:] (background of 3+F values) or zeros (background of 3).  features=None is rasterize_gaussians."""
        if means3D.ndim != 2 or means3D.shape[1] != 3:
            raise RuntimeError("means3D must have dimensions (num_points, 3)")
        if scales.ndim != 2 or scales.shape[1] != 2:
            raise RuntimeError("scales must have dimensions (num_points, 2)")
        if rotations.ndim != 2 or rotations.shape[1] != 4:
            raise RuntimeError("rotations must have dimensions (num_points, 4)")
        if transMat_precomp is not None and transMat_precomp.numel() != 0:
            raise RuntimeError("precomputed transMat / cov3D is not supported (the reference path for it is "
                               "broken: forward.cu:214-218 leaves the normal uninitialised)")
        background = _f32c(background, "background"); means3D = _f32c(means3D, "means3D")
        colors = _f32c(colors, "colors"); opacity = _f32c(opacity, "opacity")
        scales = _f32c(scales, "scales"); rotations = _f32c(rotations, "rotations")
        viewmatrix = _f32c(viewmatrix, "viewmatrix"); projmatrix = _f32c(projmatrix, "projmatrix")
        sh = _f32c(sh, "sh"); campos = _f32c(campos, "campos")
        if features is not None:
            _check_features(features, int(means3D.shape[0]), background)
            features = _f32c(features, "features")
        # one frame: M = 1 explicitly (viewmatrix is (4,4), campos (3,)), outputs without a frame dimension
        out = _forward(1, False, {}, background, means3D, sh, colors, opacity, scales, rotations, features, viewmatrix,
                       projmatrix, campos, int(image_height), int(image_width), degree, tan_fovx, tan_fovy, scale_modifier,
                       prefiltered, debug)
        return (-1 if out[0] == -1 else out[0][0],) + out[1:7]

    @staticmethod
    def rasterize_gaussians_backward(background, means3D, radii, colors, scales, rotations, scale_modifier,
                                     transMat_precomp, viewmatrix, projmatrix, tan_fovx, tan_fovy,
                                     dL_dout_color, dL_dout_others, sh, degree, campos, geomBuffer, R,
                                     binningBuffer, imageBuffer, debug):
        return _CNamespace.rasterize_gaussians_features_backward(
            background, means3D, radii, colors, scales, rotations, scale_modifier, transMat_precomp, viewmatrix,
            projmatrix, tan_fovx, tan_fovy, dL_dout_color, dL_dout_others, sh, degree, campos, geomBuffer, R,
            binningBuffer, imageBuffer, debug, None)

    @staticmethod
    def rasterize_gaussians_features_backward(background, means3D, radii, colors, scales, rotations, scale_modifier,
                                              transMat_precomp, viewmatrix, projmatrix, tan_fovx, tan_fovy,
                                              dL_dout_color, dL_dout_others, sh, degree, campos, geomBuffer, R,
                                              binningBuffer, imageBuffer, debug, features):
        """Backward of rasterize_gaussians_features: dL_dout_color is (3+F,H,W); returns the eight gradients of
        rasterize_gaussians_backward and dL_dfeatures (P,F).  features=None is rasterize_gaussians_backward."""
        if features is not None:
            F = _check_features(features, int(means3D.shape[0]), background)
            features = _f32c(features, "features")
            H, W = int(dL_dout_color.shape[1]), int(dL_dout_color.shape[2])
            if tuple(dL_dout_color.shape) != (3 + F, H, W):
                raise RuntimeError(f"dL_dout_color must be (3+F,H,W) = {(3 + F, H, W)}, got {tuple(dL_dout_color.shape)}")
        background = _f32c(background, "background"); means3D = _f32c(means3D, "means3D")
        colors = _f32c(colors, "colors"); scales = _f32c(scales, "scales"); rotations = _f32c(rotations, "rotations")
        viewmatrix = _f32c(viewmatrix, "viewmatrix"); projmatrix = _f32c(projmatrix, "projmatrix")
        sh = _f32c(sh, "sh"); campos = _f32c(campos, "campos")
        dL_dout_color = _f32c(dL_dout_color, "dL_dout_color"); dL_dout_others = _f32c(dL_dout_others, "dL_dout_others")
        return _backward(1, False, {}, background, means3D, sh, colors, scales, rotations, features, viewmatrix, projmatrix,
                         campos, radii, dL_dout_color, None, dL_dout_others, geomBuffer, binningBuffer, imageBuffer, degree,
                         tan_fovx, tan_fovy, scale_modifier, debug)

    # ---- batched entry points (SURVEY.md 8(f) N1): M frames in one launch set -------------------------------------
    @staticmethod
    def rasterize_gaussians_batch(background, means3D, colors, opacity, scales, rotations, scale_modifier, viewmatrix,
                                  projmatrix, tan_fovx, tan_fovy, image_height, image_width, sh, degree, campos,
                                  prefiltered=False, debug=False, features=None, concat=True, intrinsics=None):
        """M frames at once.  viewmatrix / projmatrix (M,4,4), campos (M,3).  Every per-surfel input is either shared by
        all frames -- the single-frame shape, e.g. means3D (P,3) -- or per frame with a leading M, e.g. (M,P,3) (Stage 3:
        each frame rasterizes its own warped copy of the surfels).  Returns (num_rendered (list of M ints, or -1 in nosync
        mode), out_color (M,3,H,W), out_others (M,8,H,W), radii (M,P), geomBuffer, binningBuffer, imgBuffer).
        features (P,F) shared or (M,P,F) per frame, 1 <= F <= 32: an eighth element, the (M,F,H,W) feature planes, is
        returned; with concat=True out_color is (M,3+F,H,W) and the feature planes are its view [:, 3:], with concat=False
        the two are separate tensors.
        intrinsics: optional (M,4) float32 CUDA table, frame m's row (tan_fovx, tan_fovy, cx_off, cy_off) with the principal
        point at (W/2 + cx_off, H/2 + cy_off) (include/surfel_camera.h; renderer.camera_table builds it from K).  The kernels
        read it from device memory, so tan_fovx / tan_fovy are not read, nothing synchronises, and a captured call renders
        with what the table holds at replay."""
        M = int(viewmatrix.shape[0])
        if viewmatrix.ndim != 3 or viewmatrix.shape[1:] != (4, 4) or campos.shape != (M, 3):
            raise RuntimeError("batched cameras: viewmatrix must be (M,4,4) and campos (M,3)")
        background = _f32c(background, "background"); viewmatrix = _f32c(viewmatrix, "viewmatrix")
        projmatrix = _f32c(projmatrix, "projmatrix"); campos = _f32c(campos, "campos")
        if features is not None:
            _check_features(features, int(means3D.shape[-2]), background, batched=True)
        intrinsics = _check_intrinsics(intrinsics, M, means3D)
        ins, strides = _batch_inputs(M, means3D=(means3D, (3,)), sh=(sh, None), colors=(colors, (3,)), opacity=(opacity, (1,)),
                                     scales=(scales, (2,)), rotations=(rotations, (4,)), features=(features, None))
        out = _forward(M, True, strides, background, ins["means3D"], ins["sh"], ins["colors"], ins["opacity"], ins["scales"],
                       ins["rotations"], ins["features"], viewmatrix, projmatrix, campos, int(image_height),
                       int(image_width), degree, tan_fovx, tan_fovy, scale_modifier, prefiltered, debug, concat, intrinsics)
        return out if features is not None else out[:7]

    @staticmethod
    def rasterize_gaussians_backward_batch(background, means3D, radii, colors, scales, rotations, scale_modifier, viewmatrix,
                                           projmatrix, tan_fovx, tan_fovy, dL_dout_color, dL_dout_others, sh, degree, campos,
                                           geomBuffer, binningBuffer, imageBuffer, grad_scale=None, debug=False,
                                           sum_shared=False, opacity_shared=True, want_transmat=True, outs=None,
                                           features=None, dL_dout_features=None, features_grad_scale=None, intrinsics=None):
        """Backward of rasterize_gaussians_batch.  dL_dout_color (M,3,H,W), dL_dout_others (M,8,H,W); grad_scale: optional
        0-d device tensor multiplying both (the upstream scalar of a fused loss).  Returns the eight gradient tensors
        (dL_dmeans2D, dL_dcolors, dL_dopacity, dL_dmeans3D, dL_dtransMat, dL_dsh, dL_dscales, dL_drotations), each with a
        leading M: (M,P,.).  With sum_shared=True the gradients of inputs the frames SHARE come back summed over the frames
        with the input's own shape (P,.) -- the per-surfel kernel accumulates them in place, nothing (M,P,.)-sized is
        written or reduced; `opacity_shared` says whether the forward's opacities were shared (they are not an input of
        the backward); dL_dmeans2D stays (M,P,3); want_transmat=False skips the (M,P,9) by-product.
        outs: optional {"dL_dmeans3D" | "dL_dsh" | "dL_dopacity" | "dL_dscales" | "dL_drotations" | "dL_dcolors": tensor}
        of pre-allocated, suitably shaped and aligned outputs (e.g. views of the flat buffer an all-reduce runs over).
        features (P,F) or (M,P,F): the gradient of the feature planes is either the tail of dL_dout_color (M,3+F,H,W) or a
        separate dL_dout_features (M,F,H,W) (then dL_dout_color is (M,3,H,W)); features_grad_scale (optional 0-d device
        tensor) multiplies it instead of grad_scale.  A ninth gradient, dL_dfeatures, is returned: (M,P,F), or (P,F) for
        shared features with sum_shared=True.  intrinsics: the forward's (M,4) camera table, or None."""
        M = int(viewmatrix.shape[0])
        H, W = int(dL_dout_color.shape[-2]), int(dL_dout_color.shape[-1])
        background = _f32c(background, "background"); viewmatrix = _f32c(viewmatrix, "viewmatrix")
        projmatrix = _f32c(projmatrix, "projmatrix"); campos = _f32c(campos, "campos")
        dL_dout_color = _f32c(dL_dout_color, "dL_dout_color"); dL_dout_others = _f32c(dL_dout_others, "dL_dout_others")
        if features is not None:
            F = _check_features(features, int(means3D.shape[-2]), background, batched=True)
            if dL_dout_features is None:
                if tuple(dL_dout_color.shape) != (M, 3 + F, H, W):
                    raise RuntimeError(f"dL_dout_color must be (M,3+F,H,W) = {(M, 3 + F, H, W)} without dL_dout_features")
            else:
                dL_dout_features = _f32c(dL_dout_features, "dL_dout_features")
                if tuple(dL_dout_features.shape) != (M, F, H, W) or tuple(dL_dout_color.shape) != (M, 3, H, W):
                    raise RuntimeError("dL_dout_color must be (M,3,H,W) and dL_dout_features (M,F,H,W)")
        intrinsics = _check_intrinsics(intrinsics, M, means3D)
        ins, strides = _batch_inputs(M, means3D=(means3D, (3,)), sh=(sh, None), colors=(colors, (3,)),
                                     scales=(scales, (2,)), rotations=(rotations, (4,)), features=(features, None))
        strides["opacity"] = 0 if (opacity_shared or M == 1) else int(ins["means3D"].shape[-2])
        return _backward(M, True, strides, background, ins["means3D"], ins["sh"], ins["colors"], ins["scales"],
                         ins["rotations"], ins["features"], viewmatrix, projmatrix, campos, radii, dL_dout_color,
                         dL_dout_features, dL_dout_others, geomBuffer, binningBuffer, imageBuffer, degree, tan_fovx,
                         tan_fovy, scale_modifier, debug, grad_scale, features_grad_scale, sum_shared, want_transmat, outs,
                         intrinsics)

    @staticmethod
    def mark_visible(means3D, viewmatrix, projmatrix):
        dev = means3D.device
        P = int(means3D.shape[0])
        present = torch.zeros((P,), dtype=torch.bool, device=dev)
        if P:
            means3D = _f32c(means3D, "means3D"); viewmatrix = _f32c(viewmatrix, "viewmatrix")
            projmatrix = _f32c(projmatrix, "projmatrix")
            _capi.call("sr_mark_visible", dev, P, _ptr(means3D), _ptr(viewmatrix), _ptr(projmatrix), present)
        return present


_C = _CNamespace()


def cpu_deep_copy_tuple(input_tuple):
    return tuple(item.cpu().clone() if isinstance(item, torch.Tensor) else item for item in input_tuple)


def rasterize_gaussians(means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                        raster_settings, features=None):
    """features (P,F), 1 <= F <= 32: the colour output is (3+F,H,W), feature planes after the colour planes."""
    return _RasterizeGaussians.apply(means3D, means2D, sh, colors_precomp, opacities, scales, rotations,
                                     cov3Ds_precomp, raster_settings, features)


class _RasterizeGaussians(torch.autograd.Function):
    @staticmethod
    def forward(ctx, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                raster_settings, features=None):
        args = (raster_settings.bg, means3D, colors_precomp, opacities, scales, rotations,
                raster_settings.scale_modifier, cov3Ds_precomp, raster_settings.viewmatrix,
                raster_settings.projmatrix, raster_settings.tanfovx, raster_settings.tanfovy,
                raster_settings.image_height, raster_settings.image_width, sh, raster_settings.sh_degree,
                raster_settings.campos, raster_settings.prefiltered, raster_settings.debug)
        fwd = _C.rasterize_gaussians if features is None else \
            (lambda *a: _C.rasterize_gaussians_features(*a, features))  # noqa: E731
        if raster_settings.debug:
            cpu_args = cpu_deep_copy_tuple(args)
            try:
                num_rendered, color, depth, radii, geomBuffer, binningBuffer, imgBuffer = fwd(*args)
            except Exception as ex:
                torch.save(cpu_args, "snapshot_fw.dump")
                print("\nAn error occured in forward. Please forward snapshot_fw.dump for debugging.")
                raise ex
        else:
            num_rendered, color, depth, radii, geomBuffer, binningBuffer, imgBuffer = fwd(*args)
        ctx.raster_settings = raster_settings
        ctx.num_rendered = num_rendered
        ctx.has_features = features is not None
        # only inputs + private buffers are saved (never our own outputs): the caller edits `color` in place
        # before backward (deformable_gaussian.py:188-190)
        ctx.save_for_backward(colors_precomp, means3D, scales, rotations, cov3Ds_precomp, radii, sh, geomBuffer,
                              binningBuffer, imgBuffer, features)
        ctx.mark_non_differentiable(radii)
        return color, radii, depth

    @staticmethod
    def backward(ctx, grad_out_color, grad_radii, grad_depth):
        num_rendered = ctx.num_rendered
        raster_settings = ctx.raster_settings
        (colors_precomp, means3D, scales, rotations, cov3Ds_precomp, radii, sh, geomBuffer, binningBuffer, imgBuffer,
         features) = ctx.saved_tensors
        F = int(features.shape[-1]) if ctx.has_features else 0
        if grad_out_color is None:
            grad_out_color = torch.zeros((3 + F, raster_settings.image_height, raster_settings.image_width),
                                         dtype=torch.float32, device=means3D.device)
        if grad_depth is None:
            grad_depth = torch.zeros((8, raster_settings.image_height, raster_settings.image_width),
                                     dtype=torch.float32, device=means3D.device)
        args = (raster_settings.bg, means3D, radii, colors_precomp, scales, rotations, raster_settings.scale_modifier,
                cov3Ds_precomp, raster_settings.viewmatrix, raster_settings.projmatrix, raster_settings.tanfovx,
                raster_settings.tanfovy, grad_out_color, grad_depth, sh, raster_settings.sh_degree,
                raster_settings.campos, geomBuffer, num_rendered, binningBuffer, imgBuffer, raster_settings.debug)
        bwd = _C.rasterize_gaussians_backward if not F else \
            (lambda *a: _C.rasterize_gaussians_features_backward(*a, features))  # noqa: E731
        if raster_settings.debug:
            cpu_args = cpu_deep_copy_tuple(args)
            try:
                grads8 = bwd(*args)
            except Exception as ex:
                torch.save(cpu_args, "snapshot_bw.dump")
                print("\nAn error occured in backward. Writing snapshot_bw.dump for debugging.\n")
                raise ex
        else:
            grads8 = bwd(*args)
        grad_features = grads8[8] if F else None
        grad_means2D, grad_colors_precomp, grad_opacities, grad_means3D, grad_cov3Ds_precomp, grad_sh, grad_scales, grad_rotations = grads8[:8]
        # the reference returns a gradient for every input slot, including the "not provided" empty tensors
        if colors_precomp.numel() == 0:
            grad_colors_precomp = None
        if sh.numel() == 0:
            grad_sh = None
        if cov3Ds_precomp.numel() == 0:
            grad_cov3Ds_precomp = None
        if grad_features is not None:
            grad_features = grad_features.view(features.shape)
        return (grad_means3D, grad_means2D, grad_sh, grad_colors_precomp, grad_opacities, grad_scales,
                grad_rotations, grad_cov3Ds_precomp, None, grad_features)


class BatchRasterizationSettings(NamedTuple):
    """GaussianRasterizationSettings for M frames: viewmatrix / projmatrix are (M,4,4), campos is (M,3).  intrinsics:
    optional (M,4) float32 CUDA table of per-frame (tan_fovx, tan_fovy, cx_off, cy_off); when set, tanfovx / tanfovy are
    not read (see _C.rasterize_gaussians_batch)."""
    image_height: int
    image_width: int
    tanfovx: float
    tanfovy: float
    bg: torch.Tensor
    scale_modifier: float
    viewmatrix: torch.Tensor
    projmatrix: torch.Tensor
    sh_degree: int
    campos: torch.Tensor
    prefiltered: bool = False
    debug: bool = False
    intrinsics: Optional[torch.Tensor] = None


def _reduce_like(grad, inp):
    """(M,P,.) per-frame gradient -> the input's shape: inputs shared by all frames get the sum over frames."""
    if inp is None or inp.numel() == 0:
        return None
    if grad.ndim == inp.ndim:                 # per-frame input, or already summed over the frames by the kernel
        return grad.view(inp.shape)
    return grad.sum(dim=0).view(inp.shape)


class _RasterizeGaussiansBatch(torch.autograd.Function):
    """M frames in one launch set (SURVEY.md 8(f) N1).  Inputs are shared (single-frame shape) or per frame (leading M);
    means2D is (M,P,3) and only receives the densification proxy gradient, as in the single-frame op."""

    @staticmethod
    def forward(ctx, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, rs, features=None):
        kw = {} if features is None else {"features": features}
        if getattr(rs, "intrinsics", None) is not None:     # settings without the field (GaussianRasterizationSettings) work too
            kw["intrinsics"] = rs.intrinsics
        num_rendered, color, allmap, radii, geomBuffer, binningBuffer, imgBuffer = _C.rasterize_gaussians_batch(
            rs.bg, means3D, colors_precomp, opacities, scales, rotations, rs.scale_modifier, rs.viewmatrix, rs.projmatrix,
            rs.tanfovx, rs.tanfovy, rs.image_height, rs.image_width, sh, rs.sh_degree, rs.campos, rs.prefiltered, rs.debug,
            **kw)[:7]
        ctx.rs = rs
        ctx.has_features = features is not None
        ctx.save_for_backward(colors_precomp, means3D, scales, rotations, radii, sh, opacities, geomBuffer, binningBuffer, imgBuffer,
                              features)
        ctx.mark_non_differentiable(radii)
        return color, radii, allmap

    @staticmethod
    def backward(ctx, grad_color, grad_radii, grad_allmap):
        rs = ctx.rs
        (colors_precomp, means3D, scales, rotations, radii, sh, opacities, geomBuffer, binningBuffer, imgBuffer,
         features) = ctx.saved_tensors
        M = int(rs.viewmatrix.shape[0])
        H, W = rs.image_height, rs.image_width
        F = int(features.shape[-1]) if ctx.has_features else 0
        if grad_color is None:
            grad_color = torch.zeros((M, 3 + F, H, W), dtype=torch.float32, device=means3D.device)
        if grad_allmap is None:
            grad_allmap = torch.zeros((M, 8, H, W), dtype=torch.float32, device=means3D.device)
        kw = {"features": features} if F else {}
        if getattr(rs, "intrinsics", None) is not None:     # settings without the field (GaussianRasterizationSettings) work too
            kw["intrinsics"] = rs.intrinsics
        grads = _C.rasterize_gaussians_backward_batch(
            rs.bg, means3D, radii, colors_precomp, scales, rotations, rs.scale_modifier, rs.viewmatrix, rs.projmatrix,
            rs.tanfovx, rs.tanfovy, grad_color, grad_allmap, sh, rs.sh_degree, rs.campos, geomBuffer, binningBuffer, imgBuffer,
            None, rs.debug, sum_shared=True, opacity_shared=opacities.ndim == 2, want_transmat=False, **kw)
        g2d, gcol, gop, g3d, gtm, gsh, gsc, grot = grads[:8]
        return (_reduce_like(g3d, means3D), g2d, _reduce_like(gsh, sh), _reduce_like(gcol, colors_precomp),
                _reduce_like(gop, opacities), _reduce_like(gsc, scales), _reduce_like(grot, rotations), None,
                _reduce_like(grads[8], features) if F else None)


def rasterize_gaussians_batch(means3D, means2D, shs, colors_precomp, opacities, scales, rotations, raster_settings,
                              features=None):
    """Batched twin of rasterize_gaussians: returns (color (M,3,H,W), radii (M,P), allmap (M,8,H,W)).
    features (P,F) shared or (M,P,F) per frame, 1 <= F <= 32: color is (M,3+F,H,W), feature planes after the colour."""
    dev = means3D.device
    empty = lambda: torch.empty((0,), dtype=torch.float32, device=dev)  # noqa: E731
    if (shs is None) == (colors_precomp is None):
        raise Exception('Please provide excatly one of either SHs or precomputed colors!')
    return _RasterizeGaussiansBatch.apply(means3D, means2D, empty() if shs is None else shs,
                                          empty() if colors_precomp is None else colors_precomp, opacities, scales, rotations,
                                          raster_settings, features)


class GaussianRasterizationSettings(NamedTuple):
    image_height: int
    image_width: int
    tanfovx: float
    tanfovy: float
    bg: torch.Tensor
    scale_modifier: float
    viewmatrix: torch.Tensor
    projmatrix: torch.Tensor
    sh_degree: int
    campos: torch.Tensor
    prefiltered: bool
    debug: bool


class GaussianRasterizer(nn.Module):
    def __init__(self, raster_settings):
        super().__init__()
        self.raster_settings = raster_settings

    def markVisible(self, positions):
        with torch.no_grad():
            raster_settings = self.raster_settings
            visible = _C.mark_visible(positions, raster_settings.viewmatrix, raster_settings.projmatrix)
        return visible

    def forward(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None,
                cov3D_precomp=None):
        return self._rasterize(means3D, means2D, opacities, shs, colors_precomp, scales, rotations, cov3D_precomp, None)

    def forward_features(self, means3D, means2D, opacities, features, shs=None, colors_precomp=None, scales=None,
                         rotations=None, cov3D_precomp=None):
        """forward() plus per-surfel channels (not in the reference; forward() keeps the reference's signature so that
        the class stays a drop-in): features (P,F), 1 <= F <= 32, composited with the colour's weights and independent
        of where the colour comes from.  The returned colour is (3+F,H,W) -- RGB, then the F feature planes (background:
        raster_settings.bg[3:] when bg has 3+F values, else 0)."""
        if features is None:
            raise RuntimeError("forward_features needs a features tensor (P,F)")
        return self._rasterize(means3D, means2D, opacities, shs, colors_precomp, scales, rotations, cov3D_precomp, features)

    def _rasterize(self, means3D, means2D, opacities, shs, colors_precomp, scales, rotations, cov3D_precomp, features):
        raster_settings = self.raster_settings
        if (shs is None and colors_precomp is None) or (shs is not None and colors_precomp is not None):
            raise Exception('Please provide excatly one of either SHs or precomputed colors!')
        if ((scales is None or rotations is None) and cov3D_precomp is None) or \
                ((scales is not None or rotations is not None) and cov3D_precomp is not None):
            raise Exception('Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!')
        dev = means3D.device
        empty = lambda: torch.empty((0,), dtype=torch.float32, device=dev)  # noqa: E731
        if shs is None:
            shs = empty()
        if colors_precomp is None:
            colors_precomp = empty()
        if scales is None:
            scales = empty()
        if rotations is None:
            rotations = empty()
        if cov3D_precomp is None:
            cov3D_precomp = empty()
        if features is not None:
            _check_features(features, int(means3D.shape[0]), raster_settings.bg)
        return rasterize_gaussians(means3D, means2D, shs, colors_precomp, opacities, scales, rotations,
                                   cov3D_precomp, raster_settings, features)
