"""TEST INFRASTRUCTURE -- the binning stage restated as integer NumPy: every buffer it writes, predicted exactly.

Binning turns each visible surfel's tile rectangle into (tile | depth) instances and sorts them:

  * emit_keys (csrc/preprocess.cu) emits, in ascending surfel id and row-major over the surfel's tile rectangle
    (sr_tile_rect, csrc/common.cuh), the key (tile << 32) | depth bits and the value surfel id; point_offsets is the
    inclusive scan of tiles_touched.  R, the number of instances, is the sum of the rectangles' areas; a frame with
    R > capacity is abandoned (its status word gets the overflow bit and no instance is written);
  * the onesweep LSD radix sort (csrc/sort.cu) sorts the keys stably in ceil(key_bits / 8) passes of 8 bits (the last
    pass may be narrower), key_bits = 32 + getHigherMsb(tiles).  Its plan skips a pass whose digit every key shares (and
    every pass of an empty or abandoned frame), and keeps the ping/pong parity in the sort control words;
  * ranges_gather writes each tile's [start, end) in the sorted list ((0, 0) when empty) and the 80-byte instance
    records: the sorted surfel's record with float 18 replaced by the surfel id and float 19 by the cull word
    (tests/cull_model.py);
  * tile_order lists the tiles by bucket floor(log2(len)) + 1 (0 when empty), largest bucket first; the order within a
    bucket comes from shared-memory atomics, so only that property is predicted.

The model's inputs are the per-surfel values binning reads: the rectangle's centre (surfel_rec floats 9 and 10), the
integer radius and the depth.  On the GPU those are the GPU's own records (tests/preprocess_bounds.py pins them to the
inputs); in tests/test_binning_model_cpu.py they are the reference's.
"""
import numpy as np

from . import cull_model as cm

F32 = np.float32
TILE = 16
RADIX_BITS = 8
MAX_PASSES = 8
SORT_TILE = 256 * 12                 # keys per onesweep tile (SR_SORT_TILE)
CTL_WORDS = 64
CTL_SORTED_SEL, CTL_NPASS, CTL_SKIP, CTL_SRC, CTL_TILE_COUNTER = 0, 1, 8, 16, 24


def higher_msb(n):
    """getHigherMsb (rasterizer_impl.cu), the bisection the library's sr_higher_msb runs."""
    n = int(n)
    msb = step = 16
    while step > 1:
        step //= 2
        msb = msb + step if n >> msb else msb - step
    if n >> msb:
        msb += 1
    return msb


def key_bits(tiles):
    return 32 + higher_msb(tiles)


def pass_plan(kbits):
    """[(shift, bits)] of the sort's passes: 8-bit digits from the bottom, the last one narrower if kbits % 8 != 0."""
    return [(s, min(RADIX_BITS, kbits - s)) for s in range(0, kbits, RADIX_BITS)][:MAX_PASSES]


def tile_rect(px, py, radii, gx, gy):
    """sr_tile_rect in fp32 with the kernel's operation order: (x0, y0, x1, y1) int64, each clamped to [0, grid].  The
    float-to-int conversions truncate toward zero and saturate (NaN -> 0) as cvt.rzi.s32.f32 does."""
    px, py = np.asarray(px, F32), np.asarray(py, F32)
    r = np.asarray(radii).astype(F32)
    with np.errstate(all="ignore"):
        lo_x, lo_y = (px - r) * F32(0.0625), (py - r) * F32(0.0625)
        hi_x = (((px + r) + F32(16)) - F32(1)) * F32(0.0625)
        hi_y = (((py + r) + F32(16)) - F32(1)) * F32(0.0625)

    def cvt(v, g):
        v = np.trunc(np.clip(np.nan_to_num(v.astype(np.float64), nan=0.0), -2.0 ** 31, 2.0 ** 31 - 1)).astype(np.int64)
        return np.minimum(g, np.maximum(0, v))
    return cvt(lo_x, gx), cvt(lo_y, gy), cvt(hi_x, gx), cvt(hi_y, gy)


def _pass_digits(keys, shift, bits):
    return ((keys >> np.uint64(shift)) & np.uint64((1 << bits) - 1)).astype(np.int64)


def sort_ctl(keys, R, tiles, overflow):
    """The 64 sort control words the plan and pass kernels leave: sorted_sel, npass, skip[p], src[p] and the tickets
    pass p handed out (one per 3072-key sort tile it ran)."""
    plan = pass_plan(key_bits(tiles))
    ctl = np.zeros(CTL_WORDS, np.uint32)
    dead = overflow or R == 0
    sel = 0
    for p, (shift, bits) in enumerate(plan):
        skip = dead or bool((_pass_digits(keys, shift, bits) == _pass_digits(keys[:1], shift, bits)).all())
        ctl[CTL_SRC + p] = sel
        ctl[CTL_SKIP + p] = skip
        ctl[CTL_TILE_COUNTER + p] = 0 if skip else -(-R // SORT_TILE)
        if not skip:
            sel ^= 1
    ctl[CTL_SORTED_SEL] = sel
    ctl[CTL_NPASS] = len(plan)
    return ctl


def predict(px, py, radii, depths, W, H, capacity):
    """Everything binning writes for one frame, from the centres (px, py) (fp32), integer radii (0: not visible) and fp32
    depths of its P surfels.  Returns a dict: tiles_touched, point_offsets (uint32, P), R, overflow, keys_unsorted,
    values_unsorted (emission order), keys, point_list (sorted), ranges (tiles, 2) uint32, sort_ctl (64) uint32,
    rect (x0, y0, x1, y1) and the grid (tiles_x, tiles_y).  The instance arrays are empty when the frame overflows."""
    gx, gy = (W + TILE - 1) // TILE, (H + TILE - 1) // TILE
    tiles = gx * gy
    radii = np.asarray(radii).astype(np.int64)
    vis = radii > 0
    x0, y0, x1, y1 = tile_rect(px, py, radii, gx, gy)
    w = np.where(vis, x1 - x0, 0)
    area = np.where(vis, w * (y1 - y0), 0)
    R = int(area.sum())
    overflow = R > capacity
    out = dict(tiles_touched=area.astype(np.uint32), point_offsets=np.cumsum(area).astype(np.uint32), R=R,
               overflow=overflow, rect=(x0, y0, x1, y1), grid=(gx, gy))
    if overflow:
        keys = vals = np.zeros(0, np.uint64)
    else:
        vals = np.repeat(np.arange(len(area), dtype=np.int64), area)
        t = np.arange(R, dtype=np.int64) - np.repeat(np.cumsum(area) - area, area)       # row-major index in the rectangle
        wv = w[vals]
        tile = (y0[vals] + t // np.maximum(wv, 1)) * gx + x0[vals] + t % np.maximum(wv, 1)
        dbits = np.asarray(depths, F32).view(np.uint32).astype(np.uint64)[vals]
        keys = (tile.astype(np.uint64) << np.uint64(32)) | dbits
    order = np.argsort(keys, kind="stable")
    skeys = keys[order]
    stile = (skeys >> np.uint64(32)).astype(np.int64)
    ids = np.arange(tiles)
    lo, hi = np.searchsorted(stile, ids, "left"), np.searchsorted(stile, ids, "right")
    ranges = np.where((hi > lo)[:, None], np.stack([lo, hi], 1), 0).astype(np.uint32)
    out.update(keys_unsorted=keys, values_unsorted=vals.astype(np.uint32), keys=skeys,
               point_list=vals[order].astype(np.uint32), ranges=ranges, sort_ctl=sort_ctl(keys, R, tiles, overflow))
    return out


def inst_records(surfel_rec, point_list, keys, tiles_x):
    """The instance records (R, 20) as uint32 bits: the sorted surfel's record, float 18 its id, float 19 its cull word.
    Returns (lo, hi): the records with the smallest and the largest rho-cut bits the kernel's logf may give (equal
    wherever cull_model.rho_cut_words is)."""
    rec = np.ascontiguousarray(surfel_rec, F32).view(np.uint32)
    sid = np.asarray(point_list).astype(np.int64)
    tile = (np.asarray(keys, np.uint64) >> np.uint64(32)).astype(np.int64)
    bx, by = rec[sid, 18], rec[sid, 19]
    lo_w, hi_w = cm.rho_cut_words(rec[:, 11].view(F32))
    out = []
    for words in (lo_w, hi_w):
        r = rec[sid].copy()
        r[:, 18] = sid.astype(np.uint32)
        r[:, 19] = cm.cull_word(bx, by, tile, tiles_x, words[sid])
        out.append(r)
    return out[0], out[1]


def bucket(lengths):
    """tile_order's bucket of each tile: 0 when empty, else floor(log2(len)) + 1."""
    n = np.asarray(lengths).astype(np.int64)
    return np.where(n > 0, np.frexp(n.astype(np.float64))[1], 0).astype(np.int64)    # frexp: the bit length, exactly


def check_tile_order(order, ranges):
    """The tile order is a permutation of [0, tiles) whose buckets never increase.  Returns a failure message or None."""
    order = np.asarray(order).astype(np.int64)
    rg = np.asarray(ranges).astype(np.int64)
    tiles = rg.shape[0]
    if order.shape != (tiles,) or not np.array_equal(np.sort(order), np.arange(tiles)):
        return f"not a permutation of [0, {tiles})"
    b = bucket(rg[order, 1] - rg[order, 0])
    up = np.nonzero(b[1:] > b[:-1])[0]
    if up.size:
        i = int(up[0])
        return f"bucket rises at position {i + 1}: tile {order[i]} bucket {b[i]} then tile {order[i + 1]} bucket {b[i + 1]}"
    return None
