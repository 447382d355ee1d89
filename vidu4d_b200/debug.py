"""Views into the library's opaque buffers (sr_debug_view) -- used by the parity tests to compare
(tile|depth) keys, the sorted surfel list and the tile ranges with the reference, bit for bit."""
from __future__ import annotations

import ctypes as C

import torch

from . import _capi
from .rasterizer import _capacity_from_bytes


def decode(geomBuffer, binningBuffer, imgBuffer, P: int, W: int, H: int, num_rendered: int) -> dict:
    lib = _capi.load()
    cap = _capacity_from_bytes(int(binningBuffer.numel()), W, H)
    L = _capi.SrDebugLayout()
    _capi.check(lib.sr_debug_view(P, W, H, cap, C.byref(L)), "sr_debug_view")
    N, R = W * H, int(num_rendered)
    tiles = ((W + 15) // 16) * ((H + 15) // 16)

    def view(buf, off, count, dtype):
        sz = torch.empty((), dtype=dtype).element_size()
        return buf[off:off + count * sz].view(dtype)

    ctl = view(binningBuffer, L.sort_ctl, 64, torch.int32)
    sel = int(ctl[0].item())
    out = {
        "surfel_rec": view(geomBuffer, L.surfel_rec, P * 20, torch.float32).view(P, 20),
        "depths": view(geomBuffer, L.depths, P, torch.float32),
        "tiles_touched": view(geomBuffer, L.tiles_touched, P, torch.int32),
        "point_offsets": view(geomBuffer, L.point_offsets, P, torch.int32),
        "clamped": view(geomBuffer, L.clamped, P, torch.uint8),
        "keys_unsorted": view(binningBuffer, L.keys[0], R, torch.int64),   # valid only if no pass wrote back into ping
        "keys": view(binningBuffer, L.keys[sel], R, torch.int64),
        "point_list": view(binningBuffer, L.values[sel], R, torch.int32),
        "inst_rec": view(binningBuffer, L.inst_rec, R * 20, torch.float32).view(R, 20),
        "sort_ctl": ctl,
        "final_T": view(imgBuffer, L.final_T, 3 * N, torch.float32).view(3, H, W),
        "n_contrib": view(imgBuffer, L.n_contrib, 2 * N, torch.int32).view(2, H, W),
        "ranges": view(imgBuffer, L.ranges, 2 * tiles, torch.int32).view(tiles, 2),
        "sub_last": view(imgBuffer, L.sub_last, 8 * tiles, torch.int32).view(tiles, 8),
        "contrib_masks": view(binningBuffer, L.contrib, ((cap >> 5) + tiles + 1) * 256, torch.int32).view(-1, 8, 32),
    }
    return out


def _lane_counts(dec: dict) -> torch.Tensor:
    """(tiles, 8, 32) int64: per tile, 8 x 4 sub-tile and lane, the population count of the contribution masks the
    forward recorded, over the stages the backward reads (stage s of tile t is row (range.x >> 5) + t + s; a sub-tile's
    stages end at its deepest contributor)."""
    rg = dec["ranges"].to(torch.int64)
    sl = dec["sub_last"].to(torch.int64)
    m = dec["contrib_masks"]
    tiles = rg.shape[0]
    nb = (torch.minimum(sl, (rg[:, 1] - rg[:, 0])[:, None]) + 31) >> 5            # (tiles, 8) stages per sub-tile
    base = (rg[:, 0] >> 5) + torch.arange(tiles, device=rg.device)
    maxnb = int(nb.max().item()) if tiles else 0
    total = torch.zeros((tiles, 8, 32), dtype=torch.int64, device=rg.device)
    for s in range(maxnb):
        live = nb > s                                                             # (tiles, 8)
        rows = (base + s).clamp_(max=m.shape[0] - 1)
        w = m[rows]                                                               # (tiles, 8, 32) int32
        w = w.to(torch.int64) & 0xFFFFFFFF
        w = w - ((w >> 1) & 0x55555555)
        w = (w & 0x33333333) + ((w >> 2) & 0x33333333)
        w = (w + (w >> 4)) & 0x0F0F0F0F
        cnt = ((w * 0x01010101) & 0xFFFFFFFF) >> 24
        total += cnt * live[:, :, None]
    return total


def contributing_pairs(dec: dict) -> int:
    """Number of (pixel, instance) pairs that contributed to the frame = population count of the contribution masks the
    forward recorded, over the stages the backward reads (_lane_counts)."""
    return int(_lane_counts(dec).sum().item())


def contributing_pairs_per_pixel(dec: dict, W: int, H: int) -> torch.Tensor:
    """(counts, outside): contributing_pairs split by pixel, an (H, W) int64 tensor, and the number of pairs recorded for
    lanes outside the image (none, if the cull rectangles hold).  Lane l of sub-tile w of tile t is pixel
    (16 (t % tiles_x) + 8 (w & 1) + (l & 7), 16 (t // tiles_x) + 4 (w >> 1) + (l >> 3))."""
    c = _lane_counts(dec)
    tx, ty = (W + 15) // 16, (H + 15) // 16
    img = c.view(ty, tx, 4, 2, 4, 8).permute(0, 2, 4, 1, 3, 5).reshape(ty * 16, tx * 16)
    return img[:H, :W], int(img.sum().item()) - int(img[:H, :W].sum().item())
