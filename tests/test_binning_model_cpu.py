"""CPU: tests/binning_model.py reproduces the reference's binning bit for bit, and its sort plan the hand-worked passes.

Fed each golden fixture's reference centres (ref_geom_means2D), radii (ref_radii, the radii the reference returns; its
geometry state's internal_radii is never written by its forward) and depths (ref_geom_depths), the model must give the
reference's tiles_touched, its emitted (unsorted) keys and values, its sorted keys and point list (CUB's stable radix
sort) and its tile ranges, element for element."""
import numpy as np
import pytest

from . import binning_model as bm
from .conftest import GOLDEN_CASES, load_golden


@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_model_reproduces_reference_binning(name):
    g = load_golden(name)
    P, W, H = [int(v) for v in g["in_meta"][:3]]
    radii = g["ref_radii"].astype(np.int64)
    xy = g["ref_geom_means2D"]
    m = bm.predict(xy[:, 0], xy[:, 1], radii, g["ref_geom_depths"], W, H, capacity=1 << 29)
    R = int(g["ref_num_rendered"][0])
    assert m["R"] == R and not m["overflow"]
    np.testing.assert_array_equal(m["tiles_touched"], g["ref_geom_tiles_touched"].astype(np.uint32))
    np.testing.assert_array_equal(m["point_offsets"][-1:], np.array([R], np.uint32))
    np.testing.assert_array_equal(m["keys_unsorted"], g["ref_bin_keys_unsorted"].view(np.uint64))
    np.testing.assert_array_equal(m["values_unsorted"], g["ref_bin_point_list_unsorted"].view(np.uint32))
    np.testing.assert_array_equal(m["keys"], g["ref_bin_keys"].view(np.uint64))
    np.testing.assert_array_equal(m["point_list"], g["ref_bin_point_list"].view(np.uint32))
    np.testing.assert_array_equal(m["ranges"], g["ref_img_ranges"].view(np.uint32))
    assert int(m["sort_ctl"][bm.CTL_NPASS]) in (5, 6)               # the golden frames' keys: 37 to 43 bits
    tiles = ((W + 15) // 16) * ((H + 15) // 16)
    ok = bm.check_tile_order(np.argsort(-bm.bucket(m["ranges"][:, 1] - m["ranges"][:, 0]), kind="stable"), m["ranges"])
    assert ok is None and m["ranges"].shape == (tiles, 2), ok


@pytest.mark.parametrize("tiles,kbits,npass,last", [(1, 33, 5, 1), (255, 40, 5, 8), (256, 41, 6, 1), (65535, 48, 6, 8),
                                                    (65536, 49, 7, 1)])
def test_key_width_and_pass_plan(tiles, kbits, npass, last):
    assert bm.key_bits(tiles) == kbits
    plan = bm.pass_plan(kbits)
    assert len(plan) == npass and plan[-1][1] == last
    assert [s for s, _ in plan] == list(range(0, 8 * npass, 8))
    assert sum(b for _, b in plan) == kbits


def _keys(tile, depth_bits):
    return (np.asarray(tile, np.uint64) << np.uint64(32)) | np.asarray(depth_bits, np.uint64)


def _z(v):
    return np.asarray(v, np.float32).view(np.uint32)


@pytest.mark.parametrize("tiles,keys,skip", [
    # one tile, one depth: every pass an identity
    (1, _keys([0, 0, 0], _z([2.0] * 3)), [1, 1, 1, 1, 1]),
    # depth byte 0 only; byte 1 only; the exponent bytes only
    (1, _keys([0] * 4, _z(2.0 + np.arange(4) * 2.0 ** -22)), [0, 1, 1, 1, 1]),
    (1, _keys([0] * 4, _z(2.0 + np.arange(4) * 2.0 ** -14)), [1, 0, 1, 1, 1]),
    (1, _keys([0] * 4, _z([2.0, 4.0, 8.0, 16.0])), [1, 1, 0, 0, 1]),
    # 255 tiles: all 8 tile bits run; 256 tiles: tile bit 8 is never set, so the 1-bit pass is an identity
    (255, _keys([0, 254], _z([2.0, 2.0])), [1, 1, 1, 1, 0]),
    (256, _keys([0, 255], _z([2.0, 2.0])), [1, 1, 1, 1, 0, 1]),
    # 65535 tiles with the top tile byte constant; alternating runs and skips (the ping/pong parity flips thrice)
    (65535, _keys([0, 200], _z([2.0, 2.0])), [1, 1, 1, 1, 0, 1]),
    (256, _keys([0, 0, 7], [0x40000000, 0x40100003, 0x40000001]), [0, 1, 0, 1, 0, 1]),
    # all keys but one share digit 0: the pass runs
    (1, _keys([0] * 5, _z([2.0] * 4 + [2.0 + 2.0 ** -22])), [0, 1, 1, 1, 1]),
    (65536, _keys([0, 65535], _z([2.0, 2.0])), [1, 1, 1, 1, 0, 0, 1]),
])
def test_sort_plan_skips_and_parity(tiles, keys, skip):
    R = len(keys)
    ctl = bm.sort_ctl(keys, R, tiles, overflow=False)
    n = len(skip)
    assert int(ctl[bm.CTL_NPASS]) == n
    assert ctl[bm.CTL_SKIP:bm.CTL_SKIP + n].tolist() == skip
    sel, src = 0, []
    for s in skip:
        src.append(sel)
        sel ^= 1 - s
    assert ctl[bm.CTL_SRC:bm.CTL_SRC + n].tolist() == src and int(ctl[bm.CTL_SORTED_SEL]) == sel
    assert ctl[bm.CTL_TILE_COUNTER:bm.CTL_TILE_COUNTER + n].tolist() == [0 if s else 1 for s in skip]
    # dead frames: every pass skipped, nothing handed out
    for dead in (bm.sort_ctl(keys, R, tiles, overflow=True), bm.sort_ctl(keys[:0], 0, tiles, overflow=False)):
        assert dead[bm.CTL_SKIP:bm.CTL_SKIP + n].tolist() == [1] * n and int(dead[bm.CTL_SORTED_SEL]) == 0
        assert not dead[bm.CTL_TILE_COUNTER:].any()


def test_tile_order_check_rejects_wrong_orders():
    rg = np.array([[0, 0], [0, 5], [5, 6], [6, 6], [6, 40]], np.uint32)
    good = np.array([4, 1, 2, 0, 3])
    assert bm.check_tile_order(good, rg) is None
    assert bm.check_tile_order(good[::-1], rg) is not None                     # shortest first
    assert bm.check_tile_order(np.array([4, 1, 2, 0, 0]), rg) is not None      # not a permutation
    assert list(bm.bucket([0, 1, 2, 3, 4, 1 << 20, (1 << 20) - 1])) == [0, 1, 2, 2, 3, 21, 20]


def test_emission_order_and_clamping():
    """Row-major emission over each rectangle, clamped rectangles at every grid edge, and an overflowed frame."""
    W, H = 64, 48                                   # 4 x 3 tiles
    px = np.array([8.0, 60.0, 30.0, 30.0, -500.0], np.float32)
    py = np.array([8.0, 40.0, 24.0, 24.0, 24.0], np.float32)
    radii = np.array([3, 20, 100, 0, 10], np.int64)
    depths = np.array([1.0, 2.0, 3.0, 0.5, 1.0], np.float32)
    m = bm.predict(px, py, radii, depths, W, H, capacity=1 << 20)
    assert m["tiles_touched"].tolist() == [1, 2 * 2, 12, 0, 0]
    tile = (m["keys_unsorted"] >> np.uint64(32)).astype(np.int64).tolist()
    assert tile == [0, 6, 7, 10, 11] + list(range(12))
    assert m["point_offsets"].tolist() == [1, 5, 17, 17, 17]
    assert m["ranges"][0].tolist() == [0, 2] and m["ranges"][11].tolist() == [15, 17]
    o = bm.predict(px, py, radii, depths, W, H, capacity=16)
    assert o["overflow"] and o["R"] == 17 and not o["ranges"].any() and o["keys"].size == 0
    assert o["sort_ctl"][bm.CTL_SKIP:bm.CTL_SKIP + 5].tolist() == [1] * 5
