"""The ordering argument of DESIGN.md 3.2 as an executable statement: the reference sorts every (Gaussian, tile) instance by
the 64-bit key tile << 32 | depth_bits with a STABLE radix sort over instances emitted in ascending Gaussian index
(rasterizer_impl.cu:88-107, 303-308).  The product sorts the P Gaussians by depth bits first (stable, so equal depths keep
ascending index), emits instances in that order and then splits them by tile with a stable sort on the tile id alone.  Both
give the same per-tile sequence -- including depth ties, empty tiles and Gaussians touching many tiles."""
import numpy as np


def _scene(rng, n_gauss, n_tiles, max_touch):
    depth_bits = rng.integers(0x3E4CCCCD, 0x3E4CCCCD + 40, size=n_gauss, dtype=np.uint64)  # few distinct values: many ties
    tiles = [np.sort(rng.choice(n_tiles, size=rng.integers(0, max_touch + 1), replace=False)) for _ in range(n_gauss)]
    return depth_bits, tiles


def _reference_order(depth_bits, tiles):
    keys, vals = [], []
    for g, ts in enumerate(tiles):  # duplicateWithKeys: ascending Gaussian index, the rectangle's tiles row-major
        for t in ts:
            keys.append((np.uint64(t) << np.uint64(32)) | depth_bits[g])
            vals.append(g)
    keys, vals = np.array(keys, dtype=np.uint64), np.array(vals, dtype=np.int64)
    order = np.argsort(keys, kind="stable")
    return keys[order] >> np.uint64(32), vals[order]


def _product_order(depth_bits, tiles):
    by_depth = np.argsort(depth_bits, kind="stable")  # depth sort of the P Gaussians, payload = index
    tile_keys, vals = [], []
    for g in by_depth:  # emit_sorted_kernel: instances in depth order
        for t in tiles[g]:
            tile_keys.append(t)
            vals.append(g)
    tile_keys, vals = np.array(tile_keys, dtype=np.int64), np.array(vals, dtype=np.int64)
    order = np.argsort(tile_keys, kind="stable")  # stable split by tile id only
    return tile_keys[order].astype(np.uint64), vals[order]


def _lsd(keys, vals, digit_bits, passes):
    """What gsb_radix.cuh does: `passes` stable counting passes over `digit_bits`-wide digits, low digit first."""
    for p in range(passes):
        d = (keys >> np.uint64(digit_bits * p)) & np.uint64((1 << digit_bits) - 1)
        order = np.argsort(d, kind="stable")
        keys, vals = keys[order], vals[order]
    return keys, vals


def test_depth_presort_plus_stable_tile_split_equals_reference_order():
    rng = np.random.default_rng(3)
    for n_gauss, n_tiles, max_touch in [(400, 37, 9), (1500, 300, 20), (50, 5, 5), (1, 1, 1)]:
        depth_bits, tiles = _scene(rng, n_gauss, n_tiles, max_touch)
        rt, rv = _reference_order(depth_bits, tiles)
        pt, pv = _product_order(depth_bits, tiles)
        np.testing.assert_array_equal(pt, rt)
        np.testing.assert_array_equal(pv, rv)


def test_digit_widths_do_not_change_a_stable_lsd_sort():
    """8+5-bit and 7+6-bit digits (the radix sort's even split) sort 13-bit tile ids identically; 4 x 8 bits sort 32-bit
    depth keys."""
    rng = np.random.default_rng(4)
    tile = rng.integers(0, 7500, size=20000).astype(np.uint64)
    vals = np.arange(20000)
    want = np.argsort(tile, kind="stable")
    for digit_bits, passes in [(8, 2), (7, 2), (13, 1)]:
        k, v = _lsd(tile, vals, digit_bits, passes)
        np.testing.assert_array_equal(v, want)
        assert (np.diff(k.astype(np.int64)) >= 0).all()
    depth = rng.integers(0, 1 << 32, size=5000, dtype=np.uint64)
    _, v = _lsd(depth, np.arange(5000), 8, 4)
    np.testing.assert_array_equal(v, np.argsort(depth, kind="stable"))
