"""CPU checks of the host restatements the TSDF edge-case tests rely on (tests/tsdf_host.py) and of the oracle's fp32-colour
variant (oracle/tsdf_oracle.cpp, variant bit 3)."""
import numpy as np

from tests import tsdf_host as th


def test_brick_key_packs_three_biased_21_bit_indices():
    assert th.brick_key((-th.BIAS, -th.BIAS, -th.BIAS)) == 0
    assert th.brick_key((th.BIAS - 1,) * 3) == (1 << 63) - 1  # never the all-ones empty marker
    assert th.brick_key((0, 0, 0)) == (th.BIAS << 42) | (th.BIAS << 21) | th.BIAS
    assert th.brick_key((1, -2, 3)) - th.brick_key((0, -2, 3)) == 1 << 42


def test_brick_hash_scalar_and_vectorised_agree():
    rng = np.random.default_rng(0)
    bricks = rng.integers(-th.BIAS, th.BIAS, (2000, 3))
    keys = [th.brick_key(b) for b in bricks]
    for mask in (15, 1023, (1 << 20) - 1, 0xFFFFFFFF):
        want = np.array([th.brick_hash(k, mask) for k in keys])
        np.testing.assert_array_equal(th.brick_hash_np(np.array(keys, np.uint64), mask), want)
        assert want.max() <= mask
    assert th.brick_hash(0, 0xFFFFFFFF) == 0  # the splitmix64 finaliser fixes 0
    # spread: 2000 keys over 4096 slots occupy far more than half of the slots a perfect hash would
    assert len(set(th.brick_hash(k, 4095) for k in keys)) > 1400


def test_linear_probing_occupancy_does_not_depend_on_order():
    rng = np.random.default_rng(1)
    homes = rng.integers(0, 32, 20)
    homes[:4] = 31  # a chain that must wrap to slot 0
    pos = th.linear_probe_positions(homes, 32)
    assert len(set(pos.tolist())) == 20 and (pos < homes).any()
    for _ in range(5):
        perm = rng.permutation(20)
        assert set(th.linear_probe_positions(homes[perm], 32).tolist()) == set(pos.tolist())


def test_oracle_fp32_colour_variant(oracle):
    """Variant bit 3 keeps colour as the fp32 running mean (c*w + rgb)/(w + 1), one rounding per operation; the default
    keeps Open3D's fp64 mean.  A fronto-parallel wall seen 9 times with one colour per frame: every updated voxel carries the
    recurrence over all 9 frames."""
    W, H, FX = 32, 24, 30.0
    depth = np.full((H, W), 1.0, np.float32)
    seq = np.array([[200, 3, 77], [1, 254, 128], [99, 100, 101], [255, 0, 7], [13, 31, 211],
                    [64, 192, 5], [250, 251, 252], [0, 9, 18], [77, 66, 55]], np.uint8)

    def fuse(bits):
        oracle.tsdf_set_variant(bits)
        try:
            vol = oracle.OracleTSDFVolume(1.0 / 64, 0.05, with_color=True)
            for c in seq:
                vol.integrate(depth, np.broadcast_to(c, (H, W, 3)), W, H, FX, FX, W / 2, H / 2, np.eye(4))
        finally:
            oracle.tsdf_set_variant(0)
        cols = [vol.unit_data(i) for i in range(vol.num_units)]
        w = np.concatenate([u[1] for u in cols])
        return w, np.concatenate([u[2] for u in cols])

    w32, c32 = fuse(8)
    w64, c64 = fuse(0)
    np.testing.assert_array_equal(w32, w64)
    full = w32 == len(seq)
    assert full.sum() > 1000 and set(np.unique(w32)) <= {0.0, float(len(seq))}
    f32, f64 = np.zeros(3, np.float32), np.zeros(3, np.float64)
    for k, c in enumerate(seq):
        w = np.float32(k)
        f32 = (f32 * w + c.astype(np.float32)) / (w + np.float32(1))
        f64 = (f64 * np.float64(w) + c.astype(np.float64)) / np.float64(w + np.float32(1))
    assert f32.dtype == np.float32
    np.testing.assert_array_equal(c32[full], np.broadcast_to(f32.astype(np.float64), (int(full.sum()), 3)))
    np.testing.assert_array_equal(c64[full], np.broadcast_to(f64, (int(full.sum()), 3)))
    assert (f32.astype(np.float64) != f64).any() and np.abs(f32 - f64).max() < 1e-4
