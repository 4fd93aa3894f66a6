"""The point grid's sizing (gs2mesh_b200.evaluate.grid_layout) and ring-range arithmetic on the CPU, the brute-force
nearest neighbour of oracle/eval_oracle.py, and the C ABI's refusal of grids the ring bound's margin does not cover."""
import ctypes as C
import math

import numpy as np
import pytest

from gs2mesh_b200.evaluate import grid_layout
from oracle import eval_oracle as eo

FAR = 2.0 ** 40  # gsb_eval.cu kFarCells


def _layout(ref, **kw):
    ref = np.asarray(ref, np.float64).reshape(-1, 3)
    srt = np.sort(ref, 0)
    m = len(srt)
    core = srt[min(m - 1, int(0.99 * m))] - srt[int(0.01 * m)]
    lo, hi = ref.min(0), ref.max(0)
    cell, dims = grid_layout(lo, hi, core, len(ref), **kw)
    return lo, cell, dims


def _rings(origin, cell, dims, q):
    """ring_nearest's query cell (clamped in double, then converted) and its first and last ring, in Python integers."""
    with np.errstate(over="ignore"):
        c = np.floor((np.asarray(q, np.float64) - origin) / cell)  # may overflow to +-inf, which the clamp catches
    qc = [int(min(max(c[a], -FAR), dims[a] - 1 + FAR)) for a in range(3)]
    k0 = max([0] + [max(-qc[a], qc[a] - (dims[a] - 1)) for a in range(3)])
    k1 = max([0] + [max(qc[a], dims[a] - 1 - qc[a]) for a in range(3)])
    return qc, k0, k1


DEGENERATE = {
    "one": [[1.0, 2.0, 3.0]],
    "copies": [[1.0, 2.0, 3.0]] * 1000,
    "origin": [[0.0, 0.0, 0.0]],
    "big": [[-3e200, 1e200, 7.0]],
    "ulp500": [[500.0, 0, 0], [np.nextafter(500.0, np.inf), 0, 0]],
    "ulp1e6": [[1e6, 0, 0], [np.nextafter(1e6, np.inf), 0, 0]],
    "subnormal_extent": [[0.0, 0, 0], [5e-324, 0, 0]],
}


@pytest.mark.parametrize("kind", sorted(DEGENERATE))
def test_degenerate_layout_and_ring_range(kind):
    """A reference whose points coincide gets a cell of max(|lo|, |hi|, 1) * 2^-30 (a normal number) and one cell per
    axis; for every query out to 1e300 the clamped cell index keeps k and qc +- k far inside int64, and the rings walked
    stay within the grid's size."""
    ref = np.asarray(DEGENERATE[kind], np.float64)
    lo, cell, dims = _layout(ref)
    assert cell >= 2.0 ** -1022 and max(dims) <= 1_000_001
    if (ref.max(0) - ref.min(0)).max() <= 1e-294:
        assert cell == max(np.abs(ref).max(), 1.0) * 2.0 ** -30 and dims == [1, 1, 1]
    for s in (1e-300, 1e-12, 1.0, 1e12, 1e300):
        for d in ((1, 0, 0), (-1, 0, 0), (0, 1, 0), (0, -1, 0), (0, 0, -1), (1, 1, 1), (-1, -1, -1), (1, -1, 1)):
            q = ref[0] + s * np.asarray(d, np.float64)
            if not np.isfinite(q).all():
                continue
            qc, k0, k1 = _rings(lo, cell, dims, q)
            assert k0 <= k1 <= FAR + max(dims)
            assert k1 - k0 <= max(dims)
            assert all(abs(c) + k1 < 2 ** 62 for c in qc)


def test_layout_unchanged_for_extended_clouds():
    """Clouds with extent keep the spacing-based cell (never the magnitude floor), and the 1e-6 floor caps every axis."""
    rng = np.random.default_rng(0)
    ref = rng.uniform(-50, 50, size=(10000, 3))
    lo, cell, dims = _layout(ref)
    assert cell == pytest.approx((100.0 ** 3 * 0.98 ** 3 / (4 * 10000)) ** (1 / 3), rel=0.05)
    line = np.zeros((2000, 3))
    line[:, 0] = rng.uniform(0, 7, 2000)
    lo, cell, dims = _layout(line, cells_per_point=1e15)
    assert cell == float(line[:, 0].max() - line[:, 0].min()) * 1e-6
    assert 1_000_000 <= dims[0] <= 1_000_001 < 2 ** 21 and dims[1:] == [1, 1]
    lo, cell, dims = _layout(ref, max_cells=8)
    assert int(np.prod(dims)) <= 8


def test_nearest_exact_ties_and_non_finite():
    ref = np.array([[1.0, 0, 0], [-1.0, 0, 0], [0, 1.0, 0], [0.0, 0, 0], [0.0, 0, 0]])
    q = np.array([[0.0, 0, 0], [0.5, 0.5, 5], [np.nan, 0, 0], [np.inf, 0, 0], [0, -np.inf, 0], [1e300, 0, 0]])
    d, i = eo.nearest_exact(q, ref)
    assert i.tolist() == [3, 0, -1, -1, -1, -1]  # exact duplicates and equal distances: the lowest index
    assert d[0] == 0.0 and d[1] == math.sqrt((0.25 + 0.25) + 25.0) and np.isinf(d[2:]).all()
    d, i = eo.nearest_exact(q[:2], ref, max_dist=d[1])
    assert i.tolist() == [3, -1]
    assert eo.nearest_exact(q, np.zeros((0, 3)))[1].tolist() == [-1] * len(q)


def test_nearest_exact_equals_kd_tree_and_chunking():
    rng = np.random.default_rng(3)
    ref = rng.uniform(-1, 1, size=(3000, 3))
    q = np.concatenate([rng.uniform(-1.5, 1.5, size=(2000, 3)), ref[:50]])
    d, i = eo.nearest_exact(q, ref)
    kd, ki = eo.nearest(q, ref)
    assert (d <= kd).all() and np.array_equal(d, eo.distance(q, ref[i]))
    assert np.mean(i == ki) > 0.999
    d2, i2 = eo.nearest_exact(q, ref, chunk=1)  # one query per block
    assert np.array_equal(d.view(np.uint64), d2.view(np.uint64)) and np.array_equal(i, i2)


def test_grid_axis_limit_is_refused(gsb_lib):
    """Every grid call refuses an axis over 2^21 cells, before touching the device."""
    from gs2mesh_b200 import _lib

    L = gsb_lib
    fake = C.c_void_p(256)
    for dims, ok in (((1 << 21) + 1, False), (1 << 21, True)):
        g = _lib.GsbPointGrid((C.c_double * 3)(0, 0, 0), 1.0, (C.c_int32 * 3)(dims, 1, 1), 256, 1, 256, 256)
        rc = L.gsb_eval_nearest(C.byref(g), fake, 0, 1.0, fake, fake, None)
        assert (rc == _lib.GSB_OK) == ok
        if not ok:
            assert L.gsb_eval_icp_correspond(C.byref(g), fake, 0, 1.0, fake, fake, None) == _lib.GSB_ERR_INVALID
            assert L.gsb_eval_grid_build(C.byref(g), fake, 1 << 30, None) == _lib.GSB_ERR_INVALID
    # a grid without points: the 27-cell searches would return at once, so only the descriptor check can refuse it
    g = _lib.GsbPointGrid((C.c_double * 3)(0, 0, 0), 1.0, (C.c_int32 * 3)((1 << 21) + 1, 1, 1), 256, 0, 256, 256)
    assert L.gsb_eval_radius_downsample(C.byref(g), 0.5, fake, fake, fake, None, None) == _lib.GSB_ERR_INVALID
    assert L.gsb_eval_poisson_neighbours(C.byref(g), 0.5, 0.0, fake, None, None, None, None) == _lib.GSB_ERR_INVALID
