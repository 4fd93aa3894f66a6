"""Point-cloud cleaning and downsampling without a GPU: the restatement (tests/pcd_oracle.py) against literal per-point
loops and scipy, Open3D's quirks that follow from its formulas, the argument errors PointCloud raises before touching a
device, the workspace sizes and every refusal of the new C entry points."""
import ctypes as C
import math

import numpy as np
import pytest

from gs2mesh_b200 import _lib
from gs2mesh_b200.mesh import PointCloud
from tests import pcd_oracle as po


# ------------------------------------------------------------------------------------------------ literal restatements
def _statistical_loop(points, k, std_ratio):
    """RemoveStatisticalOutliers one point at a time in Python floats, with the fixed-order sums."""
    p = [tuple(float(c) for c in row) for row in np.asarray(points, np.float64)]
    n = len(p)
    means = []
    for i in range(n):
        d2 = sorted((((p[i][0] - q[0]) * (p[i][0] - q[0]) + (p[i][1] - q[1]) * (p[i][1] - q[1])) +
                     (p[i][2] - q[2]) * (p[i][2] - q[2]), j) for j, q in enumerate(p))
        c = min(k, n)
        s = 0.0
        for d, _ in d2[:c]:
            s = s + math.sqrt(d)
        means.append(s / float(c))

    def S(vals):
        total = 0.0
        for a in range(0, n, po.CHUNK):
            part = 0.0
            for v in vals[a:a + po.CHUNK]:
                part = part + v
            total = total + part
        return total

    mean = S([m if m > 0 else 0.0 for m in means]) / float(n)
    sq = S([(m - mean) * (m - mean) if m > 0 else 0.0 for m in means])
    std = math.sqrt(sq / float(n - 1)) if n > 1 else math.nan
    thr = mean + std_ratio * std
    return np.array(means), np.array([m > 0 and m < thr for m in means]), np.array([mean, std, thr])


def _radius_loop(points, r):
    p = np.asarray(points, np.float64)
    r2 = r * r
    out = []
    for i in range(len(p)):
        c = 0
        for j in range(len(p)):
            d = p[i] - p[j]
            c += ((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]) < r2
        out.append(c)
    return np.array(out)


def _clouds():
    rng = np.random.default_rng(5)
    lattice = np.stack(np.meshgrid(*[np.arange(4.0)] * 3, indexing="ij"), -1).reshape(-1, 3)
    dup = np.concatenate([rng.normal(size=(40, 3)), np.repeat(rng.normal(size=(3, 3)), 6, axis=0)])
    return {"random": rng.normal(size=(150, 3)), "lattice": lattice, "duplicates": dup,
            "far": rng.normal(size=(60, 3)) * 1e-3 + 1e6}


@pytest.mark.parametrize("k", [1, 2, 5, 20, 32])
@pytest.mark.parametrize("name", ["random", "lattice", "duplicates", "far"])
def test_statistical_oracle_matches_loop(name, k):
    pts = _clouds()[name]
    m, keep, stats = po.statistical(pts, k, 1.5)
    m2, keep2, stats2 = _statistical_loop(pts, k, 1.5)
    assert np.array_equal(m, m2)
    assert np.array_equal(keep, keep2)
    assert np.array_equal(stats, stats2, equal_nan=True)


def test_fixed_sum_crosses_chunks():
    rng = np.random.default_rng(0)
    for n in (1, 1023, 1024, 1025, 3000):
        v = rng.uniform(size=n) * 10.0 ** rng.integers(-8, 8, size=n)
        ref = 0.0
        for a in range(0, n, po.CHUNK):
            part = 0.0
            for x in v[a:a + po.CHUNK].tolist():
                part = part + x
            ref = ref + part
        assert po.fixed_sum(v) == ref


@pytest.mark.parametrize("r", [0.5, 1.0, float(np.nextafter(1.0, 2.0)), 1.5, 10.0])
@pytest.mark.parametrize("name", ["random", "lattice", "duplicates"])
def test_radius_oracle_matches_loop(name, r):
    pts = _clouds()[name]
    assert np.array_equal(po.radius_counts(pts, r), _radius_loop(pts, r))


def test_lattice_radius_one_excludes_face_neighbours():
    lattice = _clouds()["lattice"]
    assert (po.radius_counts(lattice, 1.0) == 1).all()
    c = po.radius_counts(lattice, float(np.nextafter(1.0, 2.0)))
    assert c.min() == 4 and c.max() == 7  # corners: itself + 3 faces; interior: itself + 6 faces


def test_oracle_matches_scipy_away_from_ties():
    from scipy.spatial import cKDTree

    rng = np.random.default_rng(11)
    pts = rng.uniform(size=(3000, 3))
    tree = cKDTree(pts)
    d, _ = tree.query(pts, 8)
    m = po.mean_distances(pts, 8)
    assert np.allclose(m, d.mean(axis=1), rtol=1e-12, atol=0)
    counts = po.radius_counts(pts, 0.05)
    ref = np.array([len(x) for x in tree.query_ball_point(pts, 0.05)])
    assert np.array_equal(counts, ref)  # no pair lies within rounding of the radius here


# ---------------------------------------------------------------------------------------------------------- quirks
def test_statistical_quirks():
    rng = np.random.default_rng(2)
    pts = rng.normal(size=(50, 3))
    _, keep, _ = po.statistical(pts, 1, 2.0)
    assert not keep.any()  # k = 1: every m_i is the point's own distance, 0
    m, keep, stats = po.statistical(pts[:1], 5, 2.0)
    assert m[0] == 0.0 and math.isnan(stats[2]) and not keep.any()
    dup = np.concatenate([pts, np.repeat(pts[:1], 4, axis=0)])  # point 0 and its 4 copies: 5 coincident points
    m, keep, _ = po.statistical(dup, 5, 2.0)
    assert (m[[0, 50, 51, 52, 53]] == 0.0).all() and not keep[[0, 50, 51, 52, 53]].any()
    m, keep, stats = po.statistical(dup, 6, 2.0)
    assert m[0] > 0.0
    # the mean divides by n, not by the number of positive means
    m, _, stats = po.statistical(dup, 5, 2.0)
    assert stats[0] == po.fixed_sum(np.where(m > 0, m, 0.0)) / float(len(dup))
    assert stats[0] < m[m > 0].mean()


def test_voxel_attributes_match_loop():
    rng = np.random.default_rng(3)
    pts = np.round(rng.uniform(size=(400, 3)) * 8) / 8
    col = rng.uniform(size=(400, 3))
    nrm = rng.normal(size=(400, 3))
    nrm[::7, 1] = np.nan
    out, oc, on = po.voxel_down_sample(pts, 0.3, col, nrm)
    lo = pts.min(axis=0) - 0.15
    groups = {}
    for i, p in enumerate(pts):
        groups.setdefault(tuple(np.floor((p - lo) / 0.3).astype(np.int64)), []).append(i)
    keys = sorted(groups)
    assert len(keys) == len(out)
    for v, key in enumerate(keys):
        ids = groups[key]
        for arr, ref_src, skip in ((out, pts, False), (oc, col, False), (on, nrm, True)):
            s = [0.0, 0.0, 0.0]
            for i in ids:
                if skip and np.isnan(ref_src[i]).any():
                    continue
                s = [s[a] + float(ref_src[i][a]) for a in range(3)]
            assert np.array_equal(arr[v], np.array(s) / float(len(ids)))


def test_select_and_uniform_oracles():
    assert po.select(6, [4, 1, 1, 3]).tolist() == [1, 3, 4]
    assert po.select(6, [4, 1, 1, 3], invert=True).tolist() == [0, 2, 5]
    assert po.select(3, []).tolist() == []


# -------------------------------------------------------------------------------------- errors before the device
def test_argument_errors_before_any_device_work():
    pcd = PointCloud(np.zeros((4, 3)))
    for k, ratio in ((0, 2.0), (5, 0.0), (5, -1.0), (5, float("nan"))):
        with pytest.raises(RuntimeError, match="Illegal input parameters, number of neighbors and standard deviation"):
            pcd.remove_statistical_outlier(k, ratio)
    with pytest.raises(TypeError):
        pcd.remove_statistical_outlier(-1, 2.0)
    with pytest.raises(TypeError):
        pcd.remove_statistical_outlier(2.5, 2.0)
    with pytest.raises(ValueError, match="32"):
        pcd.remove_statistical_outlier(33, 2.0)
    for nb, r in ((0, 1.0), (3, 0.0), (3, -2.0)):
        with pytest.raises(RuntimeError, match="Illegal input parameters, number of points and radius must be positive"):
            pcd.remove_radius_outlier(nb, r)
    with pytest.raises(TypeError):
        pcd.remove_radius_outlier(-3, 1.0)
    for r in (float("inf"), float("nan")):
        with pytest.raises(ValueError):
            pcd.remove_radius_outlier(3, r)
    with pytest.raises(RuntimeError, match=r"^\[UniformDownSample\] Illegal sample rate\.$"):
        pcd.uniform_down_sample(0)
    for s in (0.0, -1.0, float("nan")):
        with pytest.raises(RuntimeError, match=r"^voxel_size <= 0\.$"):
            pcd.voxel_down_sample(s)
    bad = PointCloud(np.zeros((4, 3)), colors=np.zeros((3, 3)))
    nan = PointCloud(np.array([[0.0, 0.0, np.nan]]))
    for cloud in (bad, nan):
        with pytest.raises(ValueError):
            cloud.remove_statistical_outlier(2, 2.0)
        with pytest.raises(ValueError):
            cloud.remove_radius_outlier(2, 1.0)
        with pytest.raises(ValueError):
            cloud.voxel_down_sample(0.1)
        with pytest.raises(ValueError):
            cloud.select_by_index([0])
        with pytest.raises(ValueError):
            cloud.compute_nearest_neighbor_distance()


def test_facade_inherits_the_methods():
    import gs2mesh_b200.o3d_compat as o3d

    for name in ("remove_statistical_outlier", "remove_radius_outlier", "select_by_index", "voxel_down_sample",
                 "uniform_down_sample", "compute_nearest_neighbor_distance", "compute_point_cloud_distance"):
        assert getattr(o3d.geometry.PointCloud, name) is getattr(PointCloud, name)


# ----------------------------------------------------------------------------------------------- the C entry points
def test_statistical_workspace_bytes(gsb_lib):
    L = gsb_lib
    assert L.gsb_pcd_statistical_workspace_bytes(-1) == 0
    assert L.gsb_pcd_statistical_workspace_bytes(2**31) == 0
    assert L.gsb_pcd_statistical_workspace_bytes(0) == 0
    for n, chunks in ((1, 1), (1024, 1), (1025, 2), (1048577, 1025), (2**31 - 1, 2**21)):
        b = L.gsb_pcd_statistical_workspace_bytes(n)
        assert b >= 8 * chunks and b % 256 == 0 and b - 8 * chunks < 256


def test_c_entry_points_refuse_bad_arguments(gsb_lib):
    L = gsb_lib
    fake = C.c_void_p(256)  # never dereferenced: every refusal happens before any device work
    g = _lib.GsbPointGrid((C.c_double * 3)(0, 0, 0), 1.0, (C.c_int32 * 3)(1, 1, 1), 256, 10, 256, 256)
    ws = L.gsb_pcd_statistical_workspace_bytes(10)
    ok = dict(k=5, ratio=2.0)
    for k, ratio in ((0, 2.0), (33, 2.0), (-1, 2.0), (5, 0.0), (5, -1.0), (5, float("nan"))):
        assert L.gsb_pcd_statistical_outliers(C.byref(g), k, ratio, fake, ws, fake, fake, fake, None) == _lib.GSB_ERR_INVALID
    assert L.gsb_pcd_statistical_outliers(None, ok["k"], 2.0, fake, ws, fake, fake, fake, None) == _lib.GSB_ERR_INVALID
    for missing in range(4):
        args = [fake, fake, fake, fake]
        args[missing] = None
        w, m, kp, st = args
        assert L.gsb_pcd_statistical_outliers(C.byref(g), 5, 2.0, w, ws, m, kp, st, None) == _lib.GSB_ERR_INVALID
    assert L.gsb_pcd_statistical_outliers(C.byref(g), 5, 2.0, fake, ws - 1, fake, fake, fake, None) == _lib.GSB_ERR_WORKSPACE
    big = _lib.GsbPointGrid((C.c_double * 3)(0, 0, 0), 1.0, (C.c_int32 * 3)(1, 1, 1), 256, 2**31, 256, 256)
    assert L.gsb_pcd_statistical_outliers(C.byref(big), 5, 2.0, fake, 2**40, fake, fake, fake, None) == _lib.GSB_ERR_INVALID
    empty = _lib.GsbPointGrid((C.c_double * 3)(0, 0, 0), 1.0, (C.c_int32 * 3)(1, 1, 1), None, 0, 256, None)
    assert L.gsb_pcd_statistical_outliers(C.byref(empty), 5, 2.0, None, 0, None, None, None, None) == _lib.GSB_OK

    for nb, r in ((0, 0.5), (-1, 0.5), (3, 0.0), (3, -0.5), (3, float("inf")), (3, float("nan")), (3, 1.0)):
        assert L.gsb_pcd_radius_outliers(C.byref(g), nb, r, fake, None) == _lib.GSB_ERR_INVALID  # r = 1.0: cell too small
    assert L.gsb_pcd_radius_outliers(C.byref(g), 3, 0.5, None, None) == _lib.GSB_ERR_INVALID
    assert L.gsb_pcd_radius_outliers(None, 3, 0.5, fake, None) == _lib.GSB_ERR_INVALID
    assert L.gsb_pcd_radius_outliers(C.byref(empty), 3, 0.5, None, None) == _lib.GSB_OK

    lo, hi = (C.c_double * 3)(0, 0, 0), (C.c_double * 3)(1, 1, 1)
    vws = L.gsb_eval_voxel_workspace_bytes(10)
    call = lambda pts, col, nrm, n, lo_, hi_, s, w, wb, out, oc, on, cnt: L.gsb_pcd_voxel_downsample(
        pts, col, nrm, n, lo_, hi_, s, w, wb, out, oc, on, cnt, None)
    assert call(fake, fake, None, 10, lo, hi, 0.1, fake, vws, fake, None, None, fake) == _lib.GSB_ERR_INVALID
    assert call(fake, None, fake, 10, lo, hi, 0.1, fake, vws, fake, None, None, fake) == _lib.GSB_ERR_INVALID
    assert call(fake, None, None, 10, lo, hi, 0.1, fake, vws, fake, fake, None, fake) == _lib.GSB_ERR_INVALID
    assert call(fake, None, None, 10, lo, hi, 0.1, fake, vws, fake, None, fake, fake) == _lib.GSB_ERR_INVALID
    for s in (0.0, -1.0, float("nan"), float("inf")):
        assert call(fake, fake, fake, 10, lo, hi, s, fake, vws, fake, fake, fake, fake) == _lib.GSB_ERR_INVALID
    assert b"pcd_voxel_downsample" in L.gsb_last_error()
    assert call(fake, fake, fake, -1, lo, hi, 0.1, fake, vws, fake, fake, fake, fake) == _lib.GSB_ERR_INVALID
    assert call(fake, fake, fake, 2**31, lo, hi, 0.1, fake, vws, fake, fake, fake, fake) == _lib.GSB_ERR_INVALID
    nan = (C.c_double * 3)(0, float("nan"), 0)
    assert call(fake, fake, fake, 10, nan, hi, 0.1, fake, vws, fake, fake, fake, fake) == _lib.GSB_ERR_INVALID
    far = (C.c_double * 3)(1e3, 0, 0)
    assert call(fake, fake, fake, 10, lo, far, 1e-7, fake, vws, fake, fake, fake, fake) == _lib.GSB_ERR_INVALID
    assert b"voxel_size is too small" in L.gsb_last_error()
    huge = (C.c_double * 3)(2e9, 2e9, 2e9)
    assert call(fake, fake, fake, 10, lo, huge, 1.0, fake, vws, fake, fake, fake, fake) == _lib.GSB_ERR_INVALID
    assert b"63 bits" in L.gsb_last_error()
    assert call(fake, fake, fake, 10, lo, hi, 0.1, fake, vws - 1, fake, fake, fake, fake) == _lib.GSB_ERR_WORKSPACE
