"""Density clustering without a GPU: the restatement (tests/dbscan_oracle.py) against a literal restatement of Open3D's
sequential loop and against sklearn's DBSCAN, the edge behaviour that follows from the definition, the argument errors
PointCloud.cluster_dbscan raises before touching a device, the workspace size and every refusal of gsb_pcd_dbscan."""
import ctypes as C

import numpy as np
import pytest

from gs2mesh_b200 import _lib
from gs2mesh_b200.mesh import PointCloud
from tests import dbscan_oracle as do

EPS = [0.0, 0.25, float(np.nextafter(0.25, 1.0)), 0.3, 0.5]


def _small_clouds(count, seed):
    """(points, eps, min_points): random clouds and quarter lattices (distance ties exactly at eps = 0.25, 0.5)."""
    rng = np.random.default_rng(seed)
    for trial in range(count):
        n = int(rng.integers(1, 300))
        p = rng.random((n, 3)) * rng.choice([1.0, 2.0, 4.0])
        if trial % 3 == 0:
            p = np.round(p * 4) / 4
        yield p, EPS[trial % len(EPS)], int(rng.integers(0, 9))


def test_restatement_matches_open3d_loop():
    for k, (p, eps, mp) in enumerate(_small_clouds(300, 0)):
        labels, nc = do.dbscan(p, eps, mp)
        ref, ref_nc = do.open3d_loop(p, eps, mp, seed=k)
        assert labels.dtype == np.int32
        assert np.array_equal(labels, ref), (k, len(p), eps, mp)
        assert nc == ref_nc


def test_restatement_matches_open3d_loop_on_crafted_clouds():
    # clusters of cores 3..6 and 7..10; point 0 is a border point of both, below every core index; 1 is noise; border
    # point 2 reaches only the second cluster
    x = [5.0, 50.0, 7.5, 4.2, 3.9, 3.6, 3.3, 5.8, 6.1, 6.4, 6.7]
    pts = np.array([[v, 0.0, 0.0] for v in x])
    labels, nc = do.dbscan(pts, 1.0, 4)
    assert labels.tolist() == [0, -1, 1, 0, 0, 0, 0, 1, 1, 1, 1] and nc == 2
    for seed in range(5):
        assert np.array_equal(do.open3d_loop(pts, 1.0, 4, seed=seed)[0], labels)


def test_restatement_matches_sklearn_away_from_ties():
    cluster = pytest.importorskip("sklearn.cluster")
    rng = np.random.default_rng(3)
    for trial in range(40):
        n = int(rng.integers(1, 2000))
        p = rng.random((n, 3)) * rng.choice([1.0, 3.0])
        eps = float(rng.choice([0.05, 0.1, 0.2]))
        mp = int(rng.integers(1, 12))
        labels, _ = do.dbscan(p, eps, mp)
        ref = cluster.DBSCAN(eps=eps, min_samples=mp).fit_predict(p)
        assert np.array_equal(labels, ref), (trial, n, eps, mp)  # no pair lies within rounding of eps here


def test_edge_behaviour():
    rng = np.random.default_rng(1)
    p = rng.random((50, 3))
    assert np.array_equal(do.dbscan(p, 0.0, 0)[0], np.arange(50))  # nothing is within eps = 0, not even the point
    assert (do.dbscan(p, 0.0, 1)[0] == -1).all()
    assert (do.dbscan(p, 10.0, 51)[0] == -1).all()  # min_points > n
    assert (do.dbscan(p, 10.0, 50)[0] == 0).all()
    one, _ = do.dbscan(p, 1e-9, 1)  # min_points 1: every point core, its own cluster
    assert np.array_equal(one, np.arange(50))
    dup = np.repeat(p[:3], 4, axis=0)  # exact duplicates count separately: each group of 4 is a cluster at min_points 4
    labels, nc = do.dbscan(dup, 1e-9, 4)
    assert labels.tolist() == [0] * 4 + [1] * 4 + [2] * 4 and nc == 3
    assert (do.dbscan(dup, 1e-9, 5)[0] == -1).all()
    assert do.dbscan(np.zeros((0, 3)), 1.0, 3)[0].dtype == np.int32


def test_within_pairs_in_chunks():
    rng = np.random.default_rng(2)
    p = np.round(rng.random((3000, 3)) * 8) / 8
    counts, pairs = do.within_pairs(p, 0.25)
    c2, p2 = do.within_pairs(p, 0.25, chunk=64 * 7)
    assert np.array_equal(counts, c2) and np.array_equal(pairs, p2)
    d = p[pairs[:, 0]] - p[pairs[:, 1]]
    assert ((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2] < 0.0625).all()
    assert (pairs[:, 0] < pairs[:, 1]).all()
    assert np.array_equal(counts, 1 + np.bincount(pairs.ravel(), minlength=3000))


# -------------------------------------------------------------------------------------- errors before the device
def test_argument_errors_before_any_device_work():
    pcd = PointCloud(np.zeros((4, 3)))
    for mp in (-1, 2.5, "3"):
        with pytest.raises(TypeError):
            pcd.cluster_dbscan(0.1, mp)
    for eps in (-0.1, float("nan"), float("inf"), -float("inf")):
        with pytest.raises(ValueError, match="eps"):
            pcd.cluster_dbscan(eps, 3)
    for cloud in (PointCloud(np.zeros((4, 3)), colors=np.zeros((3, 3))), PointCloud(np.array([[0.0, np.inf, 0.0]]))):
        with pytest.raises(ValueError):
            cloud.cluster_dbscan(0.1, 3)
    empty = PointCloud(np.zeros((0, 3))).cluster_dbscan(0.1, 3, print_progress=True)
    assert empty.dtype == np.int32 and empty.shape == (0,)


def test_facade_inherits_cluster_dbscan():
    import gs2mesh_b200.o3d_compat as o3d

    assert o3d.geometry.PointCloud.cluster_dbscan is PointCloud.cluster_dbscan


# ----------------------------------------------------------------------------------------------- the C entry point
def test_dbscan_workspace_bytes(gsb_lib):
    L = gsb_lib
    assert L.gsb_pcd_dbscan_workspace_bytes(-1) == 0
    assert L.gsb_pcd_dbscan_workspace_bytes(0) == 0
    assert L.gsb_pcd_dbscan_workspace_bytes(2**31) == 0
    prev = 0
    for n in (1, 255, 256, 1025, 1048577, 2**31 - 1):
        b = L.gsb_pcd_dbscan_workspace_bytes(n)
        assert b % 256 == 0 and b >= 13 * n and b >= prev  # core flags, parents, root flags, ordinals, scan scratch
        prev = b


def test_c_entry_refuses_bad_arguments(gsb_lib):
    L = gsb_lib
    fake = C.c_void_p(256)  # never dereferenced: every refusal happens before any device work
    g = _lib.GsbPointGrid((C.c_double * 3)(0, 0, 0), 1.0, (C.c_int32 * 3)(1, 1, 1), 256, 10, 256, 256)
    ws = L.gsb_pcd_dbscan_workspace_bytes(10)
    call = lambda grid, eps, mp, w, wb, lab, cnt: L.gsb_pcd_dbscan(grid, eps, mp, w, wb, lab, cnt, None)
    for eps in (-0.5, -1e-300, float("nan"), float("inf"), 1.0):
        assert call(C.byref(g), eps, 3, fake, ws, fake, fake) == _lib.GSB_ERR_INVALID  # 1.0: the cell is too small
    assert b"pcd_dbscan" in L.gsb_last_error()
    assert call(C.byref(g), 0.5, -1, fake, ws, fake, fake) == _lib.GSB_ERR_INVALID
    assert call(None, 0.5, 3, fake, ws, fake, fake) == _lib.GSB_ERR_INVALID
    bad_dims = _lib.GsbPointGrid((C.c_double * 3)(0, 0, 0), 1.0, (C.c_int32 * 3)(0, 1, 1), 256, 10, 256, 256)
    assert call(C.byref(bad_dims), 0.5, 3, fake, ws, fake, fake) == _lib.GSB_ERR_INVALID
    no_cell = _lib.GsbPointGrid((C.c_double * 3)(0, 0, 0), 0.0, (C.c_int32 * 3)(1, 1, 1), 256, 10, 256, 256)
    assert call(C.byref(no_cell), 0.0, 3, fake, ws, fake, fake) == _lib.GSB_ERR_INVALID
    for missing in range(3):
        args = [fake, fake, fake]
        args[missing] = None
        w, lab, cnt = args
        assert call(C.byref(g), 0.5, 3, w, ws, lab, cnt) == _lib.GSB_ERR_INVALID
    big = _lib.GsbPointGrid((C.c_double * 3)(0, 0, 0), 1.0, (C.c_int32 * 3)(1, 1, 1), 256, 2**31, 256, 256)
    assert call(C.byref(big), 0.5, 3, fake, 2**40, fake, fake) == _lib.GSB_ERR_INVALID
    assert call(C.byref(g), 0.5, 3, fake, ws - 1, fake, fake) == _lib.GSB_ERR_WORKSPACE
    assert call(C.byref(g), 0.5, 3, fake, 0, fake, fake) == _lib.GSB_ERR_WORKSPACE
    empty = _lib.GsbPointGrid((C.c_double * 3)(0, 0, 0), 1.0, (C.c_int32 * 3)(1, 1, 1), None, 0, 256, None)
    assert call(C.byref(empty), 0.5, 3, None, 0, None, None) == _lib.GSB_OK
    assert call(C.byref(empty), 0.0, 2**62, None, 0, None, None) == _lib.GSB_OK
