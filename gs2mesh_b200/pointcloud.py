"""Point-cloud cleaning and downsampling on the GPU: Open3D 0.17's PointCloud.remove_statistical_outlier,
remove_radius_outlier, cluster_dbscan, select_by_index, voxel_down_sample (with colours and normals),
uniform_down_sample, compute_nearest_neighbor_distance and compute_point_cloud_distance, for
gs2mesh_b200.mesh.PointCloud (whose methods call these functions).  DESIGN.md section 7, "Point-cloud cleaning and
downsampling" and "Density clustering", restates each operation and its doubt points; tests/pcd_oracle.py and
tests/dbscan_oracle.py restate them in numpy.

The neighbour searches run on the shared point grid (evaluate.PointGrid): gsb_pcd_statistical_outliers and
gsb_pcd_radius_outliers of include/gs2mesh_b200.h for the outlier tests, gsb_pcd_dbscan for the clusters,
gsb_pcd_voxel_downsample for the voxel means.
Index selection and the final compaction are torch gathers on the device.  Every function runs on the cloud's device
(the current CUDA device for a cloud built from host arrays), returns a new cloud of the caller's class holding host
arrays with that device set, and leaves the cloud it was given unchanged.
"""
from __future__ import annotations

import ctypes as C
import math
import operator

import numpy as np
import torch

from . import _lib
from ._lib import ptr
from .evaluate import PointGrid
from .tnt import _voxel_downsample, compute_point_cloud_distance as _cloud_distance

MAX_POINTS = 2**31 - 1


def _size_t(value, name):
    """pybind11's size_t conversion: a non-integer or negative count is a TypeError."""
    v = operator.index(value)
    if v < 0:
        raise TypeError(f"{name} must be a non-negative integer, got {v}")
    return v


def _check(pcd, what):
    """ValueError unless the cloud's points are finite, colours and normals have one row per point, and the cloud has
    fewer than 2^31 points."""
    n = len(pcd.points)
    if n > MAX_POINTS:
        raise ValueError(f"{what}: {n} points; at most 2^31 - 1 are supported")
    for name in ("colors", "normals"):
        a = getattr(pcd, name)
        if a is not None and len(a) != n:
            raise ValueError(f"{what}: {name} must have one row per point")
    if not np.isfinite(pcd.points).all():
        raise ValueError(f"{what}: the points are not finite")
    return n


def _upload(pcd, dev):
    up = lambda a: None if a is None else torch.as_tensor(a).to(dev).contiguous()
    return up(pcd.points), up(pcd.colors), up(pcd.normals)


def _new(pcd, dev, xyz, rgb, nrm):
    host = lambda t: None if t is None else t.cpu().numpy()
    return type(pcd)(host(xyz), host(rgb), host(nrm), device=dev)


def _select(pcd, dev, mask):
    """The points where the device bool mask is set, in index order, with their attributes."""
    xyz, rgb, nrm = _upload(pcd, dev)
    pick = lambda t: None if t is None else t[mask]
    return _new(pcd, dev, pick(xyz), pick(rgb), pick(nrm))


def statistical_outliers(pcd, nb_neighbors, std_ratio):
    """The device arrays of gsb_pcd_statistical_outliers: (keep bool [n], mean_dist fp64 [n], stats fp64 [3] = (mean,
    std, threshold)); None for an empty cloud.  Argument errors as remove_statistical_outlier."""
    k = _size_t(nb_neighbors, "nb_neighbors")
    ratio = float(std_ratio)
    if k < 1 or not ratio > 0.0:
        raise RuntimeError("Illegal input parameters, number of neighbors and standard deviation ratio must be positive")
    if k > _lib.KNN_MAX_K:
        raise ValueError(f"remove_statistical_outlier: nb_neighbors is at most {_lib.KNN_MAX_K}, got {k}")
    n = _check(pcd, "remove_statistical_outlier")
    if n == 0:
        return None
    dev = _lib.device(pcd.device)
    L = _lib.lib()
    with torch.cuda.device(dev):
        grid = PointGrid(torch.as_tensor(pcd.points).to(dev))
        work = torch.empty(int(L.gsb_pcd_statistical_workspace_bytes(n)), dtype=torch.uint8, device=dev)
        mean_dist = torch.empty(n, dtype=torch.float64, device=dev)
        keep = torch.empty(n, dtype=torch.uint8, device=dev)
        stats = torch.empty(3, dtype=torch.float64, device=dev)
        _lib.check(L.gsb_pcd_statistical_outliers(C.byref(grid.desc), k, ratio, ptr(work), work.numel(), ptr(mean_dist),
                                                  ptr(keep), ptr(stats), _lib.stream(dev)), invalid_is_value_error=True)
    return keep.bool(), mean_dist, stats


def remove_statistical_outlier(pcd, nb_neighbors, std_ratio, print_progress=False):
    """(cloud, indices): the points whose mean distance m_i to their nb_neighbors nearest points (themselves included) is
    positive and below mean + std_ratio * std of the positive means, the mean and std taken over the whole cloud's
    count; indices int64 ascending.  RuntimeError as Open3D's for nb_neighbors < 1 or std_ratio <= 0 (or NaN),
    TypeError for a negative count, ValueError for nb_neighbors > 32."""
    r = statistical_outliers(pcd, nb_neighbors, std_ratio)
    if r is None:
        return _empty_like(pcd), np.zeros(0, np.int64)
    keep = r[0]
    dev = keep.device
    with torch.cuda.device(dev):
        return _select(pcd, dev, keep), keep.nonzero()[:, 0].cpu().numpy()


def radius_outliers(pcd, nb_points, radius):
    """keep (device bool [n]) of gsb_pcd_radius_outliers, None for an empty cloud; argument errors as
    remove_radius_outlier."""
    nb = _size_t(nb_points, "nb_points")
    r = float(radius)
    if nb < 1 or r <= 0.0:
        raise RuntimeError("Illegal input parameters, number of points and radius must be positive")
    if not math.isfinite(r):
        raise ValueError(f"remove_radius_outlier: radius must be finite, got {r}")
    n = _check(pcd, "remove_radius_outlier")
    if n == 0:
        return None
    dev = _lib.device(pcd.device)
    with torch.cuda.device(dev):
        grid = PointGrid(torch.as_tensor(pcd.points).to(dev), radius=r)
        keep = torch.empty(n, dtype=torch.uint8, device=dev)
        _lib.check(_lib.lib().gsb_pcd_radius_outliers(C.byref(grid.desc), nb, r, ptr(keep), _lib.stream(dev)),
                   invalid_is_value_error=True)
    return keep.bool()


def remove_radius_outlier(pcd, nb_points, radius, print_progress=False):
    """(cloud, indices): the points with more than nb_points points (themselves included) at squared distance strictly
    below radius * radius; indices int64 ascending.  RuntimeError as Open3D's for nb_points < 1 or radius <= 0,
    TypeError for a negative count, ValueError for a non-finite radius."""
    keep = radius_outliers(pcd, nb_points, radius)
    if keep is None:
        return _empty_like(pcd), np.zeros(0, np.int64)
    dev = keep.device
    with torch.cuda.device(dev):
        return _select(pcd, dev, keep), keep.nonzero()[:, 0].cpu().numpy()


def dbscan(pcd, eps, min_points):
    """(labels device int32 [n], n_clusters device int32 [1]) of gsb_pcd_dbscan, None for an empty cloud; argument
    errors as cluster_dbscan."""
    e = float(eps)
    m = _size_t(min_points, "min_points")
    if not (math.isfinite(e) and e >= 0.0):
        raise ValueError(f"cluster_dbscan: eps must be finite and >= 0, got {e}")
    n = _check(pcd, "cluster_dbscan")
    if n == 0:
        return None
    dev = _lib.device(pcd.device)
    L = _lib.lib()
    with torch.cuda.device(dev):
        grid = PointGrid(torch.as_tensor(pcd.points).to(dev), radius=e)
        work = torch.empty(int(L.gsb_pcd_dbscan_workspace_bytes(n)), dtype=torch.uint8, device=dev)
        labels = torch.empty(n, dtype=torch.int32, device=dev)
        n_clusters = torch.empty(1, dtype=torch.int32, device=dev)
        # min_points past n + 1 makes no point core, like n + 1 does
        _lib.check(L.gsb_pcd_dbscan(C.byref(grid.desc), e, min(m, n + 1), ptr(work), work.numel(), ptr(labels),
                                    ptr(n_clusters), _lib.stream(dev)), invalid_is_value_error=True)
    return labels, n_clusters


def cluster_dbscan(pcd, eps, min_points, print_progress=False):
    """int32 numpy [n]: Open3D's DBSCAN labels.  Point i is core iff at least min_points points (itself included) lie at
    squared distance strictly below eps * eps; core points joined by such pairs form clusters, numbered 0, 1, ... by
    their smallest core index; a non-core point within eps of a core point takes the smallest number among those
    points' clusters, any other point -1.  TypeError for a negative or non-integer min_points, ValueError for a negative
    or non-finite eps."""
    r = dbscan(pcd, eps, min_points)
    if r is None:
        return np.zeros(0, np.int32)
    with torch.cuda.device(r[0].device):
        return r[0].cpu().numpy()


def _empty_like(pcd):
    empty = lambda a: None if a is None else np.zeros((0, 3))
    return type(pcd)(np.zeros((0, 3)), empty(pcd.colors), empty(pcd.normals), device=_lib.device(pcd.device))


def select_by_index(pcd, indices, invert=False):
    """The points at `indices` (invert: every other point) in ascending index order, each once; ValueError for an index
    outside [0, n)."""
    n = _check(pcd, "select_by_index")
    idx = np.asarray(indices).reshape(-1)
    if idx.size and not np.issubdtype(idx.dtype, np.integer):
        raise TypeError("select_by_index: indices must be integers")
    idx = idx.astype(np.int64)
    if idx.size and (idx.min() < 0 or idx.max() >= n):
        raise ValueError(f"select_by_index: an index lies outside [0, {n})")
    dev = _lib.device(pcd.device)
    with torch.cuda.device(dev):
        mask = torch.zeros(n, dtype=torch.bool, device=dev)
        mask[torch.as_tensor(idx).to(dev)] = True
        return _select(pcd, dev, ~mask if invert else mask)


def uniform_down_sample(pcd, every_k_points):
    """Points 0, k, 2k, ... with their attributes; RuntimeError as Open3D's for k = 0."""
    k = _size_t(every_k_points, "every_k_points")
    if k == 0:
        raise RuntimeError("[UniformDownSample] Illegal sample rate.")
    _check(pcd, "uniform_down_sample")
    dev = _lib.device(pcd.device)
    with torch.cuda.device(dev):
        xyz, rgb, nrm = _upload(pcd, dev)
        pick = lambda t: None if t is None else t[::k].contiguous()
        return _new(pcd, dev, pick(xyz), pick(rgb), pick(nrm))


def voxel_down_sample(pcd, voxel_size):
    """One point per occupied voxel of a voxel_size grid anchored half a voxel below the points' minimum, in ascending
    (x, y, z) voxel order (Open3D's order follows its hash map): the mean of its points, colours and normals, each summed
    in input order from 0.0 and divided by the point count; a normal with a NaN component adds nothing but its point
    counts.  Normals are not renormalised.  RuntimeError("voxel_size <= 0.") / ("voxel_size is too small.") as Open3D's;
    ValueError for a non-finite voxel size or a voxel box past 63-bit keys."""
    s = float(voxel_size)
    if not s > 0.0:
        raise RuntimeError("voxel_size <= 0.")
    n = _check(pcd, "voxel_down_sample")
    if n == 0:
        return _empty_like(pcd)
    dev = _lib.device(pcd.device)
    with torch.cuda.device(dev):
        try:
            out = _voxel_downsample(*_upload(pcd, dev), s)
        except ValueError as e:
            if "voxel_size is too small" in str(e):
                raise RuntimeError("voxel_size is too small.") from None
            raise
        return _new(pcd, dev, *out)


def compute_nearest_neighbor_distance(pcd):
    """fp64 numpy [n]: the distance of every point to its nearest other point, sqrt(d2) of the second entry of its k = 2
    search (0 for an exact duplicate); all zeros with fewer than 2 points."""
    n = _check(pcd, "compute_nearest_neighbor_distance")
    if n < 2:
        return np.zeros(n)
    dev = _lib.device(pcd.device)
    with torch.cuda.device(dev):
        p = torch.as_tensor(pcd.points).to(dev)
        d2, _ = PointGrid(p).knn(p, 2)
        return torch.sqrt(d2[:, 1]).cpu().numpy()


def compute_point_cloud_distance(pcd, target):
    """fp64 numpy [n]: the distance of every point to the nearest point of `target` (zeros for an empty target)."""
    n = _check(pcd, "compute_point_cloud_distance")
    _check(target, "compute_point_cloud_distance")
    if n == 0:
        return np.zeros(0)
    dev = _lib.device(pcd.device)
    with torch.cuda.device(dev):
        p = torch.as_tensor(pcd.points).to(dev)
        return _cloud_distance(p, torch.as_tensor(target.points).to(dev)).cpu().numpy()
