"""numpy restatement of the point-cloud cleaning and downsampling of gs2mesh_b200.pointcloud (test infrastructure only;
float64 throughout, every operation a single correctly rounded numpy ufunc or Python float operation, so nothing is
contracted into an FMA).  DESIGN.md section 7, "Point-cloud cleaning and downsampling", gives the semantics:
  statistical       Open3D 0.17 RemoveStatisticalOutliers: mean distances, the fixed-order sums, (mean, std, thr), keep
  radius_counts     the points at squared distance strictly below radius*radius (itself included), and the keep flags
  voxel_down_sample VoxelDownSample with colours and normals, in ascending (x, y, z) voxel order
  select / uniform / nearest_neighbor_distance  the plumbing, restated for the comparisons
"""
from __future__ import annotations

import numpy as np

from oracle import tnt_oracle
from tests import normals_oracle

CHUNK = 1024


def fixed_sum(values):
    """S: chunks of CHUNK consecutive values, each summed sequentially from 0.0, then the chunk sums sequentially from
    0.0."""
    v = np.asarray(values, np.float64).reshape(-1)
    n = len(v)
    chunks = -(-n // CHUNK)
    padded = np.zeros(chunks * CHUNK)  # +0.0 added to a sum from +0.0 of values >= 0 changes nothing
    padded[:n] = v
    padded = padded.reshape(chunks, CHUNK)
    acc = np.zeros(chunks)
    for j in range(CHUNK):
        acc = acc + padded[:, j]
    total = 0.0
    for s in acc.tolist():
        total = total + s
    return total


def mean_distances(points, k, knn=None):
    """m_i = (((0.0 + sqrt(d2_0)) + sqrt(d2_1)) + ...) / double(c), c = min(k, n), over the knn order."""
    p = np.asarray(points, np.float64).reshape(-1, 3)
    n = len(p)
    c = min(k, n)
    d2, _ = normals_oracle.knn(p, p, k) if knn is None else knn
    s = np.zeros(n)
    for j in range(c):
        s = s + np.sqrt(d2[:, j])
    return s / float(c)


def statistical(points, k, std_ratio, knn=None):
    """(mean_dist [n], keep bool [n], stats (mean, std, thr)) of RemoveStatisticalOutliers(k, std_ratio)."""
    p = np.asarray(points, np.float64).reshape(-1, 3)
    n = len(p)
    m = mean_distances(p, k, knn)
    pos = m > 0.0
    mean = fixed_sum(np.where(pos, m, 0.0)) / float(n)
    dev = m - mean
    sq = fixed_sum(np.where(pos, dev * dev, 0.0))
    with np.errstate(invalid="ignore", divide="ignore"):
        std = float(np.sqrt(np.float64(sq) / np.float64(n - 1)))
    thr = mean + float(std_ratio) * std
    keep = pos & (m < thr)
    return m, keep, np.array([mean, std, thr])


def radius_counts(points, radius, chunk=1 << 22):
    """count_i = #{j : ((dx*dx + dy*dy) + dz*dz) < radius*radius} with j = i included.  Candidates come from scipy's
    cKDTree at a slightly larger radius; the exact test decides."""
    from scipy.spatial import cKDTree

    p = np.asarray(points, np.float64).reshape(-1, 3)
    r2 = float(radius) * float(radius)
    counts = np.zeros(len(p), np.int64)
    if len(p) == 0:
        return counts
    tree = cKDTree(p)
    step = max(1, chunk // 64)
    for a in range(0, len(p), step):
        q = p[a:a + step]
        lists = tree.query_ball_point(q, float(radius) * (1 + 1e-6) + 1e-300)
        lens = np.array([len(x) for x in lists], np.int64)
        if lens.sum() == 0:
            continue
        cand = np.concatenate([np.asarray(x, np.int64) for x in lists])
        owner = np.repeat(np.arange(len(q)), lens)
        d2 = normals_oracle.sq_dist(q[owner], p[cand])
        counts[a:a + step] = np.bincount(owner[d2 < r2], minlength=len(q))
    return counts


def radius(points, nb_points, radius_):
    """keep bool [n] of RemoveRadiusOutliers(nb_points, radius): count_i > nb_points."""
    return radius_counts(points, radius_) > nb_points


def voxel_down_sample(points, voxel_size, colors=None, normals=None):
    """(points, colours or None, normals or None) in ascending (x, y, z) voxel order: the points of
    oracle/tnt_oracle.voxel_down_sample, and each voxel's colours and normals summed in input order from 0.0 (a normal
    with a NaN component adds nothing) and divided by the voxel's point count."""
    p = np.asarray(points, np.float64).reshape(-1, 3)
    out, keys = tnt_oracle.voxel_down_sample(p, voxel_size)
    if len(p) == 0:
        return out, None if colors is None else np.zeros((0, 3)), None if normals is None else np.zeros((0, 3))
    lo = p.min(axis=0) - voxel_size * 0.5
    idx = np.floor((p - lo) / voxel_size).astype(np.int64)
    k2, inverse = np.unique(idx, axis=0, return_inverse=True)
    assert np.array_equal(k2, keys)
    inverse = inverse.reshape(-1)
    counts = np.bincount(inverse, minlength=len(keys)).astype(np.float64)

    def mean(a, skip_nan):
        if a is None:
            return None
        a = np.asarray(a, np.float64).reshape(-1, 3)
        if skip_nan:
            a = np.where(np.isnan(a).any(axis=1, keepdims=True), 0.0, a)
        sums = np.zeros((len(keys), 3))
        np.add.at(sums, inverse, a)  # unbuffered: each voxel's rows are added from 0.0 in input order
        return sums / counts[:, None]

    return out, mean(colors, False), mean(normals, True)


def select(n, indices, invert=False):
    """The selected indices, ascending, each once."""
    mask = np.zeros(n, bool)
    mask[np.asarray(indices, np.int64).reshape(-1)] = True
    return np.nonzero(~mask if invert else mask)[0]


def nearest_neighbor_distance(points):
    p = np.asarray(points, np.float64).reshape(-1, 3)
    if len(p) < 2:
        return np.zeros(len(p))
    return np.sqrt(normals_oracle.knn(p, p, 2)[0][:, 1])
