"""CPU restatement of the Tanks and Temples evaluation's Open3D 0.17 operations (test infrastructure only; numpy, float64
throughout).  Operation orders are those of DESIGN.md section 7d:
  transform            PointCloud::Transform: rows ((T_r0*x + T_r1*y) + T_r2*z) + T_r3, then xyz / w
  crop_mask            SelectionPolygonVolume::CropInPolygon's loop over the polygon's edges, vectorised over points
  voxel_down_sample    VoxelDownSample as an accumulation in input order, voxels in ascending (x, y, z) order
  correspond           nanoflann's hybrid search with max_nn = 1: brute force on ((dx*dx)+dy*dy)+dz*dz < r*r
  moments / umeyama    the ICP sums in the GPU's reduction order (gsb_eval_icp_moments), then Eigen::umeyama
  registration_icp     Open3D's RegistrationICP loop
  f1_score_histo2      evaluation.py:163-205 literally, Python-float sums over a generator
"""
from __future__ import annotations

import math

import numpy as np

AXES = {"x": (1, 2, 0), "y": (0, 2, 1), "z": (0, 1, 2)}
MOMENT_BLOCKS = MOMENT_THREADS = 256


def transform(points, T):
    p = np.asarray(points, dtype=np.float64).reshape(-1, 3)
    T = np.asarray(T, dtype=np.float64).reshape(4, 4)
    v = [((T[r, 0] * p[:, 0] + T[r, 1] * p[:, 1]) + T[r, 2] * p[:, 2]) + T[r, 3] for r in range(4)]
    return np.stack([v[0] / v[3], v[1] / v[3], v[2] / v[3]], axis=1)


def crop_mask(points, orthogonal_axis, axis_min, axis_max, polygon):
    """Keep mask: axis_min <= p_w <= axis_max and an odd number of edge crossings strictly below p_u."""
    p = np.asarray(points, dtype=np.float64).reshape(-1, 3)
    P = np.asarray(polygon, dtype=np.float64).reshape(-1, 3)
    u, v, w = AXES[orthogonal_axis.lower()]
    pu, pv, pw = p[:, u], p[:, v], p[:, w]
    below = np.zeros(len(p), dtype=np.int64)
    for i in range(len(P)):
        j = (i + 1) % len(P)
        cross = ((P[i, v] < pv) & (P[j, v] >= pv)) | ((P[j, v] < pv) & (P[i, v] >= pv))
        with np.errstate(divide="ignore", invalid="ignore"):
            x = P[i, u] + (pv - P[i, v]) / (P[j, v] - P[i, v]) * (P[j, u] - P[i, u])
        below += cross & (x < pu)
    return ~((pw < axis_min) | (pw > axis_max)) & (below % 2 == 1)


def voxel_down_sample(points, voxel_size):
    """(points in ascending (x, y, z) voxel order, voxel index [M,3]); raises ValueError like Open3D when voxel_size is
    too small."""
    p = np.asarray(points, dtype=np.float64).reshape(-1, 3)
    if len(p) == 0:
        return p.copy(), np.zeros((0, 3), np.int64)
    lo = p.min(axis=0) - voxel_size * 0.5
    hi = p.max(axis=0) + voxel_size * 0.5
    if voxel_size * 2147483647 < (hi - lo).max():
        raise ValueError("voxel_size is too small")
    idx = np.floor((p - lo) / voxel_size).astype(np.int64)
    keys, inverse = np.unique(idx, axis=0, return_inverse=True)
    inverse = inverse.reshape(-1)
    sums = np.zeros((len(keys), 3))
    np.add.at(sums, inverse, p)  # unbuffered: each voxel's points are added from 0.0 in input order
    counts = np.bincount(inverse, minlength=len(keys)).astype(np.float64)
    return sums / counts[:, None], keys


def correspond(source, target, radius, chunk=1 << 22):
    """(index, d2): the nearest target point (lowest index among ties) with ((dx*dx)+dy*dy)+dz*dz < radius*radius."""
    s = np.asarray(source, dtype=np.float64).reshape(-1, 3)
    t = np.asarray(target, dtype=np.float64).reshape(-1, 3)
    r2 = radius * radius
    idx = np.full(len(s), -1, dtype=np.int64)
    d2 = np.full(len(s), np.inf)
    if len(t) == 0:
        return idx, d2
    step = max(1, chunk // len(t))
    for a in range(0, len(s), step):
        d = s[a:a + step, None, :] - t[None, :, :]
        dd = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]
        k = dd.argmin(axis=1)
        best = dd[np.arange(len(k)), k]
        hit = best < r2
        idx[a:a + step] = np.where(hit, k, -1)
        d2[a:a + step] = np.where(hit, best, np.inf)
    return idx, d2


def tree_sum(values):
    """Sums of the columns of values [n, Q] in gsb_eval_icp_moments' order: lane t = i mod (blocks*threads) adds its
    rows in turn from 0.0, then lanes halve within each block, then the block partials halve."""
    vals = np.asarray(values, dtype=np.float64)
    lanes = MOMENT_BLOCKS * MOMENT_THREADS
    rows = -(-len(vals) // lanes)
    padded = np.zeros((max(rows, 1) * lanes, vals.shape[1]))
    padded[:len(vals)] = vals
    acc = np.zeros((lanes, vals.shape[1]))
    for r in range(rows):
        acc = acc + padded[r * lanes:(r + 1) * lanes]
    a = acc.reshape(MOMENT_BLOCKS, MOMENT_THREADS, -1)
    while a.shape[1] > 1:
        h = a.shape[1] // 2
        a = a[:, :h] + a[:, h:]
    a = a[:, 0]
    while a.shape[0] > 1:
        h = a.shape[0] // 2
        a = a[:h] + a[h:]
    return a[0]


def moments(source, target, idx, d2, means=None):
    """(sums, count): pass 0 (means None) -> [sum d2, sum source xyz, sum target xyz]; pass 1 -> the 9 products
    (t - mu_t)_j (s - mu_s)_k (j-major) and the 3 squares (s - mu_s)_k^2."""
    s = np.asarray(source, dtype=np.float64).reshape(-1, 3)
    t = np.asarray(target, dtype=np.float64).reshape(-1, 3)
    hit = idx >= 0
    tp = np.zeros_like(s)
    tp[hit] = t[idx[hit]]
    if means is None:
        vals = np.concatenate([np.where(hit, d2, 0.0)[:, None], s, tp], axis=1)
    else:
        sd = s - np.asarray(means[:3])
        td = tp - np.asarray(means[3:])
        vals = np.concatenate([(td[:, :, None] * sd[:, None, :]).reshape(-1, 9), sd * sd], axis=1)
    vals[~hit] = 0.0
    return tree_sum(vals), int(hit.sum())


def umeyama(sums, n, second, with_scaling=True):
    one_over_n = 1.0 / n
    mu_s = sums[1:4] * one_over_n
    mu_t = sums[4:7] * one_over_n
    sigma = np.asarray(second[:9]).reshape(3, 3) * one_over_n
    U, D, Vt = np.linalg.svd(sigma)
    S = np.ones(3)
    if np.linalg.det(U) * np.linalg.det(Vt) < 0:
        S[2] = -1.0
    R = (U * S) @ Vt  # U diag(S) V^T
    T = np.eye(4)
    c = 1.0
    if with_scaling:
        src_var = ((second[9] + second[10]) + second[11]) * one_over_n
        c = 1.0 / src_var * ((D[0] * S[0] + D[1] * S[1]) + D[2] * S[2])
    T[:3, 3] = mu_t - (c * R) @ mu_s
    T[:3, :3] = R * c
    return T


def registration_icp(source, target, radius, init=np.eye(4), with_scaling=True, relative_fitness=1e-6,
                     relative_rmse=1e-6, max_iteration=30):
    """(T, fitness, rmse, iterations, [T after each iteration])."""
    pcd = np.asarray(source, dtype=np.float64).reshape(-1, 3)
    tgt = np.asarray(target, dtype=np.float64).reshape(-1, 3)
    init = np.asarray(init, dtype=np.float64)
    if not np.array_equal(init, np.eye(4)):
        pcd = transform(pcd, init)
    T = init.copy()
    n = len(pcd)

    def result(p):
        idx, d2 = correspond(p, tgt, radius)
        sums, cnt = moments(p, tgt, idx, d2)
        fit, rmse = (cnt / n, math.sqrt(sums[0] / cnt)) if cnt else (0.0, 0.0)
        return idx, d2, sums, cnt, fit, rmse

    idx, d2, sums, cnt, fit, rmse = result(pcd)
    history, it = [], 0
    for it in range(1, max_iteration + 1):
        if cnt:
            mu = np.concatenate([sums[1:4], sums[4:7]]) * (1.0 / cnt)
            update = umeyama(sums, cnt, moments(pcd, tgt, idx, d2, mu)[0], with_scaling)
        else:
            update = np.eye(4)
        T = update @ T
        history.append(T.copy())
        pcd = transform(pcd, update)
        f0, r0 = fit, rmse
        idx, d2, sums, cnt, fit, rmse = result(pcd)
        if abs(f0 - fit) < relative_fitness and abs(r0 - rmse) < relative_rmse:
            break
    return T, fit, rmse, it, history


def f1_score_histo2(threshold, plot_stretch, distance1, distance2):
    """evaluation.py:163-205 (precision, recall, fscore, edges_source, cum_source, edges_target, cum_target)."""
    distance1, distance2 = list(distance1), list(distance2)
    if len(distance1) and len(distance2):
        recall = float(sum(d < threshold for d in distance2)) / float(len(distance2))
        precision = float(sum(d < threshold for d in distance1)) / float(len(distance1))
        fscore = 2 * recall * precision / (recall + precision)
        bins = np.arange(0, threshold * plot_stretch, threshold / 100)
        hist, edges_source = np.histogram(distance1, bins)
        cum_source = np.cumsum(hist).astype(float) / len(distance1)
        hist, edges_target = np.histogram(distance2, bins)
        cum_target = np.cumsum(hist).astype(float) / len(distance2)
        return precision, recall, fscore, edges_source, cum_source, edges_target, cum_target
    return 0, 0, 0, np.array([0]), np.array([0]), np.array([0]), np.array([0])
