"""CPU restatement of the mesh-quality evaluators (test infrastructure only; numpy + scipy, no sklearn, no Open3D).

Written from the reference's behaviour (file:line in the gs2mesh sources):
  evaluation/DTU/eval_code/eval.py:54-65    per-triangle edge vectors, lengths, doubled area, sample counts n1/n2
  evaluation/DTU/eval_code/eval.py:10-19    grid samples kept where (i+.5)/max(n1,1e-7) + (j+.5)/max(n2,1e-7) < 1
  evaluation/DTU/eval_code/eval.py:71       data_pcd = [vertices ; samples in triangle order]
  evaluation/DTU/eval_code/eval.py:86-93    greedy radius downsampling over sklearn radius_neighbors (inclusive)
  evaluation/DTU/eval_code/eval.py:119-120  kd_tree kneighbors: distance sqrt(((dx*dx)+dy*dy)+dz*dz)
  evaluation/MobileBrick/eval_code/evaluate.py:46-63  pred_gt / accuracy / gt_pred / recall / chamfer / F1
"""
from __future__ import annotations

import numpy as np
from scipy.spatial import cKDTree


def sample_mesh(vertices, triangles, thresh):
    """data_pcd of eval.py:48-71, vectorised across triangles with the reference's elementwise expressions."""
    vertices = np.asarray(vertices, dtype=np.float64).reshape(-1, 3)
    triangles = np.asarray(triangles, dtype=np.int64).reshape(-1, 3)
    tri_vert = vertices[triangles]
    v1 = tri_vert[:, 1] - tri_vert[:, 0]
    v2 = tri_vert[:, 2] - tri_vert[:, 0]
    l1 = np.sqrt((v1[:, 0] * v1[:, 0] + v1[:, 1] * v1[:, 1]) + v1[:, 2] * v1[:, 2])
    l2 = np.sqrt((v2[:, 0] * v2[:, 0] + v2[:, 1] * v2[:, 1]) + v2[:, 2] * v2[:, 2])
    cr = np.cross(v1, v2)
    area2 = np.sqrt((cr[:, 0] * cr[:, 0] + cr[:, 1] * cr[:, 1]) + cr[:, 2] * cr[:, 2])
    keep = area2 > 0
    l1, l2, area2, v1, v2, a = l1[keep], l2[keep], area2[keep], v1[keep], v2[keep], tri_vert[keep, 0]
    thr = thresh * np.sqrt(l1 * l2 / area2)
    n1 = np.floor(l1 / thr)
    n2 = np.floor(l2 / thr)
    size = ((n1 + 1) * (n2 + 1)).astype(np.int64)  # the np.mgrid[:n1+1, :n2+1] of each triangle, i-major
    t = np.repeat(np.arange(len(size)), size)
    local = np.arange(int(size.sum())) - np.repeat(np.cumsum(size) - size, size)
    cols = (n2 + 1).astype(np.int64)[t]
    i = (local // cols).astype(np.float64)
    j = (local % cols).astype(np.float64)
    k0 = (i + 0.5) / np.maximum(n1, 1e-7)[t]
    k1 = (j + 0.5) / np.maximum(n2, 1e-7)[t]
    sel = k0 + k1 < 1
    t, k0, k1 = t[sel], k0[sel, None], k1[sel, None]
    q = v1[t] * k0 + v2[t] * k1 + a[t]
    return np.concatenate([vertices, q], axis=0)


def sample_counts(vertices, triangles, thresh):
    """Points each triangle contributes (0 for zero-area triangles)."""
    triangles = np.asarray(triangles, dtype=np.int64).reshape(-1, 3)
    return np.array([len(sample_mesh(vertices, triangles[k:k + 1], thresh)) - len(vertices) for k in range(len(triangles))],
                    dtype=np.int64)


def distance(q, p):
    """sklearn's euclidean distance in its summation order: sqrt(((dx*dx)+dy*dy)+dz*dz)."""
    d = np.asarray(q, dtype=np.float64) - np.asarray(p, dtype=np.float64)
    return np.sqrt((d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2])


def nearest(queries, reference):
    """(dist, idx): cKDTree's candidate, its distance recomputed in the reference's summation order."""
    queries = np.asarray(queries, dtype=np.float64).reshape(-1, 3)
    reference = np.asarray(reference, dtype=np.float64).reshape(-1, 3)
    _, idx = cKDTree(reference).query(queries, k=1)
    idx = np.asarray(idx, dtype=np.int64)
    return distance(queries, reference[idx]), idx


def nearest_exact(queries, reference, max_dist=np.inf, chunk=1 << 22):
    """(dist, idx) of gsb_eval_nearest by brute force in fp64: the minimum of ((dx*dx)+dy*dy)+dz*dz over every reference
    point, the lowest index among equal minima, dist = its sqrt.  Queries whose dist is not below max_dist, and queries
    with a coordinate that is not finite, get (+inf, -1).  Works on blocks of about `chunk` query-point pairs."""
    q = np.asarray(queries, dtype=np.float64).reshape(-1, 3)
    ref = np.asarray(reference, dtype=np.float64).reshape(-1, 3)
    dist = np.full(len(q), np.inf)
    idx = np.full(len(q), -1, dtype=np.int64)
    if len(ref) == 0:
        return dist, idx
    step = max(1, chunk // len(ref))
    for a in range(0, len(q), step):
        with np.errstate(over="ignore", invalid="ignore"):  # far or non-finite queries: inf / nan, handled below
            d = q[a:a + step, None, :] - ref[None, :, :]
            dd = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]
        k = dd.argmin(axis=1)  # the first minimum: the lowest index
        best = np.sqrt(dd[np.arange(len(k)), k])
        hit = (best < max_dist) & np.isfinite(q[a:a + step]).all(axis=1)
        dist[a:a + step] = np.where(hit, best, np.inf)
        idx[a:a + step] = np.where(hit, k, -1)
    return dist, idx


def radius_downsample(points, thresh):
    """Keep mask of eval.py:88-93 for points already in shuffled order: the literal sequential loop over radius neighbours,
    a neighbour being a point with ((dx*dx)+dy*dy)+dz*dz <= thresh*thresh (sklearn's radius test on reduced distances)."""
    points = np.asarray(points, dtype=np.float64).reshape(-1, 3)
    tree = cKDTree(points)
    r2 = thresh * thresh
    mask = np.ones(len(points), dtype=np.bool_)
    for curr in range(len(points)):
        if mask[curr]:
            cand = np.asarray(tree.query_ball_point(points[curr], thresh * (1 + 1e-9)), dtype=np.int64)
            d = points[cand] - points[curr]
            idxs = cand[(d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2] <= r2]
            mask[idxs] = 0
            mask[curr] = 1
    return mask


def precision_recall_f1(pred_points, gt_points, threshold):
    """MobileBrick evaluate() (evaluate.py:46-63) over oracle nearest neighbours."""
    d = nearest(pred_points, gt_points)[0]
    pred_gt_dist = np.mean(d)
    precision = np.sum(d < threshold) / len(d)
    d = nearest(gt_points, pred_points)[0]
    gt_pred_dist = np.mean(d)
    recall = np.sum(d < threshold) / len(d)
    F1 = 2 * precision * recall / (precision + recall)
    chamfer = pred_gt_dist + gt_pred_dist
    return {"pred_gt": pred_gt_dist, "accuracy": precision, "gt_pred": gt_pred_dist, "recall": recall, "chamfer": chamfer,
            "F1": F1}


def dtu_chamfer(data_pcd, stl, obs_mask, bb, res, plane, order, downsample_density=0.2, patch_size=60, max_dist=20):
    """eval.py:80-134 for data_pcd (already sampled) shuffled by the explicit permutation `order`."""
    thresh = downsample_density
    data_pcd = np.asarray(data_pcd, dtype=np.float64)[np.asarray(order)]  # eval.py:81-82
    data_down = data_pcd[radius_downsample(data_pcd, thresh)]  # eval.py:86-94
    BB = np.asarray(bb).astype(np.float32)  # eval.py:99-110
    patch = patch_size
    inbound = ((data_down >= BB[:1] - patch) & (data_down < BB[1:] + patch * 2)).sum(axis=-1) == 3
    data_in = data_down[inbound]
    data_grid = np.around((data_in - BB[:1]) / res).astype(np.int32)
    grid_inbound = ((data_grid >= 0) & (data_grid < np.expand_dims(obs_mask.shape, 0))).sum(axis=-1) == 3
    data_grid_in = data_grid[grid_inbound]
    in_obs = obs_mask[data_grid_in[:, 0], data_grid_in[:, 1], data_grid_in[:, 2]].astype(np.bool_)
    data_in_obs = data_in[grid_inbound][in_obs]
    stl = np.asarray(stl, dtype=np.float64)
    dist_d2s = nearest(data_in_obs, stl)[0]  # eval.py:119-122
    mean_d2s = dist_d2s[dist_d2s < max_dist].mean()
    stl_hom = np.concatenate([stl, np.ones_like(stl[:, :1])], -1)  # eval.py:126-134
    above = (np.asarray(plane).reshape((1, 4)) * stl_hom).sum(-1) > 0
    dist_s2d = nearest(stl[above], data_in)[0]
    mean_s2d = dist_s2d[dist_s2d < max_dist].mean()
    return {"mean_d2s": mean_d2s, "mean_s2d": mean_s2d, "overall": (mean_d2s + mean_s2d) / 2, "data_down": data_down,
            "dist_d2s": dist_d2s, "dist_s2d": dist_s2d}
