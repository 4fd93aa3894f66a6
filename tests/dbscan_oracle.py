"""numpy restatement of Open3D 0.17's PointCloud::ClusterDBSCAN as gs2mesh_b200.pointcloud.cluster_dbscan computes it
(test infrastructure only).  DESIGN.md section 7, "Density clustering", gives the semantics:
  1. core[i] = count_i >= min_points, count_i = #{j : ((dx*dx + dy*dy) + dz*dz) < eps*eps}, j = i included;
  2. core points joined by such a pair form components, numbered 0, 1, ... in the order of their smallest core index;
  3. a core point gets its component's number;
  4. a non-core point with a core point within eps gets the smallest number among those points' components, else -1.
Candidate pairs come from scipy's cKDTree at a slightly larger radius, a chunk of queries at a time, and the exact test
decides, as pcd_oracle.radius_counts does.
"""
from __future__ import annotations

import numpy as np

from tests import normals_oracle


def within_pairs(points, eps, chunk=1 << 22):
    """(count int64 [n], pairs int64 [m, 2]): each point's count (itself included) and every pair i < j with
    ((dx*dx + dy*dy) + dz*dz) < eps*eps."""
    from scipy.spatial import cKDTree

    p = np.asarray(points, np.float64).reshape(-1, 3)
    n = len(p)
    r2 = float(eps) * float(eps)
    counts = np.zeros(n, np.int64)
    pairs = [np.zeros((0, 2), np.int64)]
    if n == 0:
        return counts, pairs[0]
    tree = cKDTree(p)
    step = max(1, chunk // 64)
    for a in range(0, n, step):
        q = p[a:a + step]
        lists = tree.query_ball_point(q, float(eps) * (1 + 1e-6) + 1e-300)
        lens = np.array([len(x) for x in lists], np.int64)
        if lens.sum() == 0:
            continue
        cand = np.concatenate([np.asarray(x, np.int64) for x in lists])
        owner = np.repeat(np.arange(len(q), dtype=np.int64), lens)
        inside = normals_oracle.sq_dist(q[owner], p[cand]) < r2
        counts[a:a + step] = np.bincount(owner[inside], minlength=len(q))
        owner = owner + a
        keep = inside & (owner < cand)
        pairs.append(np.stack([owner[keep], cand[keep]], 1))
    return counts, np.concatenate(pairs)


def dbscan(points, eps, min_points, pairs=None):
    """(labels int32 [n], n_clusters) of ClusterDBSCAN(eps, min_points); `pairs` may pass within_pairs' result."""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components

    p = np.asarray(points, np.float64).reshape(-1, 3)
    n = len(p)
    if n == 0:
        return np.zeros(0, np.int32), 0
    counts, pr = within_pairs(p, eps) if pairs is None else pairs
    core = counts >= min_points
    cc = pr[core[pr[:, 0]] & core[pr[:, 1]]]
    graph = coo_matrix((np.ones(len(cc), np.int8), (cc[:, 0], cc[:, 1])), shape=(n, n))
    _, comp = connected_components(graph, directed=False)
    # the smallest core index of each component that has a core point; n elsewhere
    root = np.full(comp.max() + 1, n, np.int64)
    core_ids = np.nonzero(core)[0]
    np.minimum.at(root, comp[core_ids], core_ids)
    head = np.zeros(n + 1, np.int64)
    head[root[root < n]] = 1
    ordinal = np.cumsum(head) - head  # exclusive: the number of roots below each index
    n_clusters = int(head.sum())
    labels = np.full(n, -1, np.int64)
    labels[core] = ordinal[root[comp[core]]]
    best = np.full(n, n, np.int64)
    for a, b in ((0, 1), (1, 0)):
        m = core[pr[:, a]] & ~core[pr[:, b]]
        np.minimum.at(best, pr[m, b], root[comp[pr[m, a]]])
    border = ~core & (best < n)
    labels[border] = ordinal[best[border]]
    return labels.astype(np.int32), n_clusters


def open3d_loop(points, eps, min_points, seed=0):
    """A literal restatement of Open3D's sequential loop over Python lists, popping its frontier in a random order
    (Open3D's unordered_set order is unspecified), for small clouds."""
    p = np.asarray(points, np.float64).reshape(-1, 3)
    n = len(p)
    d = p[:, None, :] - p[None, :, :]
    inside = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2] < float(eps) * float(eps)
    nbs = [np.nonzero(row)[0].tolist() for row in inside]  # KDTreeFlann::SearchRadius: the point itself included
    rng = np.random.default_rng(seed)
    labels = [-2] * n
    c = 0
    for idx in range(n):
        if labels[idx] != -2:
            continue
        if len(nbs[idx]) < min_points:
            labels[idx] = -1
            continue
        frontier = set(nbs[idx])
        visited = {idx}
        labels[idx] = c
        while frontier:
            x = sorted(frontier)[int(rng.integers(len(frontier)))]
            frontier.discard(x)
            visited.add(x)
            if labels[x] == -1:
                labels[x] = c
            if labels[x] != -2:
                continue
            labels[x] = c
            if len(nbs[x]) >= min_points:
                frontier.update(q for q in nbs[x] if q not in visited)
        c += 1
    return np.array(labels, np.int32), c
