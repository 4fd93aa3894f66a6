"""CPU restatement of the MobileBrick evaluation's Open3D 0.17 operations (test infrastructure only; numpy with explicit
dtypes, float64 unless stated).  Operation orders are those of DESIGN.md section 7e:
  mt19937_outputs / canonical   std::mt19937(seed) and libstdc++'s generate_canonical<double, 53> over two outputs
  triangle_areas / cdf          TriangleMesh::GetSurfaceArea (sequential total) and SamplePointsUniformlyImpl's CDF
  sample_uniform                SamplePointsUniformlyImpl: std::round bounds, variates r1, r2 per sample
  neighbour_lists               nanoflann's radius search, ((dx*dx)+dy*dy)+dz*dz < r_max^2, sorted by (d2, index)
  eliminate_heap                SamplePointsPoissonDisk's priority-queue loop (ties: larger index first)
  eliminate_rounds              the same elimination as parallel greedy rounds, vectorised
  visibility                    evaluate.py:34-44's normalisation and grid_sample(nearest, zeros, align_corners) in fp32
  remove_vertices_by_mask       TriangleMesh::RemoveVerticesByMask
  evaluate_single               evaluate.py:72-108 over tnt_oracle's ICP and eval_oracle's precision / recall / F1
Sums whose order matters are explicit loops or np.cumsum (sequential), never np.sum (pairwise).
"""
from __future__ import annotations

import heapq

import numpy as np

ALPHA, BETA, GAMMA = 8.0, 0.5, 1.5


# ------------------------------------------------------------------------------------------------------ random stream
def mt19937_outputs(seed, n, skip=0):
    """Outputs skip .. skip+n-1 of std::mt19937(seed) as uint64 (numpy's legacy seeding is init_genrand)."""
    bg = np.random.RandomState(int(seed) & 0xFFFFFFFF)._bit_generator
    if skip:
        bg.random_raw(skip)
    return np.asarray(bg.random_raw(n), dtype=np.uint64)


def canonical(outputs):
    """generate_canonical<double, 53> of consecutive output pairs: (u0 + u1 * 2^32) / 2^64, then >= 1 -> nextafter(1, 0)."""
    u = np.asarray(outputs, dtype=np.uint64).reshape(-1, 2)
    s = u[:, 0].astype(np.float64) + u[:, 1].astype(np.float64) * 4294967296.0
    r = s / 18446744073709551616.0
    return np.where(r >= 1.0, np.nextafter(1.0, 0.0), r)


class Stream:
    """One std::mt19937 engine drawn from in turn."""

    def __init__(self, seed):
        self.seed, self.drawn = int(seed), 0

    def uniform(self, n):
        u = mt19937_outputs(self.seed, 2 * n, self.drawn)
        self.drawn += 2 * n
        return canonical(u)


# --------------------------------------------------------------------------------------------------------- sampling
def triangle_areas(vertices, triangles):
    v = np.asarray(vertices, np.float64)
    t = np.asarray(triangles, np.int64).reshape(-1, 3)
    a = v[t[:, 0]] - v[t[:, 1]]
    b = v[t[:, 0]] - v[t[:, 2]]
    c = np.stack([a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1], a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2],
                  a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]], 1)
    return 0.5 * np.sqrt((c[:, 0] * c[:, 0] + c[:, 1] * c[:, 1]) + c[:, 2] * c[:, 2])


def surface_area(areas):
    """GetSurfaceArea's total: added in triangle order from 0.0 (np.cumsum is sequential)."""
    a = np.asarray(areas, np.float64)
    return float(np.cumsum(a)[-1]) if len(a) else 0.0


def cdf(areas, total):
    """a[0] = area[0] / S; a[i] = area[i] / S + a[i-1]."""
    return np.cumsum(np.asarray(areas, np.float64) / total)


def std_round(x):
    """std::round for x >= 0: halves away from zero."""
    x = np.asarray(x, np.float64)
    f = np.floor(x)
    return f + (x - f >= 0.5)


def sample_bounds(areas, total, n_samples):
    """[0, round(a[0] M), round(a[1] M), ...] clamped to M (int64 [T+1])."""
    b = np.minimum(std_round(cdf(areas, total) * float(n_samples)), float(n_samples)).astype(np.int64)
    return np.concatenate([np.zeros(1, np.int64), np.maximum.accumulate(b)])


def sample_uniform(vertices, triangles, n_samples, variates):
    """SamplePointsUniformlyImpl(M = n_samples) with variates [2M] (r1, r2 of sample j at 2j, 2j+1)."""
    v = np.asarray(vertices, np.float64)
    t = np.asarray(triangles, np.int64).reshape(-1, 3)
    if len(t) == 0:
        raise ValueError("Input mesh has no triangles.")
    areas = triangle_areas(v, t)
    S = surface_area(areas)
    if not S > 0.0:
        raise ValueError("Invalid surface area")
    bounds = sample_bounds(areas, S, n_samples)
    out = np.zeros((n_samples, 3))
    j = np.arange(bounds[-1])
    tri = np.searchsorted(bounds, j, side="right") - 1
    r = np.asarray(variates, np.float64)
    r1, r2 = r[2 * j], r[2 * j + 1]
    s = np.sqrt(r1)
    a, b, c = 1.0 - s, s * (1.0 - r2), s * r2
    p0, p1, p2 = v[t[tri, 0]], v[t[tri, 1]], v[t[tri, 2]]
    out[:len(j)] = (a[:, None] * p0 + b[:, None] * p1) + c[:, None] * p2
    return out, areas, S


# ------------------------------------------------------------------------------------------------ Poisson elimination
def poisson_radii(S, N, M):
    ratio = float(N) / float(M)
    r_max = 2 * np.sqrt((S / N) / (2 * np.sqrt(3.0)))
    r_min = r_max * BETA * (1 - np.power(ratio, GAMMA))
    return float(r_max), float(r_min)


def weight_term(d2, r_min, r_max, exact_pow=False):
    d = np.sqrt(np.asarray(d2, np.float64))
    d = np.where(d < r_min, r_min, d)
    t = 1.0 - d / r_max
    if exact_pow:  # std::pow(t, 8.0), the DOUBT alternative
        return np.power(t, ALPHA)
    s = t * t
    q = s * s
    return q * q


def neighbour_lists(points, r_max, tie_shuffle_seed=None):
    """Padded [M, K] neighbour index (-1 = none) and squared distance arrays, each row sorted by (d2, index); with
    tie_shuffle_seed the order inside runs of equal d2 is shuffled instead (the DOUBT on nanoflann's tie order)."""
    from scipy.spatial import cKDTree

    p = np.asarray(points, np.float64).reshape(-1, 3)
    M = len(p)
    pairs = cKDTree(p).query_pairs(r_max * (1 + 1e-9), output_type="ndarray").astype(np.int64).reshape(-1, 2)
    i = np.concatenate([pairs[:, 0], pairs[:, 1]])
    j = np.concatenate([pairs[:, 1], pairs[:, 0]])
    d = p[i] - p[j]
    d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
    ok = d2 < r_max * r_max
    i, j, d2 = i[ok], j[ok], d2[ok]
    tie = np.zeros(len(i)) if tie_shuffle_seed is None else np.random.default_rng(tie_shuffle_seed).random(len(i))
    order = np.lexsort((j if tie_shuffle_seed is None else tie, d2, i))
    i, j, d2 = i[order], j[order], d2[order]
    counts = np.bincount(i, minlength=M)
    K = int(counts.max()) if len(counts) and len(i) else 0
    start = np.concatenate([[0], np.cumsum(counts)[:-1]]) if M else np.zeros(0, np.int64)
    col = np.arange(len(i)) - start[i]
    nbr = np.full((M, max(K, 1)), -1, np.int64)
    dd = np.zeros((M, max(K, 1)))
    nbr[i, col] = j
    dd[i, col] = d2
    return nbr, dd


def _row_weights(nbr, term, alive):
    """Sum of the live neighbours' terms, column by column (the list order), from 0.0."""
    w = np.zeros(len(nbr))
    valid = nbr >= 0
    live = valid & alive[np.where(valid, nbr, 0)]
    for k in range(nbr.shape[1]):
        w = w + np.where(live[:, k], term[:, k], 0.0)
    return w


def eliminate_rounds(nbr, term, N):
    """(kept indices ascending, removal key weights, round of each point, number of rounds)."""
    M = len(nbr)
    alive = np.ones(M, bool)
    key = np.zeros(M)
    rnd = np.zeros(M, np.int64)
    idx = np.arange(M)
    valid = nbr >= 0
    safe = np.where(valid, nbr, 0)
    w = _row_weights(nbr, term, alive)
    r = 0
    while alive.any():
        r += 1
        wq = w[safe]
        rival = valid & alive[safe] & ((wq > w[:, None]) | ((wq == w[:, None]) & (safe > idx[:, None])))
        top = alive & ~rival.any(axis=1)
        key[top] = w[top]
        rnd[top] = r
        alive &= ~top
        w = np.where(alive, _row_weights(nbr, term, alive), w)
    order = np.lexsort((idx, key))
    return np.sort(order[:N]), key, rnd, r


def eliminate_heap(nbr, term, N):
    """Open3D's loop: pop the largest (weight, index), skip stale entries, delete, recompute the neighbours' weights.
    Returns (kept indices ascending, removal key weights of the deleted points, deletion order)."""
    M = len(nbr)
    lists = [(row[row >= 0], trow[row >= 0]) for row, trow in zip(nbr, term)]
    deleted = np.zeros(M, bool)

    def weight(p):
        w = 0.0
        for q, t in zip(*lists[p]):
            if not deleted[q]:
                w = w + float(t)
        return w

    weights = [weight(p) for p in range(M)]
    heap = [(-weights[p], -p) for p in range(M)]
    heapq.heapify(heap)
    key = np.full(M, np.nan)
    order = []
    live = M
    while live > N:
        nw, np_ = heapq.heappop(heap)
        p = -np_
        if deleted[p] or -nw != weights[p]:
            continue
        deleted[p] = True
        key[p] = weights[p]
        order.append(p)
        live -= 1
        for q in lists[p][0]:
            weights[q] = weight(q)
            heapq.heappush(heap, (-weights[q], -int(q)))
    return np.flatnonzero(~deleted), key, order


def poisson_disk(vertices, triangles, N, stream, init_factor=5, exact_pow=False, tie_shuffle_seed=None, heap=False):
    """SamplePointsPoissonDisk: (kept points, kept indices into the initial samples, initial samples, rounds)."""
    M = int(init_factor * N)
    pts, _, S = sample_uniform(vertices, triangles, M, stream.uniform(2 * M))
    r_max, r_min = poisson_radii(S, N, M)
    nbr, d2 = neighbour_lists(pts, r_max, tie_shuffle_seed)
    term = weight_term(d2, r_min, r_max, exact_pow)
    if heap:
        kept, _, _ = eliminate_heap(nbr, term, N)
        rounds = None
    else:
        kept, _, _, rounds = eliminate_rounds(nbr, term, N)
    return pts[kept], kept, pts, rounds


# ------------------------------------------------------------------------------------------------- visibility, masks
def visibility_index(points, min_pts, resolution, voxel_size):
    """The voxel (i0, i1, i2) grid_sample reads for each point (int64 [N,3]; may lie outside the volume)."""
    p = np.asarray(points, np.float64).reshape(-1, 3)
    res = np.asarray(resolution, np.int64).reshape(3)
    v = (p - np.asarray(min_pts, np.float64).reshape(3)) / np.float64(voxel_size)
    g = (v / (res - 1) * 2 - 1).astype(np.float32)
    idx = np.empty((len(p), 3), np.int64)
    with np.errstate(invalid="ignore", over="ignore"):
        for a in range(3):
            x = ((g[:, a] + np.float32(1)) / np.float32(2)) * np.float32(res[a] - 1)
            # grid_sampler's safe_downgrade_to_int_range: a non-finite coordinate becomes -100, outside the volume;
            # otherwise nearbyint in fp32, then the saturating conversion
            r = np.where(np.isfinite(x), np.rint(x), -100.0).astype(np.float64)
            idx[:, a] = np.clip(r, -2 ** 31, 2 ** 31 - 1).astype(np.int64)
    return idx


def visibility(points, volume, min_pts, resolution, voxel_size):
    """keep mask (bool) of evaluate.py:34-41: fp64 normalisation, fp32 grid, nearest lookup with zero padding."""
    res = np.asarray(resolution, np.int64).reshape(3)
    vol = np.asarray(volume).reshape(tuple(res)).astype(np.float32) > 0
    idx = visibility_index(points, min_pts, res, voxel_size)
    inside = ((idx >= 0) & (idx < res)).all(axis=1)
    keep = np.zeros(len(idx), bool)
    ii = idx[inside]
    keep[inside] = vol[ii[:, 0], ii[:, 1], ii[:, 2]]
    return keep


def remove_vertices_by_mask(vertices, triangles, remove, colors=None, normals=None):
    v = np.asarray(vertices, np.float64).reshape(-1, 3)
    t = np.asarray(triangles, np.int64).reshape(-1, 3)
    keep = ~np.asarray(remove, bool)
    vmap = np.full(len(v), -1, np.int64)
    vmap[keep] = np.arange(int(keep.sum()))
    mt = vmap[t] if len(t) else np.zeros((0, 3), np.int64)
    tk = (mt >= 0).all(axis=1)
    pick = lambda a: None if a is None else np.asarray(a, np.float64).reshape(-1, 3)[keep]
    return v[keep], mt[tk], pick(colors), pick(normals)


def vertex_normals(v, t):
    """TriangleMesh::ComputeVertexNormals(normalized=true) (tests/test_gpu_mesh_volumes.py states it the same way)."""
    v = np.asarray(v, np.float64)
    t = np.asarray(t, np.int64).reshape(-1, 3)
    a, b = v[t[:, 1]] - v[t[:, 0]], v[t[:, 2]] - v[t[:, 0]]
    n = np.stack([a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1], a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2],
                  a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]], 1)
    acc = np.zeros_like(v)
    np.add.at(acc, t.reshape(-1), np.repeat(n, 3, axis=0))
    sq = (acc[:, 0] * acc[:, 0] + acc[:, 1] * acc[:, 1]) + acc[:, 2] * acc[:, 2]
    pos = sq > 0
    acc[pos] /= np.sqrt(sq[pos])[:, None]
    acc[np.isnan(acc[:, 0])] = (0.0, 0.0, 1.0)
    return acc


# ----------------------------------------------------------------------------------------------------- the pipeline
def evaluate_single(gt_vertices, gt_triangles, pred_vertices, pred_triangles, mask_dict, seed=0, number_of_points=100000,
                    pred_colors=None):
    """evaluate.py:72-108 on arrays: (the 7 numbers, the cropped mesh (vertices, triangles, colours, normals), ICP
    fitness)."""
    from oracle import eval_oracle as eo
    from oracle import tnt_oracle as to

    res = np.asarray(mask_dict["resolutions"]).reshape(3)
    stream = Stream(seed)
    gt_points = poisson_disk(gt_vertices, gt_triangles, number_of_points, stream)[0]
    T, fitness, _, _, _ = to.registration_icp(gt_vertices, pred_vertices, 0.02, np.eye(4), False, 1e-6, 1e-6, 10)
    pv = np.asarray(pred_vertices, np.float64)
    if fitness > 0.99:
        pv = to.transform(pv, np.linalg.inv(T))
    keep = visibility(pv, mask_dict["mask"], mask_dict["min_pts"], res, mask_dict["voxel_size"])
    v, t, c, _ = remove_vertices_by_mask(pv, pred_triangles, ~keep, pred_colors)
    n = vertex_normals(v, t)
    if len(t):
        pred_points = poisson_disk(v, t, number_of_points, stream)[0]
    else:
        pred_points = np.random.RandomState(seed).permutation(v)[:number_of_points]
    a = eo.precision_recall_f1(pred_points, gt_points, 0.0025)
    b = eo.precision_recall_f1(pred_points, gt_points, 0.005)
    out = [a["chamfer"], a["accuracy"], a["recall"], a["F1"], b["accuracy"], b["recall"], b["F1"]]
    return out, (v, t, c, n), fitness
