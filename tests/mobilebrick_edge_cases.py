"""Edge inputs for the MobileBrick kernels of gsb_mobilebrick.cu (host only, deterministic).  Each case names the place
where the parallel kernels could part from oracle/mobilebrick_oracle.py; tests/test_mobilebrick_edges_host.py proves on
the CPU that every case reaches its edge, tests/test_gpu_mobilebrick_edges.py compares the kernels with the oracle.

  elimination  (points [M,3], N, r_max, r_min): ties decided across many blocks, d2 = 0 with the r_min clamp, a clump
               whose lists hold every other point (one point per round, M rounds), all-zero terms, hundreds of rounds,
               round counts on both sides of the 4-round read-back batch, M around the 128-thread block, a far offset,
               points on cell faces and pairs at exactly r_max, and an N-th removal key tied with the (N+1)-th
  sampler      (vertices, triangles, bounds, variates, ns): extreme variates, zero-area runs, bounds[nt] < ns, nt = 1 and
               nt > 2^20, coordinates near 1e6, ns around the 256-thread block
  visibility   (points, volume, min_pts, res, voxel_size): fp32 rounding of g across half-integers, non-finite and huge
               points, small and odd resolutions; and a volume of more than 2^31 voxels, given as marked voxels only"""
from __future__ import annotations

import functools

import numpy as np

from oracle import mobilebrick_oracle as mo

CELL_FACTOR = 1.0000001  # gsb_eval_poisson_neighbours refuses a grid cell below r_max * CELL_FACTOR


def _radii(r_max, N, M):
    return float(r_max), float(r_max * 0.5 * (1 - (N / M) ** 1.5))


# ------------------------------------------------------------------------------------------------------ elimination
def lattice_plane_1m():
    """About 1M points on a plane quantised to 1/8, 95% of a 1060 x 1000 lattice in shuffled order: 12 neighbours of
    exactly equal d2 in the interior, so equal weights are decided by index across thousands of blocks."""
    rng = np.random.default_rng(101)
    i, j = np.meshgrid(np.arange(1060), np.arange(1000), indexing="ij")
    sites = np.stack([i.ravel(), j.ravel()], 1)
    sites = sites[rng.random(len(sites)) < 0.95]
    sites = sites[rng.permutation(len(sites))]
    p = np.concatenate([sites * 0.125, np.zeros((len(sites), 1))], 1)
    M = len(p)
    N = M // 4
    return (p, N, *_radii(0.125 * 2.1, N, M))


def duplicates_200k():
    """200 000 points on 20 000 sites: d2 = 0 between copies, every copy closer than r_min (equal clamped terms)."""
    rng = np.random.default_rng(102)
    sites = np.round(rng.uniform(0, 1, (20000, 3)) * 1024) / 1024
    p = sites[rng.integers(0, len(sites), 200000)]
    N = 40000
    return (p, N, *_radii(0.016, N, len(p)))


def clump_all_neighbours():
    """10^3 = 1000 points of a 1/16 lattice cube, all closer than r_max to each other: every list holds M - 1 entries with
    long runs of equal d2, and exactly one point goes per round (1000 rounds, 250 read-back batches)."""
    rng = np.random.default_rng(103)
    g = np.stack(np.meshgrid(*[np.arange(10)] * 3, indexing="ij"), -1).reshape(-1, 3)
    p = g[rng.permutation(len(g))] / 16.0
    N = 250
    return (p, N, *_radii(10 * 1.7321 / 16, N, len(p)))


def zero_terms():
    """r_min = r_max: every term and every weight is 0.0, so only the index orders the keys."""
    p = np.random.default_rng(104).uniform(0, 1, (5000, 3))
    return (p, 1500, 0.08, 0.08)


def gradient_100k():
    """100 chains of 1000 points, each a line whose spacing grows from about 0.3 to 0.9 r_max, in shuffled order: the
    density gradient lets each round take only a few points per chain, so the elimination runs hundreds of rounds
    across 782 blocks."""
    rng = np.random.default_rng(105)
    r = 0.01
    chains = []
    for c in range(100):
        lo, hi = 0.3 + 0.05 * rng.random(), 0.85 + 0.1 * rng.random()
        x = np.concatenate([[0.0], np.cumsum(np.linspace(lo, hi, 999) * r)])
        chains.append(np.stack([x, np.full(1000, 3 * r * c), np.zeros(1000)], 1))
    p = np.concatenate(chains)[rng.permutation(100_000)]
    N = 20000
    return (p, N, *_radii(r, N, len(p)))


ROUND_TARGETS = (1, 2, 3, 4, 5, 8, 9)


@functools.lru_cache(maxsize=None)
def round_count_clouds():
    """{target: (points, N, r_max, r_min)}: the first seed of a fixed search whose oracle round count is the target."""
    found = {}
    for s in range(4000):
        rng = np.random.default_rng(20000 + s)
        M = int(rng.integers(30, 90))
        p = rng.uniform(0, 1, (M, 3))
        r_max = 0.02 + 0.4 * (s % 40) / 40
        N = M // 3
        r_max, r_min = _radii(r_max, N, M)
        nbr, d2 = mo.neighbour_lists(p, r_max)
        rounds = mo.eliminate_rounds(nbr, mo.weight_term(d2, r_min, r_max), N)[3]
        if rounds in ROUND_TARGETS and rounds not in found:
            found[rounds] = (p, N, r_max, r_min)
            if len(found) == len(ROUND_TARGETS):
                break
    return found


def block_edge_cloud(M):
    rng = np.random.default_rng(300 + M)
    p = np.round(rng.uniform(0, 1, (M, 3)) * 64) / 64  # quantised: some equal d2
    N = M // 3
    return (p, N, *_radii(0.3, N, M))


def far_offset():
    """A 3000-point cloud moved by (1e5, -3e4, 7e3): coordinates with ulps near 1.5e-11."""
    p = np.random.default_rng(106).uniform(0, 1, (3000, 3)) + np.array([1e5, -3e4, 7e3])
    N = 700
    return (p, N, *_radii(0.1, N, len(p)))


def cell_faces():
    """r_max = 1/4.  Pairs along each axis across x = 0 (the second cell face of the hand-built grid, whose origin sits at
    -r_max * CELL_FACTOR) at exactly r_max (no neighbours) and at nextafter(r_max, 0) (neighbours), at -r_max/4 and
    3 r_max/4 so the difference is exact; plus points on that grid's cell faces.  Returns (points, N, r_max, r_min)."""
    r = 0.25
    cell = r * CELL_FACTOR
    inner = np.nextafter(r, 0.0)
    pts = [np.full(3, -cell)]  # the grid origin
    for a in range(3):
        for k, sep in enumerate([r, inner] * 4):
            q = np.zeros(3)
            b, c = (a + 1) % 3, (a + 2) % 3
            q[b] = 4 * r * (k + 1)  # pairs far enough apart not to see each other
            q[c] = 2 * r * (k % 3)
            q0, q1 = q.copy(), q.copy()
            q0[a] = -r / 4
            q1[a] = -r / 4 + sep
            pts += [q0, q1]
    rng = np.random.default_rng(107)
    k = rng.integers(0, 12, (400, 3)).astype(np.float64)
    face = -cell + k * cell  # every coordinate on a cell face of the hand-built grid
    jitter = rng.integers(0, 12, (400, 3)) * (r / 8)
    axis = rng.integers(0, 3, 400)
    face_pts = np.where(np.arange(3)[None, :] == axis[:, None], face, -cell + jitter)
    p = np.concatenate([np.array(pts), face_pts])
    N = len(p) // 3
    return (p, N, *_radii(r, N, len(p)))


def hand_grid_layout(points, r_max):
    """(origin, cell, dims) of the grid at the smallest cell gsb_eval_poisson_neighbours accepts."""
    lo = np.asarray(points, np.float64).min(0)
    hi = np.asarray(points, np.float64).max(0)
    cell = r_max * CELL_FACTOR
    dims = [int((h - l) // cell) + 1 for l, h in zip(lo, hi)]
    return lo, cell, dims


def cell_of(points, origin, cell):
    return np.floor((np.asarray(points, np.float64) - origin) / cell).astype(np.int64)


@functools.lru_cache(maxsize=None)
def nth_key_tie():
    """A quantised cloud and an N for which the N-th and (N+1)-th smallest removal keys are equal weights: the stable
    selection must keep the lower index of the two."""
    rng = np.random.default_rng(108)
    p = np.concatenate([rng.integers(0, 24, (3000, 2)) * 0.125, np.zeros((3000, 1))], 1)
    r_max, r_min = 0.3, 0.05
    nbr, d2 = mo.neighbour_lists(p, r_max)
    key = mo.eliminate_rounds(nbr, mo.weight_term(d2, r_min, r_max), len(p) // 2)[1]
    order = np.lexsort((np.arange(len(p)), key))
    ks = key[order]
    tied = np.flatnonzero((ks[1:] == ks[:-1]) & (ks[1:] > 0))  # positions n-1, n of equal keys
    N = int(tied[len(tied) // 2]) + 1
    return (p, N, r_max, r_min)


ELIMINATION_NAMES = (["lattice_plane_1m", "duplicates_200k", "clump_all_neighbours", "zero_terms", "gradient_100k"]
                     + [f"round_count_{t}" for t in ROUND_TARGETS] + [f"block_edge_{m}" for m in (127, 128, 129, 255, 256, 257)]
                     + ["far_offset", "cell_faces", "nth_key_tie"])
LARGE = ("lattice_plane_1m", "duplicates_200k", "gradient_100k")


def elimination_case(name):
    """(points, N, r_max, r_min) of a named case."""
    if name.startswith("round_count_"):
        return round_count_clouds()[int(name[len("round_count_"):])]
    if name.startswith("block_edge_"):
        return block_edge_cloud(int(name[len("block_edge_"):]))
    return globals()[name]()


def _clump_elimination(nbr, term):
    """The sequential loop on a cloud where every point neighbours every other: each step deletes the live point of
    largest (weight, index) and recomputes every live weight as the sequential sum of its live terms in list order (a
    deleted neighbour adds an exact 0.0).  Gives the round oracle's (removal keys, rounds of deletion, rounds) where one
    point goes per round, at a cost eliminate_rounds cannot reach for thousands of full lists."""
    M = len(nbr)
    alive = np.ones(M, bool)
    key = np.zeros(M)
    rnd = np.zeros(M, np.int64)
    live_rows = np.arange(M)
    for r in range(1, M + 1):
        sub = nbr[live_rows]
        w = np.cumsum(np.where(alive[sub], term[live_rows], 0.0), axis=1)[:, -1]
        best = np.lexsort((live_rows, w))[-1]
        p = live_rows[best]
        key[p], rnd[p] = w[best], r
        alive[p] = False
        live_rows = np.delete(live_rows, best)
    return key, rnd, M


@functools.lru_cache(maxsize=None)
def elimination_oracle(name):
    """dict(nbr, d2, term, kept, key, round_of, rounds) of a named case from the round oracle (the clump from
    _clump_elimination, which the host tests pin against eliminate_rounds and eliminate_heap on a smaller clump)."""
    p, N, r_max, r_min = elimination_case(name)
    nbr, d2 = mo.neighbour_lists(p, r_max)
    term = mo.weight_term(d2, r_min, r_max)
    if name == "clump_all_neighbours":
        key, rnd, rounds = _clump_elimination(nbr, term)
        kept = np.sort(np.lexsort((np.arange(len(p)), key))[:N])
    else:
        kept, key, rnd, rounds = mo.eliminate_rounds(nbr, term, N)
    return dict(nbr=nbr, d2=d2, term=term, kept=kept, key=key, round_of=rnd, rounds=rounds)


def small_clump(M, seed):
    rng = np.random.default_rng(seed)
    p = rng.integers(0, 5, (M, 3)) / 16.0
    return p, M // 4, 0.6, 0.1


# ---------------------------------------------------------------------------------------------------------- sampler
SPECIAL_VARIATES = np.array([0.0, 2.0 ** -53, 0.25, 0.5, 1.0 - 2.0 ** -53])


def _bounds_from_areas(v, t, ns):
    areas = mo.triangle_areas(v, t)
    return mo.sample_bounds(areas, mo.surface_area(areas), ns)


def _special_variates(ns):
    """(r1, r2) running through all 25 pairs of SPECIAL_VARIATES in turn."""
    k = np.arange(ns)
    return np.stack([SPECIAL_VARIATES[k % 5], SPECIAL_VARIATES[(k // 5) % 5]], 1).reshape(-1)


def _strip(n, offset=0.0):
    """n triangles of a unit-height strip, areas 0.5 each."""
    x = np.arange(n + 2, dtype=np.float64)
    v = np.concatenate([np.stack([x, np.zeros_like(x), np.zeros_like(x)], 1), np.stack([x, np.ones_like(x), x * 0], 1)])
    m = n + 2
    t = np.array([[i // 2, m + i // 2, i // 2 + 1] if i % 2 == 0 else [i // 2 + 1, m + i // 2, m + i // 2 + 1]
                  for i in range(n)], np.int64)
    return v + offset, t


def _with_zero_runs(v, t, runs):
    """Inserts runs of zero-area triangles (three copies of one vertex) at the given positions [(pos, length)]."""
    parts, last = [], 0
    for pos, length in runs:
        parts += [t[last:pos], np.full((length, 3), t[min(pos, len(t) - 1), 0], np.int64)]
        last = pos
    parts.append(t[last:])
    return v, np.concatenate(parts)


SAMPLER_NAMES = ("special_variates", "zero_area_runs", "hand_bounds_short", "hand_bounds_empty",
                 "hand_bounds_start_end_runs", "one_triangle", "one_triangle_hand_short", "over_2p20_triangles", "near_1e6",
                 "ns_255", "ns_256", "ns_257")


@functools.lru_cache(maxsize=None)
def sampler_case(name):
    """(vertices, triangles, bounds, variates, ns, bounds_from_areas) of a named case; bounds come from the triangle areas
    (mo.sample_bounds) unless the case makes them by hand."""
    from tests import mobilebrick_cases as mc

    rng = np.random.default_rng(200 + SAMPLER_NAMES.index(name))
    strip10 = _strip(10)
    v1 = np.array([[0.0, 0, 0], [1, 0, 0], [0, 1, 0]])
    bounds = None
    if name == "special_variates":
        (v, t), ns, variates = mc.grid_mesh(12, 9, seed=3), 1000, _special_variates(1000)
    elif name == "zero_area_runs":  # runs of zero-area triangles at the start, in the middle and at the end
        v, t = _with_zero_runs(*_strip(40), [(0, 6), (17, 9), (40, 5)])
        ns, variates = 997, rng.uniform(0, 1, 2 * 997)
    elif name == "hand_bounds_short":  # the last bound stops short of ns: trailing samples stay (0, 0, 0)
        (v, t), ns, variates = strip10, 64, rng.uniform(0, 1, 128)
        bounds = [0, 3, 3, 3, 10, 11, 20, 20, 25, 25, 30]
    elif name == "hand_bounds_empty":
        (v, t), ns, variates, bounds = strip10, 50, rng.uniform(0, 1, 100), np.zeros(11, np.int64)
    elif name == "hand_bounds_start_end_runs":
        (v, t), ns, variates = strip10, 40, _special_variates(40)
        bounds = [0, 0, 0, 0, 7, 9, 9, 33, 33, 33, 33]
    elif name == "one_triangle":
        v, t, ns, variates = v1, np.array([[0, 1, 2]]), 257, _special_variates(257)
    elif name == "one_triangle_hand_short":
        v, t, ns, variates, bounds = v1, np.array([[0, 1, 2]]), 257, rng.uniform(0, 1, 514), [0, 200]
    elif name == "over_2p20_triangles":  # 2 * 729^2 = 1 062 882 triangles > 2^20, 5M samples
        (v, t), ns, variates = mc.grid_mesh(730, 730, seed=4), 5_000_000, rng.uniform(0, 1, 10_000_000)
    elif name == "near_1e6":
        v, t = mc.grid_mesh(20, 20, seed=5)
        v, ns, variates = v + np.array([1e6, -1e6, 1e6 + 0.5]), 4000, rng.uniform(0, 1, 8000)
    else:  # ns around the 256-thread block
        ns = int(name[len("ns_"):])
        (v, t), variates = mc.grid_mesh(6, 5, seed=6), rng.uniform(0, 1, 2 * ns)
    v, t = np.asarray(v, np.float64), np.asarray(t, np.int64)
    from_areas = bounds is None
    b = _bounds_from_areas(v, t, ns) if from_areas else np.asarray(bounds, np.int64)
    return v, t, b, variates, ns, from_areas


def sample_formula(v, t, bounds, variates, ns):
    """The sampler's per-sample formula for any nondecreasing bounds: triangle t with bounds[t] <= j < bounds[t+1],
    a = 1 - sqrt(r1), b = sqrt(r1)(1 - r2), c = sqrt(r1) r2, (a p0 + b p1) + c p2; (0, 0, 0) from bounds[nt] on."""
    out = np.zeros((ns, 3))
    j = np.arange(min(int(bounds[-1]), ns))
    tri = np.searchsorted(bounds, j, side="right") - 1
    r1, r2 = variates[2 * j], variates[2 * j + 1]
    s = np.sqrt(r1)
    a, b, c = 1.0 - s, s * (1.0 - r2), s * r2
    out[j] = (a[:, None] * v[t[tri, 0]] + b[:, None] * v[t[tri, 1]]) + c[:, None] * v[t[tri, 2]]
    return out


# ------------------------------------------------------------------------------------------------------- visibility
def fp64_index(points, min_pts, res, voxel_size):
    """The voxel an fp64 g would pick (nearest, halves to even): what the fp32 rounding of g must be seen to differ from."""
    p = np.asarray(points, np.float64).reshape(-1, 3)
    g = (p - min_pts) / voxel_size / (np.asarray(res) - 1) * 2 - 1
    return np.rint((g + 1) / 2 * (np.asarray(res) - 1))


def _near_half_integers(min_pts, res, vs, rng, n=4000, ulps=6):
    """Points a few ulps either side of half-integer voxel coordinates on every axis."""
    k = rng.integers(0, np.asarray(res) - 1, (n, 3)) + 0.5
    p = min_pts + k * vs
    steps = rng.integers(-ulps, ulps + 1, (n, 3))
    for _ in range(ulps):
        p = np.where(steps > 0, np.nextafter(p, np.inf), np.where(steps < 0, np.nextafter(p, -np.inf), p))
        steps = steps - np.sign(steps)
    return p


VISIBILITY_NAMES = ("flip_odd", "flip_large", "non_finite_and_huge", "res_2_2_2", "res_2_3_4097", "res_odd")


@functools.lru_cache(maxsize=None)
def visibility_case(name):
    """(points, volume bool [res], min_pts, res, voxel_size) of a named case."""
    rng = np.random.default_rng(400 + VISIBILITY_NAMES.index(name))
    if name.startswith("flip_"):  # a few ulps around half-integer voxel coordinates
        res, min_pts, vs = {"flip_odd": ((7, 5, 9), [0.1, -0.2, 0.3], 0.05),
                            "flip_large": ((1001, 77, 30), [-3.7, 12.1, 0.013], 0.0013)}[name]
        res, min_pts = np.array(res), np.array(min_pts)
        vol = rng.random(tuple(res)) > 0.5
        return _near_half_integers(min_pts, res, vs, rng, 20000), vol, min_pts, res, vs
    if name == "non_finite_and_huge":  # every offset from min_pts is 0 or non-finite or far outside
        res = np.array([6, 4, 5])
        min_pts, vs = np.array([1.0, 2.0, 3.0]), 0.5
        vol = np.ones(tuple(res), bool)  # every voxel visible: only the index decides
        vals = [np.nan, np.inf, -np.inf, 1e30, -1e30, 2.0 ** 31 * vs, -(2.0 ** 31) * vs, (2.0 ** 31 - 1) * vs, 0.0]
        bad = np.array([[a, b, c] for a in vals for b in vals[:5] + [0.0] for c in (0.0, np.nan)]) + min_pts
        return bad, vol, min_pts, res, vs
    res = np.array({"res_2_2_2": (2, 2, 2), "res_2_3_4097": (2, 3, 4097), "res_odd": (11, 38, 101)}[name])
    vol = rng.random(tuple(res)) > 0.5
    vs = 0.01
    min_pts = np.array([-0.5, 0.25, 0.125])
    ijk = np.concatenate([rng.uniform(-1.2, res[None, :] + 0.2, (6000, 3)),
                          rng.integers(-1, res + 1, (2000, 3)) + 0.5,
                          rng.integers(-1, res + 1, (2000, 3)).astype(np.float64)])
    return min_pts + ijk * vs, vol, min_pts, res, vs


def grid_sample_reference(points, vol, min_pts, res, vs, device):
    """evaluate.py:36-41 literally (torch's F.grid_sample, nearest, zero padding, align_corners) -> keep mask (numpy)."""
    import torch
    import torch.nn.functional as F

    volume = torch.from_numpy(vol.astype(np.float64)).float().to(device)
    with np.errstate(invalid="ignore", over="ignore"):
        voxels = (points - min_pts) / vs
        voxels = voxels / (res - 1) * 2 - 1
    voxels = torch.from_numpy(voxels)[..., [2, 1, 0]].float().to(device)
    mask = F.grid_sample(volume.unsqueeze(0).unsqueeze(0), voxels.unsqueeze(0).unsqueeze(0).unsqueeze(0), mode="nearest",
                         padding_mode="zeros", align_corners=True)
    return mask[0, 0, 0, 0].cpu().numpy() > 0


BIG_RES = np.array([1291, 1291, 1291])  # 2 151 685 171 voxels > 2^31


def big_volume_case():
    """(points, marked flat voxel indices, min_pts, res, voxel_size) of a volume over 2^31 voxels, stored only as the few
    marked voxels: a band near the far corner, whose flat indices all lie past 2^31, and one voxel at the origin."""
    res = BIG_RES
    vs = 1.0 / 1024
    min_pts = np.array([0.5, -0.25, 2.0])
    rng = np.random.default_rng(500)
    corner = rng.integers(1280, 1291, (300, 3))
    marked_ijk = np.concatenate([corner, [[0, 0, 0], [1290, 1290, 1290], [1290, 0, 0]]])
    marked = np.unique((marked_ijk[:, 0] * res[1] + marked_ijk[:, 1]) * res[2] + marked_ijk[:, 2])
    ijk = np.concatenate([rng.integers(1270, 1291, (20000, 3)).astype(np.float64) + rng.uniform(-0.49, 0.49, (20000, 3)),
                          marked_ijk.astype(np.float64), [[1290.6, 1290.0, 1290.0], [1289.5, 1290.0, 1290.0]]])
    return min_pts + ijk * vs, marked, min_pts, res, vs


def big_volume_oracle(points, marked, min_pts, res, vs):
    idx = mo.visibility_index(points, min_pts, res, vs)
    inside = ((idx >= 0) & (idx < res)).all(1)
    flat = (idx[:, 0] * res[1] + idx[:, 1]) * res[2] + idx[:, 2]
    return inside & np.isin(flat, marked), np.where(inside, flat, -1)
