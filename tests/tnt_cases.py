"""Inputs that put the Tanks and Temples kernels (gs2mesh_b200/csrc/gsb_tnt.cu, gs2mesh_b200/tnt.py) at their edges, the
CPU predicates that show each case reaches its edge, and exact references that share no code with oracle/tnt_oracle.py:
rational arithmetic (fractions.Fraction, or Python integers over a common power of two) and math.fsum.

Every builder is seeded.  tests/test_tnt_cases_host.py asserts the predicates on the CPU; tests/test_gpu_tnt_edges.py runs
the cases on the GPU against the oracle (bit for bit) and against the exact references here."""
from __future__ import annotations

import math
from fractions import Fraction

import numpy as np

U = 2.0 ** -53  # unit roundoff of float64
EPS = 2.0 ** -52
TINY = 2.0 ** -1074  # the smallest subnormal
MIN_NORMAL = 2.0 ** -1022
INT_MAX = 2147483647
MAX_POLYGON = 2048  # GSB_EVAL_MAX_POLYGON
BLOCK = 256  # the crop and transform kernels' block size
MOMENT_LANES = 256 * 256  # gsb_eval_icp_moments: blocks x threads
AXES = {"x": (1, 2, 0), "y": (0, 2, 1), "z": (0, 1, 2)}  # (u, v, w) for each orthogonal axis


def similarity(angle, axis, scale, t):
    axis = np.asarray(axis, dtype=np.float64) / np.linalg.norm(axis)
    K = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    T = np.eye(4)
    T[:3, :3] = scale * (np.eye(3) + math.sin(angle) * K + (1 - math.cos(angle)) * K @ K)
    T[:3, 3] = t
    return T


def _dyadic(x, k):
    """x rounded to a multiple of 2^-k."""
    return np.round(np.asarray(x, np.float64) * 2.0 ** k) / 2.0 ** k


def is_negative_zero(x):
    x = np.asarray(x, np.float64)
    return (x == 0) & np.signbit(x)


def is_subnormal(x):
    x = np.abs(np.asarray(x, np.float64))
    return (x > 0) & (x < MIN_NORMAL)


# ------------------------------------------------------------------------------------------------------- transform
def transform_cases():
    """{name: (points [n, 3], T [4, 4])}."""
    rng = np.random.default_rng(70)
    sim = similarity(0.7, [1, -2, 0.5], 1.3, [12.5, -3.0, 40.0])
    cases = {f"n{n}": (rng.normal(size=(n, 3)) * 40, sim) for n in (1, 255, 256, 257)}
    pts = np.clip(rng.normal(size=(300, 3)) * 3, -6, 6)
    pts[:4] = [[0.0, 0.0, 0.0], [-0.0, -0.0, -0.0], [1.0, -1.0, 0.0], [-2.0, 0.5, 3.0]]
    T = sim.copy()
    T[3] = [0.0, 0.0, 0.0, 0.0]  # v3 = 0 for every finite point: +-inf, or NaN where v_k = 0 too
    T[0] = [0.0, 0.0, 0.0, 0.0]
    cases["w_zero"] = (pts, T)
    T = sim.copy()
    T[3] = [0.25, -0.125, 0.0, -2.0]  # v3 < 0 for |x|, |y| <= 6
    cases["w_negative"] = (pts, T)
    T = np.array([[-0.0, 1.0, -0.0, -0.0], [2.0, -0.0, 0.5, 0.0], [-0.0, -0.0, -1.0, -0.0], [-0.0, 0.0, -0.0, 1.0]])
    cases["negative_zero"] = (np.concatenate([pts, -pts]), T)
    small = rng.uniform(0.5, 1.0, size=(257, 3)) * np.array([1e-20, 1e-160, 1e-300]) * rng.choice([-1, 1], size=(257, 3))
    T = np.array([[1e-300, 1.0, 0.0, 0.0], [0.0, 1e-160, 1.0, 0.0], [3.0, 0.0, 1e-20, 0.0], [0.0, 0.0, 0.0, 1.0]])
    cases["subnormal"] = (small, T)
    bad = rng.normal(size=(257, 3))
    for k, v in enumerate([np.inf, -np.inf, np.nan]):
        bad[k::7, k] = v
    bad[3] = [np.inf, -np.inf, np.nan]
    cases["non_finite"] = (bad, sim)
    cases["non_finite_identity"] = (bad, np.eye(4))
    return cases


def transform_rows(points, T):
    """The four row sums of T (x, y, z, 1) in Fraction, and the terms |T_r0 x|, |T_r1 y|, |T_r2 z|, |T_r3| summed."""
    p = [Fraction(float(c)) for c in points]
    rows, mags = [], []
    for r in range(4):
        terms = [Fraction(float(T[r, j])) * p[j] for j in range(3)] + [Fraction(float(T[r, 3]))]
        rows.append(sum(terms))
        mags.append(sum(abs(t) for t in terms))
    return rows, mags


def transform_exact_check(points, T, got):
    """Checks every row whose inputs are finite and whose exact v3 is nonzero against the exact quotient v_k / v3: the
    computed ((a + b) + c) + d over products carries at most gamma_4 * sum|terms| (+ 3 subnormal half-steps), and the
    division one more rounding.  Returns (rows checked, rows skipped)."""
    g4 = Fraction(4) * Fraction(U) / (1 - 4 * Fraction(U))
    u = Fraction(U)
    checked = skipped = 0
    for i in range(len(points)):
        if not (np.isfinite(points[i]).all() and np.isfinite(T).all()):
            skipped += 1
            continue
        rows, mags = transform_rows(points[i], T)
        err = [g4 * m + 3 * Fraction(TINY) for m in mags]
        v3, e3 = rows[3], err[3]
        if abs(v3) <= e3:
            skipped += 1
            continue
        for k in range(3):
            g = float(got[i, k])
            assert math.isfinite(g), (i, k, g)
            q = rows[k] / v3
            bound = (abs(rows[k]) * e3 + abs(v3) * err[k]) / (abs(v3) * (abs(v3) - e3))
            bound += u * abs(Fraction(g)) / (1 - u) + Fraction(TINY)
            assert abs(Fraction(g) - q) <= bound, (i, k, g, float(q))
        checked += 1
    return checked, skipped


# ------------------------------------------------------------------------------------------------------------ crop
def star(m, r_out=8.0, r_in=5.5):
    """An m-vertex star (alternating radii), counter-clockwise, coordinates multiples of 2^-6."""
    a = 2 * np.pi * np.arange(m) / m
    r = np.where(np.arange(m) % 2 == 0, r_out, r_in) if m > 3 else np.full(m, r_out)
    return _dyadic(np.stack([r * np.cos(a), r * np.sin(a)], 1), 6)


def staircase():
    """A rectilinear polygon: horizontal and vertical edges only (counter-clockwise)."""
    return np.array([[-4, -4], [4, -4], [4, -1], [2, -1], [2, 1], [5, 1], [5, 4], [-1, 4], [-1, 2], [-4, 2]], np.float64)


def degenerate_polygon():
    """Repeated vertices (zero-length edges), a collinear run of four vertices and a spike back along an edge."""
    return np.array([[-4, -4], [-4, -4], [0, -4], [2, -4], [4, -4], [4, -4], [4, 0], [4, 4], [0, 4], [0, 4], [0, 0],
                     [-2, 2], [-4, 4], [-4, 0], [-4, -4]], np.float64)


BOWTIE = np.array([[-4.0, -4.0], [4.0, 4.0], [4.0, -4.0], [-4.0, 4.0]])


def _lift(uv, axis, w=None):
    """(u, v) vertices or points into 3-D for an orthogonal axis, with w (default 0)."""
    u, v, wa = AXES[axis]
    out = np.zeros((len(uv), 3))
    out[:, u], out[:, v] = uv[:, 0], uv[:, 1]
    out[:, wa] = 0.0 if w is None else w
    return out


def _edge_points(poly_uv, js=(1, 3, 5, 7)):
    """Points at j/8 of the way along every edge: with dyadic vertices, (p_v - a_v) / (b_v - a_v) = j/8 exactly, so the
    crossing of that edge equals p_u exactly."""
    a = poly_uv
    b = np.roll(poly_uv, -1, axis=0)
    return np.concatenate([a + (b - a) * (j / 8.0) for j in js])


def _probe_points(poly_uv, rng, n_random, span):
    """Random points on a 2^-20 grid, every vertex, points on every edge, and points left and right of every vertex on
    its horizontal line."""
    pts = [_dyadic(rng.uniform(-span, span, size=(n_random, 2)), 20), poly_uv, _edge_points(poly_uv)]
    for d in (-0.25, 0.25, 0.5, 2.0):
        pts.append(poly_uv + np.array([d, 0.0]))
    return np.concatenate(pts)


def crop_cases():
    """{name: dict(points, axis, axis_min, axis_max, polygon [m, 3])}; polygon w coordinates are nonzero, which the crop
    ignores."""
    rng = np.random.default_rng(71)
    cases = {}

    def add(name, uv_poly, uv_pts, axis="z", lo=-1.0, hi=1.0, w=None):
        w = _dyadic(rng.uniform(-1.5, 1.5, len(uv_pts)), 10) if w is None else w
        cases[name] = dict(points=_lift(uv_pts, axis, w), axis=axis, axis_min=lo, axis_max=hi,
                           polygon=_lift(uv_poly, axis, _dyadic(rng.uniform(-50, 50, len(uv_poly)), 4)))

    for m, axis in ((3, "z"), (255, "y"), (256, "z"), (257, "x"), (1024, "z"), (2048, "Y")):
        p = star(m)
        add(f"m{m}", p, _probe_points(p, rng, 3000, 9.0), axis.lower())
        cases[f"m{m}"]["axis"] = axis  # the axis name is case-insensitive
    p = star(64)[::-1].copy()
    add("clockwise", p, _probe_points(p, rng, 3000, 9.0))
    p = staircase()
    add("rectilinear", p, _probe_points(p, rng, 3000, 6.0), "x")
    p = degenerate_polygon()
    add("degenerate_edges", p, _probe_points(p, rng, 3000, 6.0), "y")
    add("bowtie", BOWTIE, np.concatenate([_probe_points(BOWTIE, rng, 3000, 6.0), [[0.0, 0.0], [1.0, 0.0]]]))
    add("bowtie_reversed", BOWTIE[::-1].copy(), _probe_points(BOWTIE, rng, 3000, 6.0))
    p = star(12)
    pts = _probe_points(p, rng, 500, 9.0)
    w = np.array([0.5, np.nextafter(0.5, 1), np.nextafter(0.5, 0)])[np.arange(len(pts)) % 3]
    add("slab_equal", p, pts, "z", 0.5, 0.5, w)
    add("slab_reversed", p, pts, "z", 1.0, -1.0, _dyadic(rng.uniform(-1.5, 1.5, len(pts)), 10))
    w = np.array([-0.0, 0.0, TINY, -TINY])[np.arange(len(pts)) % 4]
    add("zero_bounds", p, pts, "z", -0.0, 0.0, w)
    add("zero_bounds_swapped", p, pts, "z", 0.0, -0.0, w)
    big = np.array([[-1e308, -1e308], [1e308, -1e308], [1e308, 1e308], [-1e308, 1e308], [0.0, 3e307]])
    pts = np.concatenate([rng.uniform(-1.2, 1.2, size=(2000, 2)) * 1e308, big, rng.uniform(-1e300, 1e300, size=(500, 2))])
    add("huge", big, pts)
    p = star(10)
    for n in (1, 255, 256, 257):
        add(f"n{n}", p, _dyadic(rng.uniform(-9, 9, size=(n, 2)), 20))
    return cases


def crop_edges_selected(pu, pv, au, av, bu, bv):
    """The half-open crossing rule (exact in floating point: comparisons only)."""
    return ((av < pv) & (bv >= pv)) | ((bv < pv) & (av >= pv))


def _to_int(values, K):
    """Exact integers values * 2^K (Python ints in an object array)."""
    out = np.empty(len(values), dtype=object)
    for i, x in enumerate(np.asarray(values, np.float64).tolist()):
        n, d = x.as_integer_ratio()
        out[i] = n * (1 << K) // d if K >= 0 else Fraction(n, d) * Fraction(1, 1 << -K)
        assert K < 0 or out[i] * d == n * (1 << K)
    return out


def crop_exact(case, band_ulps=8):
    """Exact crossing-number test in rational arithmetic: every coordinate times a common power of two is an integer, and
    a selected edge's crossing X = a_u + (p_v - a_v)(b_u - a_u)/(b_v - a_v) lies below p_u iff
    (p_v - a_v)(b_u - a_u) < (p_u - a_u)(b_v - a_v) for b_v > a_v (reversed otherwise).  Returns (keep, band): band marks
    points with a selected edge whose exact crossing lies within band_ulps * eps * (|a_u| + |X - a_u|) of p_u without
    equalling it, or whose floating-point intermediates overflow; there the computed crossing may fall on either side."""
    u, v, w = AXES[case["axis"].lower()]
    P, pts = case["polygon"], case["points"]
    vals = np.concatenate([P[:, u], P[:, v], pts[:, u], pts[:, v]])
    nz = vals[vals != 0]
    K = int(53 - np.frexp(nz)[1].min()) if len(nz) else 0
    K = max(K, 0)
    Pu, Pv = _to_int(P[:, u], K), _to_int(P[:, v], K)
    pu, pv = _to_int(pts[:, u], K), _to_int(pts[:, v], K)
    below = np.zeros(len(pts), np.int64)
    band = np.zeros(len(pts), bool)
    m = len(P)
    for a in range(m):
        b = (a + 1) % m
        sel = crop_edges_selected(pts[:, u], pts[:, v], P[a, u], P[a, v], P[b, u], P[b, v])
        if not sel.any():
            continue
        idx = np.nonzero(sel)[0]
        den = Pv[b] - Pv[a]
        num = (pv[idx] - Pv[a]) * (Pu[b] - Pu[a])
        rhs = (pu[idx] - Pu[a]) * den
        diff = num - rhs  # = (X - p_u) * den
        lt = diff < 0 if den > 0 else diff > 0
        below[idx] += lt.astype(np.int64)
        scale = abs(Pu[a]) * abs(den) + np.abs(num)  # (|a_u| + |X - a_u|) * |den|
        near = (diff != 0) & (np.abs(diff) * (1 << 52) <= band_ulps * scale)  # X == p_u exactly is decided: not below
        with np.errstate(over="ignore", invalid="ignore"):
            overflow = not (np.isfinite(P[b, u] - P[a, u]) and np.isfinite(P[b, v] - P[a, v]))
            overflow = overflow | ~np.isfinite(pts[idx, v] - P[a, v])
        band[idx] |= near.astype(bool) | overflow
    pw = pts[:, w]
    keep = (pw >= case["axis_min"]) & (pw <= case["axis_max"]) & (below % 2 == 1)
    return keep, band


def crossing_float(pu_v, a, b):
    """The crop's crossing in its stated float64 order (the predicate that a crossing equals p_u)."""
    return a[0] + ((pu_v[1] - a[1]) / (b[1] - a[1])) * (b[0] - a[0])


# ----------------------------------------------------------------------------------------------------- voxel grid
def voxel_layout(points, vs):
    """gsb_pcd_voxel_downsample's host arithmetic restated: (lo, span, extents, bits per axis)."""
    p = np.asarray(points, np.float64)
    mn, mx = p.min(0), p.max(0)
    lo = mn - vs * 0.5
    span = float(((mx + vs * 0.5) - lo).max())
    extent = [int(math.floor((mx[a] - lo[a]) / vs)) + 1 for a in range(3)]
    bits = [next(b for b in range(64) if b == 63 or (1 << b) >= e) for e in extent]
    return lo, span, extent, bits


def voxel_cases():
    """{name: (points, voxel_size, expected)}; expected is "ok", or the words of the refusal."""
    rng = np.random.default_rng(72)
    cases = {}
    c = np.array([31.27, -12.9, 4.113])
    for n in (2, 1000, 1_000_000):
        cases[f"one_voxel_{n}"] = (c + rng.uniform(0, 0.004, size=(n, 3)), 0.01, "ok")  # extent < vs/2 on every axis
    plane = rng.normal(size=(20000, 3)) * 2
    plane[:, 2] = 1.75
    cases["planar"] = (plane, 0.05, "ok")
    line = rng.normal(size=(20000, 3)) * 2
    line[:, 1], line[:, 0] = -3.5, 0.125
    cases["linear"] = (line, 0.05, "ok")
    e = (1 << 21) - 1
    cube = rng.integers(0, e + 1, size=(50000, 3)).astype(np.float64)
    cube[:2] = [[0, 0, 0], [e, e, e]]
    cube[2:200] = cube[200:398]  # voxels holding two points
    cases["bits63"] = (cube, 1.0, "ok")
    over = cube.copy()
    over[1, 0] = e + 1
    cases["bits64"] = (over, 1.0, "63 bits")
    cases["int_max"] = (np.array([[0.0, 0, 0], [INT_MAX - 1.0, 0, 0], [12345.0, 0, 0]]), 1.0, "ok")
    cases["int_max_over"] = (np.array([[0.0, 0, 0], [float(INT_MAX), 0, 0]]), 1.0, "too small")
    for vs in (0.01, 0.005, 0.003, 0.0025, 0.0015):
        h = vs / 2  # the half-voxel lattice: every other point lies on a voxel boundary (p - lo)/vs = integer
        k = rng.integers(0, 400, size=(60000, 3)) + np.round(np.array([31.0, -12.0, 4.5]) / h).astype(np.int64)
        cases[f"lattice_{vs}"] = (k * h, vs, "ok")
    d = rng.permutation(np.stack(np.meshgrid(np.arange(40), np.arange(30), np.arange(20)), -1).reshape(-1, 3))
    cases["all_distinct"] = (d * 0.5 + 0.0625, 0.5, "ok")
    base = rng.normal(size=(500, 3))
    cases["duplicates"] = (base[rng.integers(0, 500, 20000)], 0.25, "ok")
    z = np.array([[0.0, 0.0, 0.0], [-0.0, -0.0, -0.0], [-0.0, 0.0, -0.0], [0.0, -0.0, 0.0], [0.125, -0.0, 0.0],
                  [1.0, 1.0, 1.0]])
    cases["signed_zero"] = (z, 1.0, "ok")
    return cases


def voxel_quotients(points, vs):
    lo = voxel_layout(points, vs)[0]
    return (np.asarray(points) - lo) / vs, lo


def voxel_exact(points, vs):
    """(keys [M, 3] ascending, groups (list of point-index arrays), boundary count).  A point's voxel is the floor of its
    exact quotient (p - lo) / vs; the float quotient is within 2.5 ulp of it, so only quotients within that of an integer
    are decided in Fraction.  A point whose exact quotient lies within one ulp of an integer is a boundary point: Open3D's
    floating-point quotient defines its voxel and it keeps that one (lo itself is Open3D's rounded min - vs/2)."""
    p = np.asarray(points, np.float64)
    q, lo = voxel_quotients(p, vs)
    fl = np.floor(q)
    key = fl.astype(np.int64)
    r = np.rint(q)
    near = np.abs(q - r) <= 4 * EPS * np.maximum(np.abs(q), 1.0)
    boundary = np.zeros(len(p), bool)
    F_vs = Fraction(float(vs))
    for i, a in zip(*np.nonzero(near)):
        qe = (Fraction(float(p[i, a])) - Fraction(float(lo[a]))) / F_vs
        n = round(qe)
        if abs(qe - n) <= EPS * abs(qe):
            boundary[i] = True  # keeps the floating-point voxel
        else:
            key[i, a] = math.floor(qe)
    keys, inverse = np.unique(key, axis=0, return_inverse=True)
    inverse = inverse.reshape(-1)
    order = np.argsort(inverse, kind="stable")
    groups = np.split(order, np.cumsum(np.bincount(inverse, minlength=len(keys)))[:-1])
    return keys, groups, int(boundary.sum())


def exact_sum(values):
    """The exact sum of float64 values as a Fraction (integers over a common power of two)."""
    v = np.asarray(values, np.float64)
    nz = v[v != 0]
    if not len(nz):
        return Fraction(0)
    K = int(53 - np.frexp(nz)[1].min())
    scaled = np.ldexp(v, K) if K < 1000 else None
    if scaled is not None and np.isfinite(scaled).all() and np.abs(scaled).max() < 2.0 ** 62:
        total = sum(scaled.astype(np.int64).tolist())
        return Fraction(total) / Fraction(2) ** K
    return sum((Fraction(x) for x in v.tolist()), Fraction(0))


def voxel_mean_check(points, groups, got):
    """Each computed mean within count * eps * sum|p| / count of the exact mean of its voxel's points."""
    p = np.asarray(points, np.float64)
    assert len(got) == len(groups)
    single = np.array([len(g) == 1 for g in groups], bool)
    if single.any():  # one point: 0.0 + p, divided by 1, is p (+0.0 for -0.0)
        first = np.array([g[0] for g in groups])
        assert np.array_equal(np.asarray(got)[single], p[first[single]])
    worst = 0.0
    for g, mean in zip(groups, got):
        c = len(g)
        if c == 1:
            continue
        for a in range(3):
            col = p[g, a]
            exact = exact_sum(col) / c
            bound = c * Fraction(EPS) * exact_sum(np.abs(col)) / c
            err = abs(Fraction(float(mean[a])) - exact)
            assert err <= bound, (g[:4], a, float(mean[a]), float(exact))
            if bound:
                worst = max(worst, float(err / bound))
    return worst


# ---------------------------------------------------------------------------------------------------------- moments
def moment_cases():
    """{name: (source [n,3], target [m,3], index [n], d2 [n])}."""
    rng = np.random.default_rng(73)
    cases = {}

    def random_case(n, offset=0.0):
        src = rng.normal(size=(n, 3)) * 5 + offset
        tgt = rng.normal(size=(4097, 3)) * 5 + offset
        idx = np.where(rng.random(n) < 0.8, rng.integers(0, len(tgt), n), -1)
        idx[n // 2] = len(tgt) - 1  # the last target row
        d2 = rng.random(n)
        d2[::97] = 0.0
        d2[1::97] = TINY * rng.integers(1, 1 << 20, size=len(d2[1::97]))  # subnormal
        return src, tgt, idx, d2

    for n in (65535, 65536, 65537, 131073):
        cases[f"n{n}"] = random_case(n)
    cases["far"] = random_case(65537, np.array([3.0e4, -1.0e5, 250.0]))
    src, tgt, idx, d2 = random_case(65537)
    cases["no_correspondence"] = (src, tgt, np.full(len(src), -1, np.int64), d2)
    src, tgt, _, d2 = random_case(65536)
    idx = np.full(65536, -1, np.int64)
    idx[MOMENT_LANES - 1] = len(tgt) - 1  # lane 255 of block 255
    cases["last_lane"] = (src, tgt, idx, d2)
    return cases


def moment_values(src, tgt, idx, d2, means=None):
    """The per-correspondence values the moments sum (each product rounded once), rows of non-correspondences removed."""
    hit = idx >= 0
    s, t = src[hit], tgt[idx[hit]]
    if means is None:
        return np.concatenate([d2[hit, None], s, t], 1)
    sd, td = s - means[:3], t - means[3:]
    return np.concatenate([(td[:, :, None] * sd[:, None, :]).reshape(-1, 9), sd * sd], 1)


def moment_fsum_check(values, n, got):
    """Every column within (ceil(n / 65536) + 16) * eps * sum|x| of math.fsum: a lane adds ceil(n / 65536) values, then
    16 halvings follow (8 within a block, 8 across blocks)."""
    depth = -(-n // MOMENT_LANES) + 16
    worst = 0.0
    for q in range(values.shape[1]):
        col = values[:, q].tolist()
        ref = math.fsum(col)
        bound = depth * EPS * math.fsum(abs(x) for x in col)
        err = abs(float(got[q]) - ref)
        assert err <= bound, (q, float(got[q]), ref, bound)
        if bound:
            worst = max(worst, err / bound)
    return worst


# -------------------------------------------------------------------------------------------------------------- ICP
def surface(n_side, extent=1.5):
    g = np.linspace(-extent, extent, n_side)
    x, y = np.meshgrid(g, g)
    return np.stack([x.ravel(), y.ravel(), (0.3 * np.sin(3 * x) * np.cos(2 * y) + 0.1 * x ** 2).ravel()], 1)


RIGID = similarity(0.02, [1, 2, 3], 1.0, [0.01, -0.005, 0.008])


def icp_cases():
    """{name: dict(source, target, radius, init, with_scaling, max_iteration, relative)}."""
    rng = np.random.default_rng(74)
    cases = {}

    def add(name, source, target, radius, init=None, with_scaling=True, max_iteration=30, relative=1e-6):
        cases[name] = dict(source=np.asarray(source, np.float64).reshape(-1, 3),
                           target=np.asarray(target, np.float64).reshape(-1, 3), radius=radius,
                           init=np.eye(4) if init is None else init, with_scaling=with_scaling,
                           max_iteration=max_iteration, relative=relative)

    gt = surface(61)
    inv = np.linalg.inv(RIGID)
    scan = gt[rng.permutation(len(gt))[:1500]]
    moved = np.stack([((inv[r, 0] * scan[:, 0] + inv[r, 1] * scan[:, 1]) + inv[r, 2] * scan[:, 2]) + inv[r, 3]
                      for r in range(3)], 1)
    add("rigid", moved, gt, 0.1, with_scaling=False, max_iteration=100, relative=1e-12)
    xy = np.stack(np.meshgrid(np.linspace(-1, 1, 21), np.linspace(-1, 1, 21)), -1).reshape(-1, 2)
    slab = np.concatenate([xy, rng.uniform(0.005, 0.02, size=(len(xy), 1)) * rng.choice([-1, 1], (len(xy), 1))], 1)
    add("mirror", slab, slab * np.array([1.0, 1.0, -1.0]), 0.05, max_iteration=5)
    add("mirror_rigid", slab, slab * np.array([1.0, 1.0, -1.0]), 0.05, with_scaling=False, max_iteration=5)
    one = np.tile([[0.5, 0.25, -1.0]], (4, 1))
    near = np.array([[0.5, 0.25, -1.0]]) + rng.normal(scale=0.01, size=(50, 3))
    add("one_source_point", one, near, 0.2)
    add("one_source_point_rigid", one, near, 0.2, with_scaling=False)
    t = _dyadic(rng.uniform(-1, 1, 200), 10)[:, None]
    line = t * np.array([[1.0, 2.0, -1.0]])
    add("collinear", line, line + np.array([0.015625, 0.03125, -0.015625]), 0.1)
    add("max_iteration_0", gt[:500], gt, 0.1, max_iteration=0)
    add("empty_source", np.zeros((0, 3)), gt[:100], 0.1)
    add("empty_target", gt[:100], np.zeros((0, 3)), 0.1)
    init = np.eye(4)
    init[0, 1] = init[1, 3] = init[2, 0] = init[3, 2] = -0.0
    add("negative_zero_init", gt[::3] + np.array([0.01, 0.0, -0.01]), gt, 0.1, init=init)
    return cases


def first_umeyama_inputs(case):
    """The first iteration's pass-0 and pass-1 moments, in the oracle's order (the host predicates' view of a case)."""
    from oracle import tnt_oracle as to

    src, tgt = case["source"], case["target"]
    idx, d2 = to.correspond(src, tgt, case["radius"])
    sums, cnt = to.moments(src, tgt, idx, d2)
    mu = np.concatenate([sums[1:4], sums[4:7]]) * (1.0 / cnt)
    return sums, cnt, to.moments(src, tgt, idx, d2, mu)[0]
