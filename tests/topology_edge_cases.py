"""Edge cases of the topology queries (DESIGN.md section 7, "Topology queries"), shared by
tests/test_topology_edges_host.py and tests/test_gpu_topology_edges.py.

- exact_tri_tri: closed-set triangle-triangle intersection on integer coordinates, from orientation signs alone (not
  from Moeller's algorithm), and robust_class, which sorts a pair into separated / crossing / contact by testing it again
  with both triangles grown and shrunk about their centroids.
- Lattice soups and crafted branch families (vertex on face, vertex on edge, edge on edge, vertex on vertex, an edge in
  the other plane, coplanar overlap / edge touch / containment / disjoint in planes whose normalised normals tie), and
  epsilon pairs on either side of NoDivTriTriIsect's 1e-6 clamp.
- Grid cases for the self-intersection broad phase, each stating the level and registrations the grid rule must reach,
  with a numpy port of the kernel's cell_of and level rule."""
import numpy as np

from tests import topology_oracle as to

SEPARATED, CROSSING, CONTACT = 0, 1, 2
ROBUST_SCALE = 500  # robust_class grows and shrinks by 1 +- 1/ROBUST_SCALE


# --- exact closed-set intersection on integers ------------------------------------------------------------------------

def _orient3d(a, b, c, d):
    """sign of det[b - a, c - a, d - a] per row (int64 rows of 3)."""
    u, v, w = b - a, c - a, d - a
    det = (u[:, 0] * (v[:, 1] * w[:, 2] - v[:, 2] * w[:, 1]) - u[:, 1] * (v[:, 0] * w[:, 2] - v[:, 2] * w[:, 0])
           + u[:, 2] * (v[:, 0] * w[:, 1] - v[:, 1] * w[:, 0]))
    return np.sign(det)


def _orient2d(a, b, c):
    return np.sign((b[:, 0] - a[:, 0]) * (c[:, 1] - a[:, 1]) - (b[:, 1] - a[:, 1]) * (c[:, 0] - a[:, 0]))


def _seg_seg_2d(p, q, r, s):
    """closed segments pq and rs meet (2-D rows)."""
    d1, d2 = _orient2d(r, s, p), _orient2d(r, s, q)
    d3, d4 = _orient2d(p, q, r), _orient2d(p, q, s)
    proper = (d1 * d2 <= 0) & (d3 * d4 <= 0)
    collinear = (d1 == 0) & (d2 == 0)
    overlap = np.ones(len(p), bool)
    for a in range(2):
        overlap &= (np.maximum(np.minimum(p[:, a], q[:, a]), np.minimum(r[:, a], s[:, a]))
                    <= np.minimum(np.maximum(p[:, a], q[:, a]), np.maximum(r[:, a], s[:, a])))
    return np.where(collinear, overlap, proper)


def _point_in_tri_2d(p, a, b, c):
    """p in the closed non-degenerate triangle abc."""
    s = np.stack([_orient2d(a, b, p), _orient2d(b, c, p), _orient2d(c, a, p)], axis=1)
    return (s >= 0).all(axis=1) | (s <= 0).all(axis=1)


def _drop_axis(T):
    """the two axes kept when projecting triangle rows T (n, 3, 3) along their normal's largest component."""
    n = np.cross(T[:, 1] - T[:, 0], T[:, 2] - T[:, 0])
    k = np.argmax(np.abs(n), axis=1)
    keep = np.array([[1, 2], [0, 2], [0, 1]])[k]
    return keep


def _proj(X, keep):
    return np.take_along_axis(X, keep, axis=1)


def _seg_tri_2d(a, b, T, keep):
    A, B = _proj(a, keep), _proj(b, keep)
    C = [_proj(T[:, k], keep) for k in range(3)]
    hit = _point_in_tri_2d(A, *C) | _point_in_tri_2d(B, *C)
    for k in range(3):
        hit |= _seg_seg_2d(A, B, C[k], C[(k + 1) % 3])
    return hit


def _tri_tri_2d(P, Q, keep):
    Pp = [_proj(P[:, k], keep) for k in range(3)]
    Qp = [_proj(Q[:, k], keep) for k in range(3)]
    hit = _point_in_tri_2d(Pp[0], *Qp) | _point_in_tri_2d(Qp[0], *Pp)
    for i in range(3):
        for j in range(3):
            hit |= _seg_seg_2d(Pp[i], Pp[(i + 1) % 3], Qp[j], Qp[(j + 1) % 3])
    return hit


def _seg_tri(a, b, T):
    """closed segment ab meets the closed non-degenerate triangle T (n, 3, 3)."""
    c, d, e = T[:, 0], T[:, 1], T[:, 2]
    oa, ob = _orient3d(c, d, e, a), _orient3d(c, d, e, b)
    in_plane = (oa == 0) & (ob == 0)
    reaches = oa * ob <= 0
    s = np.stack([_orient3d(a, b, c, d), _orient3d(a, b, d, e), _orient3d(a, b, e, c)], axis=1)
    through = (s >= 0).all(axis=1) | (s <= 0).all(axis=1)  # the line ab meets the triangle (not all zero: ab crosses its plane)
    hit = reaches & ~in_plane & through
    if in_plane.any():
        m = in_plane
        hit[m] = _seg_tri_2d(a[m], b[m], T[m], _drop_axis(T[m]))
    return hit


def degenerate(T):
    """rows of T (n, 3, 3) whose corners are collinear (exact on integers)."""
    T = np.asarray(T, np.int64)
    return (np.cross(T[:, 1] - T[:, 0], T[:, 2] - T[:, 0]) == 0).all(axis=1)


def exact_tri_tri(P, Q):
    """Closed triangles P, Q (n, 3, 3), integer coordinates, neither degenerate: do they share a point?  Not coplanar:
    iff an edge of one meets the other (the intersection lies on the planes' common line, and its ends lie on the
    boundary of one triangle).  Coplanar: projected along the normal's largest component, iff an edge pair meets or a
    corner of one lies in the other.  Orientation signs in int64: |coordinates| below 2^19, so
    every determinant (at most 6 (2^20)^3) is exact."""
    P, Q = np.asarray(P, np.int64), np.asarray(Q, np.int64)
    assert not degenerate(P).any() and not degenerate(Q).any()
    assert np.abs(P).max(initial=0) < 2 ** 19 and np.abs(Q).max(initial=0) < 2 ** 19
    coplanar = np.ones(len(P), bool)
    for k in range(3):
        coplanar &= _orient3d(P[:, 0], P[:, 1], P[:, 2], Q[:, k]) == 0
    hit = np.zeros(len(P), bool)
    g = ~coplanar
    if g.any():
        Pg, Qg = P[g], Q[g]
        h = np.zeros(len(Pg), bool)
        for k in range(3):
            h |= _seg_tri(Pg[:, k], Pg[:, (k + 1) % 3], Qg) | _seg_tri(Qg[:, k], Qg[:, (k + 1) % 3], Pg)
        hit[g] = h
    if coplanar.any():
        hit[coplanar] = _tri_tri_2d(P[coplanar], Q[coplanar], _drop_axis(P[coplanar]))
    return hit


def _scaled(T, num, den):
    """T scaled about its centroid by num / den, in units of 1 / (3 den): integers."""
    T = np.asarray(T, np.int64) * 3 * den
    c = T.sum(axis=1, keepdims=True) // 3
    return c + (T - c) * num // den


def robust_class(P, Q):
    """SEPARATED if P and Q still miss with both grown by 1 + delta about their centroids, CROSSING if they still meet
    with both shrunk by 1 - delta, else CONTACT (delta = 1 / ROBUST_SCALE; the scaling is exact in integers)."""
    d = ROBUST_SCALE
    grown = exact_tri_tri(_scaled(P, d + 1, d), _scaled(Q, d + 1, d))
    shrunk = exact_tri_tri(_scaled(P, d - 1, d), _scaled(Q, d - 1, d))
    return np.where(~grown, SEPARATED, np.where(shrunk, CROSSING, CONTACT))


# --- soups and pairs as meshes ----------------------------------------------------------------------------------------

def soup_mesh(T):
    """Triangles (n, 3, 3) as a mesh in which every triangle has its own three vertex ids."""
    T = np.asarray(T, np.float64).reshape(-1, 3, 3)
    return T.reshape(-1, 3), np.arange(3 * len(T), dtype=np.int64).reshape(-1, 3)


def lattice_soup(seed, n=800, side=6):
    """n random non-degenerate triangles with integer corners in [0, side]^3."""
    rng = np.random.default_rng(seed)
    T = rng.integers(0, side + 1, size=(3 * n, 3, 3))
    T = T[~degenerate(T)][:n]
    assert len(T) == n
    return T


def box_pairs(T):
    """(i, j), i < j, of the triangles whose boxes overlap, touching included: the restatement's candidates for a
    soup (no shared ids)."""
    T = np.asarray(T, np.float64)
    lo, hi = T.min(axis=1), T.max(axis=1)
    i, j = np.triu_indices(len(T), 1)
    ok = ~((hi[i] < lo[j]) | (lo[i] > hi[j])).any(axis=1)
    return i[ok], j[ok]


def pair_flags(pairs, i, j, n):
    """For each candidate (i, j), is it among pairs (k, 2)?"""
    have = np.zeros(0, np.int64) if len(pairs) == 0 else pairs[:, 0] * n + pairs[:, 1]
    return np.isin(i * n + j, have)


# --- crafted branch families ------------------------------------------------------------------------------------------
# Each family is an exact-contact instance with its push vector: the pair as built, Q moved by -push (pushed in) and
# Q moved by +push (pushed apart).  P is z = 0 unless stated.

_FLOOR = np.array([[0, 0, 0], [8, 0, 0], [0, 8, 0]])

FAMILIES = {
    # Q's first corner on P's face
    "vertex_on_face": (_FLOOR, [[2, 2, 0], [3, 2, 5], [2, 3, 5]], [0, 0, 1]),
    # Q's first corner on P's edge y = 0
    "vertex_on_edge": (_FLOOR, [[4, 0, 0], [5, -2, 4], [3, -2, 4]], [0, -1, 1]),
    # Q's edge along y through P's bottom edge; P in the plane y = 0
    "edge_on_edge": ([[0, 0, 0], [8, 0, 0], [4, 0, 8]], [[4, -4, 0], [4, 4, 0], [4, 0, -8]], [0, 0, -1]),
    # one position under two ids
    "vertex_on_vertex": (_FLOOR, [[0, 0, 0], [-3, 1, 5], [1, -3, 5]], [-1, -1, 1]),
    # Q's edge (first and last corners) lies in P's plane and crosses P's interior
    "edge_in_plane": (_FLOOR, [[-2, 4, 0], [1, 1, 6], [4, -2, 0]], [0, 0, 1]),
    # Q's edge lies in P's plane beside P, on a line that cuts P (so P straddles Q's plane and the interval code runs):
    # separated; pushed in, it touches P's long edge
    "edge_in_plane_beside": (_FLOOR, [[6, 3, 0], [7, 5, 6], [6, 7, 0]], [0, 1, 0]),
}


def _rotations(T):
    T = np.asarray(T)
    return [T[[k, (k + 1) % 3, (k + 2) % 3]] for k in range(3)]


def branch_family_pairs():
    """{family: (P, Q) (n, 3, 3)}: every family as built, pushed in and pushed apart, with both triangles in each of
    their three corner rotations and in both orders, so every vertex / edge lands in every slot of the interval code."""
    out = {}
    for name, (P, Q, push) in FAMILIES.items():
        P, Q, push = np.asarray(P), np.asarray(Q), np.asarray(push)
        Ps, Qs = [], []
        for s in (0, -1, 1):
            Qm = Q + s * push
            for Pr in _rotations(P):
                for Qr in _rotations(Qm):
                    Ps += [Pr, Qr]
                    Qs += [Qr, Pr]
        out[name] = (np.array(Ps, np.int64), np.array(Qs, np.int64))
    return out


# Coplanar configurations in 2-D (a, b), each with its push: P = (0,0), (8,0), (0,8).
_P2 = [[0, 0], [8, 0], [0, 8]]
COPLANAR_2D = {
    "overlap": ([[2, 2], [10, 2], [2, 10]], [1, 1]),
    "edge_touch": ([[8, 0], [0, 8], [8, 8]], [1, 1]),
    "q_in_p": ([[1, 1], [5, 1], [1, 5]], [-1, -1]),      # strictly inside, pushed further in, pushed out through an edge
    "p_in_q": ([[-2, -2], [14, -2], [-2, 14]], [-1, -1]),
    "disjoint": ([[6, 6], [14, 6], [6, 14]], [1, 1]),
    "vertex_touch": ([[8, 0], [12, -2], [12, 2]], [1, 0]),
}

# Plane bases (e1, e2) with e1 x e2 along the tie; every family is embedded as 6 * (a e1 + b e2) + origin so the
# per-axis sums of the six corners are multiples of 6 (the normalisation's mean is exact).
TIE_PLANES = {
    (1, 1, 0): ([1, -1, 0], [0, 0, 1]),
    (1, 0, 1): ([-1, 0, 1], [0, 1, 0]),  # e1 x e2 = (-1, 0, -1)
    (0, 1, 1): ([0, 1, -1], [1, 0, 0]),  # (0, -1, -1)
    (1, -1, 0): ([1, 1, 0], [0, 0, 1]),
}

# Möller's coplanar projection on a tie: A0 > A1 ? (A0 > A2 ? (1, 2) : (0, 1)) : (A2 > A1 ? (0, 1) : (0, 2)).
TIE_AXES = {(1, 1, 0): (0, 2), (1, 0, 1): (0, 1), (0, 1, 1): (0, 2), (1, -1, 0): (0, 2), (1, 1, 1): (0, 2)}


def _embed(T2, e1, e2, origin):
    T2 = np.asarray(T2, np.int64)
    return 6 * (T2[..., :1] * np.asarray(e1) + T2[..., 1:] * np.asarray(e2)) + np.asarray(origin)


def _cyclic(a):
    """The triangle a, rot a, rot^2 a with rot(x, y, z) = (y, z, x): its normal is along (1, 1, 1)."""
    a = np.asarray(a, np.int64)
    return np.stack([a, a[[1, 2, 0]], a[[2, 0, 1]]])


def _normalised_normal(P, Q):
    q = to.normalise(P, Q)
    return np.abs(to._cross(q[:, 1] - q[:, 0], q[:, 2] - q[:, 0]))


def ties(P, Q, tie):
    """Rows whose normalised |N1| has the tie's nonzero components exactly equal and the others smaller."""
    A = _normalised_normal(P, Q)
    nz = [k for k in range(3) if tie[k]]
    ok = np.ones(len(P), bool)
    for k in nz[1:]:
        ok &= A[:, k] == A[:, nz[0]]
    for k in range(3):
        if not tie[k]:
            ok &= A[:, k] < A[:, nz[0]]
    return ok


def tie_family_pairs():
    """{(tie, config): (P, Q)}: the coplanar configurations as built, pushed in and pushed apart, in every tie plane,
    kept where the normalised normal ties exactly (all rows for the two-axis ties, whose planes keep the per-axis
    deviations equal up to sign; a search over centred cyclic triangles for (1, 1, 1))."""
    out = {}
    for tie, (e1, e2) in TIE_PLANES.items():
        for name, (Q2, push) in COPLANAR_2D.items():
            Ps, Qs = [], []
            for s in (0, -1, 1):
                Qm = np.asarray(Q2) + s * np.asarray(push)
                P3, Q3 = _embed(_P2, e1, e2, [6, 12, 18]), _embed(Qm, e1, e2, [6, 12, 18])
                for Pr in _rotations(P3):
                    Ps += [Pr, Q3]
                    Qs += [Q3, Pr]
            out[(tie, name)] = (np.array(Ps), np.array(Qs))
    # (1, 1, 1): cyclic triangles about the axis x = y = z, in the plane x + y + z = 3m (the per-axis multisets of
    # the six corners are equal, so the per-axis sigmas are); ties of the rounded normal are searched for
    rng = np.random.default_rng(111)
    Ps, Qs = [], []
    while len(Ps) < 400:
        a = rng.integers(-12, 13, size=2)
        b = rng.integers(-12, 13, size=2)
        a = np.array([a[0], a[1], -a[0] - a[1]]) * 2 + 10  # coordinate sums 30: the mean of six is exact
        b = np.array([b[0], b[1], -b[0] - b[1]]) * 2 + 10
        P, Q = _cyclic(a), _cyclic(b)
        if degenerate(P[None])[0] or degenerate(Q[None])[0]:
            continue
        if ties(P[None], Q[None], (1, 1, 1))[0]:
            Ps.append(P)
            Qs.append(Q)
    out[((1, 1, 1), "cyclic")] = (np.array(Ps), np.array(Qs))
    return out


# --- epsilon pairs ----------------------------------------------------------------------------------------------------

def epsilon_pairs():
    """(P, Q, du0): P in the plane z = y / 2, Q with its first corner hovering over P's interior point (1, 1, 1/2) at a
    normalised plane distance du0 of +-0.9e-6 and +-1.1e-6 (found by the secant method on the restatement's own
    arithmetic), the other two corners well to the same side.  Below 1e-6 the clamp puts the corner on the plane and
    the pair touches; above, Q lies wholly on one side.  P is tilted so the two boxes overlap and the pair reaches the
    narrow phase."""
    P = np.array([[0.0, 0, 0], [4, 0, 0], [0, 4, 2]])
    rows = []
    for target in (0.9e-6, 1.1e-6, -0.9e-6, -1.1e-6):
        def du(h):
            Q = np.array([[1.0, 1, 0.5 + h], [2, 1, 0.5 + 3 * np.sign(target)], [1, 2, 1 + 3 * np.sign(target)]])
            return to.plane_distances(P[None], Q[None])[0][0, 0], Q

        h0, h1 = 1e-7 * np.sign(target), 2e-7 * np.sign(target)
        for _ in range(30):
            f0, f1 = du(h0)[0] - target, du(h1)[0] - target
            if f1 == f0 or abs(f1) < 1e-12 * abs(target):
                break
            h0, h1 = h1, h1 - f1 * (h1 - h0) / (f1 - f0)
        d, Q = du(h1)
        assert abs(d - target) < 1e-3 * abs(target)
        rows.append((P, Q, d))
    return rows


# --- grid cases -------------------------------------------------------------------------------------------------------
LEVELS = 22
REGS_PER_TRIANGLE = 4


def cell_of(x, o, extent, level):
    """The kernel's cell_of: floor(clamp((x - o) / extent, 0, 1) * 2^(20 - level))."""
    u = np.clip((np.asarray(x, np.float64) - o) / extent, 0.0, 1.0)
    return np.floor(np.ldexp(u, 20 - level)).astype(np.int64)


def grid_extent(v, t):
    """(origin, extent) over the referenced vertices, with the kernel's 1.0 for a zero or non-finite extent."""
    p = np.asarray(v, np.float64)[np.asarray(t, np.int64).reshape(-1)]
    lo, hi = p.min(axis=0), p.max(axis=0)
    e = float((hi - lo).max())
    return lo, (e if e > 0 and np.isfinite(e) else 1.0)


def grid_level(v, t):
    """(level, registrations) of the grid rule: the finest level whose registrations (cells per triangle box, summed)
    are at most 4 n."""
    v, t = np.asarray(v, np.float64), np.asarray(t, np.int64)
    o, e = grid_extent(v, t)
    p = v[t]
    lo, hi = p.min(axis=1), p.max(axis=1)
    for L in range(LEVELS):
        n = np.prod(cell_of(hi, o, e, L) - cell_of(lo, o, e, L) + 1, axis=1)
        regs = int(np.minimum(n, 2 ** 32).sum())
        if regs <= REGS_PER_TRIANGLE * len(t) or L == LEVELS - 1:
            return L, regs


# Two triangles crossing inside the unit cube, each with the box [0, 1]^3 (one in the plane x = y).
_CROSS_PAIR = np.array([[[0, 0, 0], [1, 1, 0], [0.5, 0.5, 1]], [[1, 0, 0], [0, 1, 1], [1, 0, 1]]])
_ANCHOR = np.array([[0, 0, 0.5], [0.5, 0, 0], [0, 0.5, 0.25]])  # box [0, 1/2]^3


def _in_box(T, lo, size):
    return np.asarray(lo, np.float64) + np.asarray(T, np.float64) * size


def _anchors(c):
    """Triangles with boxes [0, c/2]^3 and [1 - c/2, 1]^3: the bounds are exactly [0, 1]^3, one corner at min_bound,
    one at max_bound (u = 1 on every axis, the extra cell 2^(20 - L))."""
    return [_in_box(_ANCHOR, 0.0, c), 1.0 - _in_box(_ANCHOR, 0.0, c)]


def level_case(L, pairs=3):
    """A mesh in [0, 1]^3 reaching grid level L: `pairs` crossing pairs, each pair with the box [k c + c/4, k c + 3c/4]^3
    (c = 2^(L - 20), one cell at level L, 2 per axis at L - 1) in its own cell, plus the two anchors (1 and 8 cells at
    level L).  Registrations at L: 2 pairs + 9 <= 4 n; at every finer level at least 8 per crossing triangle > 4 n.
    L = 21: every triangle spans [0, 1]^3 (8 cells at level 20, one at 21).
    Returns (triangles (n, 3, 3), level, registrations, crossing pairs)."""
    if L == 21:
        T = [_CROSS_PAIR[k] for _ in range(pairs) for k in range(2)]
        return np.array(T, np.float64), 21, len(T), [(2 * i, 2 * i + 1) for i in range(pairs)]
    c = 2.0 ** (L - 20)
    ks = np.unique(np.linspace(0, 2 ** (20 - L) - 1, pairs).astype(np.int64))  # one pair at level 20
    T = []
    for k in ks:
        for tri in _CROSS_PAIR:
            T.append(_in_box(tri, k * c + c / 4, c / 2))
    T += _anchors(c)
    return np.array(T), L, 2 * len(ks) + 9, [(2 * i, 2 * i + 1) for i in range(len(ks))]


def threshold_case(L=10, over=False):
    """Registrations at level L exactly 4 n (over=False: level L is chosen) or 4 n + 1 (over=True: level L + 1).
    Three one-cell crossing-type triangles, two triangles with the box [k c + c/2, k c + 3c/2]^3 (8 cells at L, k even
    so one cell at L + 1) and the anchors: 3 + 16 + 9 = 28 = 4 * 7.  over=True stretches one one-cell triangle across a
    cell face in x (2 cells at L, one at L + 1): 29 at L, 3 + 2 + 9 = 14 at L + 1."""
    c = 2.0 ** (L - 20)
    T = [_in_box(_CROSS_PAIR[0], k * c + c / 4, c / 2) for k in (100, 200, 300)]
    if over:
        T[0] = T[0].copy()
        T[0][:, 0] = 100 * c + c / 2 + _CROSS_PAIR[0][:, 0] * c
    T += [_in_box(_CROSS_PAIR[1], k * c + c / 2, c) for k in (400, 600)]
    T += _anchors(c)
    return np.array(T), (L + 1 if over else L), (14 if over else 28)


def boundary_case(n=800):
    """Boxes whose faces, and whose pairwise intersections' minimum corners, lie on cell faces of the chosen level:
    triangles flat on one axis at an integer plane, spanning one unit square [b, b + 1]^2 on the other two, corners on
    the integer lattice of [0, 8]^3 (bounds exactly [0, 8]^3, so level 17 has cells of one unit).  Each box registers
    2 x 2 x 1 cells at level 17, exactly 4 n, and 3 x 3 x 1 at level 16.  Crossing, coplanar and touching pairs meet
    on cell faces.  Returns (triangles, level, registrations)."""
    rng = np.random.default_rng(17)
    T = [np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]]), np.array([[8, 8, 8], [7, 8, 8], [8, 7, 8]])]
    square = np.array([[0, 0], [1, 0], [0, 1], [1, 1]])
    while len(T) < n:
        flat = rng.integers(0, 3)
        corners = square[rng.choice(4, size=3, replace=False)] + rng.integers(0, 8, size=2)
        tri = np.insert(corners, flat, rng.integers(0, 9), axis=1)
        T.append(tri)
    return np.array(T, np.int64), 17, 4 * n


def flat_case(axes):
    """Triangles flat in `axes` (1: z = 0.25 for all; 2: y = z = 0.25, degenerate triangles on a line; 3: all corners
    on one point).  For 1 and 2 the x (and y) layout of level_case(10)'s cells: (level, registrations) from the cell
    counts per axis, see the test."""
    if axes == 3:  # zero extent: the kernel's extent 1.0, every corner in cell 0 at every level
        return np.full((40, 3, 3), 0.375), 0, 40
    T, _, _, _ = level_case(10)
    T = T.copy()
    T[:, :, 2] = 0.25
    if axes == 2:
        T[:, :, 1] = 0.25
    # level_case(10) at one flat axis: every box spans 2 x 2 cells at level 9 (4 n, which fits) and 3 x 3 at level 8.
    # At two flat axes: 2, 3 and 5 cells per box at levels 9, 8 and 7, so level 8 with 3 n.
    n = len(T)
    return (T, 9, 4 * n) if axes == 1 else (T, 8, 3 * n)
