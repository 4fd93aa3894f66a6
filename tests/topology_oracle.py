"""numpy restatement of the mesh topology queries (DESIGN.md section 7, "Topology queries"): Open3D 0.17.0's
GetNonManifoldEdges, IsOrientable, EulerPoincareCharacteristic, GetNonManifoldVertices, GetSelfIntersectingTriangles,
GetSurfaceArea and GetVolume.

Graphs are solved with scipy's connected_components, the self-intersection broad phase is a sort-and-sweep along x
(not the GPU's grid), and the narrow phase is Moeller's NoDivTriTriIsect written once over arrays of pairs.  Every float
operation is one numpy fp64 operation in the GPU's order, so results agree bit for bit."""
import numpy as np
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components

EPSILON = 1e-6
SUM_THREADS = 256  # the block of the fixed-shape sum


def _tri(t):
    return np.asarray(t, dtype=np.int64).reshape(-1, 3)


def _incidences(t, nv):
    """(key, triangle, direction) of the 3 nt edge incidences in triangle-major order, sorted stably by key."""
    t = _tri(t)
    a = t.reshape(-1)
    b = t[:, [1, 2, 0]].reshape(-1)
    stride = nv + 1
    key = np.minimum(a, b) * stride + np.maximum(a, b)
    order = np.argsort(key, kind="stable")
    return key[order], (order // 3), (a > b)[order], stride


def edges(t, nv, allow_boundary_edges=True):
    """(non-manifold edges int64 (k, 2) ascending, distinct edge count)."""
    key, _, _, stride = _incidences(t, nv)
    uniq, counts = np.unique(key, return_counts=True)
    bad = counts > 2 if allow_boundary_edges else counts != 2
    k = uniq[bad]
    return np.stack([k // stride, k % stride], axis=1).astype(np.int64).reshape(-1, 2), len(uniq)


def is_orientable(t, nv):
    """Union-find over the double cover (2t: as given, 2t + 1: flipped); one constraint per incidence of an edge (a, b),
    a != b, against the edge's first incidence in (triangle, corner) order."""
    key, tri, direction, stride = _incidences(t, nv)
    nt = len(_tri(t))
    if nt == 0:
        return True
    head = np.ones(len(key), bool)
    head[1:] = key[1:] != key[:-1]
    centre = np.maximum.accumulate(np.where(head, np.arange(len(key)), 0))
    m = ~head & (key // stride != key % stride)
    u, c = tri[m], tri[centre[m]]
    same = direction[m] == direction[centre[m]]
    src = np.concatenate([2 * u, 2 * u + 1])
    dst = np.concatenate([2 * c + same, 2 * c + 1 - same])
    g = coo_matrix((np.ones(len(src), np.int8), (src, dst)), shape=(2 * nt, 2 * nt))
    _, label = connected_components(g, directed=False)
    return bool((label[0::2] != label[1::2]).all())


def euler_poincare(t, nv):
    return nv + len(_tri(t)) - edges(t, nv)[1]


def link_edges(t):
    """(vertex, x, y) rows: for every triangle and each distinct vertex v of it, Open3D's chain (t0, t1) / (t0, t2) /
    (t1, t2), the first pair without v; none if every pair holds v."""
    t = _tri(t)
    rows = []
    for k in range(3):
        v = t[:, k]
        first = np.ones(len(t), bool) if k == 0 else (t[:, :k] != v[:, None]).all(axis=1)
        c01 = (t[:, 0] != v) & (t[:, 1] != v)
        c02 = ~c01 & (t[:, 0] != v) & (t[:, 2] != v)
        c12 = ~c01 & ~c02 & (t[:, 1] != v) & (t[:, 2] != v)
        x = np.where(c01 | c02, t[:, 0], t[:, 1])
        y = np.where(c01, t[:, 1], t[:, 2])
        m = first & (c01 | c02 | c12)
        rows.append(np.stack([v[m], x[m], y[m]], axis=1))
    return np.concatenate(rows).reshape(-1, 3)


def non_manifold_vertices(t, nv):
    e = link_edges(t)
    if len(e) == 0:
        return np.zeros(0, np.int64)
    keys = np.concatenate([e[:, 0] * nv + e[:, 1], e[:, 0] * nv + e[:, 2]])
    nodes, inv = np.unique(keys, return_inverse=True)
    g = coo_matrix((np.ones(len(e), np.int8), (inv[:len(e)], inv[len(e):])), shape=(len(nodes), len(nodes)))
    _, label = connected_components(g, directed=False)
    owner = nodes // nv
    comps = np.unique(np.stack([owner, label], axis=1), axis=0)[:, 0]
    v, n = np.unique(comps, return_counts=True)
    return v[n > 1].astype(np.int64)


# --- narrow phase: IntersectionTest::TriangleTriangle3d over arrays of pairs --------------------------------------------

def _dot(a, b):
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def _cross(a, b):
    return np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1],
                     a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                     a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], axis=-1)


def _pick(a, i):
    return np.take_along_axis(a, i[:, None], axis=1)[:, 0]


def _edge_edge(Ax, Ay, V0, U0, U1, i0, i1):
    Bx, By = _pick(U0, i0) - _pick(U1, i0), _pick(U0, i1) - _pick(U1, i1)
    Cx, Cy = _pick(V0, i0) - _pick(U0, i0), _pick(V0, i1) - _pick(U0, i1)
    f = Ay * Bx - Ax * By
    d = By * Cx - Bx * Cy
    e = Ax * Cy - Ay * Cx
    first = ((f > 0) & (d >= 0) & (d <= f)) | ((f < 0) & (d <= 0) & (d >= f))
    second = np.where(f > 0, (e >= 0) & (e <= f), (e <= 0) & (e >= f))
    return first & second


def _edge_against_tri(V0, V1, U0, U1, U2, i0, i1):
    Ax, Ay = _pick(V1, i0) - _pick(V0, i0), _pick(V1, i1) - _pick(V0, i1)
    return _edge_edge(Ax, Ay, V0, U0, U1, i0, i1) | _edge_edge(Ax, Ay, V0, U1, U2, i0, i1) | _edge_edge(Ax, Ay, V0, U2, U0, i0, i1)


def _side(V, Q, P, i0, i1):
    a = _pick(P, i1) - _pick(Q, i1)
    b = -(_pick(P, i0) - _pick(Q, i0))
    c = (-a) * _pick(Q, i0) - b * _pick(Q, i1)
    return (a * _pick(V, i0) + b * _pick(V, i1)) + c


def _point_in_tri(V0, U0, U1, U2, i0, i1):
    d0, d1, d2 = _side(V0, U0, U1, i0, i1), _side(V0, U1, U2, i0, i1), _side(V0, U2, U0, i0, i1)
    return (d0 * d1 > 0) & (d0 * d2 > 0)


coplanar_axes_hook = None  # called as hook(|N|, i0, i1) by every coplanar test (tests/test_topology_edges_host.py)


def _coplanar(N, V0, V1, V2, U0, U1, U2):
    A = np.abs(N)
    i0 = np.where(A[:, 0] > A[:, 1], np.where(A[:, 0] > A[:, 2], 1, 0), 0)
    i1 = np.where(A[:, 0] > A[:, 1], np.where(A[:, 0] > A[:, 2], 2, 1), np.where(A[:, 2] > A[:, 1], 1, 2))
    if coplanar_axes_hook is not None:
        coplanar_axes_hook(A, i0, i1)
    return (_edge_against_tri(V0, V1, U0, U1, U2, i0, i1) | _edge_against_tri(V1, V2, U0, U1, U2, i0, i1)
            | _edge_against_tri(V2, V0, U0, U1, U2, i0, i1) | _point_in_tri(V0, U0, U1, U2, i0, i1)
            | _point_in_tri(U0, V0, V1, V2, i0, i1))


def _intervals(VV0, VV1, VV2, D0, D1, D2, D0D1, D0D2):
    """NEWCOMPUTE_INTERVALS: (A, B, C, X0, X1, coplanar) per pair."""
    b1 = D0D1 > 0
    b2 = ~b1 & (D0D2 > 0)
    b3 = ~b1 & ~b2 & ((D1 * D2 > 0) | (D0 != 0))
    b4 = ~b1 & ~b2 & ~b3 & (D1 != 0)
    b5 = ~b1 & ~b2 & ~b3 & ~b4 & (D2 != 0)
    cop = ~(b1 | b2 | b3 | b4 | b5)
    # branch 1 and 5 pivot on vertex 2, 2 and 4 on vertex 1, 3 on vertex 0
    on2, on1 = b1 | b5, b2 | b4
    P = np.where(on2, VV2, np.where(on1, VV1, VV0))
    DP = np.where(on2, D2, np.where(on1, D1, D0))
    Q0 = np.where(on2 | on1, VV0, VV1)
    Q1 = np.where(on2, VV1, VV2)
    E0 = np.where(on2 | on1, D0, D1)
    E1 = np.where(on2, D1, D2)
    return P, (Q0 - P) * DP, (Q1 - P) * DP, DP - E0, DP - E1, cop


def _no_div_tri_tri(V0, V1, V2, U0, U1, U2):
    N1 = _cross(V1 - V0, V2 - V0)
    d1 = -_dot(N1, V0)
    du = [_dot(N1, U) + d1 for U in (U0, U1, U2)]
    du = [np.where(np.abs(x) < EPSILON, 0.0, x) for x in du]
    du0du1, du0du2 = du[0] * du[1], du[0] * du[2]
    alive = ~((du0du1 > 0) & (du0du2 > 0))
    N2 = _cross(U1 - U0, U2 - U0)
    d2 = -_dot(N2, U0)
    dv = [_dot(N2, V) + d2 for V in (V0, V1, V2)]
    dv = [np.where(np.abs(x) < EPSILON, 0.0, x) for x in dv]
    dv0dv1, dv0dv2 = dv[0] * dv[1], dv[0] * dv[2]
    alive &= ~((dv0dv1 > 0) & (dv0dv2 > 0))
    D = np.abs(_cross(N1, N2))
    index = np.where(D[:, 1] > D[:, 0], 1, 0)
    index = np.where(D[:, 2] > np.maximum(D[:, 0], D[:, 1]), 2, index)
    vp = [_pick(V, index) for V in (V0, V1, V2)]
    up = [_pick(U, index) for U in (U0, U1, U2)]
    a, b, c, x0, x1, cop1 = _intervals(*vp, *dv, dv0dv1, dv0dv2)
    d, e, f, y0, y1, cop2 = _intervals(*up, *du, du0du1, du0du2)
    xx, yy = x0 * x1, y0 * y1
    xxyy = xx * yy
    tmp = a * xxyy
    s10, s11 = tmp + (b * x1) * yy, tmp + (c * x0) * yy
    tmp = d * xxyy
    s20, s21 = tmp + (e * xx) * y1, tmp + (f * xx) * y0
    s10, s11 = np.minimum(s10, s11), np.maximum(s10, s11)
    s20, s21 = np.minimum(s20, s21), np.maximum(s20, s21)
    general = ~((s11 < s20) | (s21 < s10))
    cop = cop1 | cop2
    out = np.where(cop, False, general)
    if cop.any():
        m = cop & alive
        out[m] = _coplanar(N1[m], V0[m], V1[m], V2[m], U0[m], U1[m], U2[m])
    return alive & out


def normalise(P, Q):
    """TriangleTriangle3d's frame for arrays P, Q (n, 3, 3): the six points (n, 6, 3) less their mean, divided per axis
    by sqrt(sum of squares / 5) + 1e-12."""
    pts = np.concatenate([np.asarray(P, np.float64), np.asarray(Q, np.float64)], axis=1)  # (n, 6, 3)
    s = pts[:, 0]
    for k in range(1, 6):
        s = s + pts[:, k]
    mu = s / 6.0
    ss = (pts[:, 0] - mu) * (pts[:, 0] - mu)
    for k in range(1, 6):
        ss = ss + (pts[:, k] - mu) * (pts[:, k] - mu)
    sigma = np.sqrt(ss / 5.0) + 1e-12
    return (pts - mu[:, None]) / sigma[:, None]


def plane_distances(P, Q):
    """NoDivTriTriIsect's (du, dv) in the normalised frame, before the epsilon clamp: Q's vertices against P's plane and
    P's against Q's, each (n, 3)."""
    q = normalise(P, Q)
    V, U = q[:, :3], q[:, 3:]
    N1, N2 = _cross(V[:, 1] - V[:, 0], V[:, 2] - V[:, 0]), _cross(U[:, 1] - U[:, 0], U[:, 2] - U[:, 0])
    d1, d2 = -_dot(N1, V[:, 0]), -_dot(N2, U[:, 0])
    return (np.stack([_dot(N1, U[:, k]) + d1 for k in range(3)], axis=1),
            np.stack([_dot(N2, V[:, k]) + d2 for k in range(3)], axis=1))


def tri_tri(P, Q):
    """TriangleTriangle3d for arrays P, Q (n, 3, 3): normalise, then NoDivTriTriIsect."""
    q = normalise(P, Q)
    return _no_div_tri_tri(*(q[:, k] for k in range(6)))


def candidate_pairs(v, t, chunk=1 << 22):
    """Sort-and-sweep along x: yields (t0, t1) arrays, t0 < t1, of the pairs whose boxes overlap (touching included) and
    that share no vertex id."""
    v, t = np.asarray(v, np.float64), _tri(t)
    if len(t) < 2:
        return
    p = v[t]
    lo, hi = p.min(axis=1), p.max(axis=1)
    order = np.argsort(lo[:, 0], kind="stable")
    slo = lo[order, 0]
    end = np.searchsorted(slo, hi[order, 0], side="right")  # sorted positions whose lo_x <= this hi_x
    n_after = end - np.arange(len(t)) - 1
    cum = np.concatenate([[0], np.cumsum(n_after)])
    i = 0
    while i < len(t):
        j = int(np.searchsorted(cum, cum[i] + chunk, side="right")) - 1
        j = max(j, i + 1)
        cnt = n_after[i:j]
        a = np.repeat(np.arange(i, j), cnt)
        b = a + 1 + (np.arange(len(a)) - np.repeat(cum[i:j] - cum[i], cnt))
        ta, tb = order[a], order[b]
        t0, t1 = np.minimum(ta, tb), np.maximum(ta, tb)
        ok = ~((hi[t0] < lo[t1]) | (lo[t0] > hi[t1])).any(axis=1)
        ok &= ~(t[t0][:, :, None] == t[t1][:, None, :]).any(axis=(1, 2))
        yield t0[ok], t1[ok]
        i = j


def self_intersecting_triangles(v, t):
    """int64 (k, 2), t0 < t1, ascending by (t0, t1)."""
    v, t = np.asarray(v, np.float64), _tri(t)
    found = []
    for t0, t1 in candidate_pairs(v, t):
        if len(t0):
            hit = tri_tri(v[t[t0]], v[t[t1]])
            found.append(np.stack([t0[hit], t1[hit]], axis=1))
    if not found:
        return np.zeros((0, 2), np.int64)
    pairs = np.concatenate(found)
    return pairs[np.lexsort((pairs[:, 1], pairs[:, 0]))].astype(np.int64)


# --- area and volume ----------------------------------------------------------------------------------------------

def triangle_terms(v, t):
    """(0.5 ||(p0 - p1) x (p0 - p2)||, p0 . (p1 x p2) / 6) per triangle, Eigen's cross and dot."""
    v, t = np.asarray(v, np.float64), _tri(t)
    p0, p1, p2 = v[t[:, 0]], v[t[:, 1]], v[t[:, 2]]
    c = _cross(p0 - p1, p0 - p2)
    return 0.5 * np.sqrt(_dot(c, c)), _dot(p0, _cross(p1, p2)) / 6.0


def _tree(x):
    """x (..., 256) -> (...): x[i] = x[i] + x[i + w] for w = 128, ..., 1."""
    x = x.copy()
    w = SUM_THREADS // 2
    while w:
        x[..., :w] = x[..., :w] + x[..., w:2 * w]
        w //= 2
    return x[..., 0]


def fixed_sum(terms):
    """The GPU's two-stage sum: 256-term blocks (0.0 past the end) by _tree, then thread i of one block adds partials
    i, i + 256, ... from 0.0 in order, then _tree."""
    terms = np.asarray(terms, np.float64)
    if len(terms) == 0:
        return 0.0
    nb = -(-len(terms) // SUM_THREADS)
    x = np.zeros(nb * SUM_THREADS)
    x[:len(terms)] = terms
    partial = _tree(x.reshape(nb, SUM_THREADS))
    rows = -(-nb // SUM_THREADS)
    y = np.zeros(rows * SUM_THREADS)
    y[:nb] = partial
    acc = np.zeros(SUM_THREADS)
    for r in y.reshape(rows, SUM_THREADS):
        acc = acc + r
    return float(_tree(acc))


def surface_area(v, t):
    return fixed_sum(triangle_terms(v, t)[0])


def signed_volume(v, t):
    return fixed_sum(triangle_terms(v, t)[1])
