"""The topology restatement (tests/topology_oracle.py) against literal transcriptions of Open3D's loops: the all-pairs
self-intersection loop with a scalar NoDivTriTriIsect, the per-vertex BFS of GetNonManifoldVertices and the BFS of
OrientTriangleHelper; known answers on hand-built meshes; and the C ABI's workspace sizes and argument checks, which
refuse bad input before anything is enqueued (no GPU needed)."""
import math
from collections import deque

import numpy as np
import pytest

from gs2mesh_b200 import _lib
from tests import topology_oracle as to

P = 256  # any non-NULL pointer: validation only checks pointers for NULL and dereferences none of them


# --- literal transcriptions -------------------------------------------------------------------------------------------

def _sub(a, b):
    return [a[0] - b[0], a[1] - b[1], a[2] - b[2]]


def _cross(a, b):
    return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]


def _dot(a, b):
    return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]


def _coplanar_tri_tri(N, V0, V1, V2, U0, U1, U2):
    A = [abs(N[0]), abs(N[1]), abs(N[2])]
    if A[0] > A[1]:
        i0, i1 = (1, 2) if A[0] > A[2] else (0, 1)
    else:
        i0, i1 = (0, 1) if A[2] > A[1] else (0, 2)

    def edge_edge(Ax, Ay, V0, U0, U1):
        Bx, By = U0[i0] - U1[i0], U0[i1] - U1[i1]
        Cx, Cy = V0[i0] - U0[i0], V0[i1] - U0[i1]
        f = Ay * Bx - Ax * By
        d = By * Cx - Bx * Cy
        if (f > 0 and d >= 0 and d <= f) or (f < 0 and d <= 0 and d >= f):
            e = Ax * Cy - Ay * Cx
            if f > 0:
                if e >= 0 and e <= f:
                    return True
            else:
                if e <= 0 and e >= f:
                    return True
        return False

    def edge_against_tri_edges(V0, V1):
        Ax, Ay = V1[i0] - V0[i0], V1[i1] - V0[i1]
        return edge_edge(Ax, Ay, V0, U0, U1) or edge_edge(Ax, Ay, V0, U1, U2) or edge_edge(Ax, Ay, V0, U2, U0)

    def point_in_tri(V0, U0, U1, U2):
        a = U1[i1] - U0[i1]
        b = -(U1[i0] - U0[i0])
        c = -a * U0[i0] - b * U0[i1]
        d0 = a * V0[i0] + b * V0[i1] + c
        a = U2[i1] - U1[i1]
        b = -(U2[i0] - U1[i0])
        c = -a * U1[i0] - b * U1[i1]
        d1 = a * V0[i0] + b * V0[i1] + c
        a = U0[i1] - U2[i1]
        b = -(U0[i0] - U2[i0])
        c = -a * U2[i0] - b * U2[i1]
        d2 = a * V0[i0] + b * V0[i1] + c
        return d0 * d1 > 0.0 and d0 * d2 > 0.0

    if edge_against_tri_edges(V0, V1) or edge_against_tri_edges(V1, V2) or edge_against_tri_edges(V2, V0):
        return True
    return point_in_tri(V0, U0, U1, U2) or point_in_tri(U0, V0, V1, V2)


class _Coplanar(Exception):
    pass


def _intervals(VV0, VV1, VV2, D0, D1, D2, D0D1, D0D2):
    if D0D1 > 0.0:
        return VV2, (VV0 - VV2) * D2, (VV1 - VV2) * D2, D2 - D0, D2 - D1
    if D0D2 > 0.0:
        return VV1, (VV0 - VV1) * D1, (VV2 - VV1) * D1, D1 - D0, D1 - D2
    if D1 * D2 > 0.0 or D0 != 0.0:
        return VV0, (VV1 - VV0) * D0, (VV2 - VV0) * D0, D0 - D1, D0 - D2
    if D1 != 0.0:
        return VV1, (VV0 - VV1) * D1, (VV2 - VV1) * D1, D1 - D0, D1 - D2
    if D2 != 0.0:
        return VV2, (VV0 - VV2) * D2, (VV1 - VV2) * D2, D2 - D0, D2 - D1
    raise _Coplanar


def _no_div_tri_tri_isect(V0, V1, V2, U0, U1, U2):
    E1, E2 = _sub(V1, V0), _sub(V2, V0)
    N1 = _cross(E1, E2)
    d1 = -_dot(N1, V0)
    du0, du1, du2 = _dot(N1, U0) + d1, _dot(N1, U1) + d1, _dot(N1, U2) + d1
    du0 = 0.0 if abs(du0) < 1e-6 else du0
    du1 = 0.0 if abs(du1) < 1e-6 else du1
    du2 = 0.0 if abs(du2) < 1e-6 else du2
    du0du1, du0du2 = du0 * du1, du0 * du2
    if du0du1 > 0.0 and du0du2 > 0.0:
        return False
    E1, E2 = _sub(U1, U0), _sub(U2, U0)
    N2 = _cross(E1, E2)
    d2 = -_dot(N2, U0)
    dv0, dv1, dv2 = _dot(N2, V0) + d2, _dot(N2, V1) + d2, _dot(N2, V2) + d2
    dv0 = 0.0 if abs(dv0) < 1e-6 else dv0
    dv1 = 0.0 if abs(dv1) < 1e-6 else dv1
    dv2 = 0.0 if abs(dv2) < 1e-6 else dv2
    dv0dv1, dv0dv2 = dv0 * dv1, dv0 * dv2
    if dv0dv1 > 0.0 and dv0dv2 > 0.0:
        return False
    D = _cross(N1, N2)
    mx, index = abs(D[0]), 0
    bb, cc = abs(D[1]), abs(D[2])
    if bb > mx:
        mx, index = bb, 1
    if cc > mx:
        mx, index = cc, 2
    try:
        a, b, c, x0, x1 = _intervals(V0[index], V1[index], V2[index], dv0, dv1, dv2, dv0dv1, dv0dv2)
        d, e, f, y0, y1 = _intervals(U0[index], U1[index], U2[index], du0, du1, du2, du0du1, du0du2)
    except _Coplanar:
        return _coplanar_tri_tri(N1, V0, V1, V2, U0, U1, U2)
    xx, yy = x0 * x1, y0 * y1
    xxyy = xx * yy
    tmp = a * xxyy
    isect1 = [tmp + b * x1 * yy, tmp + c * x0 * yy]
    tmp = d * xxyy
    isect2 = [tmp + e * xx * y1, tmp + f * xx * y0]
    isect1.sort()
    isect2.sort()
    return not (isect1[1] < isect2[0] or isect2[1] < isect1[0])


def _triangle_triangle_3d(p0, p1, p2, q0, q1, q2):
    pts = [p0, p1, p2, q0, q1, q2]
    mu = [(((((p0[a] + p1[a]) + p2[a]) + q0[a]) + q1[a]) + q2[a]) / 6 for a in range(3)]
    sigma = []
    for a in range(3):
        s = 0.0
        for k, p in enumerate(pts):
            s = (p[a] - mu[a]) * (p[a] - mu[a]) if k == 0 else s + (p[a] - mu[a]) * (p[a] - mu[a])
        sigma.append(math.sqrt(s / 5) + 1e-12)
    n = [[(p[a] - mu[a]) / sigma[a] for a in range(3)] for p in pts]
    return _no_div_tri_tri_isect(*n)


def _literal_self_intersections(v, t):
    """GetSelfIntersectingTriangles: every pair tidx0 < tidx1 without a shared index, AABBAABB then TriangleTriangle3d."""
    v, t = np.asarray(v).tolist(), np.asarray(t).tolist()
    out = []
    for i in range(len(t) - 1):
        P = [v[k] for k in t[i]]
        lo1 = [min(P[0][a], min(P[1][a], P[2][a])) for a in range(3)]
        hi1 = [max(P[0][a], max(P[1][a], P[2][a])) for a in range(3)]
        for j in range(i + 1, len(t)):
            if set(t[i]) & set(t[j]):
                continue
            Q = [v[k] for k in t[j]]
            lo2 = [min(Q[0][a], min(Q[1][a], Q[2][a])) for a in range(3)]
            hi2 = [max(Q[0][a], max(Q[1][a], Q[2][a])) for a in range(3)]
            if any(hi1[a] < lo2[a] or lo1[a] > hi2[a] for a in range(3)):
                continue
            if _triangle_triangle_3d(*P, *Q):
                out.append((i, j))
    return np.array(out, dtype=np.int64).reshape(-1, 2)


def _literal_non_manifold_vertices(t, nv):
    """GetNonManifoldVertices: per vertex, the link edges of its triangle set, then a BFS from one link vertex."""
    t = np.asarray(t).tolist()
    vert_to_tris = [set() for _ in range(nv)]
    for i, tri in enumerate(t):
        for x in tri:
            vert_to_tris[x].add(i)
    out = []
    for v in range(nv):
        if not vert_to_tris[v]:
            continue
        edges = {}
        for i in vert_to_tris[v]:
            a, b, c = t[i]
            if a != v and b != v:
                edges.setdefault(a, set()).add(b), edges.setdefault(b, set()).add(a)
            elif a != v and c != v:
                edges.setdefault(a, set()).add(c), edges.setdefault(c, set()).add(a)
            elif b != v and c != v:
                edges.setdefault(b, set()).add(c), edges.setdefault(c, set()).add(b)
        if not edges:  # Open3D dereferences edges.begin() here; we report nothing
            continue
        start = next(iter(edges))
        visited, queue = {start}, deque([start])
        while queue:
            x = queue.popleft()
            for y in edges[x]:
                if y not in visited:
                    visited.add(y)
                    queue.append(y)
        if len(visited) != len(edges):
            out.append(v)
    return np.array(out, dtype=np.int64)


def _literal_is_orientable(t):
    """OrientTriangleHelper: BFS over edge-adjacent triangles, flipping a triangle that runs an edge the way an earlier
    one did, and failing when an edge is then seen twice in one direction.  One deliberate difference: a degenerate edge
    (a, a) has no direction and is never a conflict (`or a == b`), as in the restatement (DESIGN.md section 7, "Topology
    queries", point 3); Open3D's VerifyAndAdd, as remembered, fails on a second (a, a)."""
    t = [list(x) for x in np.asarray(t).tolist()]
    ordered = lambda a, b: (min(a, b), max(a, b))
    orientation, adjacent = {}, {}
    for i, (a, b, c) in enumerate(t):
        for e in ((a, b), (b, c), (c, a)):
            adjacent.setdefault(ordered(*e), []).append(i)
    unvisited = set(range(len(t)))
    queue = deque()

    def verify_and_add(a, b):
        key = ordered(a, b)
        if key in orientation:
            return orientation[key] == (b, a) or a == b
        orientation[key] = (a, b)
        return True

    while unvisited:
        i = queue.popleft() if queue else min(unvisited)
        if i not in unvisited:
            continue
        unvisited.discard(i)
        a, b, c = t[i]
        if any(orientation.get(ordered(x, y)) == (x, y) and x != y for x, y in ((a, b), (b, c), (c, a))):
            a, c = c, a
        for x, y in ((a, b), (b, c), (c, a)):
            if not verify_and_add(x, y):
                return False
        for x, y in ((a, b), (b, c), (c, a)):
            queue.extend(adjacent[ordered(x, y)])
    return True


def _literal_non_manifold_edges(t, allow):
    counts = {}
    for a, b, c in np.asarray(t).tolist():
        for x, y in ((a, b), (b, c), (c, a)):
            k = (min(x, y), max(x, y))
            counts[k] = counts.get(k, 0) + 1
    bad = sorted(k for k, n in counts.items() if (n > 2 if allow else n != 2))
    return np.array(bad, dtype=np.int64).reshape(-1, 2), len(counts)


# --- meshes ---------------------------------------------------------------------------------------------------------

def tetrahedron():
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]], np.float64)
    t = np.array([[0, 2, 1], [0, 1, 3], [0, 3, 2], [1, 2, 3]])
    return v, t


def cube(s=0.5):
    v = np.array([[x, y, z] for x in (0, s) for y in (0, s) for z in (0, s)], np.float64)  # id = 4x + 2y + z
    q = [(0, 1, 3, 2), (4, 6, 7, 5), (0, 4, 5, 1), (2, 3, 7, 6), (0, 2, 6, 4), (1, 5, 7, 3)]  # outward quads
    t = np.array([f for a, b, c, d in q for f in ((a, b, c), (a, c, d))])
    return v, t


def uv_sphere(n_lat=12, n_lon=16, r=1.0):
    v = [[0, 0, r]]
    for i in range(1, n_lat):
        th = math.pi * i / n_lat
        for j in range(n_lon):
            ph = 2 * math.pi * j / n_lon
            v.append([r * math.sin(th) * math.cos(ph), r * math.sin(th) * math.sin(ph), r * math.cos(th)])
    v.append([0, 0, -r])
    ring = lambda i, j: 1 + (i - 1) * n_lon + j % n_lon
    t = [[0, ring(1, j), ring(1, j + 1)] for j in range(n_lon)]
    for i in range(1, n_lat - 1):
        for j in range(n_lon):
            a, b, c, d = ring(i, j), ring(i, j + 1), ring(i + 1, j), ring(i + 1, j + 1)
            t += [[a, c, d], [a, d, b]]
    south = len(v) - 1
    t += [[south, ring(n_lat - 1, j + 1), ring(n_lat - 1, j)] for j in range(n_lon)]
    return np.array(v, np.float64), np.array(t, np.int64)


def torus(n=16, m=10, R=2.0, r=0.6):
    v = np.array([[(R + r * math.cos(2 * math.pi * j / m)) * math.cos(2 * math.pi * i / n),
                   (R + r * math.cos(2 * math.pi * j / m)) * math.sin(2 * math.pi * i / n),
                   r * math.sin(2 * math.pi * j / m)] for i in range(n) for j in range(m)])
    idx = lambda i, j: (i % n) * m + j % m
    t = [f for i in range(n) for j in range(m)
         for f in ((idx(i, j), idx(i + 1, j), idx(i + 1, j + 1)), (idx(i, j), idx(i + 1, j + 1), idx(i, j + 1)))]
    return v, np.array(t, np.int64)


def moebius(n=24, w=0.3):
    v = []
    for i in range(n):
        u = 2 * math.pi * i / n
        for s in (-w, w):
            v.append([(1 + s * math.cos(u / 2)) * math.cos(u), (1 + s * math.cos(u / 2)) * math.sin(u), s * math.sin(u / 2)])
    t = []
    for i in range(n):
        a, b = 2 * i, 2 * i + 1
        c, d = (2 * (i + 1), 2 * (i + 1) + 1) if i + 1 < n else (1, 0)  # the half twist swaps the sides
        t += [[a, c, d], [a, d, b]]
    return np.array(v, np.float64), np.array(t, np.int64)


def _random_soup(seed, nv=60, nt=120, scale=1.0):
    rng = np.random.default_rng(seed)
    v = rng.normal(size=(nv, 3)) * scale
    v[5] = v[6]  # one shared position under two ids
    t = rng.integers(0, nv, size=(nt, 3))
    t[:4, 1] = t[:4, 0]  # degenerate (a, a, b)
    return v, t


# --- the restatement equals the literal loops -------------------------------------------------------------------------

@pytest.mark.parametrize("seed", range(4))
def test_self_intersections_equal_the_all_pairs_loop(seed):
    v, t = _random_soup(seed, nt=150 + 100 * seed)
    want = _literal_self_intersections(v, t)
    got = to.self_intersecting_triangles(v, t)
    assert got.dtype == np.int64 and got.tolist() == want.tolist() and len(want) > 10


def test_self_intersections_equal_the_loop_on_closed_and_coplanar_meshes():
    rng = np.random.default_rng(7)
    cases = [uv_sphere(), torus(), cube(), tetrahedron()]
    # a noisy sphere folds through itself; a plane of grid triangles shifted in-plane overlaps coplanar triangles
    v, t = uv_sphere(20, 30)
    cases.append((v + rng.normal(scale=0.08, size=v.shape), t))
    g = np.array([[x, y, 0.0] for x in range(8) for y in range(8)])
    gt = np.array([[8 * x + y, 8 * x + y + 8, 8 * x + y + 9] for x in range(7) for y in range(7)])
    cases.append((np.concatenate([g, g + [0.3, 0.2, 0.0]]), np.concatenate([gt, gt + 64])))
    for v, t in cases:
        assert to.self_intersecting_triangles(v, t).tolist() == _literal_self_intersections(v, t).tolist()
    assert len(to.self_intersecting_triangles(*cases[4])) > 0 and len(to.self_intersecting_triangles(*cases[5])) > 50


def test_self_intersections_on_2000_triangles():
    v, t = uv_sphere(32, 32)
    v = v + np.random.default_rng(8).normal(scale=0.05, size=v.shape)
    assert len(t) > 1900
    want = _literal_self_intersections(v, t)
    assert to.self_intersecting_triangles(v, t).tolist() == want.tolist() and len(want) > 0


@pytest.mark.parametrize("seed", range(6))
def test_vertices_edges_and_orientation_equal_the_loops(seed):
    rng = np.random.default_rng(100 + seed)
    meshes = [_random_soup(seed, nv=40, nt=60), uv_sphere(), torus(), moebius(), cube()]
    # a sphere with a few triangles removed, one flipped, and a fan glued on at one vertex
    v, t = uv_sphere(10, 14)
    t = t[rng.permutation(len(t))][:-3]
    t[0] = t[0, ::-1]
    meshes.append((v, t))
    for v, t in meshes:
        nv = len(v)
        assert to.non_manifold_vertices(t, nv).tolist() == _literal_non_manifold_vertices(t, nv).tolist()
        for allow in (True, False):
            got, e = to.edges(t, nv, allow)
            want, we = _literal_non_manifold_edges(t, allow)
            assert got.tolist() == want.tolist() and e == we
        if len(to.edges(t, nv, True)[0]) == 0:  # on edge-manifold meshes the answer does not depend on BFS order
            assert to.is_orientable(t, nv) == _literal_is_orientable(t)


def test_orientation_on_random_manifold_patches():
    """Edge-manifold meshes with randomly flipped triangles: orientable ones stay so, the Moebius strip never is."""
    rng = np.random.default_rng(9)
    for v, t in (uv_sphere(), torus(), moebius(), moebius(25)):
        for _ in range(5):
            f = t.copy()
            flip = rng.random(len(t)) < 0.3
            f[flip] = f[flip][:, ::-1]
            f = f[rng.permutation(len(f))]
            assert to.is_orientable(f, len(v)) == _literal_is_orientable(f)


# --- known answers -------------------------------------------------------------------------------------------------

def test_tetrahedron_and_cube():
    v, t = tetrahedron()
    area, vol = to.surface_area(v, t), to.signed_volume(v, t)
    assert abs(vol) == 1 / 6 or abs(abs(vol) - 1 / 6) < 1e-16
    assert abs(area - (1.5 + math.sqrt(3) / 2)) < 1e-15
    assert to.is_orientable(t, 4) and to.euler_poincare(t, 4) == 2
    v, t = cube(0.5)
    assert abs(to.signed_volume(v, t)) == 0.125 and to.surface_area(v, t) == 1.5  # dyadic: exact
    assert to.edges(t, 8, False)[0].shape == (0, 2) and to.non_manifold_vertices(t, 8).shape == (0,)
    assert to.self_intersecting_triangles(v, t).shape == (0, 2) and to.euler_poincare(t, 8) == 2


def test_sphere_and_torus_are_watertight():
    for (v, t), chi in ((uv_sphere(), 2), (torus(), 0)):
        nv = len(v)
        assert to.euler_poincare(t, nv) == chi
        assert len(to.edges(t, nv, False)[0]) == 0 and len(to.non_manifold_vertices(t, nv)) == 0
        assert len(to.self_intersecting_triangles(v, t)) == 0 and to.is_orientable(t, nv)
    v, t = uv_sphere(40, 60)
    assert abs(abs(to.signed_volume(v, t)) - 4 / 3 * math.pi) < 0.02


def test_moebius_strip_is_not_orientable():
    v, t = moebius()
    assert not to.is_orientable(t, len(v)) and not _literal_is_orientable(t)
    assert len(to.edges(t, len(v), True)[0]) == 0 and len(to.edges(t, len(v), False)[0]) > 0  # a boundary, no fin


def test_two_tetrahedra_sharing_a_vertex():
    v, t = tetrahedron()
    w = v.copy() * -1  # mirrored through vertex 0 = the origin
    t2 = t.copy() + 3
    t2[t2 == 3] = 0  # the second tetrahedron's corner 0 is the first one's vertex 0
    vv = np.concatenate([v, w[1:]])
    tt = np.concatenate([t, t2])
    assert to.non_manifold_vertices(tt, 7).tolist() == [0]
    assert len(to.edges(tt, 7, False)[0]) == 0 and to.euler_poincare(tt, 7) == 3


def test_fin_and_boundary_edges():
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1]], np.float64)
    fin = np.array([[0, 1, 2], [1, 0, 3], [0, 1, 4]])
    assert to.edges(fin, 5, True)[0].tolist() == [[0, 1]]
    bad, e = to.edges(fin, 5, False)
    assert bad.tolist() == [[0, 1], [0, 2], [0, 3], [0, 4], [1, 2], [1, 3], [1, 4]] and e == 7
    one = np.array([[0, 1, 2]])
    assert to.edges(one, 5, True)[0].shape == (0, 2) and to.edges(one, 5, False)[0].tolist() == [[0, 1], [0, 2], [1, 2]]
    # (a, a, b) puts two incidences on (a, b), and (a, a) counts as an edge
    assert to.edges([[0, 0, 1]], 2, False)[0].tolist() == [[0, 0]] and to.edges([[0, 0, 1]], 2, True)[1] == 2


def test_crossing_coplanar_and_touching_triangles():
    v = np.array([[0, 0, 0], [2, 0, 0], [0, 2, 0],          # 0: in z = 0
                  [0.5, 0.5, -1], [0.5, 0.5, 1], [1.5, 1.5, 0.3],  # 1: pierces 0
                  [0.2, 0.2, 0], [1.0, 0.2, 0], [0.2, 1.0, 0],   # 2: coplanar inside 0
                  [5, 5, 5], [6, 5, 5], [5, 6, 5]], np.float64)  # 3: far away
    t = np.array([[0, 1, 2], [3, 4, 5], [6, 7, 8], [9, 10, 11]])
    got = to.self_intersecting_triangles(v, t)
    assert got.tolist() == [[0, 1], [0, 2], [1, 2]] == _literal_self_intersections(v, t).tolist()
    # touching at one position: distinct ids are tested and reported, a shared id is skipped
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 0], [-1, 0, 0.5], [0, -1, 0.5]], np.float64)
    assert to.self_intersecting_triangles(v, [[0, 1, 2], [3, 4, 5]]).tolist() == [[0, 1]]
    assert to.self_intersecting_triangles(v, [[0, 1, 2], [0, 4, 5]]).shape == (0, 2)


def test_empty_and_degenerate_inputs():
    e = np.zeros((0, 3), np.int64)
    assert to.self_intersecting_triangles(np.zeros((0, 3)), e).shape == (0, 2)
    assert to.edges(e, 3, False)[0].shape == (0, 2) and to.is_orientable(e, 3) and to.euler_poincare(e, 3) == 3
    assert to.non_manifold_vertices(e, 3).shape == (0,) and to.surface_area(np.zeros((3, 3)), e) == 0.0
    # a vertex whose every triangle repeats it has an empty link graph and is not reported
    assert to.non_manifold_vertices([[0, 0, 0], [1, 1, 2]], 3).tolist() == _literal_non_manifold_vertices([[0, 0, 0], [1, 1, 2]], 3).tolist()


def test_fixed_sum_shape():
    rng = np.random.default_rng(10)
    for n in (1, 255, 256, 257, 70_000):
        x = rng.random(n)
        assert abs(to.fixed_sum(x) - math.fsum(x)) <= 1e-12 * n
    # the shape: a pairwise tree inside each 256-term block
    x = rng.random(256)
    t = x.copy()
    w = 128
    while w:
        t[:w] = t[:w] + t[w:2 * w]
        w //= 2
    assert to.fixed_sum(x) == 0.0 + t[0]


# --- the C ABI ------------------------------------------------------------------------------------------------------

def test_workspace_bytes(gsb_lib):
    for f in (gsb_lib.gsb_mesh_edge_topology_workspace_bytes, gsb_lib.gsb_mesh_vertex_topology_workspace_bytes,
              gsb_lib.gsb_mesh_area_volume_workspace_bytes):
        assert f(-1, 10) == 0 and f(10, -1) == 0 and f(357913942, 10) == 0 and f(10, 2**31) == 0 and f(5, 0) == 0
        assert f(357913941, 2**31 - 1) > 0 and 0 < f(1, 3) <= f(1000, 3000) <= f(10**6, 3 * 10**6)
    g = gsb_lib.gsb_mesh_self_intersections_workspace_bytes
    assert g(100, 50, -1) == 0 and g(100, 50, 4951) == 0 and g(357913942, 10, 0) == 0
    assert 0 < g(100, 50, 0) < g(100, 50, 4950)
    assert gsb_lib.gsb_mesh_edge_topology_workspace_bytes(10**6, 10) >= 3 * 10**6 * 24  # keys and values, double-buffered


def test_argument_validation_without_gpu(gsb_lib):
    import ctypes as C

    launches = gsb_lib.gsb_kernel_launch_count()
    lo, hi = (C.c_double * 3)(0, 0, 0), (C.c_double * 3)(1, 1, 1)
    bad_lo = (C.c_double * 3)(0, float("nan"), 0)
    inf_hi = (C.c_double * 3)(1, 1, float("inf"))
    we = gsb_lib.gsb_mesh_edge_topology_workspace_bytes(100, 50)
    wv = gsb_lib.gsb_mesh_vertex_topology_workspace_bytes(100, 50)
    wi = gsb_lib.gsb_mesh_self_intersections_workspace_bytes(100, 50, 7)
    wa = gsb_lib.gsb_mesh_area_volume_workspace_bytes(100, 50)

    def edges(tri=P, nt=100, nv=50, work=P, wsb=we, out=P, sizes=P):
        return gsb_lib.gsb_mesh_edge_topology(tri, nt, nv, 1, work, wsb, out, sizes, None), "mesh_edge_topology: "

    def verts(tri=P, nt=100, nv=50, work=P, wsb=wv, out=P, count=P):
        return gsb_lib.gsb_mesh_non_manifold_vertices(tri, nt, nv, work, wsb, out, count, None), "mesh_non_manifold_vertices: "

    def isect(xyz=P, nv=50, tri=P, nt=100, lo=lo, hi=hi, work=P, wsb=wi, out=P, cap=7, stats=P):
        return (gsb_lib.gsb_mesh_self_intersections(xyz, nv, tri, nt, lo, hi, work, wsb, out, cap, stats, None),
                "mesh_self_intersections: ")

    def area(xyz=P, nv=50, tri=P, nt=100, work=P, wsb=wa, out=P):
        return gsb_lib.gsb_mesh_area_volume(xyz, nv, tri, nt, work, wsb, out, None), "mesh_area_volume: "

    sizes = [dict(nt=-1), dict(nv=-1), dict(nt=357913942), dict(nv=2**31), dict(nv=0)]
    for fn in (edges, verts, isect, area):
        for kw in sizes + [dict(tri=None), dict(work=None)]:
            (rc, prefix) = fn(**kw)
            msg = gsb_lib.gsb_last_error().decode()
            assert rc == _lib.GSB_ERR_INVALID and msg.startswith(prefix), (fn.__name__, kw, msg)
        assert "32-bit" in (fn(nt=357913942), gsb_lib.gsb_last_error().decode())[1]
        rc, prefix = fn(wsb={edges: we, verts: wv, isect: wi, area: wa}[fn] - 1)
        assert rc == _lib.GSB_ERR_WORKSPACE and gsb_lib.gsb_last_error().decode().startswith(prefix)
    for kw in (dict(sizes=None),):
        assert edges(**kw)[0] == _lib.GSB_ERR_INVALID
    assert verts(count=None)[0] == _lib.GSB_ERR_INVALID
    for kw in (dict(xyz=None), dict(out=None), dict(stats=None), dict(lo=None), dict(hi=None), dict(cap=-1),
               dict(cap=4951), dict(lo=bad_lo), dict(hi=inf_hi), dict(lo=hi, hi=lo)):
        assert isect(**kw)[0] == _lib.GSB_ERR_INVALID, kw
    assert "not finite" in (isect(lo=bad_lo), gsb_lib.gsb_last_error().decode())[1]
    for kw in (dict(xyz=None), dict(out=None)):
        assert area(**kw)[0] == _lib.GSB_ERR_INVALID
    # edges and vertices may skip the list; the counting self-intersection pass needs no output
    assert edges(out=None, wsb=we - 1)[0] == _lib.GSB_ERR_WORKSPACE
    assert verts(out=None, wsb=wv - 1)[0] == _lib.GSB_ERR_WORKSPACE
    wi0 = gsb_lib.gsb_mesh_self_intersections_workspace_bytes(100, 50, 0)
    assert wi0 < wi and isect(out=None, cap=0, wsb=wi0 - 1)[0] == _lib.GSB_ERR_WORKSPACE
    assert gsb_lib.gsb_kernel_launch_count() == launches  # nothing was enqueued
