"""The smoothing and sharpening restatement (tests/filter_oracle.py) against a literal per-vertex loop of its formulas,
its adjacency against a set-of-pairs construction, known answers, and the C ABI's workspace sizes and argument checks,
which refuse bad input before anything is enqueued (no GPU needed)."""
import ctypes as C
import math

import numpy as np
import pytest

from gs2mesh_b200 import _lib
from tests import filter_oracle as fo

P = 256  # any non-NULL pointer: validation only checks pointers for NULL and dereferences none of them
KINDS = [fo.SIMPLE, fo.LAPLACIAN, fo.TAUBIN, fo.SHARPEN]
SCOPES = [fo.ALL, fo.COLOR, fo.NORMAL, fo.VERTEX]


def _neighbour_sets(triangles, nv):
    sets = [set() for _ in range(nv)]
    for tri in np.asarray(triangles).reshape(-1, 3).tolist():
        for i in range(3):
            for j in range(3):
                if i != j:
                    sets[tri[i]].add(tri[j])
    return [sorted(s) for s in sets]


def _literal(kind, v, t, iterations, p0, p1, scope, colors, normals):
    """The formulas of tests/filter_oracle.py, one Python float operation at a time, vertex by vertex."""
    N = _neighbour_sets(t, len(v))
    cur = [np.asarray(v, dtype=np.float64).tolist()] + [None if a is None else np.asarray(a, np.float64).tolist()
                                                        for a in (colors, normals)]
    filtered = [a for a, on in enumerate([scope in (fo.ALL, fo.VERTEX), colors is not None and scope in (fo.ALL, fo.COLOR),
                                          normals is not None and scope in (fo.ALL, fo.NORMAL)]) if on]

    def one_pass(op, param, cur):
        new = [None if a is None else [row[:] for row in a] for a in cur]
        p = cur[0]
        for i in range(len(v)):
            ws = []
            for u in N[i]:
                d = [p[i][c] - p[u][c] for c in range(3)]
                ws.append(1.0 / (math.sqrt((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]) + 1e-12))
            W = 0.0
            for w in ws:
                W = W + w
            for a in filtered:
                x = cur[a]
                for c in range(3):
                    s = 0.0
                    if op == fo.SIMPLE:
                        for u in N[i]:
                            s = s + x[u][c]
                        new[a][i][c] = (x[i][c] + s) / float(1 + len(N[i]))
                    elif op == fo.SHARPEN:
                        for u in N[i]:
                            s = s + (x[i][c] - x[u][c])
                        new[a][i][c] = x[i][c] + param * s
                    elif N[i]:
                        for w, u in zip(ws, N[i]):
                            s = s + w * x[u][c]
                        new[a][i][c] = x[i][c] + param * (s / W - x[i][c])
        return new

    passes = [(fo.LAPLACIAN, p0), (fo.LAPLACIAN, p1)] if kind == fo.TAUBIN else [(kind, p0)]
    for _ in range(iterations):
        for op, param in passes:
            cur = one_pass(op, param, cur)
    return [None if a is None else np.array(a, dtype=np.float64).reshape(-1, 3) for a in cur]


def _small_adversarial(seed, nv=24):
    """Random vertices, with a repeated position, a degenerate (a,a,b), (a,b,b) and (a,a,a), repeated, reversed and
    rotated triangles, and two vertices no triangle uses."""
    rng = np.random.default_rng(seed)
    v = rng.normal(size=(nv, 3))
    v[3] = v[4]
    t = rng.integers(0, nv - 2, size=(30, 3))
    t = np.concatenate([t, [[0, 0, 1], [2, 5, 5], [6, 6, 6]], t[:4, ::-1], t[4:8, [1, 2, 0]], t[:3]])
    return v, t[rng.permutation(len(t))], rng.random(v.shape), rng.normal(size=v.shape)


def _params(kind):
    return {fo.SIMPLE: (0.0, 0.0), fo.LAPLACIAN: (0.37, 0.0), fo.TAUBIN: (0.5, -0.53), fo.SHARPEN: (0.3, 0.0)}[kind]


def _same(a, b):
    if a is None or b is None:
        assert a is None and b is None
        return
    assert a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("seed", range(3))
def test_restatement_equals_the_literal_loop(kind, seed):
    v, t, col, nrm = _small_adversarial(seed)
    p0, p1 = _params(kind)
    for scope in SCOPES:
        for iterations in range(4):
            for c, n in ((col, nrm), (None, nrm), (col, None), (None, None)):
                got = fo.filter_mesh(kind, v, t, iterations, p0, p1, scope, c, n)
                want = _literal(kind, v, t, iterations, p0, p1, scope, c, n)
                for g, w in zip(got, want):
                    _same(g, w)


def test_adjacency_equals_set_of_pairs():
    rng = np.random.default_rng(4)
    for nv in (1, 5, 40):
        t = rng.integers(0, max(nv - 1, 1), size=(3 * nv, 3))
        t = np.concatenate([t, t[:, ::-1], t[:, [1, 2, 0]], t[:2]])
        offsets, nb = fo.adjacency(t, nv)
        sets = _neighbour_sets(t, nv)
        assert offsets.tolist() == np.concatenate([[0], np.cumsum([len(s) for s in sets])]).tolist()
        assert nb.tolist() == [u for s in sets for u in s] and nb.dtype == np.int64
    # (a,a,b) makes a its own neighbour (and b's), (c,c,c) makes c its own; reversed and repeated triangles add nothing;
    # vertex 4 is unreferenced
    offsets, nb = fo.adjacency([[0, 0, 1], [2, 2, 2], [1, 0, 0], [0, 0, 1], [3, 1, 2], [2, 1, 3]], 5)
    runs = [nb[offsets[i]:offsets[i + 1]].tolist() for i in range(5)]
    assert runs == [[0, 1], [0, 2, 3], [1, 2, 3], [1, 2], []]
    offsets, nb = fo.adjacency(np.zeros((0, 3), np.int64), 3)
    assert offsets.tolist() == [0, 0, 0, 0] and nb.shape == (0,)


def test_identities():
    v, t, col, nrm = _small_adversarial(5)
    for kind in KINDS:
        got = fo.filter_mesh(kind, v, t, 0, 0.5, -0.53, fo.ALL, col, nrm)
        for g, w in zip(got, (v, col, nrm)):
            _same(g, w)
    for iterations in (1, 3):
        got = fo.filter_mesh(fo.SHARPEN, v, t, iterations, 0.0, 0.0, fo.ALL, col, nrm)
        for g, w in zip(got, (v, col, nrm)):
            _same(g, w)
    # attributes outside the scope are returned unchanged
    for scope, keep in ((fo.COLOR, (0, 2)), (fo.NORMAL, (0, 1)), (fo.VERTEX, (1, 2))):
        got = fo.filter_mesh(fo.TAUBIN, v, t, 2, 0.5, -0.53, scope, col, nrm)
        for a in keep:
            _same(got[a], (v, col, nrm)[a])


def _planar_grid(n, rng=None):
    """(n x n) vertices at integer (i - n//2, j - n//2, 0), two triangles per quad, ids in row order."""
    g = np.arange(n * n).reshape(n, n)
    a, b, c, d = g[:-1, :-1].ravel(), g[:-1, 1:].ravel(), g[1:, :-1].ravel(), g[1:, 1:].ravel()
    t = np.concatenate([np.stack([a, b, d], 1), np.stack([a, d, c], 1)])
    xy = np.stack(np.meshgrid(np.arange(n) - n // 2, np.arange(n) - n // 2, indexing="ij"), -1).reshape(-1, 2)
    v = np.concatenate([xy, np.zeros((n * n, 1))], 1).astype(np.float64)
    if rng is not None:
        v[:, :2] += rng.uniform(-0.3, 0.3, size=(n * n, 2))
    return v, t


def test_interior_vertex_of_a_regular_grid_is_a_fixed_point():
    v, t = _planar_grid(7)
    interior = np.array([i * 7 + j for i in range(1, 6) for j in range(1, 6)])
    got = fo.filter_mesh(fo.SIMPLE, v, t, 1)[0]
    _same(got[interior], v[interior])  # integer sums of a centrally symmetric neighbourhood divide exactly
    assert (got != v).any()
    centre = 3 * 7 + 3  # three rings from the boundary: still fixed after two passes
    assert fo.filter_mesh(fo.SIMPLE, v, t, 2)[0][centre].tolist() == v[centre].tolist()
    # the Laplacian's weights 1 / (1 + 1e-12) and 1 / (sqrt(2) + 1e-12) are rounded, so its fixed point is to rounding
    got = fo.filter_mesh(fo.LAPLACIAN, v, t, 1, 0.5)[0]
    np.testing.assert_allclose(got[interior], v[interior], rtol=0, atol=1e-14)
    assert np.abs(got - v).max() > 0.1  # the boundary moves


def test_a_plane_stays_planar_under_taubin():
    v, t = _planar_grid(12, np.random.default_rng(6))
    for iterations in (1, 5, 20):
        got = fo.filter_mesh(fo.TAUBIN, v, t, iterations, 0.5, -0.53)[0]
        assert (got[:, 2] == 0.0).all() and np.abs(got[:, :2] - v[:, :2]).max() > 1e-3


def test_vertices_without_neighbours_keep_their_values():
    rng = np.random.default_rng(8)
    v = rng.normal(size=(6, 3))
    col, nrm = rng.random((6, 3)), rng.normal(size=(6, 3))
    t = np.array([[0, 1, 2], [2, 1, 3]])  # 4 and 5 unreferenced
    for kind in KINDS:
        for iterations in (1, 2, 3):
            got = fo.filter_mesh(kind, v, t, iterations, 0.5, -0.53, fo.ALL, col, nrm)
            for g, w in zip(got, (v, col, nrm)):
                _same(g[4:], w[4:])
                assert np.isfinite(g).all()
    # no triangles at all
    for kind in KINDS:
        got = fo.filter_mesh(kind, v, np.zeros((0, 3), np.int64), 2, 0.5, -0.53, fo.ALL, col, None)
        _same(got[0], v)
        _same(got[1], col)


def test_workspace_bytes(gsb_lib):
    f = gsb_lib.gsb_mesh_filter_workspace_bytes
    assert f(-1, 0, 0) == 0 and f(2**31, 1, 1) == 0 and f(-5, 1, 0) == 0
    sizes = [f(n, c, m) for n in (1, 1000, 1_000_000) for c, m in ((0, 0), (1, 0), (1, 1))]
    assert all(a <= b for a, b in zip(sizes, sizes[1:])) and sizes[0] > 0
    assert f(1000, 0, 1) == f(1000, 1, 0)
    # one ping-pong copy per attribute: 24 B per vertex each
    assert f(1_000_000, 1, 1) >= 3 * 24 * 1_000_000 and f(1_000_000, 0, 0) >= 24 * 1_000_000
    assert f(2**31 - 1, 0, 0) >= 24 * (2**31 - 1)


def test_argument_validation_without_gpu(gsb_lib):
    launches = gsb_lib.gsb_kernel_launch_count()
    ws = gsb_lib.gsb_mesh_filter_workspace_bytes(100, 1, 1)

    def call(kind=_lib.GSB_FILTER_TAUBIN, xyz=P, col=P, nrm=P, nv=100, off=P, nb=P, it=2, scope=0, work=P, wsb=ws, ov=P, oc=P,
             on=P):
        rc = gsb_lib.gsb_mesh_filter(kind, xyz, col, nrm, nv, off, nb, it, 0.5, -0.53, scope, work, wsb, ov, oc, on, None)
        return rc, gsb_lib.gsb_last_error().decode()

    bad = [dict(kind=-1), dict(kind=4), dict(scope=-1), dict(scope=4), dict(it=-1), dict(it=-(2**31)), dict(nv=-1),
           dict(nv=2**31), dict(nv=2**40), dict(xyz=None), dict(ov=None), dict(off=None), dict(work=None),
           dict(oc=None), dict(on=None), dict(col=None), dict(nrm=None), dict(col=None, nrm=None),
           dict(nv=0, col=None, oc=P), dict(nv=0, nrm=None, on=P)]
    for kw in bad:
        rc, msg = call(**kw)
        assert rc == _lib.GSB_ERR_INVALID and msg.startswith("mesh_filter: "), (kw, msg)
    assert "unknown kind" in call(kind=4)[1] and "unknown scope" in call(scope=4)[1] and "< 0" in call(it=-1)[1]
    assert "32-bit" in call(nv=2**31)[1] and "32-bit" in call(nv=-1)[1] and "without its input" in call(col=None)[1]
    rc, msg = call(wsb=ws - 1)
    assert rc == _lib.GSB_ERR_WORKSPACE and msg.startswith("mesh_filter: ")
    # the workspace follows the attributes given: positions only need less
    ws1 = gsb_lib.gsb_mesh_filter_workspace_bytes(100, 0, 0)
    assert ws1 < ws and call(col=None, oc=None, nrm=None, on=None, wsb=ws1 - 1)[0] == _lib.GSB_ERR_WORKSPACE
    # an empty mesh needs no pointers and enqueues nothing
    assert call(nv=0, xyz=None, col=None, nrm=None, off=None, nb=None, work=None, wsb=0, ov=None, oc=None, on=None)[0] == _lib.GSB_OK
    assert gsb_lib.gsb_kernel_launch_count() == launches  # nothing was enqueued
