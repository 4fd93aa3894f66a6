"""Known answers of the vertex-clustering restatement (tests/simplify_oracle.py) on hand-built meshes, and the C ABI's
workspace sizes and argument checks, which refuse bad input before anything is enqueued (no GPU needed)."""
import ctypes as C

import numpy as np
import pytest

from gs2mesh_b200 import _lib
from tests import simplify_oracle as so

P = 256  # any non-NULL pointer: validation only checks pointers for NULL and dereferences none of them


def _grid_4x4():
    """16 vertices at x, y in {0, 0.25, 1, 1.25}, z = 0, id = 4 i + j; 3 x 3 quads, two triangles each."""
    c = np.array([0.0, 0.25, 1.0, 1.25])
    v = np.array([[c[i], c[j], 0.0] for i in range(4) for j in range(4)])
    g = np.arange(16).reshape(4, 4)
    a, b, cc, d = g[:-1, :-1].ravel(), g[:-1, 1:].ravel(), g[1:, :-1].ravel(), g[1:, 1:].ravel()
    return v, np.concatenate([np.stack([a, b, d], 1), np.stack([a, d, cc], 1)])


def test_two_by_two_cell_grid():
    v, t = _grid_4x4()
    out_v, out_t, col, nrm, nq = so.simplify(v, t, 1.0, colors=v / 2, normals=-v)
    # m = -0.5: 0 and 0.25 fall into cell 0, 1 and 1.25 into cell 1; numbered by first vertex id: (0,0), (0,1), (1,0),
    # (1,1)
    want = np.array([[0.125, 0.125, 0], [0.125, 1.125, 0], [1.125, 0.125, 0], [1.125, 1.125, 0]])
    assert out_v.tolist() == want.tolist()
    assert col.tolist() == (want / 2).tolist() and nrm.tolist() == (-want).tolist() and nq == 0
    # only the middle quad touches four cells; its two triangles (a, b, d), (a, d, c) keep their winding
    assert out_t.tolist() == [[0, 1, 3], [0, 3, 2]] and out_t.dtype == np.int64


def _cyclic(tri):
    return min(tri[k:] + tri[:k] for k in range(3))


def test_numbering_by_first_appearance_under_shuffled_ids():
    rng = np.random.default_rng(0)
    v, t = _grid_4x4()
    for _ in range(5):
        perm = rng.permutation(16)
        pv = np.empty_like(v)
        pv[perm] = v
        out_v, out_t, _, _, _ = so.simplify(pv, perm[t][rng.permutation(len(t))], 1.0)
        cell = np.floor((pv + 0.5) / 1.0).astype(int)
        firsts = sorted({tuple(c): i for i, c in reversed(list(enumerate(cell.tolist())))}.items(), key=lambda kv: kv[1])
        for k, (c, _) in enumerate(firsts):
            members = (cell == c).all(1)
            assert out_v[k].tolist() == (np.cumsum(np.concatenate([[[0, 0, 0]], pv[members]]), 0)[-1] / members.sum()).tolist()
        # the middle quad's two triangles, as cells, with their winding
        as_cells = {_cyclic(tuple(map(tuple, np.floor(out_v[r] + 0.5).astype(int)[:, :2].tolist()))) for r in out_t}
        assert as_cells == {_cyclic(((0, 0), (0, 1), (1, 1))), _cyclic(((0, 0), (1, 1), (1, 0)))}
        assert len(out_t) == 2 and all(r[0] < r[1] and r[0] < r[2] for r in out_t.tolist())


def _three_cells():
    # ids 0..2 in cells x = 0, 1, 2; ids 3..5 again in cells 0, 1, 2
    return np.array([[0, 0, 0], [1, 0, 0], [2, 0, 0], [0.1, 0, 0], [1.1, 0, 0], [2.1, 0, 0]], dtype=np.float64)


def test_rotations_merge_and_opposite_windings_stay():
    v = _three_cells()
    t = np.array([[1, 2, 0], [0, 1, 2], [4, 5, 3], [2, 0, 1], [0, 2, 1], [5, 4, 3], [2, 1, 0]])
    _, out_t, _, _, _ = so.simplify(v, t, 1.0)
    # (1,2,0) rotates to (0,1,2) and is the first occurrence; (0,2,1) is the other winding, (5,4,3) and (2,1,0) repeat it
    assert out_t.tolist() == [[0, 1, 2], [0, 2, 1]]


def test_degenerate_and_collapsing_triangles():
    v = _three_cells()
    t = np.array([[0, 0, 1], [0, 3, 1], [2, 2, 2], [1, 4, 5], [3, 1, 2], [2, 5, 0]])
    _, out_t, _, _, _ = so.simplify(v, t, 1.0)
    assert out_t.tolist() == [[0, 1, 2]]
    assert so.simplify(v, t[:3], 1.0)[1].shape == (0, 3)


def test_boundary_exact_and_negative_coordinates():
    # s = 0.5, lo = -1 -> m = -1.25: (v - m) / s is exact for these, and a vertex on a boundary opens the upper cell
    v = np.array([[-1.0, -1.0, -1.0], [-0.75, -1.0, -1.0], [-0.25, -1.0, -1.0], [-0.2500000000000001, -1.0, -1.0],
                  [0.25, -0.75, -1.0]])
    m, c, dims = so.cells(v, 0.5)
    assert m.tolist() == [-1.25] * 3
    assert c.tolist() == [[0, 0, 0], [1, 0, 0], [2, 0, 0], [1, 0, 0], [3, 1, 0]] and dims.tolist() == [4, 2, 1]
    out_v, _, _, _, _ = so.simplify(v, np.zeros((0, 3), np.int64), 0.5)
    assert out_v.tolist() == [[-1, -1, -1], [(-0.75 + -0.2500000000000001) / 2, -1, -1], [-0.25, -1, -1], [0.25, -0.75, -1]]


def test_unreferenced_vertices_keep_their_cells():
    v = np.concatenate([_three_cells(), [[5.0, 5.0, 5.0]]])
    out_v, out_t, _, _, _ = so.simplify(v, np.array([[0, 1, 2]]), 1.0)
    assert len(out_v) == 4 and out_v[3].tolist() == [5, 5, 5] and out_t.tolist() == [[0, 1, 2]]
    out_v, out_t, col, _, _ = so.simplify(v, np.zeros((0, 3), np.int64), 1.0, colors=np.ones_like(v))
    assert len(out_v) == 4 and out_t.shape == (0, 3) and col.tolist() == [[1, 1, 1]] * 4
    out_v, out_t, col, nrm, nq = so.simplify(np.zeros((0, 3)), np.zeros((0, 3), np.int64), 1.0, colors=np.zeros((0, 3)))
    assert out_v.shape == (0, 3) and out_t.shape == (0, 3) and col.shape == (0, 3) and nrm is None and nq == 0


def test_errors():
    v = _three_cells()
    for s in (0.0, -1.0, float("nan")):
        with pytest.raises(RuntimeError, match=r"^voxel_size <= 0\.0$"):
            so.simplify(v, np.zeros((0, 3), np.int64), s)
    with pytest.raises(RuntimeError, match=r"^voxel_size is too small\.$"):
        so.simplify(np.array([[0.0, 0, 0], [1e7, 0, 0]]), np.zeros((0, 3), np.int64), 1e-3)
    # a voxel just large enough: (2.1 + s/2) - (0 - s/2) <= s * INT_MAX
    so.simplify(v, np.zeros((0, 3), np.int64), 2.2 / 2147483646.0)
    with pytest.raises(ValueError, match="63 bits"):
        so.simplify(np.array([[0.0, 0, 0], [1e7, 1e7, 1e7]]), np.zeros((0, 3), np.int64), 1.0)
    with pytest.raises(ValueError, match="not finite"):
        so.simplify(np.array([[0.0, 0, 0], [np.inf, 0, 0]]), np.zeros((0, 3), np.int64), 1.0)
    with pytest.raises(ValueError, match="not finite"):
        so.simplify(v, np.zeros((0, 3), np.int64), np.inf)


def _rotation(rng):
    q, r = np.linalg.qr(rng.normal(size=(3, 3)))
    return q * np.sign(np.diag(r))


def test_quadric_cube_corner_is_invertible():
    """Three faces of a unit cube meeting at a corner, rotated and moved: the quadric's minimum is the corner."""
    rng = np.random.default_rng(7)
    for _ in range(10):
        R, corner = _rotation(rng), rng.normal(size=3)
        local = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1], [1, 1, 0], [0, 1, 1], [1, 0, 1]], dtype=np.float64)
        v = local @ R.T + corner
        t = np.array([[0, 1, 4], [0, 4, 2], [0, 2, 5], [0, 5, 3], [0, 3, 6], [0, 6, 1]])
        out_v, out_t, _, _, nq = so.simplify(v, t, 10.0, so.QUADRIC)  # one cell holds every vertex
        assert nq == 1 and len(out_v) == 1 and out_t.shape == (0, 3)
        A = sum(so.triangle_quadrics(v, t)[k, :9].reshape(3, 3) for k in range(6))
        assert abs(np.linalg.det(A)) > 1e-4
        np.testing.assert_allclose(out_v[0], corner, rtol=0, atol=1e-12)


def test_quadric_flat_patch_takes_the_average():
    v, t = _grid_4x4()
    v = v + [0, 0, 0.5]
    out_v, _, _, _, nq = so.simplify(v, t, 10.0, so.QUADRIC)
    assert nq == 0 and out_v.tolist() == so.simplify(v, t, 10.0)[0].tolist()


def test_ldlt_solve_matches_numpy():
    """The restated LDLT against np.linalg.solve on plane-quadric sums, random SPD matrices and ones whose pivots
    reorder, to 1e-9 relative."""
    rng = np.random.default_rng(3)
    for k in range(300):
        if k % 3 == 0:
            n = rng.normal(size=(5, 3))
            n /= np.linalg.norm(n, axis=1, keepdims=True)
            A = sum(w * np.outer(x, x) for w, x in zip(rng.random(5) + 0.1, n))
        elif k % 3 == 1:
            B = rng.normal(size=(3, 3))
            A = B @ B.T + 0.01 * np.eye(3)
        else:
            A = np.diag(rng.random(3) * 10.0 ** rng.integers(-3, 4, size=3)) + 1e-3 * rng.normal(size=(3, 3))
            A = (A + A.T) / 2
        b = rng.normal(size=3)
        got = np.array(so.ldlt_solve(A.reshape(-1), b))
        want = np.linalg.solve(A, b)
        np.testing.assert_allclose(got, want, rtol=1e-9, atol=1e-9 * np.abs(want).max())
        assert so.det3(A.reshape(-1)) == ((A[0, 0] * (A[1, 1] * A[2, 2] - A[1, 2] * A[2, 1])
                                           - A[0, 1] * (A[1, 0] * A[2, 2] - A[1, 2] * A[2, 0]))
                                          + A[0, 2] * (A[1, 0] * A[2, 1] - A[1, 1] * A[2, 0]))


def test_quadric_counts_shared_triangles_per_vertex():
    """A triangle with two corners in the cell is added twice, a degenerate (a, a, b) once for a."""
    v = np.array([[0, 0, 0], [0.1, 0, 0], [3, 0, 0], [0, 0.2, 0.3]], dtype=np.float64)
    t = np.array([[0, 1, 2], [0, 0, 3], [3, 2, 1]])
    Q = so.triangle_quadrics(v, t)
    out_v, _, _, _, _ = so.simplify(v, t, 1.0, so.QUADRIC)
    # cell 0 holds 0, 1, 3: vertex 0 -> triangles 0, 1; vertex 1 -> 0, 2; vertex 3 -> 1, 2
    want = np.zeros(12)
    for k in (0, 1, 0, 2, 1, 2):
        want = want + Q[k]
    avg = so.simplify(v, t, 1.0)[0]
    expect = [-x for x in so.ldlt_solve(want[:9], want[9:])] if abs(so.det3(want[:9])) > 1e-4 else avg[0].tolist()
    assert out_v[0].tolist() == list(expect)


def test_segment_sums_are_sequential():
    rng = np.random.default_rng(1)
    vals = rng.normal(size=(3000, 2)) * np.exp(rng.normal(size=(3000, 2)) * 8)
    seg = np.sort(np.concatenate([np.zeros(1000, np.int64), rng.integers(1, 400, size=2000)]))  # one cell > 256
    got = so.segment_sums(vals, seg, 400)
    want = np.zeros((400, 2))
    for x, s in zip(vals, seg):
        want[s] = want[s] + x
    assert got.tobytes() == want.tobytes()


def test_workspace_bytes(gsb_lib):
    f = gsb_lib.gsb_mesh_simplify_workspace_bytes
    assert f(-1, 0) == 0 and f(0, -1) == 0 and f(2**31, 0) == 0 and f(10, 2**31) == 0 and f(0, 10) == 0
    small, big = f(1000, 2000), f(1_000_000, 2_000_000)
    # per vertex: 2 keys + 2 ids + 8 int arrays + incidence count/offset; per triangle: 2 x 3 incidence pairs, the
    # rotated triple, 2 lo keys, 2 ids, 2 hi keys, keep and position
    assert 0 < small < big and big >= 1_000_000 * (16 + 8 + 32 + 16) + 2_000_000 * (48 + 12 + 8 + 8 + 16 + 8)


def test_argument_validation_without_gpu(gsb_lib):
    launches = gsb_lib.gsb_kernel_launch_count()
    ws = gsb_lib.gsb_mesh_simplify_workspace_bytes(100, 50)
    d3 = C.c_double * 3

    def call(nv=100, nt=50, xyz=P, col=None, nrm=None, tri=P, lo=(0, 0, 0), hi=(1, 1, 1), s=0.1, mode=0, work=P, wsb=ws,
             ov=P, oc=None, on=None, ot=P, sizes=P):
        rc = gsb_lib.gsb_mesh_simplify(xyz, col, nrm, nv, tri, nt, None if lo is None else d3(*lo),
                                       None if hi is None else d3(*hi), s, mode, work, wsb, ov, oc, on, ot, sizes, None)
        return rc, gsb_lib.gsb_last_error().decode()

    bad = [dict(xyz=None), dict(tri=None), dict(work=None), dict(ov=None), dict(ot=None), dict(sizes=None),
           dict(col=P), dict(nrm=P), dict(lo=None), dict(hi=None), dict(nv=-1), dict(nt=-1), dict(nv=2**31),
           dict(nt=2**31), dict(nv=0), dict(mode=2), dict(mode=-1), dict(s=0.0), dict(s=-1.0), dict(s=float("nan")),
           dict(s=float("inf")), dict(lo=(0, float("nan"), 0)), dict(hi=(0, 0, float("inf"))),
           dict(lo=(0, 0, 0), hi=(1e7, 0, 0), s=1e-3), dict(lo=(0, 0, 0), hi=(1e7, 1e7, 1e7), s=1.0)]
    for kw in bad:
        rc, msg = call(**kw)
        assert rc == _lib.GSB_ERR_INVALID and msg.startswith("mesh_simplify: "), (kw, msg)
    assert call(s=0.0)[1] == "mesh_simplify: voxel_size <= 0.0"
    assert call(s=float("nan"))[1] == "mesh_simplify: voxel_size <= 0.0"
    assert call(hi=(1e7, 0, 0), s=1e-3)[1] == "mesh_simplify: voxel_size is too small."
    assert "63 bits" in call(hi=(1e7, 1e7, 1e7), s=1.0)[1]
    assert "32-bit" in call(nt=2**31)[1] and "no vertices" in call(nv=0)[1] and "negative" in call(nt=-1)[1]
    assert call(wsb=ws - 1)[0] == _lib.GSB_ERR_WORKSPACE
    # the span limit is inclusive: s * INT_MAX == span passes validation (and fails only on the workspace here)
    assert call(hi=(2147483646.0, 0, 0), s=1.0, wsb=0)[0] == _lib.GSB_ERR_WORKSPACE
    assert gsb_lib.gsb_kernel_launch_count() == launches  # nothing was enqueued
