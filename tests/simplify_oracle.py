"""Host restatement of Open3D 0.17.0 TriangleMesh::SimplifyVertexClustering (restated from memory: the wheel cannot be
installed here), in numpy fp64 with one rounding per operation in the order below.  gsb_mesh_simplify must match it bit
for bit.

1. Errors.  voxel_size s <= 0 or NaN: RuntimeError("voxel_size <= 0.0").  m = lo - s*0.5, M = hi + s*0.5 (lo, hi the
   component-wise min and max of the vertices); s * 2147483647 < max_k(M_k - m_k): RuntimeError("voxel_size is too
   small.").  Non-finite vertices and an infinite s are refused with ValueError (Open3D's cells would be undefined).
2. Cell of a vertex: floor((v - m) / s), one subtraction then one true division, per component.  Keys are packed over
   the cell box (c0 * d1 + c1) * d2 + c2; a box of more than 2^63 cells is a ValueError.
3. Cells are numbered in the order of their smallest vertex id.  Vertices no triangle uses still make their cell.
4. Average: each attribute's sum over the cell's vertices from 0.0 in ascending id, divided by double(count); normals
   are not renormalised.  DOUBT: Open3D sums in unordered_set<int> iteration order.
5. Quadric: per triangle, e0 = p1 - p0, e1 = p2 - p0, c = e0 x e1 (one product minus another per component),
   |c| = sqrt((cx^2 + cy^2) + cz^2); n = c / |c|, d = -((n0 p0x + n1 p0y) + n2 p0z), or the plane (0,0,0,0) if |c| == 0;
   w = 0.5 |c| (Open3D's GetTriangleArea forms (p0 - p1) x (p0 - p2), the same bits: negation is exact); A_ij =
   (w n_i) n_j, b_i = (w d) n_i.  A cell's A and b are the sums, from 0.0, over its vertices in ascending id and, for
   each, its distinct incident triangles in ascending id (a triangle with two corners in the cell counts twice; (a,a,b)
   counts once for a).  If |det A| > 1e-4 (Eigen's cofactor order, `det3`) the position is -A^-1 b by `ldlt_solve`,
   else the average.  DOUBTS: the LDLT's operation order and zero-pivot rule, the 1e-4 threshold, the summation orders.
6. Triangles: mapped through the cell numbering, dropped if two new ids are equal, rotated so the smallest id comes
   first (winding kept), one copy of each rotated triple kept -- opposite windings are different triples.  Order: first
   occurrence in input order.  DOUBT: Open3D's order is its hash set's and cannot be reproduced; the set is the same.
"""
import numpy as np

AVERAGE, QUADRIC = 0, 1
DBL_MIN = float(np.finfo(np.float64).tiny)
DET_THRESHOLD = 1e-4
_SMALL = 256  # cells up to this size are summed "k-th member of every cell" at a time, larger ones by np.cumsum


def cells(vertices, voxel_size):
    """(m, per-vertex cell [n,3] int64, cells per axis [3]) after the error checks of step 1 and 2."""
    s = float(voxel_size)
    if not s > 0.0:
        raise RuntimeError("voxel_size <= 0.0")
    if not np.isfinite(s):
        raise ValueError("voxel_size is not finite")
    v = np.asarray(vertices, dtype=np.float64).reshape(-1, 3)
    if not np.isfinite(v).all():
        raise ValueError("the vertices are not finite")
    lo = v.min(axis=0) if len(v) else np.zeros(3)
    hi = v.max(axis=0) if len(v) else np.zeros(3)
    half = s * 0.5
    m, big = lo - half, hi + half
    if s * 2147483647.0 < np.max(big - m):
        raise RuntimeError("voxel_size is too small.")
    dims = np.floor((hi - m) / s).astype(np.int64) + 1
    if int(dims[0]) * int(dims[1]) * int(dims[2]) > 2**63:
        raise ValueError(f"{dims.tolist()} cells; cell keys are limited to 63 bits")
    return m, np.floor((v - m) / s).astype(np.int64), dims


def vertex_cells(vertices, voxel_size):
    """(cell number of every vertex, number of cells): cells in the order of their smallest vertex id."""
    _, c, dims = cells(vertices, voxel_size)
    if len(c) == 0:
        return np.zeros(0, np.int64), 0
    key = (c[:, 0] * dims[1] + c[:, 1]) * dims[2] + c[:, 2]
    _, first, inverse = np.unique(key, return_index=True, return_inverse=True)
    number = np.empty(len(first), np.int64)
    number[np.argsort(first, kind="stable")] = np.arange(len(first))
    return number[inverse.reshape(-1)], len(first)


def segment_sums(values, seg, n_seg):
    """Sums of values [T,k] per segment (seg [T] ascending, terms in summation order inside a segment), each a
    sequential left-to-right sum starting from 0.0."""
    values = np.asarray(values, dtype=np.float64).reshape(len(seg), -1)
    out = np.zeros((n_seg, values.shape[1]))
    if len(seg) == 0:
        return out
    counts = np.bincount(seg, minlength=n_seg)
    starts = np.concatenate([[0], np.cumsum(counts)[:-1]])
    small = counts <= _SMALL
    for k in range(min(_SMALL, int(counts.max()))):
        sel = np.nonzero(small & (counts > k))[0]
        out[sel] = out[sel] + values[starts[sel] + k]
    for c in np.nonzero(~small)[0]:
        block = np.concatenate([np.zeros((1, values.shape[1])), values[starts[c]:starts[c] + counts[c]]])
        out[c] = np.cumsum(block, axis=0)[-1]  # add.accumulate: sequential, unlike np.sum's pairwise reduction
    return out


def triangle_quadrics(vertices, triangles):
    """[nt,12]: A (row-major, all nine entries) and b of Quadric(plane, area) per triangle."""
    v = np.asarray(vertices, dtype=np.float64).reshape(-1, 3)
    t = np.asarray(triangles, dtype=np.int64).reshape(-1, 3)
    p0, p1, p2 = v[t[:, 0]], v[t[:, 1]], v[t[:, 2]]
    a, b = p1 - p0, p2 - p0
    c = np.stack([a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1], a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2],
                  a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]], 1)
    norm = np.sqrt((c[:, 0] * c[:, 0] + c[:, 1] * c[:, 1]) + c[:, 2] * c[:, 2])
    zero = norm == 0.0
    with np.errstate(invalid="ignore", divide="ignore"):
        n = np.where(zero[:, None], 0.0, c / np.where(zero, 1.0, norm)[:, None])
    d = np.where(zero, 0.0, -((n[:, 0] * p0[:, 0] + n[:, 1] * p0[:, 1]) + n[:, 2] * p0[:, 2]))
    w = 0.5 * norm
    wn = w[:, None] * n
    A = wn[:, :, None] * n[:, None, :]
    bb = (w * d)[:, None] * n
    return np.concatenate([A.reshape(-1, 9), bb], 1)


def det3(a):
    """Eigen's 3x3 determinant over [..., 9] row-major entries."""
    a = np.asarray(a, dtype=np.float64)
    m = lambda i, j: a[..., 3 * i + j]
    h0 = m(0, 0) * (m(1, 1) * m(2, 2) - m(1, 2) * m(2, 1))
    h1 = m(0, 1) * (m(1, 0) * m(2, 2) - m(1, 2) * m(2, 0))
    h2 = m(0, 2) * (m(1, 0) * m(2, 1) - m(1, 1) * m(2, 0))
    return (h0 - h1) + h2


def ldlt_solve(A, b):
    """A^-1 b as Eigen's LDLT<Matrix3d>().solve restated, in Python floats (one IEEE rounding per operation).
    Factorisation (ldlt_inplace<Lower>, left-looking, reads the lower triangle only): at step k pivot on the largest
    |diagonal| among rows k..2 (the first on ties; the trailing diagonal is still A's, not a Schur complement), swap
    it in, t_j = D_j L_kj, D_k = A_kk - sum_j L_kj t_j, column k below the diagonal minus sum_j L_ij t_j, then divided
    by D_k when |D_k| > 0.  Solve: the transpositions in order, the unrolled unit-lower solve (y_i -= (L_i0 y_0 +
    L_i1 y_1)), y_i / D_i where |D_i| > DBL_MIN and 0 elsewhere, the unrolled unit-upper solve with L^T, the
    transpositions in reverse.  Eigen's early exit when the whole diagonal is 0 is not restated: such an A has
    det = 0 and never reaches the solve."""
    m = [[float(A[3 * i + j]) for j in range(3)] for i in range(3)]
    tr = [0, 1, 2]
    for k in range(3):
        p = k
        for i in range(k + 1, 3):
            if abs(m[i][i]) > abs(m[p][p]):
                p = i
        tr[k] = p
        if p != k:
            for j in range(k):
                m[k][j], m[p][j] = m[p][j], m[k][j]
            for i in range(p + 1, 3):
                m[i][k], m[i][p] = m[i][p], m[i][k]
            m[k][k], m[p][p] = m[p][p], m[k][k]
            for i in range(k + 1, p):
                m[i][k], m[p][i] = m[p][i], m[i][k]
        if k == 1:
            t0 = m[0][0] * m[1][0]
            m[1][1] = m[1][1] - m[1][0] * t0
            m[2][1] = m[2][1] - m[2][0] * t0
        elif k == 2:
            t0, t1 = m[0][0] * m[2][0], m[1][1] * m[2][1]
            m[2][2] = m[2][2] - (m[2][0] * t0 + m[2][1] * t1)
        if abs(m[k][k]) > 0.0:
            for i in range(k + 1, 3):
                m[i][k] = m[i][k] / m[k][k]
    y = [float(x) for x in b]
    for k in range(3):
        y[k], y[tr[k]] = y[tr[k]], y[k]
    y[1] = y[1] - m[1][0] * y[0]
    y[2] = y[2] - (m[2][0] * y[0] + m[2][1] * y[1])
    y = [y[i] / m[i][i] if abs(m[i][i]) > DBL_MIN else 0.0 for i in range(3)]
    y[1] = y[1] - m[2][1] * y[2]
    y[0] = y[0] - (m[1][0] * y[1] + m[2][0] * y[2])
    for k in (2, 1, 0):
        y[k], y[tr[k]] = y[tr[k]], y[k]
    return y


def simplify(vertices, triangles, voxel_size, contraction=AVERAGE, colors=None, normals=None):
    """-> (vertices [k,3], triangles int64 [m,3], colours or None, normals or None, cells that took the quadric solve)."""
    v = np.asarray(vertices, dtype=np.float64).reshape(-1, 3)
    t = np.asarray(triangles, dtype=np.int64).reshape(-1, 3)
    vcell, n_cells = vertex_cells(v, voxel_size)
    members = np.argsort(vcell, kind="stable")  # by cell, ascending vertex id inside a cell
    seg = vcell[members]
    count = np.bincount(vcell, minlength=n_cells).astype(np.float64)[:, None]
    avg = lambda a: None if a is None else segment_sums(np.asarray(a, dtype=np.float64).reshape(-1, 3)[members], seg,
                                                        n_cells) / count
    out_v = avg(v) if n_cells else np.zeros((0, 3))
    n_quadric = 0
    if contraction == QUADRIC and n_cells and len(t):
        flat = t.reshape(-1)
        tid = np.arange(len(flat)) // 3
        o = np.argsort(flat, kind="stable")  # by vertex, ascending triangle inside a vertex
        fv, ft = flat[o], tid[o]
        distinct = np.ones(len(fv), bool)
        distinct[1:] = (fv[1:] != fv[:-1]) | (ft[1:] != ft[:-1])
        fv, ft = fv[distinct], ft[distinct]
        order = np.lexsort((ft, fv, vcell[fv]))  # by cell, then vertex, then triangle
        q = segment_sums(triangle_quadrics(v, t)[ft[order]], vcell[fv[order]], n_cells)
        inv = np.nonzero(np.abs(det3(q[:, :9])) > DET_THRESHOLD)[0]
        for c in inv:
            out_v[c] = [-x for x in ldlt_solve(q[c, :9], q[c, 9:])]
        n_quadric = len(inv)
    colors_out = None if colors is None else (avg(colors) if n_cells else np.zeros((0, 3)))
    normals_out = None if normals is None else (avg(normals) if n_cells else np.zeros((0, 3)))
    return out_v, simplify_triangles(vcell, t), colors_out, normals_out, n_quadric


def simplify_triangles(vcell, triangles):
    """Step 6 over the cell number of every vertex."""
    t = np.asarray(triangles, dtype=np.int64).reshape(-1, 3)
    if len(t) == 0:
        return np.zeros((0, 3), np.int64)
    a, b, c = (vcell[t[:, k]] for k in range(3))
    keep = (a != b) & (a != c) & (b != c)
    r1 = (b < a) & (b < c)
    r2 = ~r1 & (c < a) & (c < b)
    tri = np.stack([np.where(r1, b, np.where(r2, c, a)), np.where(r1, c, np.where(r2, a, b)),
                    np.where(r1, a, np.where(r2, b, c))], 1)[keep]
    if len(tri) == 0:
        return np.zeros((0, 3), np.int64)
    _, first = np.unique(tri, axis=0, return_index=True)
    return tri[np.sort(first)].astype(np.int64)
