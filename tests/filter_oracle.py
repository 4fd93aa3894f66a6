"""Host restatement of Open3D 0.17.0 TriangleMesh::FilterSmoothSimple, FilterSmoothLaplacian, FilterSmoothTaubin and
FilterSharpen (restated from memory: the wheel cannot be installed here), in numpy fp64 with one rounding per operation
in the order below and no FMA.  gsb_mesh_filter must match it bit for bit.

1. Neighbours.  N(v) is the set of distinct ids u such that v and u sit at two different corner positions of some
   triangle (Open3D's ComputeAdjacencyList, which inserts all six ordered pairs of every triangle): a degenerate (a,a,b)
   makes a its own neighbour, repeated and reversed triangles add nothing new, a vertex no triangle uses has none.
   Neighbours are visited in ascending id.  DOUBT: Open3D visits them in unordered_set<int> order, which changes only the
   order of the fp64 additions, so results agree with Open3D to rounding, not bit for bit.
2. Scope (FilterScope All=0, Color=1, Normal=2, Vertex=3): positions for All and Vertex, normals for All and Normal,
   colours for All and Color, the last two only where the mesh has them.  Normals are not renormalised, colours not
   clamped.  An attribute that is not filtered is returned unchanged, and 0 iterations return a copy.  DOUBT: Open3D's
   FilterSmoothSimple may leave attributes it does not filter zero-filled.
3. Passes are Jacobi style: each reads only the previous pass's values.  Sums start from 0.0 and add in ascending
   neighbour id.  With x the attribute, p the pass's input positions and deg = |N(v)|:
   simple     x' = (x + sum_u x_u) / double(1 + deg).  DOUBT: Open3D may start its sum at x itself, ((x + x_u1) + x_u2)...
   laplacian  d = p_v - p_u, w_u = 1.0 / (sqrt((dx*dx + dy*dy) + dz*dz) + 1e-12), W = sum w_u, s = sum (w_u * x_u);
              x' = x + lambda * (s / W - x).  The weights come from the positions even when only colours or normals
              are filtered.  A self-neighbour has distance 0 and weight 1e12, as in Open3D.  A vertex with deg = 0 keeps
              x (ours: Open3D's expression gives 0/0 = NaN there).
   taubin     per iteration one Laplacian pass with lambda, then one with mu, whose weights come from the first pass's
              output positions.
   sharpen    x' = x + strength * sum_u (x - x_u).
   Simple and sharpen leave a vertex with deg = 0 at x by their formulas (up to the sign of a zero).
Non-finite inputs are not checked: they propagate as IEEE arithmetic says.
"""
import numpy as np

from tests.simplify_oracle import segment_sums

SIMPLE, LAPLACIAN, TAUBIN, SHARPEN = 0, 1, 2, 3
ALL, COLOR, NORMAL, VERTEX = 0, 1, 2, 3
WEIGHT_EPS = 1e-12

_PAIRS = ((0, 1), (0, 2), (1, 0), (1, 2), (2, 0), (2, 1))


def adjacency(triangles, n_vertices):
    """(offsets int64 [n_vertices + 1], neighbours int64): N(v) as CSR, ascending within each vertex's run."""
    t = np.asarray(triangles, dtype=np.int64).reshape(-1, 3)
    nv = int(n_vertices)
    keys = np.unique(np.concatenate([t[:, i] * nv + t[:, j] for i, j in _PAIRS])) if len(t) else np.zeros(0, np.int64)
    owner = keys // nv if nv else keys
    offsets = np.zeros(nv + 1, np.int64)
    offsets[1:] = np.cumsum(np.bincount(owner, minlength=nv))
    return offsets, keys - owner * nv


def _pass(op, param, attrs, p, owner, nb, deg):
    """One pass of op over the filtered attributes `attrs` (list of [nv,3] arrays); p are the weights' positions."""
    out = []
    sums = lambda terms: segment_sums(terms, owner, len(deg)) if len(owner) else np.zeros((len(deg), terms.shape[1]))
    if op == LAPLACIAN:
        d = p[owner] - p[nb]
        w = 1.0 / (np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]) + WEIGHT_EPS)
        W = sums(w[:, None])[:, 0]
        lone = deg == 0
    for x in attrs:
        if op == SIMPLE:
            out.append((x + sums(x[nb])) / (1 + deg).astype(np.float64)[:, None])
        elif op == SHARPEN:
            out.append(x + param * sums(x[owner] - x[nb]))
        else:
            s = sums(w[:, None] * x[nb])
            with np.errstate(invalid="ignore", divide="ignore"):
                y = x + param * (s / W[:, None] - x)
            out.append(np.where(lone[:, None], x, y))
    return out


def filter_mesh(kind, vertices, triangles, iterations=1, param0=0.0, param1=0.0, scope=ALL, colors=None, normals=None):
    """-> (vertices, colours or None, normals or None) after `iterations` iterations of filter `kind`.  param0 is
    lambda (Laplacian, Taubin) or strength (sharpen), param1 mu (Taubin)."""
    if iterations < 0:
        raise ValueError("iterations must be >= 0")
    v = np.asarray(vertices, dtype=np.float64).reshape(-1, 3).copy()
    arrays = [v] + [None if a is None else np.asarray(a, dtype=np.float64).reshape(-1, 3).copy() for a in (colors, normals)]
    filtered = [scope in (ALL, VERTEX), colors is not None and scope in (ALL, COLOR),
                normals is not None and scope in (ALL, NORMAL)]
    offsets, nb = adjacency(triangles, len(v))
    deg = np.diff(offsets)
    owner = np.repeat(np.arange(len(v)), deg)
    passes = [(LAPLACIAN, param0), (LAPLACIAN, param1)] if kind == TAUBIN else [(kind, param0)]
    for _ in range(iterations):
        for op, param in passes:
            idx = [a for a in range(3) if filtered[a]]
            new = _pass(op, param, [arrays[a] for a in idx], arrays[0], owner, nb, deg)
            for a, y in zip(idx, new):
                arrays[a] = y
    return arrays[0], arrays[1], arrays[2]
