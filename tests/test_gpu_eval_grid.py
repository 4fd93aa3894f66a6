"""The point-grid kernels of gsb_eval.cu where they branch or round, bit for bit against brute force.

Nearest neighbours (gsb_eval_nearest) and ICP correspondences (gsb_eval_icp_correspond) against
oracle/eval_oracle.py's nearest_exact and oracle/tnt_oracle.py's correspond, both exhaustive in fp64 with the lowest index
among equal minima: degenerate and flat references, queries on cell faces, the ring cut-off, ties across cells and rings,
grid-shape edges and the max_dist / radius cut-offs.  Greedy radius downsampling against the sequential loop, and mesh
sampling at the warp scan's 32-row chunk edges and the strict `< 1` boundary of its row predicate."""
import ctypes as C
import math

import numpy as np
import pytest

from oracle import eval_oracle as eo
from oracle import tnt_oracle as to
from tests.test_gpu_tnt import _correspond

pytestmark = pytest.mark.gpu


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def _dev(x, device):
    import torch

    return torch.as_tensor(np.ascontiguousarray(x, dtype=np.float64).reshape(-1, 3), device=device)


class _Grid:
    """A grid with an explicit origin, cell and dims (the C ABI's layout, not PointGrid's), so that the tests place points
    and queries at known cells and rings."""

    def __init__(self, ref, origin, cell, dims, device):
        import torch

        from gs2mesh_b200 import _lib
        from gs2mesh_b200.evaluate import _stream

        self.points = _dev(ref, device)
        n = self.points.shape[0]
        cells = int(np.prod(dims))
        self.cell_start = torch.empty(cells + 1, dtype=torch.int64, device=device)
        self.ids = torch.empty(n, dtype=torch.int64, device=device)
        self.origin, self.cell, self.dims = np.asarray(origin, np.float64), float(cell), list(dims)
        self.desc = _lib.GsbPointGrid((C.c_double * 3)(*origin), cell, (C.c_int32 * 3)(*dims), _lib.ptr(self.points), n,
                                      _lib.ptr(self.cell_start), _lib.ptr(self.ids))
        L = _lib.lib()
        ws = torch.empty(int(L.gsb_eval_grid_workspace_bytes(n, cells)), dtype=torch.uint8, device=device)
        _lib.check(L.gsb_eval_grid_build(C.byref(self.desc), _lib.ptr(ws), ws.numel(), _stream(device)))


def _nearest(grid, q, max_dist, device):
    import torch

    from gs2mesh_b200 import _lib
    from gs2mesh_b200.evaluate import _stream

    qt = _dev(q, device)
    d = torch.empty(len(q), dtype=torch.float64, device=device)
    i = torch.empty(len(q), dtype=torch.int64, device=device)
    _lib.check(_lib.lib().gsb_eval_nearest(C.byref(grid.desc), _lib.ptr(qt), len(q), float(max_dist), _lib.ptr(d),
                                           _lib.ptr(i), _stream(device)))
    return d.cpu().numpy(), i.cpu().numpy()


def _icp(grid, q, r, device):
    import torch

    from gs2mesh_b200 import _lib
    from gs2mesh_b200.evaluate import _stream

    qt = _dev(q, device)
    i = torch.empty(len(q), dtype=torch.int64, device=device)
    d2 = torch.empty(len(q), dtype=torch.float64, device=device)
    _lib.check(_lib.lib().gsb_eval_icp_correspond(C.byref(grid.desc), _lib.ptr(qt), len(q), float(r), _lib.ptr(i),
                                                  _lib.ptr(d2), _stream(device)))
    return i.cpu().numpy(), d2.cpu().numpy()


def _check(grid, q, ref, device, max_dists=(math.inf,), radii=()):
    """gsb_eval_nearest at every max_dist and gsb_eval_icp_correspond at every radius equal brute force, bit for bit."""
    q = np.asarray(q, np.float64).reshape(-1, 3)
    for md in max_dists:
        d, i = _nearest(grid, q, md, device)
        ed, ei = eo.nearest_exact(q, ref, md)
        bad = np.nonzero((_bits(d) != _bits(ed)) | (i != ei))[0]
        assert len(bad) == 0, (md, q[bad[:5]], d[bad[:5]], i[bad[:5]], ed[bad[:5]], ei[bad[:5]])
    for r in radii:
        i, d2 = _icp(grid, q, r, device)
        ei, ed2 = to.correspond(q, ref, r)
        bad = np.nonzero((_bits(d2) != _bits(ed2)) | (i != ei))[0]
        assert len(bad) == 0, (r, q[bad[:5]], d2[bad[:5]], i[bad[:5]], ed2[bad[:5]], ei[bad[:5]])


def _point_grid(ref, device, **kw):
    from gs2mesh_b200.evaluate import PointGrid

    return PointGrid(_dev(ref, device), **kw)


NON_FINITE = np.array([[np.inf, 2, 3], [-np.inf, 2, 3], [1, np.nan, 3], [1, 2, -np.inf], [np.nan] * 3, [np.inf] * 3,
                       [-np.inf, np.nan, np.inf]])


def _directions():
    d = np.stack(np.meshgrid([-1.0, 0, 1], [-1.0, 0, 1], [-1.0, 0, 1], indexing="ij"), -1).reshape(-1, 3)
    return d[np.abs(d).sum(1) > 0]  # the 6 axes, 12 edge and 8 corner diagonals


# ------------------------------------------------------------------------------------------------ degenerate references
def _degenerate(kind):
    if kind == "one":
        return np.array([[1.0, 2.0, 3.0]])
    if kind == "origin":
        return np.zeros((1, 3))
    if kind == "copies":
        return np.tile([[1.0, 2.0, 3.0]], (1000, 1))
    off = {"ulp500": 500.0, "ulp1e6": 1e6}[kind]
    return np.array([[off, -off, off], [np.nextafter(off, np.inf), -off, off]])


@pytest.mark.parametrize("kind", ["one", "origin", "copies", "ulp500", "ulp1e6"])
def test_degenerate_reference(gsb_lib, cuda_device, kind):
    """A reference whose points coincide, or lie one ulp apart: queries on both sides of every axis and on every diagonal
    at 1e-300 to 1e12, and non-finite queries, which get (+inf, -1) from both kernels."""
    ref = _degenerate(kind)
    dist = 10.0 ** np.array([-300, -150, -20, -9, -3, 0, 3, 6, 9, 12])
    q = (ref[0] + _directions()[:, None, :] * dist[None, :, None]).reshape(-1, 3)
    q = np.concatenate([q, ref, NON_FINITE])
    grid = _point_grid(ref, cuda_device)
    assert grid.dims == [1, 1, 1] or kind.startswith("ulp")
    _check(grid, q, ref, cuda_device, max_dists=(math.inf, 1.0, 1e9), radii=(1.0, 1e9))
    d, i = _nearest(grid, q, math.inf, cuda_device)
    assert np.isinf(d[-len(NON_FINITE):]).all() and (i[-len(NON_FINITE):] == -1).all()
    assert (i[:-len(NON_FINITE)] >= 0).all()
    if kind == "copies":
        assert (i[:-len(NON_FINITE)] == 0).all()
    idx, _ = _correspond(q, ref, 1e9, cuda_device)  # the ICP helper, on a grid of its own
    assert np.array_equal(idx, to.correspond(q, ref, 1e9)[0])


def test_degenerate_reference_through_public_paths(gsb_lib, cuda_device):
    from gs2mesh_b200.evaluate import nearest, precision_recall_f1

    ref = np.array([[1.0, 2.0, 3.0]])
    q = np.array([[2.0, 2, 3], [0.0, 2, 3], [1, 2, 3 + 1e12], [1, 2 - 1e-12, 3], [-1e300, 1e300, 0]])
    d, i = nearest(_dev(q, cuda_device), _dev(ref, cuda_device))
    ed, ei = eo.nearest_exact(q, ref)
    assert np.array_equal(_bits(d.cpu().numpy()), _bits(ed)) and np.array_equal(i.cpu().numpy(), ei)
    got = precision_recall_f1(_dev(q[:4], cuda_device), _dev(ref, cuda_device), 0.5)
    want = eo.precision_recall_f1(q[:4], ref, 0.5)
    assert {k: float(v) for k, v in got.items()} == {k: float(v) for k, v in want.items()}


# ------------------------------------------------------------------------------------------------ flat references
@pytest.mark.parametrize("shape", ["plane", "line"])
def test_flat_reference(gsb_lib, cuda_device, shape):
    """Points on a plane or a line (the quantile box has zero axes): queries many cells off it, and queries on cell faces
    origin + k*cell with their nextafter neighbours on each side."""
    rng = np.random.default_rng(31)
    n = 4000
    ref = np.full((n, 3), 0.3)
    if shape == "plane":
        ref[:, 0], ref[:, 1] = rng.uniform(-2, 2, n), rng.integers(-16, 16, n) * 0.125  # exact ties along y
    else:
        ref[:, 1] = rng.uniform(-5, 5, n)
    ref[:50] = ref[50:100]  # duplicates
    grid = _point_grid(ref, cuda_device)
    o, h, dims = grid.origin, grid.cell, grid.dims
    assert min(dims) == 1
    off = rng.uniform(-2, 2, size=(2000, 3))
    off[:, 2] = rng.choice([-1, 1], 2000) * h * rng.choice([1.5, 7, 100, 1e4], 2000)  # many cells off the plane / line
    k = np.stack([rng.integers(-3, d + 4, 3000) for d in dims], 1)
    face = o + k * h  # on a cell face in every coordinate
    faces = [face, np.nextafter(face, np.inf), np.nextafter(face, -np.inf)]
    mixed = face.copy()
    mixed[:, 1] = np.nextafter(mixed[:, 1], np.inf)
    q = np.concatenate([ref[::7] + off[: len(ref[::7])], *faces, mixed, ref[:200]])
    _check(grid, q, ref, cuda_device, max_dists=(math.inf, 3 * h), radii=(h, 5 * h))


# ------------------------------------------------------------------------------------------------ the ring cut-off
def _ring_case(k, h, o, rng):
    """One group per ring k: the query sits one ulp below, on, or one ulp above the upper face of its cell; the nearest
    point P lies k cells up the x axis, at (k-1)*h from the face, so its distance is (k-1)*h plus, exactly, or minus one
    ulp of the query; a runner-up R in ring k-1 (along y) lies 0.25*h farther.  Stopping one ring early returns R."""
    groups, queries = [], []
    for g in range(3):
        c = 40 * g + 8  # cell index of the query along x, one group every 40 cells
        face = o[0] + (c + 1) * h
        yq, zq = o[1] + 8.5 * h, o[2] + 8.5 * h
        p = np.array([o[0] + (c + k) * h, yq, zq])
        r = np.array([face, yq + (k - 1) * h + 0.25 * h, zq])
        groups.append(np.stack([r, p]))  # R first: the lower index
        for x in (np.nextafter(face, -np.inf), face, np.nextafter(face, np.inf)):
            queries.append([x, yq, zq])
    ref = np.concatenate(groups)
    return ref, np.array(queries)


@pytest.mark.parametrize("k", [2, 3, 6])
def test_ring_cut_off(gsb_lib, cuda_device, k):
    rng = np.random.default_rng(k)
    for h, o in ((1.0, np.zeros(3)), (0.1, np.array([0.3, -7.7, 1e3])), (2.0 ** -20, np.array([1e3, 1e3, -1e3]))):
        ref, q = _ring_case(k, h, o, rng)
        ref = np.concatenate([ref, [o, o + 16 * h]])  # anchors: the grid's box is [o, o + 16h] in y and z
        grid = _Grid(ref, o, h, [3 * 40 + 16, 17, 17], cuda_device)
        _check(grid, q, ref, cuda_device, max_dists=(math.inf, (k - 1) * h + 0.1 * h), radii=((k - 1) * h + 0.2 * h,))
        d, i = _nearest(grid, q, math.inf, cuda_device)
        assert (i == np.repeat(2 * np.arange(3) + 1, 3)).all()  # P, never the runner-up R
        # the same cases through PointGrid's own layout
        _check(_point_grid(ref, cuda_device), q, ref, cuda_device)


# ------------------------------------------------------------------------------------------------ ties
def test_ties(gsb_lib, cuda_device):
    """Equal squared distances (exact binary offsets) to points in different cells and in different rings, where the
    lowest index is in the outer ring, and exact duplicates: the lowest index wins."""
    h = 1.0  # cell; the queries sit at cell centres x.5 or on faces
    # (a) different rings, 3-4-5 offsets at distance 2.5: index 0 in ring 3, index 1 in ring 2
    qa = np.array([20.5, 20.5, 20.5])
    a = [qa + [2.5, 0, 0], qa + [1.5, 2.0, 0]]
    # (b) different cells either side of the face the query sits on: index 2 in ring 1, indices 3 and 4 in ring 0
    qb = np.array([40.0, 20.5, 20.5])
    b = [qb - [0.25, 0, 0], qb + [0.25, 0, 0], qb + [0, 0.25, 0]]
    # (c) the lowest index in the inner ring (ring 2), an equal point in ring 3 and two more in ring 2
    qc = np.array([60.5, 20.5, 20.5])
    c = [qc + [0, 1.5, -2.0], qc + [0, 2.5, 0], qc + [0, 0, -2.5], qc + [2.0, 0, 1.5]]
    # (d) exact duplicates: they share a cell, inside which the order is unspecified
    qd = np.array([80.25, 20.75, 20.5])
    d = [qd + [3.0, 0, 0], qd + [0.5, 0.5, 0.5], qd + [0.5, 0.5, 0.5], qd + [0.5, 0.5, 0.5]]
    ref = np.array(a + b + c + d + [[0.0, 0, 0], [100.0, 41, 41]])
    q = np.array([qa, qb, qc, qd])
    want = [0, 2, 5, 10]
    grid = _Grid(ref, np.zeros(3), h, [101, 42, 42], cuda_device)
    for g in (grid, _point_grid(ref, cuda_device)):
        _check(g, q, ref, cuda_device, max_dists=(math.inf, 2.5, np.nextafter(2.5, 3)), radii=(2.5, np.nextafter(2.5, 3)))
        d_, i_ = _nearest(g, q, math.inf, cuda_device)
        assert i_.tolist() == want and d_.tolist() == [2.5, 0.25, 2.5, math.sqrt(0.75)]

    # many queries over a lattice reference: every query has ties among up to 8 equidistant points
    rng = np.random.default_rng(5)
    lat = np.stack(np.meshgrid(*[np.arange(12) * 0.5] * 3, indexing="ij"), -1).reshape(-1, 3)
    lat = np.concatenate([lat[rng.permutation(len(lat))], lat[:300]])  # shuffled, then duplicates at higher indices
    ql = rng.integers(-4, 30, size=(8000, 3)) * 0.25  # lattice points, edge midpoints, face and cell centres, outside
    for g in (_point_grid(lat, cuda_device), _Grid(lat, np.zeros(3), 0.75, [8, 8, 8], cuda_device)):
        _check(g, ql, lat, cuda_device, max_dists=(math.inf, 0.25, np.nextafter(0.25, 1)), radii=(0.25, 0.5))


# ------------------------------------------------------------------------------------------------ grid-shape edges
@pytest.mark.parametrize("nq", [0, 1, 127, 128, 129, 257])
def test_query_counts(gsb_lib, cuda_device, nq):
    rng = np.random.default_rng(nq)
    ref = rng.uniform(-1, 1, size=(3000, 3))
    q = rng.uniform(-1.5, 1.5, size=(nq, 3))
    grid = _point_grid(ref, cuda_device)
    _check(grid, q, ref, cuda_device, max_dists=(math.inf, 0.05), radii=(0.05,))


@pytest.mark.parametrize("max_cells", [1, 8])
def test_cell_budget_growth(gsb_lib, cuda_device, max_cells):
    """A cell budget of 1 or 8 cells runs the 1.25x growth loop until the grid fits: 1e5 points share one cell (or eight)."""
    rng = np.random.default_rng(max_cells)
    ref = np.concatenate([rng.uniform(0, 1, size=(100_000, 3)), [[0.5, 0.5, 0.5]] * 3])
    grid = _point_grid(ref, cuda_device, max_cells=max_cells)
    assert int(np.prod(grid.dims)) <= max_cells
    q = np.concatenate([rng.uniform(-0.5, 1.5, size=(129, 3)), [[0.5, 0.5, 0.5]], NON_FINITE])
    _check(grid, q, ref, cuda_device, max_dists=(math.inf, 0.01), radii=(0.01,))


def test_axis_at_the_cell_floor(gsb_lib, cuda_device):
    """cells_per_point so large that the spacing cell falls below (hi - lo) * 1e-6: the x axis has about 1e6 cells."""
    rng = np.random.default_rng(12)
    ref = np.zeros((2000, 3))
    ref[:, 0] = np.sort(rng.uniform(0, 7, 2000))
    ref[:, 1] = rng.uniform(0, 1e-5, 2000)
    grid = _point_grid(ref, cuda_device, cells_per_point=1e15)
    assert grid.dims[0] >= 1_000_000 and grid.cell == float(ref[:, 0].max() - ref[:, 0].min()) * 1e-6
    # near the line: a query 1 unit off it would walk some 1e5 rings of 1e6-cell rows
    q = rng.uniform(-0.5, 7.5, size=(3000, 3)) * [1, 1e-5, 1e-5]
    _check(grid, q, ref, cuda_device, max_dists=(math.inf, 1e-3), radii=(1e-3,))


def test_one_cell_of_1e5_points(gsb_lib, cuda_device):
    rng = np.random.default_rng(13)
    ref = np.concatenate([rng.uniform(0.2, 0.3, size=(100_000, 3)), [[0.0, 0, 0], [1.0, 1, 1]]])
    grid = _Grid(ref, np.zeros(3), 0.5, [3, 3, 3], cuda_device)
    q = np.concatenate([rng.uniform(-1, 2, size=(129, 3)), ref[:64]])
    _check(grid, q, ref, cuda_device, max_dists=(math.inf,), radii=(0.05,))


# ------------------------------------------------------------------------------------------------ cut-offs
def test_max_dist_and_radius_edges(gsb_lib, cuda_device):
    """The nearest point exactly at max_dist misses and one ulp inside hits; the ICP radius misses at d2 == r*r and hits
    one ulp above; queries farther than max_dist from the grid's box stop at the first ring that can reach it."""
    rng = np.random.default_rng(14)
    ref = rng.uniform(0, 1, size=(5000, 3))
    grid = _point_grid(ref, cuda_device)
    q = rng.uniform(-0.2, 1.2, size=(64, 3))
    d, i = eo.nearest_exact(q, ref)
    for t in range(8):
        md = d[t]
        for m in (md, np.nextafter(md, np.inf), np.nextafter(md, 0)):
            got_d, got_i = _nearest(grid, q[t:t + 1], m, cuda_device)
            assert (got_i[0] == i[t]) == (d[t] < m) and (got_i[0] == -1) == (d[t] >= m)
        d2 = float(((q[t] - ref[i[t]]) ** 2)[0] + ((q[t] - ref[i[t]]) ** 2)[1] + ((q[t] - ref[i[t]]) ** 2)[2])
        r = math.sqrt(d2)
        for rr in (r, np.nextafter(r, np.inf), np.nextafter(r, 0)):
            got_i, got_d2 = _icp(grid, q[t:t + 1], rr, cuda_device)
            ei, ed2 = to.correspond(q[t:t + 1], ref, rr)
            assert got_i[0] == ei[0] and _bits(got_d2)[0] == _bits(ed2)[0]
    _check(grid, q, ref, cuda_device, max_dists=tuple(d[:8]) + tuple(np.nextafter(d[:8], np.inf)), radii=(0.5,))
    # a lattice 2 apart, queries 0.5 off a lattice point along an axis: the nearest lies at exactly 0.5 (d2 == r*r)
    lat = rng.integers(-10, 10, size=(3000, 3)) * 2.0
    at_r = lat[:500] + rng.choice([-0.5, 0.5], size=(500, 1)) * np.eye(3)[rng.integers(0, 3, 500)]
    lgrid = _point_grid(lat, cuda_device)
    _check(lgrid, at_r, lat, cuda_device, max_dists=(0.5, np.nextafter(0.5, 1)), radii=(0.5, np.nextafter(0.5, 1)))
    assert (_nearest(lgrid, at_r, 0.5, cuda_device)[1] == -1).all()
    assert (_nearest(lgrid, at_r, np.nextafter(0.5, 1), cuda_device)[1] >= 0).all()
    # far outside the box: every ring up to k0 is skipped; max_dist decides between a miss and a full search
    far = np.concatenate([rng.uniform(-1, 1, size=(200, 3)) * 50, [[5.0, 0.5, 0.5], [-3.0, -3, -3]]])
    _check(grid, far, ref, cuda_device, max_dists=(1.0, 4.0, math.inf), radii=(1.0, 4.0))
    dd, ii = _nearest(grid, far, 1.0, cuda_device)
    assert np.isinf(dd).all() and (ii == -1).all()


# ------------------------------------------------------------------------------------------------ radius downsampling
def _downsample(points, radius, device):
    """gsb_eval_radius_downsample in index order, with the rounds it took."""
    import torch

    from gs2mesh_b200 import _lib
    from gs2mesh_b200.evaluate import PointGrid, _stream

    p = _dev(points, device)
    n = p.shape[0]
    keep = torch.zeros(n, dtype=torch.uint8, device=device)
    grid = PointGrid(p, min_cell=float(radius) * 1.001)
    counters = torch.empty(4, dtype=torch.int32, device=device)
    host = torch.empty(1, dtype=torch.int32).pin_memory()
    rounds = C.c_int32(-1)
    _lib.check(_lib.lib().gsb_eval_radius_downsample(C.byref(grid.desc), float(radius), _lib.ptr(keep), _lib.ptr(counters),
                                                     _lib.ptr(host), C.byref(rounds), _stream(device)))
    return keep.cpu().numpy().astype(bool), rounds.value


def _exact_r_pairs(r, rng):
    """Pairs (a, b), one per site of a 5r lattice so that pairs never interact, with b - a along an edge or corner
    diagonal: r = 105/128 and b - a a signed permutation of r/3 (1, 2, 2), r/5 (3, 4, 0) or r/7 (2, 3, 6), all exact in
    binary, with a on a 2^-7 grid, so ((dx*dx)+dy*dy)+dz*dz is exactly r*r.  In the second half b moves one ulp outward
    along its largest component.  Returns the points (a, b interleaved) and the number of pairs in each half."""
    assert r == 105 / 128
    m = 2000
    site = np.stack(np.unravel_index(rng.permutation(40 ** 3)[:m], (40, 40, 40)), 1)
    a = site * (5 * r) + 2.0 + rng.integers(0, 128, size=(m, 3)) / 128  # b >= 1: an ulp moves d2 past r*r
    a = np.round(a * 128) / 128
    base = np.array([[1, 2, 2], [3, 4, 0], [2, 3, 6]]) * np.array([[r / 3], [r / 5], [r / 7]])
    d = base[rng.integers(0, 3, m)]
    d = np.take_along_axis(d, np.argsort(rng.random((m, 3)), 1), 1) * rng.choice([-1.0, 1.0], size=(m, 3))
    b = a + d
    dd = b - a
    assert ((dd[:, 0] * dd[:, 0] + dd[:, 1] * dd[:, 1]) + dd[:, 2] * dd[:, 2] == r * r).all()
    ok = np.arange(m)
    half = m // 2
    u = d
    out = ok[half:]
    ax = np.abs(u[out]).argmax(1)
    b[out, ax] = np.nextafter(b[out, ax], np.sign(u[out, ax]) * np.inf)
    return np.stack([a[ok], b[ok]], 1).reshape(-1, 3), half, len(ok) - half


@pytest.mark.parametrize("case", ["chain", "chain_reversed", "clump", "exact_r", "radius0", "n1", "n2"])
def test_radius_downsample_edges(gsb_lib, cuda_device, case):
    from gs2mesh_b200.evaluate import radius_downsample

    rng = np.random.default_rng(17)
    r = 0.2
    order = None
    if case.startswith("chain"):
        n = 20_000
        pts = np.zeros((n, 3))
        pts[:, 0] = np.arange(n) * (0.6 * r)  # each point within r of its predecessor only
        pts = pts[rng.permutation(n)]
        order = np.argsort(pts[:, 0])[:: -1 if case == "chain_reversed" else 1]
    elif case == "clump":
        pts = rng.uniform(0, r / 2, size=(5000, 3))  # every pair within r: only the first point survives
    elif case == "exact_r":
        r = 105 / 128
        pts, n_at, n_out = _exact_r_pairs(r, rng)
        assert n_at > 100 and n_out > 100
    elif case == "radius0":
        pts = rng.integers(1, 9, size=(3000, 3)) * 0.5
        pts = np.concatenate([pts, np.nextafter(pts[:500], np.inf)])  # exact duplicates, and neighbours one ulp away
        r = 0.0
    else:
        pts = rng.uniform(0, 1, size=(int(case[1:]), 3))
    if order is None:
        order = rng.permutation(len(pts))
    shuffled = pts[order]
    want = eo.radius_downsample(shuffled, r)
    keep, rounds = _downsample(shuffled, r, cuda_device)
    assert np.array_equal(keep, want), int((keep != want).sum())
    got_pts, got_keep = radius_downsample(_dev(pts, cuda_device), r, order=order)
    assert np.array_equal(_bits(got_pts.cpu().numpy()), _bits(shuffled))
    assert np.array_equal(got_keep.cpu().numpy(), want)
    n = len(pts)
    assert 1 <= rounds <= n + 3 or (rounds == 0 and n == 0)
    print(f"radius downsample {case}: n={n} kept={int(want.sum())} rounds={rounds}")
    if case.startswith("chain"):
        assert want.sum() == n // 2
    if case == "clump":
        assert want.sum() == 1
    if case == "exact_r":
        assert want.sum() == n_at + 2 * n_out  # one point of each pair at r, both one ulp beyond
    if case == "radius0":
        assert want.sum() == len(np.unique(pts, axis=0))


# ------------------------------------------------------------------------------------------------ mesh sampling
def _right_triangle(l1, l2, base, rot=None):
    """Legs l1 along x and l2 along y from `base` (v1 _|_ v2, so thr = thresh and n1 = floor(l1 / thresh))."""
    a = np.zeros(3)
    b, c = np.array([l1, 0.0, 0.0]), np.array([0.0, l2, 0.0])
    v = np.stack([a, b, c])
    if rot is not None:
        v = v @ rot.T
    return v + base


def _base(rng):
    return rng.integers(-5, 5, 3).astype(np.float64)  # small integers: the edge vectors stay exact


def _sampling_mesh(rng):
    tris, zero_area = [], []
    # rows n1 + 1 = 1, 31, 32, 33, 64, 65 (legs n + 0.5: floor(l / 1.0) = n), square and wide
    for n1 in (0, 30, 31, 32, 63, 64):
        for n2 in (n1, 40, 3):
            tris.append(_right_triangle(n1 + 0.5, n2 + 0.5, _base(rng)))
    # long rows: n2 >= 1e4 with n1 = 0, 1, 2
    for n1 in (0, 1, 2):
        tris.append(_right_triangle(n1 + 0.5, 10_000.5 + 37 * n1, _base(rng)))
    # right isosceles with n1 == n2 = n: k0 + k1 = (i + j + 1) / n lands on 1 exactly for powers of two, rounds otherwise;
    # legs of exactly n make l / thr integral
    for n in (1, 2, 3, 4, 5, 7, 8, 10, 31, 32, 33, 64, 100):
        tris.append(_right_triangle(float(n), float(n), _base(rng)))
        tris.append(_right_triangle(n + 0.999, n + 0.999, _base(rng)))
    # n1 or n2 zero
    tris += [_right_triangle(0.5, 10.5, np.zeros(3)), _right_triangle(10.5, 0.5, np.zeros(3))]
    # rotated and at a 1e6 offset, where b - a cancels
    th = 0.7
    rot = np.array([[math.cos(th), -math.sin(th), 0], [math.sin(th), math.cos(th), 0], [0, 0, 1]])
    for n in (31, 32, 33, 64):
        tris.append(_right_triangle(n + 0.5, n / 2 + 0.5, np.array([1e6, -1e6, 1e6]), rot))
        tris.append(_right_triangle(float(n), float(n), np.array([1e6, 1e6, -1e6])))
    tris.append(rng.normal(size=(3, 3)) * 20 + 1e6)
    v = np.concatenate(tris)
    t = np.arange(len(v)).reshape(-1, 3)
    # zero-area triangles interleaved: collinear, and with a repeated vertex index
    line = np.array([[0.0, 0, 0], [1.0, 1, 1], [3.0, 3, 3]])
    v = np.concatenate([v, line])
    L = len(v) - 3
    out = []
    for k, tri in enumerate(t):
        out.append(tri)
        if k % 3 == 0:
            out.append([L, L + 1, L + 2] if k % 2 == 0 else [tri[0], tri[0], tri[1]])
    return v, np.array(out)


def test_sampling_edges(gsb_lib, cuda_device):
    import torch

    from gs2mesh_b200 import _lib
    from gs2mesh_b200.evaluate import _stream, sample_mesh_points

    rng = np.random.default_rng(19)
    v, t = _sampling_mesh(rng)
    for thresh in (1.0, 0.5, 0.3):
        got = sample_mesh_points(torch.as_tensor(v, device=cuda_device), torch.as_tensor(t, device=cuda_device),
                                 thresh).cpu().numpy()
        ref = eo.sample_mesh(v, t, thresh)
        assert got.shape == ref.shape and np.array_equal(_bits(got), _bits(ref))
        vt, tt = _dev(v, cuda_device), torch.as_tensor(t, device=cuda_device)
        counts = torch.empty(len(t), dtype=torch.int64, device=cuda_device)
        _lib.check(_lib.lib().gsb_eval_sample_count(_lib.ptr(vt), len(v), _lib.ptr(tt), len(t), thresh, _lib.ptr(counts),
                                                    _stream(cuda_device)))
        want = eo.sample_counts(v, t, thresh)
        assert np.array_equal(counts.cpu().numpy(), want)
        if thresh == 1.0:
            assert (want == 0).sum() > len(t) // 5 and want.max() > 10_000
    # the isosceles counts at thresh 1 are the lattice's: (i + j + 1) / n < 1 exactly when i + j <= n - 2 for n = 2^m
    iso = {n: eo.sample_counts(_right_triangle(float(n), float(n), np.zeros(3)), [[0, 1, 2]], 1.0)[0] for n in (4, 8, 64)}
    assert iso == {n: n * (n - 1) // 2 for n in (4, 8, 64)}


def test_sampling_zero_triangles(gsb_lib, cuda_device):
    import torch

    from gs2mesh_b200.evaluate import sample_mesh_points

    v = np.random.default_rng(20).normal(size=(10, 3))
    got = sample_mesh_points(torch.as_tensor(v, device=cuda_device), torch.zeros((0, 3), dtype=torch.int64,
                                                                                 device=cuda_device)).cpu().numpy()
    assert np.array_equal(_bits(got), _bits(v))
    assert np.array_equal(_bits(eo.sample_mesh(v, np.zeros((0, 3), np.int64), 0.2)), _bits(v))
