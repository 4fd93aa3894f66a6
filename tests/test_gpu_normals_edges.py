"""ring_knn and FastEigen3x3 at their edges on the GPU (tests/normals_edge_cases.py builds the inputs, and
tests/test_normals_edges_host.py shows on the CPU that each is where it says): gsb_eval_knn against brute force,
gsb_eval_estimate_normals and gsb_pcd_statistical_outliers against the numpy oracles, bit for bit, with NaN equal to
NaN by position."""
import ctypes as C

import numpy as np
import pytest

from tests import normals_edge_cases as ec
from tests import normals_oracle as no
from tests import pcd_oracle as po
from tests.test_gpu_eval_grid import _Grid, _dev, _point_grid
from tests.test_normals_edges_host import RING_CASES_PRESENT, _same

pytestmark = pytest.mark.gpu


def _knn(grid, q, k, device):
    import torch

    from gs2mesh_b200 import _lib
    from gs2mesh_b200.evaluate import _stream

    qt = _dev(q, device)
    d2 = torch.empty((len(q), k), dtype=torch.float64, device=device)
    idx = torch.empty((len(q), k), dtype=torch.int64, device=device)
    _lib.check(_lib.lib().gsb_eval_knn(C.byref(grid.desc), _lib.ptr(qt), len(q), k, _lib.ptr(d2), _lib.ptr(idx),
                                       _stream(device)))
    return d2.cpu().numpy(), idx.cpu().numpy()


def _normals(grid, pts, k, device):
    import torch

    from gs2mesh_b200 import _lib
    from gs2mesh_b200.evaluate import _stream

    pt = _dev(pts, device)
    out = torch.empty((len(pts), 3), dtype=torch.float64, device=device)
    _lib.check(_lib.lib().gsb_eval_estimate_normals(C.byref(grid.desc), _lib.ptr(pt), len(pts), k, _lib.ptr(out),
                                                    _stream(device)))
    return out.cpu().numpy()


def _statistical(grid, k, ratio, device):
    import torch

    from gs2mesh_b200 import _lib
    from gs2mesh_b200.evaluate import _stream

    n = grid.points.shape[0]
    L = _lib.lib()
    ws = torch.empty(int(L.gsb_pcd_statistical_workspace_bytes(n)), dtype=torch.uint8, device=device)
    m = torch.empty(n, dtype=torch.float64, device=device)
    keep = torch.empty(n, dtype=torch.uint8, device=device)
    stats = torch.empty(3, dtype=torch.float64, device=device)
    _lib.check(L.gsb_pcd_statistical_outliers(C.byref(grid.desc), k, float(ratio), _lib.ptr(ws), ws.numel(), _lib.ptr(m),
                                              _lib.ptr(keep), _lib.ptr(stats), _stream(device)))
    return m.cpu().numpy(), keep.cpu().numpy().astype(bool), stats.cpu().numpy()


def _check_knn(grid, q, ref, k, device):
    d2, idx = _knn(grid, q, k, device)
    ed2, eidx = no.knn_brute(q, ref, k)
    bad = np.nonzero((d2.view(np.uint64) != ed2.view(np.uint64)).any(1) | (idx != eidx).any(1))[0]
    assert len(bad) == 0, (q[bad[:3]], idx[bad[:3]], eidx[bad[:3]])
    return idx


def _grids(ref, o, h, dims, device):
    return [_Grid(ref, o, h, dims, device), _point_grid(ref, device)]


# ------------------------------------------------------------------------------------------------ k nearest neighbours
@pytest.mark.parametrize("k", ec.KNN_KS)
def test_ring_bound_ties(gsb_lib, cuda_device, k):
    """The k-th distance below, at or above the bound of the stop test before ring K, tied with a lower-index point in
    ring K: the search walks ring K and keeps that point.  Statistical outlier removal on the same grids."""
    for (h, K), present in RING_CASES_PRESENT.items():
        for rel in sorted(present):
            ref, q, o, dims = ec.ring_bound_case(K, k, h, rel)
            for grid in _grids(ref, o, h, dims, cuda_device):
                idx = _check_knn(grid, q, ref, k, cuda_device)
                assert idx[0, k - 1] == 0, (h, K, rel)
            grid = _Grid(ref, o, h, dims, cuda_device)
            m, keep, stats = _statistical(grid, k, 1.0, cuda_device)
            wm, wkeep, wstats = po.statistical(ref, k, 1.0)
            assert _same(m, wm) and np.array_equal(keep, wkeep) and _same(stats, wstats)


def _three_ring_ties(h):
    """Ties at the k-th place spread over rings 1, 2 and 3 (3-4-5 offsets at distance 2.5h), lowest index outermost."""
    o = np.array([0.0, 0.0, 0.0])
    q = np.array([[20.5, 20.5, 20.5]]) * h
    offs = [[2.5, 0, 0], [2.0, 1.5, 0], [0, 1.5, 2.0], [1.5, 2.0, 0], [0, 0, -2.5], [0, -2.0, 1.5]]
    near = [[0.25 * j, 0, 0] for j in range(1, 8)]
    ref = np.concatenate([q + np.array(offs) * h, q + np.array(near) * h, [o, o + 41 * h]])
    return ref, q, o, [42, 42, 42]


@pytest.mark.parametrize("k", [2, 5, 8, 10])
def test_ties_over_three_rings(gsb_lib, cuda_device, k):
    for h in (1.0, 2.0 ** -20):
        ref, q, o, dims = _three_ring_ties(h)
        for grid in _grids(ref, o, h, dims, cuda_device):
            _check_knn(grid, q, ref, k, cuda_device)


@pytest.mark.parametrize("k", ec.KNN_KS)
def test_more_ties_than_k_and_duplicates(gsb_lib, cuda_device, k):
    ref, q = ec.shell_case(k)
    for h in (1.0, 3.0, 8.0):
        for grid in _grids(ref, np.zeros(3), h, [int(30 / h) + 1] * 3, cuda_device):
            _check_knn(grid, q, ref, k, cuda_device)
    ref, q = ec.duplicates_case(k)
    for grid in _grids(ref, np.array([-1.0, -6.0, -0.5]), 0.25, [32, 32, 32], cuda_device):
        idx = _check_knn(grid, q, ref, k, cuda_device)
        assert idx[0].tolist() == list(range(30, 30 + k))


@pytest.mark.parametrize("k", ec.KNN_KS)
def test_point_counts_around_k(gsb_lib, cuda_device, k):
    rng = np.random.default_rng(k)
    for n in (k - 1, k, k + 1):
        ref = rng.integers(-4, 5, size=(n, 3)) * 0.5 + [7.0, -3.0, 2.0]
        q = np.concatenate([ref, rng.uniform(-3, 3, size=(20, 3)) + [7.0, -3.0, 2.0]])
        for grid in _grids(ref, np.array([4.5, -5.5, -0.5]), 0.5, [11, 11, 11], cuda_device):
            _check_knn(grid, q, ref, k, cuda_device)


def test_far_queries_and_the_last_ring(gsb_lib, cuda_device):
    """Queries 1 cell, 10^3 cells and more than 2^40 cells outside the grid (query_cell's clamp), and queries in one
    corner whose neighbours all lie in the last ring k1, at the opposite corner."""
    o, h, dims = np.array([1.0, 2.0, 3.0]), 0.5, [9, 7, 5]
    rng = np.random.default_rng(3)
    ref = o + rng.integers(0, 9, size=(200, 3)) * [h, h * 6 / 8, h * 4 / 8]
    far = []
    for cells in (1.5, 1000.5, 2.0 ** 41, 2.0 ** 60, 1e300):
        for a in range(3):
            for s in (-1.0, 1.0):
                p = o + 2.0 * h
                p[a] = (o[a] - cells * h) if s < 0 else (o[a] + (dims[a] + cells) * h)
                far.append(p)
    for k in ec.KNN_KS:
        for grid in _grids(ref, o, h, dims, cuda_device):
            _check_knn(grid, np.array(far), ref, k, cuda_device)
    corner = np.array([o + 0.1 * h * j for j in range(3)])
    ref = np.concatenate([o + (np.array(dims) - 0.5) * h + rng.uniform(-0.4, 0.4, size=(40, 3)) * h])
    for k in ec.KNN_KS:
        _check_knn(_Grid(ref, o, h, dims, cuda_device), corner, ref, k, cuda_device)


@pytest.mark.parametrize("nq", [127, 128, 129, 257])
def test_query_counts(gsb_lib, cuda_device, nq):
    rng = np.random.default_rng(nq)
    ref = rng.integers(0, 6, size=(300, 3)) * 0.5
    q = rng.integers(-2, 14, size=(nq, 3)) * 0.25
    for k in ec.KNN_KS:
        for grid in _grids(ref, np.zeros(3), 0.75, [4, 4, 4], cuda_device):
            _check_knn(grid, q, ref, k, cuda_device)


# ------------------------------------------------------------------------------------------------ normals
@pytest.mark.parametrize("name", sorted(ec.EIGEN_CASES))
def test_eigen_cases(gsb_lib, cuda_device, name):
    from gs2mesh_b200.tnt import estimate_normals

    pts = np.asarray(ec.EIGEN_CASES[name], np.float64)
    k = len(pts)
    want = no.estimate_normals(pts, k)
    assert _same(estimate_normals(_dev(pts, cuda_device), k).cpu().numpy(), want)
    trace = np.array([ec.trace_normal(c, k)[0] for c in no.covariances(pts, no.knn(pts, pts, k)[1])])
    assert _same(trace, want)


def test_c_entry_with_queries_off_the_grid(gsb_lib, cuda_device):
    """Normals at points that are not grid points, non-finite ones included, which get (0, 0, 1): Python refuses them,
    the C entry does not."""
    rng = np.random.default_rng(9)
    ref = np.concatenate([rng.integers(-6, 7, size=(400, 3)) * 0.5, rng.normal(size=(400, 3)) * [2.0, 2.0, 0.1]])
    q = np.concatenate([rng.uniform(-4, 4, size=(300, 3)), rng.integers(-12, 13, size=(200, 3)) * 0.25,
                        [[np.nan, 0, 0], [0, np.inf, 0], [0, 0, -np.inf], [np.nan] * 3, [1e30, -1e30, 0.0]]])
    for k in (1, 2, 3, 5, 20, 32):
        idx = no.knn(q, ref, k)[1]
        want = no.fast_eigen3x3(no.covariances(ref, idx))
        zero = ((want[:, 0] * want[:, 0] + want[:, 1] * want[:, 1]) + want[:, 2] * want[:, 2]) == 0.0
        want[zero] = (0.0, 0.0, 1.0)
        for grid in _grids(ref, np.array([-3.0, -3.0, -3.0]), 0.5, [13, 13, 13], cuda_device):
            got = _normals(grid, q, k, cuda_device)
            assert _same(got, want), k
            assert (got[-5:-1] == [0.0, 0.0, 1.0]).all()
