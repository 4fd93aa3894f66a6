"""The MobileBrick kernels (gsb_mobilebrick.cu) at the edges of tests/mobilebrick_edge_cases.py, bit for bit against
oracle/mobilebrick_oracle.py: the neighbour lists themselves (counts, offsets, ids, terms; on PointGrid's grid and on a
hand-built grid at the smallest accepted cell), the elimination's kept set, removal keys, rounds of deletion and round
count, the uniform sampler on crafted bounds and variates, the visibility lookup against the oracle and the reference's
literal F.grid_sample expression, a volume of more than 2^31 voxels, and repeatability of the largest eliminations."""
import ctypes as C

import numpy as np
import pytest

from oracle import mobilebrick_oracle as mo
from tests import mobilebrick_edge_cases as ec

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _peak_memory():
    import time

    t0 = time.perf_counter()
    yield
    import torch

    if torch.cuda.is_available():
        print(f"\ntest_gpu_mobilebrick_edges: {time.perf_counter() - t0:.1f} s, peak torch memory "
              f"{torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def _dev(x, device, dtype=None):
    import torch

    return torch.as_tensor(np.ascontiguousarray(x), device=device, dtype=dtype)


def _hand_grid(p, r_max):
    """A GsbPointGrid over p at cell r_max * 1.0000001, built by gsb_eval_grid_build (the tensors stay alive on it)."""
    import torch

    from gs2mesh_b200 import _lib
    from gs2mesh_b200._lib import ptr

    origin, cell, dims = ec.hand_grid_layout(p.cpu().numpy(), r_max)
    n = p.shape[0]
    g = type("HandGrid", (), {})()
    g.points = p
    g.cell_start = torch.empty(dims[0] * dims[1] * dims[2] + 1, dtype=torch.int64, device=p.device)
    g.ids = torch.empty(n, dtype=torch.int64, device=p.device)
    g.desc = _lib.GsbPointGrid((C.c_double * 3)(*origin.tolist()), cell, (C.c_int32 * 3)(*dims), ptr(p), n,
                               ptr(g.cell_start), ptr(g.ids))
    L = _lib.lib()
    ws = torch.empty(int(L.gsb_eval_grid_workspace_bytes(n, g.cell_start.numel() - 1)), dtype=torch.uint8, device=p.device)
    _lib.check(L.gsb_eval_grid_build(C.byref(g.desc), ptr(ws), ws.numel(), _lib.stream(p.device)))
    return g


def _neighbour_lists(grid, M, r_max, r_min, device):
    """gsb_eval_poisson_neighbours in count mode, then emit mode -> (counts, offsets, ids, terms) on the host."""
    import torch

    from gs2mesh_b200 import _lib
    from gs2mesh_b200._lib import ptr

    L = _lib.lib()
    s = _lib.stream(device)
    counts = torch.full((M,), -7, dtype=torch.int64, device=device)
    _lib.check(L.gsb_eval_poisson_neighbours(C.byref(grid.desc), r_max, r_min, ptr(counts), None, None, None, s))
    offsets = torch.zeros(M + 1, dtype=torch.int64, device=device)
    torch.cumsum(counts, 0, out=offsets[1:])
    total = int(offsets[-1].item())
    nbr = torch.full((max(total, 1),), -7, dtype=torch.int32, device=device)
    terms = torch.full((max(total, 1),), -7.0, dtype=torch.float64, device=device)
    _lib.check(L.gsb_eval_poisson_neighbours(C.byref(grid.desc), r_max, r_min, None, ptr(offsets), ptr(nbr), ptr(terms), s))
    return counts.cpu().numpy(), offsets.cpu().numpy(), nbr[:total].cpu().numpy(), terms[:total].cpu().numpy()


def _check_lists(got, o):
    counts, offsets, ids, terms = got
    valid = o["nbr"] >= 0
    assert np.array_equal(counts, valid.sum(1))
    assert offsets[0] == 0 and np.array_equal(np.diff(offsets), counts)
    assert np.array_equal(ids, o["nbr"][valid])  # row-major: each point's list in (d2, index) order
    assert np.array_equal(_bits(terms), _bits(o["term"][valid]))


NEIGHBOUR_CASES = [n for n in ec.ELIMINATION_NAMES if n != "lattice_plane_1m"] + ["lattice_plane_1m"]


@pytest.mark.parametrize("name", NEIGHBOUR_CASES)
def test_neighbour_lists(gsb_lib, cuda_device, name):
    from gs2mesh_b200.evaluate import PointGrid

    p, N, r_max, r_min = ec.elimination_case(name)
    o = ec.elimination_oracle(name)
    pd = _dev(p, cuda_device)
    _check_lists(_neighbour_lists(PointGrid(pd, r_max), len(p), r_max, r_min, cuda_device), o)
    if name in ("cell_faces", "far_offset", "duplicates_200k", "clump_all_neighbours") or name.startswith("block_edge"):
        _check_lists(_neighbour_lists(_hand_grid(pd, r_max), len(p), r_max, r_min, cuda_device), o)


def _eliminate(p, N, r_max, r_min, device):
    from gs2mesh_b200 import mobilebrick as mb

    kept, info = mb.eliminate(_dev(p, device), N, r_max, r_min, return_info=True)
    return kept.cpu().numpy(), info["keys"].cpu().numpy(), info["round_of"].cpu().numpy(), info["rounds"]


@pytest.mark.parametrize("name", ec.ELIMINATION_NAMES)
def test_elimination(gsb_lib, cuda_device, name):
    p, N, r_max, r_min = ec.elimination_case(name)
    o = ec.elimination_oracle(name)
    kept, key, rnd, rounds = _eliminate(p, N, r_max, r_min, cuda_device)
    assert rounds == o["rounds"]
    assert np.array_equal(rnd, o["round_of"])
    assert np.array_equal(_bits(key), _bits(o["key"]))
    assert np.array_equal(kept, o["kept"])
    if name in ec.LARGE:  # repeatability: the same bytes again
        again = _eliminate(p, N, r_max, r_min, cuda_device)
        assert np.array_equal(again[0], kept) and np.array_equal(again[2], rnd) and again[3] == rounds
        assert np.array_equal(_bits(again[1]), _bits(key))


# ---------------------------------------------------------------------------------------------------------- sampler
@pytest.mark.parametrize("name", ec.SAMPLER_NAMES)
def test_sampler(gsb_lib, cuda_device, name):
    import torch

    from gs2mesh_b200 import _lib
    from gs2mesh_b200._lib import ptr

    v, t, bounds, variates, ns, from_areas = ec.sampler_case(name)
    vd, td, bd, var = (_dev(v, cuda_device), _dev(t, cuda_device), _dev(bounds, cuda_device), _dev(variates, cuda_device))
    out = torch.full((ns, 3), float("nan"), dtype=torch.float64, device=cuda_device)
    L = _lib.lib()
    if from_areas:
        areas = torch.empty(len(t), dtype=torch.float64, device=cuda_device)
        _lib.check(L.gsb_eval_triangle_areas(ptr(vd), len(v), ptr(td), len(t), ptr(areas), _lib.stream(cuda_device)))
        assert np.array_equal(_bits(areas.cpu().numpy()), _bits(mo.triangle_areas(v, t)))
    _lib.check(L.gsb_eval_sample_uniform(ptr(vd), len(v), ptr(td), len(t), ptr(bd), ptr(var), ns, ptr(out),
                                         _lib.stream(cuda_device)))
    got = out.cpu().numpy()
    want = mo.sample_uniform(v, t, ns, variates)[0] if from_areas else ec.sample_formula(v, t, bounds, variates, ns)
    assert np.array_equal(_bits(got), _bits(want))
    if not from_areas:
        assert (got[bounds[-1]:] == 0).all()


# ------------------------------------------------------------------------------------------------------- visibility
@pytest.mark.parametrize("name", ec.VISIBILITY_NAMES)
def test_visibility(gsb_lib, cuda_device, name):
    """Against the oracle and against evaluate.py:36-41 literally on the device, on every row: NaN and infinite
    coordinates are invisible, as torch's sampler makes them."""
    from gs2mesh_b200 import mobilebrick as mb

    points, vol, min_pts, res, vs = ec.visibility_case(name)
    got = mb.visibility_test(_dev(points, cuda_device), vol.reshape(-1), min_pts, res, vs).cpu().numpy()
    assert np.array_equal(got, mo.visibility(points, vol, min_pts, res, vs))
    assert np.array_equal(got, ec.grid_sample_reference(points, vol, min_pts, res, vs, cuda_device))
    if name == "non_finite_and_huge":
        assert got.any() and not got[~np.isfinite(points).all(1)].any()


def test_visibility_refuses_bad_volume_parameters(gsb_lib, cuda_device):
    from gs2mesh_b200 import mobilebrick as mb

    vol = np.ones(8, bool)
    pts = _dev(np.zeros((4, 3)), cuda_device)
    for vs, mins in ((0.0, [0, 0, 0]), (float("nan"), [0, 0, 0]), (-1.0, [0, 0, 0]), (float("inf"), [0, 0, 0]),
                     (0.1, [0, float("inf"), 0]), (0.1, [float("nan"), 0, 0])):
        with pytest.raises(ValueError, match="voxel_size"):
            mb.visibility_test(pts, vol, mins, [2, 2, 2], vs)


def test_visibility_over_2p31_voxels(gsb_lib, cuda_device):
    """1291^3 uint8 voxels (2.15 GB) on the device, marked near the far corner; compared with the oracle's index."""
    import torch

    from gs2mesh_b200 import _lib
    from gs2mesh_b200._lib import ptr

    points, marked, min_pts, res, vs = ec.big_volume_case()
    want, flat = ec.big_volume_oracle(points, marked, min_pts, res, vs)
    vol = torch.zeros(int(np.prod(res)), dtype=torch.uint8, device=cuda_device)
    try:
        vol[_dev(marked, cuda_device)] = 1
        pd = _dev(points, cuda_device)
        keep = torch.full((len(points),), 7, dtype=torch.uint8, device=cuda_device)
        rc = _lib.lib().gsb_eval_visibility(ptr(pd), len(points), (C.c_double * 3)(*min_pts.tolist()), vs,
                                            (C.c_int32 * 3)(*[int(r) for r in res]), ptr(vol), ptr(keep),
                                            _lib.stream(cuda_device))
        _lib.check(rc)
        got = keep.cpu().numpy().astype(bool)
    finally:
        del vol
        torch.cuda.empty_cache()
    assert np.array_equal(got, want)
    assert got[flat >= 2 ** 31].any()
