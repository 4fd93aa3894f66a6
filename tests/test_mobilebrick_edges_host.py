"""The MobileBrick edge cases of tests/mobilebrick_edge_cases.py reach their edges (checked with the oracle on the CPU),
the round oracle keeps the heap loop's set on every case small enough for the heap, and every MobileBrick C entry refuses
its bad arguments before it enqueues anything."""
import ctypes as C

import numpy as np
import pytest

from gs2mesh_b200 import _lib
from oracle import mobilebrick_oracle as mo
from tests import mobilebrick_edge_cases as ec


# ------------------------------------------------------------------------------------------------------ elimination
def test_elimination_cases_reach_their_edges():
    o = ec.elimination_oracle("lattice_plane_1m")
    p = ec.elimination_case("lattice_plane_1m")[0]
    assert len(p) > 1_000_000 and (o["nbr"] >= 0).sum(1).max() == 12
    w0 = o["key"][o["round_of"] == 1]
    assert len(w0) > 1000 and len(np.unique(w0)) < len(w0) // 100  # round 1 is decided among equal weights
    o = ec.elimination_oracle("duplicates_200k")
    p, N, r_max, r_min = ec.elimination_case("duplicates_200k")
    valid = o["nbr"] >= 0
    assert len(p) == 200_000 and len(np.unique(p, axis=0)) <= 20_000
    assert (o["d2"][valid] == 0).sum() > 100_000 and (np.sqrt(o["d2"][valid]) < r_min).mean() > 0.5
    o = ec.elimination_oracle("clump_all_neighbours")
    M = len(ec.elimination_case("clump_all_neighbours")[0])
    assert ((o["nbr"] >= 0).sum(1) == M - 1).all() and o["rounds"] == M and M // 4 >= 250
    assert np.array_equal(np.sort(o["round_of"]), np.arange(1, M + 1))  # one point per round
    assert len(np.unique(o["d2"])) < M  # long runs of equal d2
    o = ec.elimination_oracle("zero_terms")
    assert (o["term"] == 0).all() and (o["key"] == 0).all() and o["rounds"] > 4
    o = ec.elimination_oracle("gradient_100k")
    assert o["rounds"] >= 400 and len(ec.elimination_case("gradient_100k")[0]) == 100_000
    for t in ec.ROUND_TARGETS:
        r = ec.elimination_oracle(f"round_count_{t}")["rounds"]
        assert r == t
    assert sorted({t % 4 for t in ec.ROUND_TARGETS}) == [0, 1, 2, 3]  # every position in a read-back batch
    for m in (127, 128, 129, 255, 256, 257):
        assert len(ec.elimination_case(f"block_edge_{m}")[0]) == m
    p = ec.elimination_case("far_offset")[0]
    assert (np.abs(p).max(0) > [9e4, 2e4, 6e3]).all() and ec.elimination_oracle("far_offset")["rounds"] > 1


def test_cell_faces_reach_their_edges():
    p, N, r_max, r_min = ec.elimination_case("cell_faces")
    o = ec.elimination_oracle("cell_faces")
    d = p[:, None, :] - p[None, :, :]
    full = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]
    at = np.argwhere(np.triu(full == r_max * r_max))
    inner = np.argwhere(np.triu(full == np.nextafter(r_max, 0.0) ** 2))
    assert len(at) >= 12 and len(inner) >= 12
    origin, cell, dims = ec.hand_grid_layout(p, r_max)
    assert cell == r_max * ec.CELL_FACTOR and np.array_equal(origin, np.full(3, -cell))
    for pairs in (at, inner):  # the pairs straddle a cell face of the hand-built grid
        c = ec.cell_of(p, origin, cell)
        assert (c[pairs[:, 0]] != c[pairs[:, 1]]).any(1).sum() >= 12
    nbr = o["nbr"]
    for i, j in at:
        assert j not in nbr[i]
    for i, j in inner:
        assert j in nbr[i] and i in nbr[j]
    u = (p - origin) / cell
    assert (np.abs(u - np.rint(u)) == 0).any(1).sum() > 300  # points exactly on the grid's cell faces


def test_nth_key_tie():
    p, N, r_max, r_min = ec.elimination_case("nth_key_tie")
    o = ec.elimination_oracle("nth_key_tie")
    order = np.lexsort((np.arange(len(p)), o["key"]))
    a, b = order[N - 1], order[N]
    assert o["key"][a] == o["key"][b] and a < b
    assert a in o["kept"] and b not in o["kept"]


@pytest.mark.parametrize("name", [n for n in ec.ELIMINATION_NAMES if n not in ec.LARGE + ("clump_all_neighbours",)])
def test_round_oracle_keeps_the_heap_set(name):
    p, N, r_max, r_min = ec.elimination_case(name)
    assert len(p) <= 30_000
    o = ec.elimination_oracle(name)
    kept, key, order = mo.eliminate_heap(o["nbr"], o["term"], N)
    assert np.array_equal(kept, o["kept"])
    assert np.array_equal(key[order], o["key"][order])


@pytest.mark.parametrize("M,seed", [(60, 1), (150, 2)])
def test_clump_restatement(M, seed):
    """The clump's fast sequential loop equals eliminate_rounds and the heap loop on smaller clumps."""
    p, N, r_max, r_min = ec.small_clump(M, seed)
    nbr, d2 = mo.neighbour_lists(p, r_max)
    assert ((nbr >= 0).sum(1) == M - 1).all()
    term = mo.weight_term(d2, r_min, r_max)
    key, rnd, rounds = ec._clump_elimination(nbr, term)
    kept_r, key_r, rnd_r, rounds_r = mo.eliminate_rounds(nbr, term, N)
    assert rounds == rounds_r == M and np.array_equal(rnd, rnd_r) and np.array_equal(key, key_r)
    assert np.array_equal(mo.eliminate_heap(nbr, term, N)[0], kept_r)


# ---------------------------------------------------------------------------------------------------------- sampler
def test_sampler_cases_reach_their_edges():
    cases = {name: ec.sampler_case(name) for name in ec.SAMPLER_NAMES}
    v, t, b, var, ns, _ = cases["special_variates"]
    pairs = {(a, c) for a, c in var.reshape(-1, 2).tolist()}
    assert len(pairs) == 25
    v, t, b, var, ns, _ = cases["zero_area_runs"]
    zero = mo.triangle_areas(v, t) == 0
    assert zero[:6].all() and zero[23:32].all() and zero[-5:].all() and zero.sum() == 20
    assert (np.diff(b)[zero] == 0).all()
    for name in ("hand_bounds_short", "hand_bounds_empty", "hand_bounds_start_end_runs", "one_triangle_hand_short"):
        v, t, b, var, ns, from_areas = cases[name]
        assert not from_areas and b[-1] < ns and len(b) == len(t) + 1 and (np.diff(b) >= 0).all() and b[0] == 0
    assert len(cases["one_triangle"][1]) == 1
    v, t, b, var, ns, _ = cases["over_2p20_triangles"]
    assert len(t) > 2 ** 20 and ns >= 5_000_000 and b[-1] == ns
    assert np.abs(cases["near_1e6"][0]).min() > 9e5
    assert [cases[f"ns_{n}"][4] for n in (255, 256, 257)] == [255, 256, 257]


def test_sample_formula_matches_the_oracle():
    """The numpy formula the GPU test uses for hand-made bounds equals mo.sample_uniform where bounds come from areas."""
    for name in ec.SAMPLER_NAMES:
        v, t, b, var, ns, from_areas = ec.sampler_case(name)
        if from_areas:
            want = mo.sample_uniform(v, t, ns, var)[0]
            assert np.array_equal(ec.sample_formula(v, t, b, var, ns), want), name


# ------------------------------------------------------------------------------------------------------- visibility
def test_visibility_cases_reach_their_edges():
    cases = {name: ec.visibility_case(name) for name in ec.VISIBILITY_NAMES}
    for name in ("flip_odd", "flip_large"):
        p, vol, mins, res, vs = cases[name]
        i32 = mo.visibility_index(p, mins, res, vs)
        with np.errstate(invalid="ignore"):
            i64 = ec.fp64_index(p, mins, res, vs)
        flips = (i32 != i64).any(1)
        assert flips.sum() > 10, name  # the fp32 g picks another voxel than the fp64 one would
        # and in at least one the other voxel's flag differs, so the keep mask sees the flip
        inside = ((i32 >= 0) & (i32 < res)).all(1) & ((i64 >= 0) & (i64 < res)).all(1) & flips
        a, b = i32[inside], i64[inside].astype(np.int64)
        assert (vol[a[:, 0], a[:, 1], a[:, 2]] != vol[b[:, 0], b[:, 1], b[:, 2]]).any(), name
    p, vol, mins, res, vs = cases["non_finite_and_huge"]
    assert np.isnan(p).any() and np.isinf(p).any() and (np.abs(p[np.isfinite(p)]) >= 1e30).any()
    idx = mo.visibility_index(p, mins, res, vs)
    assert (idx == 0).any() and (np.abs(idx) >= 2 ** 31 - 1).any() and (idx == -100).any()
    keep = mo.visibility(p, vol, mins, res, vs)
    # every voxel is marked and each offset from min_pts is 0 or far outside: visible iff all offsets are 0
    assert keep.any() and np.array_equal(keep, (p == mins).all(1))
    assert not keep[np.isnan(p).any(1)].any() and not keep[np.isinf(p).any(1)].any()
    assert list(cases["res_2_2_2"][3]) == [2, 2, 2] and list(cases["res_2_3_4097"][3]) == [2, 3, 4097]


@pytest.mark.parametrize("name", ec.VISIBILITY_NAMES)
def test_visibility_oracle_matches_grid_sample_on_the_cpu(name):
    """The oracle equals the reference's literal F.grid_sample expression on every row, NaN and infinite rows included
    (torch's CPU sampler guards non-finite coordinates as its CUDA one does)."""
    points, vol, min_pts, res, vs = ec.visibility_case(name)
    ref = ec.grid_sample_reference(points, vol, min_pts, res, vs, "cpu")
    assert np.array_equal(mo.visibility(points, vol, min_pts, res, vs), ref)


def test_big_volume_reaches_past_2p31():
    p, marked, mins, res, vs = ec.big_volume_case()
    assert np.prod(res.astype(np.float64)) > 2 ** 31
    keep, flat = ec.big_volume_oracle(p, marked, mins, res, vs)
    assert (flat >= 2 ** 31).sum() > 2000 and (marked >= 2 ** 31).sum() > 40
    assert keep[flat >= 2 ** 31].any() and not keep.all()
    assert keep[flat == 0].all() and (flat == -1).any()  # the voxel at the origin, and a point outside


# ------------------------------------------------------------------------------------------------------ C refusals
def test_c_entry_points_refuse_bad_arguments(gsb_lib):
    L = gsb_lib
    fake = C.c_void_p(256)  # never dereferenced: every refusal happens before any device work
    bad = _lib.GSB_ERR_INVALID
    # gsb_eval_triangle_areas
    assert L.gsb_eval_triangle_areas(fake, -1, fake, 1, fake, None) == bad
    assert L.gsb_eval_triangle_areas(fake, 3, fake, -1, fake, None) == bad
    for args in ((None, fake, fake), (fake, None, fake), (fake, fake, None)):
        assert L.gsb_eval_triangle_areas(args[0], 3, args[1], 1, args[2], None) == bad
    assert L.gsb_eval_triangle_areas(None, 0, None, 0, None, None) == _lib.GSB_OK
    # gsb_eval_sample_uniform
    for nt in (0, -1):
        assert L.gsb_eval_sample_uniform(fake, 3, fake, nt, fake, fake, 10, fake, None) == bad
    assert L.gsb_eval_sample_uniform(fake, -1, fake, 1, fake, fake, 10, fake, None) == bad
    assert L.gsb_eval_sample_uniform(fake, 3, fake, 1, fake, fake, -1, fake, None) == bad
    for k in range(5):
        a = [fake] * 5
        a[k] = None
        assert L.gsb_eval_sample_uniform(a[0], 3, a[1], 1, a[2], a[3], 10, a[4], None) == bad
    assert L.gsb_eval_sample_uniform(None, 3, None, 1, None, None, 0, None, None) == _lib.GSB_OK
    # gsb_eval_poisson_neighbours
    def grid(cell=1.0, n=10):
        return _lib.GsbPointGrid((C.c_double * 3)(0, 0, 0), cell, (C.c_int32 * 3)(1, 1, 1), 256, n, 256, 256)

    g = grid()
    for r_max, r_min in ((0.0, 0.0), (float("inf"), 0.0), (float("nan"), 0.0), (-1.0, 0.0), (0.5, -1e-300),
                         (0.5, np.nextafter(0.5, 1.0)), (0.5, float("nan"))):
        assert L.gsb_eval_poisson_neighbours(C.byref(g), r_max, r_min, fake, None, None, None, None) == bad
        assert L.gsb_eval_poisson_neighbours(C.byref(g), r_max, r_min, None, fake, fake, fake, None) == bad
    tight = grid(cell=0.5 * ec.CELL_FACTOR)
    assert L.gsb_eval_poisson_neighbours(C.byref(grid(cell=np.nextafter(0.5 * ec.CELL_FACTOR, 0.0))), 0.5, 0.1, fake,
                                         None, None, None, None) == bad
    assert L.gsb_eval_poisson_neighbours(C.byref(grid(n=2 ** 31 - 1)), 0.5, 0.1, fake, None, None, None, None) == bad
    assert L.gsb_eval_poisson_neighbours(C.byref(grid(n=2 ** 31)), 0.5, 0.1, fake, None, None, None, None) == bad
    assert L.gsb_eval_poisson_neighbours(C.byref(tight), 0.5, 0.1, None, None, None, None, None) == bad  # count mode
    assert L.gsb_eval_poisson_neighbours(C.byref(tight), 0.5, 0.1, None, fake, None, fake, None) == bad  # emit mode
    assert L.gsb_eval_poisson_neighbours(C.byref(tight), 0.5, 0.1, None, fake, fake, None, None) == bad
    assert L.gsb_eval_poisson_neighbours(None, 0.5, 0.1, fake, None, None, None, None) == bad
    assert L.gsb_eval_poisson_neighbours(C.byref(grid(n=0)), 0.5, 0.5, None, None, None, None, None) == _lib.GSB_OK
    assert L.gsb_eval_poisson_neighbours(C.byref(grid(n=0, cell=0.5 * ec.CELL_FACTOR)), 0.5, 0.0, None, None, None, None,
                                         None) == _lib.GSB_OK  # the smallest accepted cell, r_min = 0
    # gsb_eval_poisson_eliminate
    live = C.c_int32(0)
    assert L.gsb_eval_poisson_eliminate(fake, fake, fake, -1, fake, fake, fake, fake, C.byref(live), None) == bad
    assert L.gsb_eval_poisson_eliminate(fake, fake, fake, 2 ** 31 - 1, fake, fake, fake, fake, C.byref(live), None) == bad
    for k in range(7):
        a = [fake] * 7
        a[k] = None
        assert L.gsb_eval_poisson_eliminate(a[0], a[1], a[2], 10, a[3], a[4], a[5], a[6], None, None) == bad
    live = C.c_int32(7)
    assert L.gsb_eval_poisson_eliminate(None, None, None, 0, None, None, None, None, C.byref(live), None) == _lib.GSB_OK
    assert live.value == 0
    # gsb_eval_visibility
    mins = (C.c_double * 3)(0, 0, 0)
    res = lambda a, b, c: (C.c_int32 * 3)(a, b, c)  # noqa: E731
    for r in ((1, 2, 2), (2, 1, 2), (2, 2, 1), (0, 5, 5), (-2, 5, 5), (300000, 300000, 300000)):
        assert L.gsb_eval_visibility(fake, 10, mins, 0.1, res(*r), fake, fake, None) == bad
    for vs in (0.0, -0.1, float("nan"), float("inf"), -float("inf")):
        assert L.gsb_eval_visibility(fake, 10, mins, vs, res(4, 4, 4), fake, fake, None) == bad
        assert L.gsb_eval_visibility(None, 0, mins, vs, res(4, 4, 4), None, None, None) == bad
    assert b"voxel_size" in L.gsb_last_error()
    for m in (float("nan"), float("inf"), -float("inf")):
        for a in range(3):
            mm = [0.0, 0.0, 0.0]
            mm[a] = m
            assert L.gsb_eval_visibility(fake, 10, (C.c_double * 3)(*mm), 0.1, res(4, 4, 4), fake, fake, None) == bad
    assert L.gsb_eval_visibility(fake, -1, mins, 0.1, res(4, 4, 4), fake, fake, None) == bad
    assert L.gsb_eval_visibility(fake, 10, None, 0.1, res(4, 4, 4), fake, fake, None) == bad
    assert L.gsb_eval_visibility(fake, 10, mins, 0.1, None, fake, fake, None) == bad
    for k in range(3):
        a = [fake] * 3
        a[k] = None
        assert L.gsb_eval_visibility(a[0], 10, mins, 0.1, res(4, 4, 4), a[1], a[2], None) == bad
    assert L.gsb_eval_visibility(None, 0, mins, 0.1, res(4, 4, 4), None, None, None) == _lib.GSB_OK

