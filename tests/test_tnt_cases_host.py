"""The Tanks and Temples edge cases of tests/tnt_cases.py reach their edges (CPU only), and the CPU oracle
(oracle/tnt_oracle.py) agrees with the exact references on them."""
import math

import numpy as np
import pytest

from oracle import tnt_oracle as to
from tests import tnt_cases as tc

TRANSFORM = tc.transform_cases()
CROP = tc.crop_cases()
VOXEL = tc.voxel_cases()
MOMENTS = tc.moment_cases()
ICP = tc.icp_cases()


def test_transform_cases_reach_their_edges():
    assert {len(TRANSFORM[f"n{n}"][0]) for n in (1, 255, 256, 257)} == {1, 255, 256, 257}
    pts, T = TRANSFORM["w_zero"]
    assert all(tc.transform_rows(p, T)[0][3] == 0 for p in pts)
    assert any(tc.transform_rows(p, T)[0][0] == 0 for p in pts)  # 0 / 0
    assert np.all((T[3] == 0) & ~np.signbit(T[3]))
    pts, T = TRANSFORM["w_negative"]
    assert all(tc.transform_rows(p, T)[0][3] < 0 for p in pts)
    pts, T = TRANSFORM["negative_zero"]
    assert tc.is_negative_zero(T).sum() >= 8
    assert tc.is_negative_zero(T[None, :3, :3] * pts[:, None, :]).any()  # -0.0 * x = -0.0 and -0.0 * -x = +0.0
    pts, T = TRANSFORM["subnormal"]
    prods = T[None, :3, :3] * pts[:, None, :]
    assert tc.is_subnormal(prods).sum() >= len(pts)
    pts, _ = TRANSFORM["non_finite"]
    assert np.isposinf(pts).any() and np.isneginf(pts).any() and np.isnan(pts).any()


@pytest.mark.parametrize("name", sorted(set(TRANSFORM) - {"non_finite", "non_finite_identity", "w_zero"}))
def test_transform_oracle_within_exact_bound(name):
    pts, T = TRANSFORM[name]
    checked, skipped = tc.transform_exact_check(pts, T, to.transform(pts, T))
    assert checked == len(pts) and skipped == 0


def _uv(case):
    u, v, _ = tc.AXES[case["axis"].lower()]
    return u, v


def test_crop_cases_reach_their_edges():
    for m in (3, 255, 256, 257, 1024, 2048):
        assert len(CROP[f"m{m}"]["polygon"]) == m
    assert all(len(CROP[f"m{m}"]["polygon"]) > tc.BLOCK for m in (257, 1024, 2048))  # a second copy pass
    assert 8 * 2 * tc.MAX_POLYGON == 32 * 1024  # the largest polygon's (u, v) fill 32 KB of shared memory
    for name, case in CROP.items():
        P, pts = case["polygon"], case["points"]
        u, v = _uv(case)
        w = 3 - u - v
        assert (P[:, w] != 0).any(), name  # the crop ignores the polygon's w
        if name.startswith(("m", "clockwise", "rectilinear", "degenerate", "bowtie")):
            vert = {(a, b) for a, b in P[:, [u, v]].tolist()}
            on = [(a, b) in vert for a, b in pts[:, [u, v]].tolist()]
            assert sum(on) >= len(vert), name  # every vertex is a point
            assert np.isin(pts[:, v], P[:, v]).sum() >= 4 * len(vert), name  # p_v equals a vertex's v
            # crossings equal to p_u exactly, on an edge the rule selects
            exact = 0
            for k in range(len(P)):
                a, b = P[k, [u, v]], P[(k + 1) % len(P), [u, v]]
                pv, pu = pts[:, v], pts[:, u]
                sel = tc.crop_edges_selected(pu, pv, a[0], a[1], b[0], b[1])
                with np.errstate(divide="ignore", invalid="ignore"):
                    x = tc.crossing_float(np.stack([pu, pv]), a, b)
                exact += int((sel & (x == pu)).sum())
            assert exact >= len(P), name
    stair = CROP["rectilinear"]
    u, v = _uv(stair)
    P = stair["polygon"][:, [u, v]]
    nxt = np.roll(P, -1, 0)
    assert (P[:, 1] == nxt[:, 1]).sum() == 5 and (P[:, 0] == nxt[:, 0]).sum() == 5  # horizontal and vertical edges
    deg = CROP["degenerate_edges"]
    u, v = _uv(deg)
    P = deg["polygon"][:, [u, v]]
    nxt = np.roll(P, -1, 0)
    assert (np.all(P == nxt, axis=1)).sum() >= 3  # zero-length edges
    a, b, c = P, nxt, np.roll(P, -2, 0)
    cross = (b[:, 0] - a[:, 0]) * (c[:, 1] - a[:, 1]) - (b[:, 1] - a[:, 1]) * (c[:, 0] - a[:, 0])
    assert ((cross == 0) & ~np.all(a == b, axis=1) & ~np.all(b == c, axis=1)).sum() >= 2  # collinear runs

    def area(case):
        u, v = _uv(case)
        x, y = case["polygon"][:, u], case["polygon"][:, v]
        return 0.5 * float(np.sum(x * np.roll(y, -1) - np.roll(x, -1) * y))

    assert area(CROP["m256"]) > 0 and area(CROP["clockwise"]) < 0  # both windings
    B = tc.BOWTIE  # edges 0-1 and 2-3 cross at the origin
    side = [float(np.linalg.det(np.stack([B[1] - B[0], B[k] - B[0]]))) for k in (2, 3)]
    assert side[0] * side[1] < 0
    assert CROP["slab_equal"]["axis_min"] == CROP["slab_equal"]["axis_max"]
    assert (CROP["slab_equal"]["points"][:, 2] == 0.5).any()
    assert CROP["slab_reversed"]["axis_min"] > CROP["slab_reversed"]["axis_max"]
    for name in ("zero_bounds", "zero_bounds_swapped"):
        c = CROP[name]
        assert c["axis_min"] == 0 == c["axis_max"] and np.signbit(c["axis_min"]) != np.signbit(c["axis_max"])
        assert tc.is_negative_zero(c["points"][:, 2]).any()
    P = CROP["huge"]["polygon"]
    with np.errstate(over="ignore"):
        assert np.isinf(np.roll(P, -1, 0) - P).any()  # (b_u - a_u) overflows
    assert [len(CROP[f"n{n}"]["points"]) for n in (1, 255, 256, 257)] == [1, 255, 256, 257]


@pytest.mark.parametrize("name", sorted(CROP))
def test_crop_oracle_agrees_with_exact_outside_the_band(name):
    case = CROP[name]
    keep, band = tc.crop_exact(case)
    with np.errstate(over="ignore", invalid="ignore"):
        got = to.crop_mask(case["points"], case["axis"], case["axis_min"], case["axis_max"], case["polygon"])
    assert np.array_equal(got[~band], keep[~band])
    if name != "huge":
        assert band.sum() == 0  # dyadic inputs: every crossing is either exact or far from p_u
    if name.startswith("m") or name == "rectilinear":
        assert 0 < keep.sum() < len(keep)
    if name == "slab_reversed":
        assert not keep.any()


def test_voxel_cases_reach_their_edges():
    for n in (2, 1000, 1_000_000):
        pts, vs, _ = VOXEL[f"one_voxel_{n}"]
        assert len(pts) == n and tc.voxel_layout(pts, vs)[3] == [0, 0, 0]  # begin_bit == end_bit: CUB copies
    assert tc.voxel_layout(*VOXEL["planar"][:2])[3][2] == 0
    assert tc.voxel_layout(*VOXEL["linear"][:2])[3][:2] == [0, 0]
    lo, span, extent, bits = tc.voxel_layout(*VOXEL["bits63"][:2])
    assert extent == [1 << 21] * 3 and sum(bits) == 63
    assert sum(tc.voxel_layout(*VOXEL["bits64"][:2])[3]) == 64
    lo, span, extent, bits = tc.voxel_layout(*VOXEL["int_max"][:2])
    assert span == 1.0 * tc.INT_MAX and bits[0] == 31
    assert tc.voxel_layout(*VOXEL["int_max_over"][:2])[1] > 1.0 * tc.INT_MAX
    for vs in (0.01, 0.005, 0.003, 0.0025, 0.0015):
        pts = VOXEL[f"lattice_{vs}"][0]
        assert np.abs(pts).max() > 30
        q, _ = tc.voxel_quotients(pts, vs)
        r = np.rint(q)
        near = np.abs(q - r) < 1e-9
        assert (near & (q < r)).sum() > 100 and (near & (q >= r)).sum() > 100  # both sides of the voxel boundary
    pts, vs, _ = VOXEL["all_distinct"]
    assert len(tc.voxel_exact(pts, vs)[0]) == len(pts)
    pts = VOXEL["duplicates"][0]
    assert len(np.unique(pts, axis=0)) < len(pts)
    pts = VOXEL["signed_zero"][0]
    assert tc.is_negative_zero(pts[:4]).any() and (pts[:4] == 0).all() and (~np.signbit(pts[:4])).any()


@pytest.mark.parametrize("name", sorted(set(VOXEL) - {"one_voxel_1000000"}))
def test_voxel_oracle_against_exact(name):
    pts, vs, expect = VOXEL[name]
    if expect == "too small":
        with pytest.raises(ValueError, match="too small"):
            to.voxel_down_sample(pts, vs)
        return
    got = to.voxel_down_sample(pts, vs)[0]
    keys, groups, n_boundary = tc.voxel_exact(pts, vs)
    assert len(got) == len(keys)
    tc.voxel_mean_check(pts, groups, got)
    if name.startswith("lattice"):
        assert n_boundary > 0
    elif not name.startswith("bits") and name != "int_max":
        assert n_boundary == 0


def test_moment_cases_reach_their_edges():
    for n in (65535, 65536, 65537, 131073):
        assert len(MOMENTS[f"n{n}"][0]) == n
    for name, (src, tgt, idx, d2) in MOMENTS.items():
        if name not in ("no_correspondence", "last_lane"):
            assert idx.max() == len(tgt) - 1 and (d2[idx >= 0] == 0).any() and tc.is_subnormal(d2[idx >= 0]).any()
    assert (MOMENTS["no_correspondence"][2] == -1).all()
    idx = MOMENTS["last_lane"][2]
    (i,) = np.nonzero(idx >= 0)[0]
    assert i % tc.MOMENT_LANES == tc.MOMENT_LANES - 1 and i // 256 == 255 and i % 256 == 255  # block 255, lane 255
    assert np.abs(MOMENTS["far"][0]).min(0).max() > 1e4


@pytest.mark.parametrize("name", ["n65537", "far", "last_lane"])
def test_moment_oracle_within_fsum_bound(name):
    src, tgt, idx, d2 = MOMENTS[name]
    sums, cnt = to.moments(src, tgt, idx, d2)
    assert cnt == int((idx >= 0).sum())
    tc.moment_fsum_check(tc.moment_values(src, tgt, idx, d2), len(src), sums)
    mu = np.concatenate([sums[1:4], sums[4:7]]) * (1.0 / cnt)
    tc.moment_fsum_check(tc.moment_values(src, tgt, idx, d2, mu), len(src), to.moments(src, tgt, idx, d2, mu)[0])


def test_icp_cases_reach_their_edges():
    for name in ("mirror", "mirror_rigid"):
        sums, cnt, second = tc.first_umeyama_inputs(ICP[name])
        assert cnt == len(ICP[name]["source"])
        U, D, Vt = np.linalg.svd(second[:9].reshape(3, 3) * (1.0 / cnt))
        assert np.linalg.det(U) * np.linalg.det(Vt) < 0  # S = diag(1, 1, -1)
    for name in ("one_source_point", "one_source_point_rigid"):
        sums, cnt, second = tc.first_umeyama_inputs(ICP[name])
        assert cnt == 4 and np.all(second == 0)  # src_var = 0 and sigma = 0
    sums, cnt, second = tc.first_umeyama_inputs(ICP["collinear"])
    D = np.linalg.svd(second[:9].reshape(3, 3))[1]
    assert cnt > 100 and D[1] <= 1e-12 * D[0]
    assert ICP["max_iteration_0"]["max_iteration"] == 0
    assert len(ICP["empty_source"]["source"]) == 0 and len(ICP["empty_target"]["target"]) == 0
    init = ICP["negative_zero_init"]["init"]
    assert np.array_equal(init, np.eye(4)) and tc.is_negative_zero(init).sum() == 4
    assert ICP["rigid"]["with_scaling"] is False


@pytest.mark.parametrize("name", sorted(ICP))
def test_icp_oracle_on_the_cases(name):
    c = ICP[name]
    with np.errstate(divide="ignore", invalid="ignore"):
        T, fit, rmse, it, hist = to.registration_icp(c["source"], c["target"], c["radius"], c["init"], c["with_scaling"],
                                                     c["relative"], c["relative"], c["max_iteration"])
    assert len(hist) == it
    if name == "rigid":
        assert fit == 1.0 and it < c["max_iteration"] and np.abs(T - tc.RIGID).max() < 1e-9
    if name == "one_source_point":
        # c = (1 / 0) * 0 = NaN: the first update's top rows are NaN, no NaN point corresponds, and the identity update
        # of the second iteration (NaN * 0 in the product) leaves every entry NaN
        assert np.isnan(hist[0][:3]).all() and np.array_equal(hist[0][3], [0, 0, 0, 1])
        assert it == 2 and np.isnan(T).all() and fit == 0.0 and rmse == 0.0
    if name == "one_source_point_rigid":
        assert np.isfinite(T).all() and fit == 1.0
    if name == "max_iteration_0":
        assert it == 0 and np.array_equal(T, np.eye(4))
    if name.startswith("empty"):
        assert (fit, rmse, it) == (0.0, 0.0, 1) and np.array_equal(T, np.eye(4))
    if name == "negative_zero_init":
        assert fit > 0.9 and math.isfinite(rmse)
