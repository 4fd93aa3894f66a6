"""CPU checks that every rasterizer edge case of tests/raster_cases.py reaches the edge it is named for (computed with the
CPU oracle's preprocess and the host restatements there), and the image-side limit refusal, which needs no GPU."""
import ctypes as C

import numpy as np
import pytest

from tests import raster_cases as rc


def test_higher_msb_restatement(oracle):
    for n in [1, 2, 3, 255, 256, 257, 8191, 8192, 8193, 65535, 65536, 65537, 1 << 20, 8191 * 8191]:
        assert rc.higher_msb(n) == oracle.higher_msb(n), n
    assert rc.tile_sort_shape(1) == (1, 1, 1)
    assert rc.tile_sort_shape(65535) == (16, 2, 8)
    assert rc.tile_sort_shape(65536) == (17, 3, 6)  # 65536 tiles already need a 17th bit
    assert rc.tile_sort_shape(8191 * 129) == (21, 3, 7)
    assert rc.tile_sort_shape(8191 * 8191) == (26, 4, 7)  # the largest frame the API accepts


def test_sort_sizes_straddle_the_kernel_boundaries():
    P = rc.SORT_SIZES
    assert P[0] == rc.SMALL_SORT and P[1] == rc.SMALL_SORT + 1  # radix_pass_kernel<8> / <16> for the depth sort
    assert -(-P[2] // rc.SCAN_BLOCK) > rc.SCAN_WINDOW + 1  # the scan's last block looks back past one 32-block window
    assert {p % rc.DEPTH_SORT_BLOCK for p in P[3:5]} == {1, rc.DEPTH_SORT_BLOCK - 1}
    assert {p % rc.SCAN_BLOCK for p in P[5:7]} == {1, rc.SCAN_BLOCK - 1}


@pytest.mark.parametrize("P", [rc.SMALL_SORT + 1, rc.SORT_SIZES[2]])
def test_sort_size_cases_are_mostly_visible(oracle, P):
    case = rc.sort_size(P)
    assert case.P == P
    sub = np.random.default_rng(0).choice(P, 50_000, replace=False)
    part = rc.Case(case.name, rc.cloud(case.cloud.xyz[sub], case.cloud.scaling[sub, 0], case.cloud.opacity[sub],
                                      np.full((len(sub), 3), 0.5)), case.vt, case.focal, case.tz)
    pre = rc.preprocess(oracle, part)
    assert (pre["radii"] > 0).mean() > 0.95


def test_depth_ties_have_one_view_depth(oracle):
    case = rc.depth_ties()
    pre = rc.preprocess(oracle, case)
    assert case.P >= 300 and (pre["radii"] > 0).all()
    assert np.unique(pre["depths"].view(np.uint32)).size == 1 and pre["depths"][0] == np.float32(3.0)
    assert np.unique(case.cloud.features.reshape(case.P, 3), axis=0).shape[0] == case.P  # distinct colours
    hits = rc.tile_hits(rc.tile_rects(pre["xy"], pre["radii"], case.W, case.H), case.W, case.H)
    assert hits.max() >= 250  # heavily overlapping


def test_depth_key_digit_patterns(oracle):
    shared = rc.keys_shared_upper()
    keys = rc.preprocess(oracle, shared)["depths"].view(np.uint32)
    assert np.unique(keys >> 8).size == 1 and np.unique(keys & 255).size == 256
    w = keys[: 16 * 32].reshape(16, 32)
    assert (w == w[:, :1]).all()  # 16 warps with one key: match-all in every pass
    spread = rc.keys_spread()
    pre = rc.preprocess(oracle, spread)
    assert (pre["radii"] > 0).mean() > 0.9
    keys = pre["depths"].view(np.uint32)
    for p in range(3):
        assert np.unique((keys >> (8 * p)) & 255).size == 256, p
    assert np.unique(keys >> 24).size >= 4


@pytest.mark.parametrize("W,H", rc.TILE_FRAMES)
def test_tile_frames_touch_first_and_last_tile(oracle, W, H):
    case = rc.tile_frame(W, H)
    gx, gy = rc.grid(W, H)
    pre = rc.preprocess(oracle, case)
    r = rc.tile_rects(pre["xy"], pre["radii"], W, H)
    vis = pre["radii"] > 0
    assert vis.mean() > 0.99
    first = (r[:, 0] == 0) & (r[:, 1] == 0) & vis
    last = (r[:, 2] == gx) & (r[:, 3] == gy) & vis
    assert first.any() and last.any()
    bits, passes, digit = rc.tile_sort_shape(gx * gy)
    assert passes * digit >= bits and passes <= 4
    if gx * gy <= 70_000:  # every tile column and row is covered
        assert set(np.concatenate([np.arange(a, b) for a, b in r[vis][:, [0, 2]]])) == set(range(gx))
        assert set(np.concatenate([np.arange(a, b) for a, b in r[vis][:, [1, 3]]])) == set(range(gy))
    if "x0_last" in case.info:
        idx = case.info["x0_last"]
        ex = rc.exact_rects(pre, W, H, idx)[idx]
        for rr in (r[idx], ex):
            assert (rr[:, 0] == 8190).all() and (rr[:, 2] == 8191).all()
            assert ((rr[:, 3] - rr[:, 1]) == 64).sum() >= 32
        assert (rc.rect_margin(pre["xy"][idx], pre["radii"][idx]) > 1e-3).sum() >= 32


def test_side_limit_frames():
    assert (rc.SIDE_LIMIT, 16) in rc.TILE_FRAMES and (16, rc.SIDE_LIMIT) in rc.TILE_FRAMES
    assert rc.grid(rc.SIDE_LIMIT, 16) == (8191, 1) and rc.grid(16, rc.SIDE_LIMIT) == (1, 8191)


def test_side_above_limit_is_refused(gsb_lib):
    from gs2mesh_b200 import _lib

    ptrs = {f: 256 for f in ("background", "means3D", "shs", "opacities", "scales", "rotations", "viewmatrix", "projmatrix",
                             "cam_pos", "out_color")}
    for W, H in ((rc.SIDE_LIMIT + 1, 16), (16, rc.SIDE_LIMIT + 1), (rc.SIDE_LIMIT + 1, rc.SIDE_LIMIT + 1)):
        a = _lib.GsbRasterArgs(P=10, sh_degree=0, sh_coeffs=1, width=W, height=H, scale_modifier=1.0, tan_fovx=0.5, tan_fovy=0.5,
                               flags=0, workspace=4096, workspace_bytes=1 << 40, max_instances=1000, **ptrs)
        assert gsb_lib.gsb_raster_forward(C.byref(a), None) == _lib.GSB_ERR_INVALID
        assert b"exceeds %d pixels" % rc.SIDE_LIMIT in gsb_lib.gsb_last_error()
        assert gsb_lib.gsb_raster_forward_pair(C.byref(a), C.byref(a), None, None) == _lib.GSB_ERR_INVALID


def test_rect_case_shapes(oracle):
    case = rc.rects(oracle)
    pre = rc.preprocess(oracle, case)
    W, H = case.W, case.H
    ref = rc.tile_rects(pre["xy"], pre["radii"], W, H)
    ex = rc.exact_rects(pre, W, H)
    sr, se = rc.rect_shape(ref), rc.rect_shape(ex)
    a_ref, a_ex = sr.prod(1), se.prod(1)
    assert (pre["radii"] > 0).all()
    full = case.info["full_masks"]
    assert list(full) == list(range(32))  # one whole warp
    for s in (sr, se):
        assert (s[full] == 8).all()  # 8 x 8 = 64 tiles in both modes
    mixed = np.arange(32, 64)
    for a in (a_ref, a_ex):
        assert (a[mixed[0::2]] > 64).all() and (a[mixed[1::2]] <= 4).all() and (a[mixed[1::2]] > 0).all()
    shapes = case.info["shapes"]
    for want in rc.RECT_SHAPES:
        hit = [i for i in shapes if tuple(sr[i]) == want and tuple(se[i]) == want]
        assert len(hit) >= 2, want
    assert {63, 64, 65} <= set(a_ref[shapes]) and (sr[shapes][:, 0] == 64).any()
    faint = case.info["faint"]
    assert (a_ref[faint] > 0).all() and (a_ex[faint] == 0).all()  # exact culling leaves nothing of them
    assert (rc.rect_margin(pre["xy"], pre["radii"])[: faint[0]] > 1e-3).all()


@pytest.mark.parametrize("W,H", rc.HIT_FRAMES)
def test_hit_count_tiles(oracle, W, H):
    case = rc.tile_hit_counts(W, H)
    assert W % 16 in (1, 8, 9, 15) and H % 16 in (1, 8, 9, 15)
    pre = rc.preprocess(oracle, case)
    assert (pre["radii"] > 0).all()
    r = rc.tile_rects(pre["xy"], pre["radii"], W, H)
    hits = rc.tile_hits(r, W, H)
    assert list(hits[: len(rc.HIT_COUNTS)]) == rc.HIT_COUNTS
    assert hits[-1] == 33
    own = case.info["tile_of"] < len(rc.HIT_COUNTS)
    assert (pre["tiles_touched"][own] == 1).all()
    assert (rc.rect_margin(pre["xy"], pre["radii"])[own] > 1e-3).all()
    # no pixel saturates: even the 65-Gaussian tile keeps T well above 1e-4 at its most covered pixel
    for t in range(len(rc.HIT_COUNTS) + 2):
        assert np.prod(1.0 - pre["conic_opacity"][case.info["tile_of"] == t, 3].astype(np.float64)) > 1e-3


def _centre(oracle, case):
    pre = rc.preprocess(oracle, case)
    assert (pre["xy"] == np.float32(8.0)).all()  # exactly on the centre pixel: power = 0, alpha = opacity
    assert np.unique(pre["depths"].view(np.uint32)).size == 1
    return pre


def test_alpha_threshold_stack(oracle):
    case = rc.alpha_threshold()
    _centre(oracle, case)
    a = case.info["centre_alphas"]
    assert a[0] < rc.ALPHA_MIN == a[1] < a[2]
    assert np.nextafter(a[0], np.float32(1)) == a[1] and np.nextafter(a[1], np.float32(1)) == a[2]
    T, k = rc.blend_pixel(a)
    assert k is None and T == np.float32(np.float32(1) - a[1]) * np.float32(np.float32(1) - a[2])


@pytest.mark.parametrize("k", rc.SATURATE_AT)
def test_saturation_stacks(oracle, k):
    case = rc.saturate_at(k)
    _centre(oracle, case)
    T, hit = rc.blend_pixel(case.info["centre_alphas"])
    assert hit == k and T >= rc.T_MIN
    if k > 2:  # 1e-4 sits well inside (T_k, T_{k-1}): a few ulp of alpha cannot move the crossing
        a = np.float64(case.info["centre_alphas"][0])
        assert (1 - a) ** (k - 1) > 1.05e-4 and (1 - a) ** k < 0.95e-4
