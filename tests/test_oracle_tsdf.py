"""Known-answer tests of the TSDF oracle (Open3D-0.17 restatement; parity unpinned, see
oracle/tsdf_oracle.cpp header).  KATs 6-9 of SURVEY.md section 8(c)."""
import os

import numpy as np
import pytest

W, H, FX, FY, CX, CY = 64, 48, 60.0, 60.0, 32.0, 24.0
VL, TRUNC = 1.0 / 64, 0.05


def _plane(d0):
    return np.full((H, W), d0, np.float32)


def _lookup(vol, p):
    """(tsdf, weight) of the voxel containing world point p, or None if its unit is not allocated."""
    idx = np.floor(np.asarray(p) / (16 * VL)).astype(int)
    units = vol.unit_indices()
    hit = np.where((units == idx).all(axis=1))[0]
    if len(hit) == 0:
        return None
    t, w, _ = vol.unit_data(int(hit[0]))
    loc = np.floor(np.asarray(p) / VL).astype(int) - idx * 16
    k = (loc[0] * 16 + loc[1]) * 16 + loc[2]
    return float(t[k]), float(w[k])


def test_fronto_parallel_plane_closed_form(oracle):
    d0 = 1.0
    vol = oracle.OracleTSDFVolume(VL, TRUNC, with_color=False)
    n = vol.integrate(_plane(d0), None, W, H, FX, FY, CX, CY, np.eye(4))
    assert n == vol.num_units and n > 0
    rng = np.random.default_rng(0)
    checked = 0
    for _ in range(400):
        z = rng.uniform(d0 - 0.06, d0 + 0.06)
        x, y = rng.uniform(-0.2, 0.2, 2) * z
        # voxel centre containing (x,y,z)
        c = (np.floor(np.array([x, y, z]) / VL) + 0.5) * VL
        got = _lookup(vol, c)
        if got is None:
            continue
        u = int(c[0] * FX / c[2] + CX + 0.5)
        v = int(c[1] * FY / c[2] + CY + 0.5)
        mult = np.sqrt(((u - CX) / FX) ** 2 + ((v - CY) / FY) ** 2 + 1)
        sdf = (d0 - c[2]) * mult
        if sdf > -TRUNC:
            assert got[1] == 1.0
            assert got[0] == pytest.approx(min(1.0, sdf / TRUNC), abs=2e-5)
            checked += 1
        else:
            assert got == (0.0, 0.0)
    assert checked > 50


def test_repeated_integration_keeps_tsdf_and_counts_weight(oracle):
    vol = oracle.OracleTSDFVolume(VL, TRUNC, with_color=True)
    rgb = np.full((H, W, 3), 200, np.uint8)
    for _ in range(3):
        vol.integrate(_plane(1.0), rgb, W, H, FX, FY, CX, CY, np.eye(4))
    t1 = oracle.OracleTSDFVolume(VL, TRUNC, with_color=False)
    t1.integrate(_plane(1.0), None, W, H, FX, FY, CX, CY, np.eye(4))
    for i in range(vol.num_units):
        t, w, c = vol.unit_data(i)
        t0, w0, _ = t1.unit_data(i)
        np.testing.assert_array_equal(w, 3 * w0)
        np.testing.assert_allclose(t, t0, atol=1e-6)
        np.testing.assert_allclose(c[w > 0], 200.0, atol=1e-9)


def test_depth_convert_scale_and_trunc(oracle):
    d = np.array([[0.5, 1.0, 2.0, 4.0]], np.float32)
    out = oracle.depth_convert(d, depth_scale=2.0, depth_trunc=1.0)
    np.testing.assert_array_equal(out, [[0.25, 0.5, 0.0, 0.0]])  # d/scale >= trunc -> 0 (>=, not >)


def test_zero_and_truncated_depth_contribute_nothing(oracle):
    vol = oracle.OracleTSDFVolume(VL, TRUNC, with_color=False)
    assert vol.integrate(np.zeros((H, W), np.float32), None, W, H, FX, FY, CX, CY, np.eye(4)) == 0
    assert vol.integrate(_plane(5.0), None, W, H, FX, FY, CX, CY, np.eye(4), depth_trunc=3.0) == 0
    assert vol.num_units == 0


def test_stride4_sampling_drives_allocation(oracle):
    """Only pixels with i,j = 0 mod 4 open volume units (depth_sampling_stride=4)."""
    d = np.zeros((H, W), np.float32)
    d[5, 7] = 1.0  # not on the stride-4 lattice
    vol = oracle.OracleTSDFVolume(VL, TRUNC, with_color=False)
    assert vol.integrate(d, None, W, H, FX, FY, CX, CY, np.eye(4)) == 0
    d[8, 12] = 1.0
    assert vol.integrate(d, None, W, H, FX, FY, CX, CY, np.eye(4)) > 0


def _rot_y(deg):
    a = np.radians(deg)
    e = np.eye(4)
    e[0, 0], e[0, 2], e[2, 0], e[2, 2] = np.cos(a), np.sin(a), -np.sin(a), np.cos(a)
    return e


def test_view_order_independence_and_merge_oracle_of_shards(oracle):
    """Fusing the views in another order, or in two shards merged by the multi-GPU merge's host restatement, opens the same
    units as sequential fusion, with bit-equal weights and tsdf within 1e-6."""
    from tests.merge_oracle import merge_oracle

    views = []
    for k, ang in enumerate([-8, -3, 4, 9]):
        e = _rot_y(ang)
        e[2, 3] = 0.1 * k
        views.append((_plane(1.0 + 0.01 * k), e))

    def fuse(order):
        """{(bx,by,bz): (tsdf, weight) [4096,2]} of every unit the views open."""
        vol = oracle.OracleTSDFVolume(VL, TRUNC, with_color=False)
        for i in order:
            vol.integrate(views[i][0], None, W, H, FX, FY, CX, CY, views[i][1])
        return {tuple(int(v) for v in k): np.stack(vol.unit_data(i)[:2], -1) for i, k in enumerate(vol.unit_indices())}

    def same(got, want):
        assert set(got) == set(want)
        for k in want:
            np.testing.assert_array_equal(got[k][:, 1], want[k][:, 1])
            np.testing.assert_allclose(got[k][:, 0], want[k][:, 0], atol=1e-6)

    seq = fuse([0, 1, 2, 3])
    same(fuse([2, 0, 3, 1]), seq)
    shards = [{k: (tw, None) for k, tw in fuse(order).items()} for order in ([0, 2], [1, 3])]
    merged = merge_oracle(shards, None, len(set(shards[0]) | set(shards[1])))[0].merged
    same({k: tw[0] for k, (tw, _) in merged.items()}, seq)  # two ranks: one candidate per voxel


def _blob_mask(rng, h, w):
    m = rng.random((h, w)) < 0.02
    yy, xx = np.mgrid[0:h, 0:w]
    m |= (yy - h * 0.5) ** 2 + (xx - w * 0.4) ** 2 < (0.3 * min(h, w)) ** 2
    m &= rng.random((h, w)) > 0.05  # pin holes that the closing must fill
    return m


def test_mask_morphology_matches_cv2(oracle):
    """oracle.mask_morphology / filter_object_mask vs OpenCV itself (the calls of tsdf_utils.py:73-77)."""
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(5)
    for (h, w), k in (((37, 53), 10), ((64, 64), 3), ((20, 90), 7), ((9, 9), 10), ((31, 17), 1), ((40, 40), 4)):
        m = _blob_mask(rng, h, w)
        kern = np.ones((k, k), np.uint8)
        np.testing.assert_array_equal(oracle.mask_morphology(m, k, True), cv2.dilate(m.astype(np.uint8), kern))
        np.testing.assert_array_equal(oracle.mask_morphology(m, k, False), cv2.erode(m.astype(np.uint8), kern, iterations=1))
        closing = cv2.morphologyEx(m.astype(np.uint8), cv2.MORPH_CLOSE, kern)
        want = cv2.erode(closing, kern, iterations=1) > 0.5
        np.testing.assert_array_equal(oracle.filter_object_mask(m, k, k), want)
    m = _blob_mask(rng, 48, 60)
    closing = cv2.morphologyEx((~m).astype(np.uint8), cv2.MORPH_CLOSE, np.ones((10, 10), np.uint8))
    np.testing.assert_array_equal(oracle.filter_object_mask(m, 10, 5, invert=True), cv2.erode(closing, np.ones((5, 5), np.uint8)) > 0.5)


# ---------------------------------------------------------------------------------------------------------------
# Fixture-backed pin against the REAL open3d==0.17.0 wheel (tests/golden/make_tsdf_golden.py writes the fixtures).
# open3d 0.17.0 publishes no wheel for Python 3.12, so these skip until somebody with the
# wheel runs the generator; GSB_TSDF_GOLDEN_DIR points the tests at a directory produced with `--backend oracle` to check
# the comparison code itself.
GOLDEN_DIR = os.environ.get("GSB_TSDF_GOLDEN_DIR", os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
GOLDEN_CASES = ["centred", "offcentre", "scaled_shifted"]


def _load_golden(case):
    path = os.path.join(GOLDEN_DIR, f"tsdf_o3d_{case}.npz")
    if not os.path.exists(path):
        pytest.skip("no open3d==0.17.0 fixture (0.17.0 publishes no Python 3.12 wheel) -- "
                    "TSDF parity stays unpinned until tests/golden/make_tsdf_golden.py has been run with the wheel")
    return np.load(path, allow_pickle=False)


def _sorted_rows(points, *cols, quantum):
    key = np.round(np.asarray(points) / quantum).astype(np.int64)
    order = np.lexsort((key[:, 2], key[:, 1], key[:, 0]))
    return (np.asarray(points)[order],) + tuple(np.asarray(c)[order] for c in cols)


@pytest.mark.parametrize("case", GOLDEN_CASES)
def test_open3d_golden_voxel_values(oracle, case):
    """extract_voxel_point_cloud() of the wheel == the restatement: same voxel set (block discovery T1, truncation band T2) and
    bit-identical tsdf values.  Settles the two DOUBT marks of oracle/tsdf_oracle.cpp (Eigen 4x4 * 4x1 summation order,
    sdf * (1/trunc))."""
    from tests.golden import make_tsdf_golden as g

    z = _load_golden(case)
    vol = g.oracle_volume(case, g.frames_from_npz(z))
    got = g.oracle_readback(case, vol)
    vl = g.CASES[case]["voxel"] / 512
    wp, wv = _sorted_rows(z["voxel_points"], z["voxel_tsdf01"], quantum=vl / 4)
    gp, gv = _sorted_rows(got["voxel_points"], got["voxel_tsdf01"], quantum=vl / 4)
    assert len(wp) == len(gp) and len(wp) > 1000
    np.testing.assert_allclose(gp, wp, rtol=0, atol=1e-9)
    np.testing.assert_array_equal(gv, wv)  # (tsdf + 1) / 2 in fp64 is exact for |tsdf| < 0.98: bit-identical tsdf


def test_golden_generator_inputs_are_reproducible():
    """The fixtures carry their inputs; the generator's seeded frames must reproduce them (runs without the wheel)."""
    from tests.golden import make_tsdf_golden as g

    for case in GOLDEN_CASES:
        a, b = g.make_frames(case), g.make_frames(case)
        assert all(np.array_equal(x["depth"], y["depth"]) and np.array_equal(x["rgb"], y["rgb"]) for x, y in zip(a, b))
        assert all((f["depth"] > 0).mean() > 0.15 for f in a)
        vol = g.oracle_volume(case, a)
        assert vol.num_units > 50
        if case == "scaled_shifted":  # scene centred at (5,-3,2) / TSDF_scale 0.1: units far from the origin
            assert np.abs(vol.unit_indices()).max() > 40


def _sphere_depth(w, h, fx, fy, cx, cy, pose_c2w, radius=0.8):
    """Metric z-depth of a sphere of `radius` at the world origin seen by a pinhole camera (0 where the ray misses)."""
    jj, ii = np.meshgrid(np.arange(w), np.arange(h))
    d_cam = np.stack([(jj - cx) / fx, (ii - cy) / fy, np.ones_like(jj, dtype=np.float64)], -1)
    R, t = pose_c2w[:3, :3], pose_c2w[:3, 3]
    d = d_cam @ R.T
    b = d @ t
    a = (d * d).sum(-1)
    disc = b * b - a * (t @ t - radius * radius)
    s = np.where(disc > 0, (-b - np.sqrt(np.maximum(disc, 0))) / a, 0.0)  # point = t + s * d, z_cam = s
    return np.where((disc > 0) & (s > 0), s, 0.0).astype(np.float32)


def test_doubt_sensitivity(oracle):
    """How much hangs on the two DOUBT points of the restatement (oracle/tsdf_oracle.cpp: the fp32 summation order of
    Eigen's 4x4 * 4x1 product, `sdf * (1/trunc)` vs `sdf / trunc`) while the Open3D wheel is unobtainable: the same three
    oblique views of a sphere fused under each alternative reading.  The unit set never changes (block discovery is fp64),
    a few voxels per million sit close enough to a decision boundary (truncation band, pixel rounding) to change their
    weight, and the values of all others move by at most a few ulp of a number in [-1, 1].  The numbers are printed for
    DESIGN.md section 5; the bounds asserted are ~10x what is observed."""
    w, h, fx, fy, cx, cy = 320, 240, 300.0, 300.0, 163.2, 117.9
    vl, trunc = 2.0 / 512, 0.04
    poses = []
    for k, (az, el) in enumerate([(0.3, 0.2), (1.7, -0.35), (3.9, 0.5)]):
        c = 2.4 * np.array([np.cos(el) * np.cos(az), np.cos(el) * np.sin(az), np.sin(el)])
        fwd = -c / np.linalg.norm(c)
        right = np.cross(fwd, [0.0, 0.0, 1.0])
        right /= np.linalg.norm(right)
        down = np.cross(fwd, right)
        pose = np.eye(4)
        pose[:3, 0], pose[:3, 1], pose[:3, 2], pose[:3, 3] = right, down, fwd, c
        poses.append(pose)

    def fuse(bits):
        oracle.tsdf_set_variant(bits)
        try:
            vol = oracle.OracleTSDFVolume(vl, trunc, with_color=False)
            for pose in poses:
                vol.integrate(_sphere_depth(w, h, fx, fy, cx, cy, pose), None, w, h, fx, fy, cx, cy, np.linalg.inv(pose), threads=8)
            units = vol.unit_indices()
            data = {tuple(int(v) for v in units[i]): vol.unit_data(i)[:2] for i in range(len(units))}
        finally:
            oracle.tsdf_set_variant(0)
        return data

    base = fuse(0)
    n_vox = sum(int((wt > 0).sum()) for _, wt in base.values())
    assert n_vox > 300_000
    report = {}
    for name, bits in (("pairwise_sum", 1), ("divide", 2), ("fma_product", 4), ("pairwise_sum+divide", 3)):
        alt = fuse(bits)
        assert set(alt) == set(base)  # the same volume units are opened
        flipped, jumped, worst = 0, 0, 0.0
        for key, (t0, w0) in base.items():
            t1, w1 = alt[key]
            same = w0 == w1
            flipped += int((~same).sum())  # in / out of the truncation band, the image, or the valid-depth mask
            both = same & (w0 > 0)
            diff = np.abs(t0[both] - t1[both])
            jumped += int((diff > 1e-4).sum())  # same weight, but some view sampled the neighbouring pixel
            if (diff <= 1e-4).any():
                worst = max(worst, float(diff[diff <= 1e-4].max()))
        report[name] = dict(weight_changed=flipped, other_pixel=jumped, worst_rounding=worst)
        assert flipped + jumped <= 3e-5 * n_vox, (name, flipped, jumped, n_vox)  # observed <= 2.7e-6
        assert worst <= 5e-5, (name, worst)  # observed 6.4e-6
    print("DOUBT sensitivity over %d updated voxels: %s" % (n_vox, report))
    # `divide` alone cannot change which pixel or which voxels a view updates, only the value
    assert report["divide"]["weight_changed"] == 0 and report["divide"]["other_pixel"] == 0
