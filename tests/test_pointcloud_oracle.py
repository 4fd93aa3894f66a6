"""The point-cloud oracle (tests/pointcloud_oracle.py, the restatement of Open3D's ExtractPointCloud and
ExtractVoxelPointCloud) on volumes whose answers are known in closed form."""
import numpy as np
import pytest

from tests.pointcloud_oracle import _tsdf_at, extract_point_cloud_from_bricks, extract_voxel_point_cloud_from_bricks

VL = 2.0 / 512
NB = (2, 2, 2)  # brick (0,0,0) and its +1 neighbours


def _window(voxels, color=None, allocated=((0, 0, 0),)):
    """Dense window over bricks [0,2)^3 with the given {(gx,gy,gz): (tsdf, weight)}; everything else weight 0."""
    tw = np.zeros((8, 4096, 2), np.float32)
    col = np.zeros((8, 4096, 3), np.float32)
    for (gx, gy, gz), (f, w) in voxels.items():
        b = ((gx >> 4) * 2 + (gy >> 4)) * 2 + (gz >> 4)
        i = ((gx & 15) * 16 + (gy & 15)) * 16 + (gz & 15)
        tw[b, i] = (f, w)
        if color is not None and (gx, gy, gz) in color:
            col[b, i] = color[(gx, gy, gz)]
    alloc = np.zeros(NB, bool)
    for b in allocated:
        alloc[b] = True
    return tw, col, alloc


def _key(g, axis):
    return ((g[0] * 32 + g[1]) * 32 + g[2]) * 3 + axis


def test_one_crossing_has_the_closed_form_point_and_colour():
    tw, col, alloc = _window({(3, 4, 5): (-0.25, 1.0), (4, 4, 5): (0.75, 2.0)},
                             color={(3, 4, 5): (255.0, 0.0, 51.0), (4, 4, 5): (0.0, 255.0, 51.0)})
    r = extract_point_cloud_from_bricks(tw, (0, 0, 0), NB, VL, color=col, allocated=alloc)
    assert r["keys"].tolist() == [_key((3, 4, 5), 0)]
    # x = (3.5 vl * 0.75 + 4.5 vl * 0.25) / 1 = 3.75 vl; every value here is dyadic, so exact
    np.testing.assert_array_equal(r["points"], [[3.75 * VL, 4.5 * VL, 5.5 * VL]])
    np.testing.assert_array_equal(r["colors"], [[0.75, 0.25, float(np.float32(0.2))]])  # a float32 quotient, widened
    assert r["points"].dtype == np.float64 and r["colors"].dtype == np.float64


@pytest.mark.parametrize("sign", [1, -1], ids=["rising", "falling"])
@pytest.mark.parametrize("axis", [0, 1, 2])
def test_planar_tsdf_gives_axis_normals_and_points_on_the_plane(axis, sign):
    f = sign * ((np.arange(16, dtype=np.float32) - np.float32(7)) * np.float32(0.25) - np.float32(0.125))
    shape = [1, 1, 1]
    shape[axis] = 16
    t = np.broadcast_to(np.clip(f, -0.9, 0.9).reshape(shape), (16, 16, 16))
    tw = np.zeros((8, 4096, 2), np.float32)
    tw[0, :, 0], tw[0, :, 1] = t.reshape(-1), 1.0
    alloc = np.zeros(NB, bool)
    alloc[0, 0, 0] = True
    r = extract_point_cloud_from_bricks(tw, (0, 0, 0), NB, VL, allocated=alloc)
    assert len(r["keys"]) == 256 and (r["keys"] % 3 == axis).all()
    want = np.zeros(3)
    want[axis] = sign
    np.testing.assert_array_equal(r["normals"], np.tile(want, (256, 1)))
    np.testing.assert_array_equal(r["points"][:, axis], np.full(256, 8.0 * VL))  # tsdf 0 halfway between voxels 7 and 8


@pytest.mark.parametrize("f0, f1, emitted", [
    (np.float32(0.98), np.float32(-0.5), False),              # f0 < 0.98f fails
    (np.nextafter(np.float32(0.98), np.float32(0)), np.float32(-0.5), True),  # 0.98f - ulp passes
    (np.float32(-0.98), np.float32(0.5), True),               # f >= -0.98f passes at -0.98f
    (np.nextafter(np.float32(-0.98), np.float32(-1)), np.float32(0.5), False),
    (np.float32(0.5), np.float32(-0.98), True),
    (np.float32(0.5), np.float32(0.98), False),
])
def test_predicate_at_plus_minus_0_98(f0, f1, emitted):
    tw, _, alloc = _window({(2, 2, 2): (f0, 1.0), (2, 2, 3): (f1, 1.0)})
    r = extract_point_cloud_from_bricks(tw, (0, 0, 0), NB, VL, allocated=alloc)
    assert r["keys"].tolist() == ([_key((2, 2, 2), 2)] if emitted else [])


@pytest.mark.parametrize("w0, w1", [(0.0, 1.0), (1.0, 0.0)])
def test_weight_zero_on_either_end_suppresses_the_point(w0, w1):
    tw, _, alloc = _window({(2, 2, 2): (-0.5, w0), (2, 3, 2): (0.5, w1)})
    assert len(extract_point_cloud_from_bricks(tw, (0, 0, 0), NB, VL, allocated=alloc)["keys"]) == 0


def test_underflowing_product_emits_nothing():
    tiny = np.float32(1e-30)
    assert tiny * -tiny == 0 and np.signbit(tiny * -tiny)  # -0 in float32
    tw, _, alloc = _window({(2, 2, 2): (tiny, 1.0), (3, 2, 2): (-tiny, 1.0), (5, 5, 5): (np.float32(1e-20), 1.0),
                            (5, 5, 6): (np.float32(-1e-10), 1.0)})
    r = extract_point_cloud_from_bricks(tw, (0, 0, 0), NB, VL, allocated=alloc)
    assert r["keys"].tolist() == [_key((5, 5, 5), 2)]  # 1e-30 float product still > float32 min subnormal


def test_zero_gradient_gives_a_zero_normal():
    """A lone crossing in an otherwise unobserved (tsdf 0) brick, with f0 = -f1: the samples are symmetric about the
    crossing, and every difference is exactly 0."""
    tw, _, alloc = _window({(7, 7, 7): (-0.5, 1.0), (8, 7, 7): (0.5, 1.0)})
    r = extract_point_cloud_from_bricks(tw, (0, 0, 0), NB, VL, allocated=alloc)
    assert len(r["keys"]) == 1
    n = r["normals"][0]
    assert n[1] == 0 and n[2] == 0 and n[0] > 0  # the x gradient is real
    # a constant field: every voxel of the brick observed with the same tsdf apart from the crossing's two
    vox = {(x, y, z): (0.25, 1.0) for x in range(16) for y in range(16) for z in range(16)}
    vox[(7, 7, 7)] = (-0.25, 1.0)
    tw, _, alloc = _window(vox)
    f = tw[0, :, 0].reshape(16, 16, 16)
    full = np.zeros((32, 32, 32), np.float32)
    full[:16, :16, :16] = f
    p = np.array([[8.0 * VL, 7.5 * VL, 7.5 * VL]])
    a = _tsdf_at(full, alloc, (0, 0, 0), NB, VL, p + [[0, 0, 0.99 * VL]])
    b = _tsdf_at(full, alloc, (0, 0, 0), NB, VL, p - [[0, 0, 0.99 * VL]])
    assert a == b
    # nothing at all around: a (0,0,0) normal, returned unchanged by normalized()
    tw, _, alloc = _window({(0, 0, 0): (-0.5, 1.0), (0, 0, 1): (0.5, 1.0)}, allocated=())
    r = extract_point_cloud_from_bricks(tw, (0, 0, 0), NB, VL, allocated=alloc)
    np.testing.assert_array_equal(r["normals"], [[0.0, 0.0, 0.0]])


def test_every_surface_point_lies_on_its_voxel_edge():
    """Up to the float32 sum r0 + r1 in the denominator: (p0 r1 + p1 r0) / (r0 + r1) scales the whole point by
    (r0 + r1 exact) / (r0 + r1 rounded), a relative error of at most 2^-24 -- far from the origin (z ~ 2^19 units here)
    that moves a point off its edge by much more than the edge's own rounding."""
    rng = np.random.default_rng(3)
    tw = np.zeros((8, 4096, 2), np.float32)
    tw[:, :, 0] = rng.uniform(-1, 1, (8, 4096))
    tw[:, :, 1] = np.where(rng.random((8, 4096)) < 0.1, 0, 1)
    alloc = np.ones(NB, bool)
    b0 = np.array([-3, 5, 1 << 19])
    for vl in (2.0 / 512, 0.3 / 512, 0.2 / 512):
        r = extract_point_cloud_from_bricks(tw, b0, NB, vl, allocated=alloc)
        assert len(r["keys"]) > 10000 and (np.diff(r["keys"]) > 0).all()
        axis = r["keys"] % 3
        v = r["keys"] // 3
        g = np.stack([v // 1024, (v // 32) % 32, v % 32], 1)
        p0 = (vl * 0.5 + vl * (g & 15)) + (b0 + (g >> 4)) * (vl * 16)
        tol = 2.0 ** -23 * (np.abs(p0) + vl)
        rows = np.arange(len(axis))
        off = r["points"] - p0
        on_axis, tol_axis = off[rows, axis], tol[rows, axis]
        assert (on_axis >= -tol_axis).all() and (on_axis <= vl + tol_axis).all()
        off[rows, axis] = 0
        assert (np.abs(off) <= tol).all()  # the other two coordinates stay on the voxel's lines
        assert np.isfinite(r["normals"]).all()


def test_voxel_cloud_grey_is_half_of_tsdf_plus_one():
    rng = np.random.default_rng(4)
    tw = np.zeros((8, 4096, 2), np.float32)
    tw[:, :, 0] = rng.uniform(-1.2, 1.2, (8, 4096))
    tw[:, :, 1] = np.where(rng.random((8, 4096)) < 0.2, 0, 1)
    r = extract_voxel_point_cloud_from_bricks(tw, (4, -2, 7), NB, VL)
    f = tw[..., 0].reshape(2, 2, 2, 16, 16, 16).transpose(0, 3, 1, 4, 2, 5).reshape(32, 32, 32)
    w = tw[..., 1].reshape(2, 2, 2, 16, 16, 16).transpose(0, 3, 1, 4, 2, 5).reshape(32, 32, 32)
    sel = (w != 0) & (f < np.float32(0.98)) & (f >= np.float32(-0.98))
    np.testing.assert_array_equal(r["keys"], np.flatnonzero(sel))
    want = (f[sel].astype(np.float64) + 1.0) / 2.0
    np.testing.assert_array_equal(r["colors"], np.stack([want] * 3, 1))
    assert (r["colors"] >= 0.01 - 1e-12).all() and (r["colors"] < 0.99).all()
