"""GPU point-cloud extraction (gsb_pcd_*, mesh.extract_point_cloud / extract_voxel_point_cloud) vs the numpy restatement
of Open3D's ExtractPointCloud / ExtractVoxelPointCloud (tests/pointcloud_oracle.py), bit for bit: keys, points, colours
and normals.

The volumes are written brick by brick, like the mesh tests' (tests/test_gpu_mesh_volumes.py): crossings on every axis
inside a brick and across each +face with the neighbour present and absent, normal samples reaching into -1 / +1 bricks
and into missing ones, tsdf values of +-0, subnormals and +-0.98, lattice indices far from the origin (where the per-unit
position formula differs from the global one) and at the ends of the 21-bit brick key, and voxel lengths that are not
dyadic.  Fused scenes come from the TSDF frame tests' ray-cast sphere."""
import numpy as np
import pytest

from tests.pointcloud_oracle import extract_point_cloud_from_bricks, extract_voxel_point_cloud_from_bricks
from tests.test_gpu_mesh_volumes import _brick

pytestmark = pytest.mark.gpu

VOXEL_LENGTHS = (2.0 / 512, 0.3 / 512, 0.1 * 2.0 / 512)
TOP = (1 << 20) - 1  # the largest brick lattice index


@pytest.fixture
def brick_volume(cuda_device):
    """units {(bx,by,bz): (tsdf_weight [4096,2], colour [4096,3] | None)} -> a TSDFVolume holding exactly those bricks."""
    import torch

    from gs2mesh_b200.tsdf import TSDFVolume

    def make(units, voxel_length, with_color):
        vol = TSDFVolume(voxel_length, 4 * voxel_length, (0, 0, 0), (1, 1, 1), with_color=with_color, device=cuda_device,
                         pool_bricks=max(64, len(units)))
        if units:
            slots = vol.find_bricks(np.array(list(units), np.int32), insert=True).long()
            assert (slots >= 0).all() and len(set(slots.tolist())) == len(units)
            vol.pool()[slots] = torch.from_numpy(np.stack([u[0] for u in units.values()])).to(cuda_device)
            if with_color:
                col = np.zeros((len(units), 4096, 4), np.float32)
                col[..., :3] = np.stack([u[1] for u in units.values()])
                vol.color.view(vol.pool_bricks, 4096, 4)[slots] = torch.from_numpy(col).to(cuda_device)
        assert vol.num_bricks() == len(units)
        torch.cuda.synchronize()
        return vol

    return make


def _window(units):
    idx = np.array(list(units), np.int64)
    lo, hi = idx.min(0), idx.max(0)
    return tuple(int(v) for v in lo), tuple(int(v) for v in hi - lo + 2)


def _dense(units, b0, nb):
    """(tsdf_weight, colour, allocated) of the window [b0, b0 + nb): row-major over (bx,by,bz), missing bricks zero."""
    total = int(np.prod(nb))
    tw = np.zeros((total, 4096, 2), np.float32)
    col = np.zeros((total, 4096, 3), np.float32)
    alloc = np.zeros(total, bool)
    for (bx, by, bz), (t, c) in units.items():
        r = (bx - b0[0], by - b0[1], bz - b0[2])
        if all(0 <= r[k] < nb[k] for k in range(3)):
            i = (r[0] * nb[1] + r[1]) * nb[2] + r[2]
            tw[i], alloc[i] = t, True
            if c is not None:
                col[i] = np.asarray(c)[:, :3]
    return tw, col, alloc


def _rekey(pcd, b0, nb, surface=True):
    """pcd.keys (inside pcd.key_window) re-expressed inside window (b0, nb), and which of them fall inside it."""
    (k0, kn) = pcd.key_window
    key = pcd.keys.astype(np.int64)
    axis, lin = (key % 3, key // 3) if surface else (0, key)
    ny, nz = kn[1] * 16, kn[2] * 16
    g = np.stack([lin // (nz * ny), (lin // nz) % ny, lin % nz], 1) + (np.array(k0) - np.array(b0)) * 16
    n = np.array(nb) * 16
    sel = ((g >= 0) & (g < n)).all(1)
    lin = (g[:, 0] * n[1] + g[:, 1]) * n[2] + g[:, 2]
    return (lin * 3 + axis if surface else lin)[sel], sel


def _compare(pcd, units, vl, with_color, b0=None, nb=None, with_normals=True):
    """The surface cloud inside window (b0, nb) (default: all of `units`) equals the oracle's; returns its size."""
    if b0 is None:
        b0, nb = _window(units)
    tw, col, alloc = _dense(units, b0, nb)
    ref = extract_point_cloud_from_bricks(tw, b0, nb, vl, color=col if with_color else None, allocated=alloc,
                                          with_normals=with_normals)
    keys, sel = _rekey(pcd, b0, nb)
    np.testing.assert_array_equal(keys, ref["keys"])
    assert pcd.points.dtype == np.float64
    np.testing.assert_array_equal(pcd.points[sel], ref["points"])
    if with_color:
        np.testing.assert_array_equal(pcd.colors[sel], ref["colors"])
    else:
        assert pcd.colors is None
    if with_normals:
        np.testing.assert_array_equal(pcd.normals[sel], ref["normals"])
    else:
        assert pcd.normals is None
    return len(keys)


def _compare_voxels(vox, units, vl, b0=None, nb=None):
    if b0 is None:
        b0, nb = _window(units)
    tw, _, _ = _dense(units, b0, nb)
    ref = extract_voxel_point_cloud_from_bricks(tw, b0, nb, vl)
    keys, sel = _rekey(vox, b0, nb, surface=False)
    np.testing.assert_array_equal(keys, ref["keys"])
    np.testing.assert_array_equal(vox.points[sel], ref["points"])
    np.testing.assert_array_equal(vox.colors[sel], ref["colors"])
    assert vox.normals is None
    return len(keys)


def _surface(vol, **kw):
    from gs2mesh_b200.mesh import extract_point_cloud

    return extract_point_cloud(vol, **kw)


def _voxels(vol):
    from gs2mesh_b200.mesh import extract_voxel_point_cloud

    return extract_voxel_point_cloud(vol)


def _crossing_rich(rng, shape=(16, 16, 16)):
    """tsdf in (-0.97, 0.97) with random signs: most edges are crossings."""
    return (rng.uniform(0.02, 0.97, shape) * rng.choice([-1.0, 1.0], shape)).astype(np.float32)


# ------------------------------------------------------------------------------------------------- brick-built volumes

def test_every_axis_and_face_in_a_block_of_bricks(gsb_lib, brick_volume):
    """3x3x3 bricks: crossings on all three axes inside bricks and across every +face, normal samples reaching into the
    -1 and +1 bricks on every side, and (on the block's outer faces) into missing bricks."""
    rng = np.random.default_rng(1)
    units = {(bx, by, bz): _brick(rng, _crossing_rich(rng)) for bx in (-1, 0, 1) for by in (-1, 0, 1) for bz in (-1, 0, 1)}
    vl = 0.3 / 512
    pcd = _surface(brick_volume(units, vl, True))
    n = _compare(pcd, units, vl, True)
    assert n > 100000
    axis = pcd.keys % 3
    g = (pcd.keys // 3)
    gz = g % (4 * 16)
    gy = (g // (4 * 16)) % (4 * 16)
    gx = g // (4 * 16 * 4 * 16)
    for k, c in enumerate((gx, gy, gz)):
        assert ((axis == k) & (c % 16 == 15)).sum() > 100  # across a +face
        assert ((axis == k) & (c % 16 < 15)).sum() > 1000
    vox = _voxels(brick_volume(units, vl, True))
    assert _compare_voxels(vox, units, vl) > 50000


NEIGHBOURS = [(1, 0, 0), (0, 1, 0), (0, 0, 1)]


@pytest.mark.parametrize("absent", NEIGHBOURS, ids=["absent_x", "absent_y", "absent_z"])
def test_missing_neighbour_and_weight0_face(gsb_lib, brick_volume, absent):
    """One +1 neighbour of brick (0,0,0) is a hash miss (no crossings across that face, zero samples there); the present
    ones have weight 0 on a third of their facing plane."""
    rng = np.random.default_rng(10 + NEIGHBOURS.index(absent))
    units = {(0, 0, 0): _brick(rng, _crossing_rich(rng))}
    for d in NEIGHBOURS + [(1, 1, 0), (0, 1, 1), (1, 0, 1), (1, 1, 1)]:
        if d == absent:
            continue
        tw, col = _brick(rng, _crossing_rich(rng))
        t = tw.reshape(16, 16, 16, 2)
        t[..., 1][(rng.random((16, 16, 16)) < 1 / 3)] = 0.0
        units[d] = (tw, col)
    vl = 2.0 / 512
    assert _compare(_surface(brick_volume(units, vl, True)), units, vl, True) > 10000


SPECIAL = np.array([0.0, -0.0, 0.98, -0.98, 0.97999996, -0.97999996, 0.5, -0.5, 0.25, -0.25, 1e-45, -1e-45, 3e-39, -3e-39,
                    1e-20, -1e-20, 1.2e-38, -1.2e-38, 0.1, -0.7], np.float32)


def _special_units(rng, with_color=True):
    """2x2x2 bricks of tsdf drawn from signed zeros, +-0.98 and the float below it, equal magnitudes and subnormals
    (whose products underflow to +-0); 5% weight 0."""
    units = {}
    for b in [(bx, by, bz) for bx in (0, 1) for by in (-1, 0) for bz in (3, 4)]:
        t = SPECIAL[rng.integers(0, len(SPECIAL), (16, 16, 16))]
        w = np.where(rng.random((16, 16, 16)) < 0.05, 0.0, rng.integers(1, 4, (16, 16, 16))).astype(np.float32)
        units[b] = _brick(rng, t, w, with_color)
    return units


@pytest.mark.parametrize("with_color", [True, False], ids=["color", "nocolor"])
@pytest.mark.parametrize("vl", VOXEL_LENGTHS, ids=["vl2", "vl0.3", "vl0.2"])
def test_special_tsdf_values(gsb_lib, brick_volume, vl, with_color):
    rng = np.random.default_rng(20)
    units = _special_units(rng, with_color)
    vol = brick_volume(units, vl, with_color)
    assert _compare(_surface(vol), units, vl, with_color) > 5000
    assert _compare_voxels(_voxels(vol), units, vl) > 10000


def test_colour_and_normals_can_be_left_out(gsb_lib, brick_volume):
    rng = np.random.default_rng(21)
    units = _special_units(rng, True)
    vl = 2.0 / 512
    vol = brick_volume(units, vl, True)
    full = _surface(vol)
    bare = _surface(vol, with_colors=False, with_normals=False)
    assert _compare(bare, units, vl, False, with_normals=False) > 5000
    np.testing.assert_array_equal(bare.points, full.points)
    with pytest.raises(ValueError, match="no colour"):
        _surface(brick_volume(units, vl, False), with_colors=True)


CLUSTERS = {
    # negative indices near the origin + a cluster near (-70000, 3, 2^20 - 2) that reaches the last brick index on z
    "far": [[(bx, by, bz) for bx in (-2, -1) for by in (-1, 0) for bz in (-3, -2)],
            [(bx, by, bz) for bx in (-70000, -69999) for by in (3, 4) for bz in (TOP - 1, TOP)]],
    # both ends of the z lattice: the key window is 2^21 + 1 bricks long
    "lattice_ends": [[(7, -5, -(1 << 20)), (7, -5, -(1 << 20) + 1)], [(7, -5, TOP - 1), (8, -5, TOP)]],
}


@pytest.mark.parametrize("vl", VOXEL_LENGTHS[1:], ids=["vl0.3", "vl0.2"])
@pytest.mark.parametrize("name", sorted(CLUSTERS))
def test_far_apart_clusters(gsb_lib, brick_volume, name, vl):
    """Bricks far from the origin and at the ends of the brick key range, compared cluster by cluster.  Far out the
    per-unit position vl/2 + vl*x + index0*U and the global vl/2 + vl*(16*index0 + x) differ in the last bits; the
    points must be the per-unit ones."""
    rng = np.random.default_rng(30)
    clusters = [{b: _brick(rng, _crossing_rich(rng)) for b in c} for c in CLUSTERS[name]]
    units = {k: v for c in clusters for k, v in c.items()}
    pcd = _surface(brick_volume(units, vl, True))
    n = [_compare(pcd, units, vl, True, *_window(c)) for c in clusters]
    assert min(n) > 1000 and sum(n) == len(pcd.points)
    # the same points with the global position vl/2 + vl*(16*index0 + x) instead: different bits far out
    for c in clusters:
        b0, nb = _window(c)
        tw, _, _ = _dense(units, b0, nb)
        keys, sel = _rekey(pcd, b0, nb)
        assert not np.array_equal(pcd.points[sel], _global_points(tw, b0, nb, vl, keys))


def _global_points(tw, b0, nb, vl, keys):
    """(p0 r1 + p1 r0) / (r0 + r1) of the given keys with p0 = vl/2 + vl*(16*index0 + x), the mesh vertices' formula."""
    n = np.array(nb) * 16
    f = np.pad(tw[..., 0].reshape(*nb, 16, 16, 16).transpose(0, 3, 1, 4, 2, 5).reshape(n), ((0, 1),) * 3)
    axis, lin = keys % 3, keys // 3
    g = np.stack([lin // (n[1] * n[2]), (lin // n[2]) % n[1], lin % n[2]], 1)
    r0 = np.abs(f[tuple(g.T)])
    r1 = np.abs(f[tuple((g + np.eye(3, dtype=np.int64)[axis]).T)])
    p0 = vl * 0.5 + vl * (g + np.array(b0) * 16).astype(np.float64)
    p1 = p0.copy()
    p1[np.arange(len(keys)), axis] += vl
    return (p0 * r1.astype(np.float64)[:, None] + p1 * r0.astype(np.float64)[:, None]) / (r0 + r1).astype(np.float64)[:, None]


@pytest.mark.parametrize("kind", ["no_bricks", "zero_weight", "all_inside", "all_outside", "signed_zeros", "beyond_0_98"])
def test_empty_clouds(gsb_lib, brick_volume, kind):
    rng = np.random.default_rng(40)
    blocks = [(bx, by, bz) for bx in (0, 1) for by in (0, 1) for bz in (0, 1)]
    tsdf = {"zero_weight": None, "all_inside": -0.5, "all_outside": 0.5,
            "signed_zeros": np.where(rng.random((16, 16, 16)) < 0.5, np.float32(0.0), np.float32(-0.0)),
            "beyond_0_98": np.where(rng.random((16, 16, 16)) < 0.5, np.float32(0.98), np.float32(-1.0))}
    units = {} if kind == "no_bricks" else {b: _brick(rng, tsdf[kind], 0.0 if kind == "zero_weight" else 1.0) for b in blocks}
    vol = brick_volume(units, 2.0 / 512, True)
    pcd = _surface(vol)
    assert pcd.points.shape == (0, 3) and pcd.colors.shape == (0, 3) and pcd.normals.shape == (0, 3)
    assert not pcd.has_colors() and not pcd.has_normals()
    vox = _voxels(vol)
    want = {"no_bricks": 0, "zero_weight": 0, "beyond_0_98": 0}.get(kind, 8 * 4096)
    assert vox.points.shape == (want, 3) and vox.colors.shape == (want, 3)


def test_key_window_limit_is_a_clear_error(gsb_lib, brick_volume):
    from gs2mesh_b200 import _lib

    rng = np.random.default_rng(50)
    units = {(0, 0, 0): _brick(rng), (1 << 17, 1 << 17, 1 << 17): _brick(rng)}
    vol = brick_volume(units, 2.0 / 512, True)
    for extract in (_surface, _voxels):
        with pytest.raises(_lib.GsbError, match=r"pcd_count: .* too large for 63-bit edge keys \(16\^3 \* nbx \* nby \* nbz \* 3 "
                                                r"must be < 9e18\)"):
            extract(vol)


def test_bad_arguments_are_refused(gsb_lib, brick_volume):
    import ctypes as C

    from gs2mesh_b200 import _lib

    vol = brick_volume({(0, 0, 0): _brick(np.random.default_rng(51))}, 2.0 / 512, False)
    L = _lib.lib()
    w = (C.c_int32 * 6)(0, 0, 0, 2, 2, 2)
    assert L.gsb_pcd_count(vol._h, w, None, 0, 2, None, None) == _lib.GSB_ERR_INVALID  # mode
    assert L.gsb_pcd_points(vol._h, w, None, 0, _lib.GSB_PCD_VOXELS, None, None, C.c_void_p(8), None) == _lib.GSB_ERR_INVALID
    assert L.gsb_pcd_points(vol._h, w, None, 0, _lib.GSB_PCD_SURFACE, None, C.c_void_p(8), None, None) == _lib.GSB_ERR_INVALID
    assert L.gsb_pcd_points(vol._h, w, None, -1, _lib.GSB_PCD_SURFACE, None, None, None, None) == _lib.GSB_ERR_INVALID


# ------------------------------------------------------------------------------------------------------- fused scenes

def _fused(dev, vl):
    """A sphere seen by three cameras, fused (no background: the key window stays the sphere's bounding box); lengths
    scale with vl so that every voxel length opens about the same bricks."""
    from tests.test_gpu_tsdf_frames import _frame, _look_at, _raycast, _volume

    s = vl / (2.0 / 512)
    W, H, fx, fy = 96, 80, 90.0, 90.0
    vol = _volume(dev, vl, 4 * vl)
    for pos in [(0.0, -1.0, 0.3), (0.8, -0.7, 0.5), (-0.7, -0.8, 0.1)]:
        w2c = _look_at(np.array(pos) * s, (0.0, 0.0, 0.0))
        depth = _raycast(W, H, fx, fy, W / 2, H / 2, w2c, (0.0, 0.0, 0.0), 0.25 * s)
        f = _frame(depth, W, H, fx, fy, W / 2, H / 2, w2c)
        vol.integrate(vol.prepare_depth(f["depth"], W, H), f["rgb"], W, H, *f["K"], f["w2c"])
    assert vol.pool_stats()["dropped"] == 0 and np.prod(_window(vol.export_units())[1]) < 4096
    return vol


@pytest.mark.parametrize("vl", [2.0 / 512, 0.3 / 512], ids=["vl2", "vl0.3"])
def test_fused_scene(gsb_lib, cuda_device, vl):
    vol = _fused(cuda_device, vl)
    units = vol.export_units()
    pcd = _surface(vol)
    assert _compare(pcd, units, vl, True) > 1000
    nz = (pcd.normals != 0).any(1)
    assert nz.sum() > 1000 and np.abs(np.linalg.norm(pcd.normals[nz], axis=1) - 1).max() < 1e-12
    again = _surface(vol)  # the same arrays on every run
    for a in ("keys", "points", "colors", "normals"):
        np.testing.assert_array_equal(getattr(again, a), getattr(pcd, a))
    assert _compare_voxels(_voxels(vol), units, vl) > 1000


def test_stage_cloud_is_scaled_like_the_mesh(gsb_lib, cuda_device):
    from types import SimpleNamespace

    from gs2mesh_b200.mesh import extract_point_cloud
    from gs2mesh_b200.tsdf import TSDF

    vol = _fused(cuda_device, 2.0 / 512)
    stage = TSDF(None, None, SimpleNamespace(TSDF_scale=0.1), "scene", device=cuda_device)
    stage.volume = vol
    got = stage.extract_point_cloud()
    raw = extract_point_cloud(vol)
    np.testing.assert_array_equal(got.points, (raw.points - 0.0) * 0.1 + 0.0)
    np.testing.assert_array_equal(got.normals, raw.normals)
    np.testing.assert_array_equal(got.colors, raw.colors)


def test_facade_and_ply_round_trip(gsb_lib, cuda_device, tmp_path):
    import gs2mesh_b200.o3d_compat as o3d
    from gs2mesh_b200.io import read_point_cloud_ply
    from gs2mesh_b200.mesh import extract_point_cloud, extract_voxel_point_cloud

    vl = 2.0 / 512
    volume = o3d.pipelines.integration.ScalableTSDFVolume(voxel_length=vl, sdf_trunc=4 * vl,
                                                          color_type=o3d.pipelines.integration.TSDFVolumeColorType.RGB8,
                                                          device=cuda_device)
    volume._vol = _fused(cuda_device, vl)
    pcd = volume.extract_point_cloud()
    assert isinstance(pcd, o3d.geometry.PointCloud) and pcd.has_colors() and pcd.has_normals()
    ref = extract_point_cloud(volume._vol)
    for a in ("points", "colors", "normals"):
        np.testing.assert_array_equal(getattr(pcd, a), getattr(ref, a))
    vox = volume.extract_voxel_point_cloud()
    vref = extract_voxel_point_cloud(volume._vol)
    np.testing.assert_array_equal(vox.points, vref.points)
    np.testing.assert_array_equal(vox.colors, vref.colors)
    assert not vox.has_normals()
    path = str(tmp_path / "cloud.ply")
    assert o3d.io.write_point_cloud(path, pcd)
    np.testing.assert_array_equal(read_point_cloud_ply(path), pcd.points)


def test_cloud_contains_the_mesh_vertices_it_should(gsb_lib, cuda_device):
    """Every mesh vertex whose edge has two end voxels that pass the point predicate is a point of the surface cloud
    (same key space) and lies close to it.  The two formulas interpolate the same edge but differ in operation order,
    and the cloud divides by the float32 sum r0 + r1, which scales the point by up to 2^-24 relative."""
    from gs2mesh_b200.mesh import extract_triangle_mesh

    vl = 0.3 / 512
    vol = _fused(cuda_device, vl)
    mesh, pcd = extract_triangle_mesh(vol), _surface(vol)
    assert mesh.key_window == pcd.key_window
    b0, nb = pcd.key_window
    tw, _, _ = _dense(vol.export_units(), b0, nb)
    n = np.array(nb) * 16
    f = tw[..., 0].reshape(*nb, 16, 16, 16).transpose(0, 3, 1, 4, 2, 5).reshape(n)
    w = tw[..., 1].reshape(*nb, 16, 16, 16).transpose(0, 3, 1, 4, 2, 5).reshape(n)
    key = mesh.edge_keys.astype(np.int64)
    axis, lin = key % 3, key // 3
    g = np.stack([lin // (n[1] * n[2]), (lin // n[2]) % n[1], lin % n[2]], 1)
    g1 = g + np.eye(3, dtype=np.int64)[axis]
    f0, w0 = f[tuple(g.T)], w[tuple(g.T)]
    f1, w1 = f[tuple(g1.T)], w[tuple(g1.T)]
    ok = lambda a, b: (b != 0) & (a < np.float32(0.98)) & (a >= np.float32(-0.98))
    want = ok(f0, w0) & ok(f1, w1) & (f0 * f1 < np.float32(0))
    assert want.sum() > 1000
    pos = np.searchsorted(pcd.keys, key[want])
    assert (pcd.keys[pos] == key[want]).all()
    d = np.abs(pcd.points[pos] - mesh.vertices[want])
    assert (d <= 2.0 ** -23 * (np.abs(mesh.vertices[want]) + vl)).all()
