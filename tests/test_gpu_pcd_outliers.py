"""GPU point-cloud cleaning and downsampling (gs2mesh_b200.pointcloud: gsb_pcd_statistical_outliers,
gsb_pcd_radius_outliers, gsb_pcd_voxel_downsample and the torch plumbing) against the numpy restatement
(tests/pcd_oracle.py), bit for bit: keep flags, indices, mean distances, (mean, std, threshold), points, colours and
normals.  Cases: random clouds across both reduction levels, integer lattices (exact ties at the k-th place and on the
radius), the count boundary of the radius test, dense clusters, duplicates, coordinates near 1e6, clouds with and
without attributes, and the facade chain from integration to a written PLY."""
import numpy as np
import pytest

from gs2mesh_b200.mesh import PointCloud
from tests import pcd_oracle as po

pytestmark = pytest.mark.gpu


def _same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


def _lattice(m):
    return np.stack(np.meshgrid(*[np.arange(float(m))] * 3, indexing="ij"), -1).reshape(-1, 3)


def _cloud(pts, rng=None, colors=True, normals=True):
    rng = np.random.default_rng(0) if rng is None else rng
    n = len(pts)
    return PointCloud(pts, rng.uniform(size=(n, 3)) if colors else None, rng.normal(size=(n, 3)) if normals else None)


def _check_statistical(dev, pts, k, ratio, **attrs):
    """The device arrays and the facade's result against the oracle; returns the oracle's keep mask."""
    import torch

    from gs2mesh_b200 import pointcloud

    pcd = _cloud(pts, **attrs)
    pcd.device = dev
    before = [None if a is None else a.copy() for a in (pcd.points, pcd.colors, pcd.normals)]
    m, keep, stats = po.statistical(pts, k, ratio)
    got_keep, got_m, got_stats = pointcloud.statistical_outliers(pcd, k, ratio)
    torch.cuda.synchronize()
    _same(got_m.cpu().numpy(), m)
    _same(got_keep.cpu().numpy(), keep)
    _same(got_stats.cpu().numpy(), stats)
    out, ind = pcd.remove_statistical_outlier(k, ratio)
    _same(ind, np.nonzero(keep)[0].astype(np.int64))
    _same(out.points, pcd.points[keep])
    for name in ("colors", "normals"):
        a = getattr(pcd, name)
        assert (getattr(out, name) is None) == (a is None)
        if a is not None:
            _same(getattr(out, name), a[keep])
    assert type(out) is type(pcd) and out.device == dev
    for a, b in zip((pcd.points, pcd.colors, pcd.normals), before):
        assert (a is None and b is None) or a.tobytes() == b.tobytes()
    return keep


def _check_radius(dev, pts, nb, r):
    pcd = _cloud(pts)
    pcd.device = dev
    keep = po.radius(pts, nb, r)
    out, ind = pcd.remove_radius_outlier(nb, r)
    _same(ind, np.nonzero(keep)[0].astype(np.int64))
    _same(out.points, pts[keep])
    _same(out.colors, pcd.colors[keep])
    _same(out.normals, pcd.normals[keep])
    return keep


# ------------------------------------------------------------------------------------------------------ statistical
@pytest.mark.parametrize("k", [1, 2, 20, 32])
@pytest.mark.parametrize("n", [1, 2, 1023, 1024, 1025])
def test_statistical_small_random(gsb_lib, cuda_device, n, k):
    pts = np.random.default_rng(n * 100 + k).normal(size=(n, 3))
    _check_statistical(cuda_device, pts, k, 1.0)


@pytest.mark.parametrize("n,k", [(100000, 1), (100000, 32), (1048577, 20)])
def test_statistical_large_random(gsb_lib, cuda_device, n, k):
    """100,000 points take 98 chunks; 1,048,577 take 1025, one past a full second level of 1024 chunk sums."""
    pts = np.random.default_rng(n + k).uniform(-1, 1, size=(n, 3))
    keep = _check_statistical(cuda_device, pts, k, 2.0, colors=False, normals=n < 1000000)
    assert k == 1 or 0.8 * n < keep.sum() < n


@pytest.mark.parametrize("k", [2, 7, 20, 32])
def test_statistical_lattice_ties(gsb_lib, cuda_device, k):
    """Integer lattices: 6 face neighbours at 1, 12 at sqrt(2), 8 at sqrt(3), so the k-th place is tied for most k."""
    for m in (6, 13):
        _check_statistical(cuda_device, _lattice(m), k, 0.5)


def test_statistical_duplicates_far_and_identical(gsb_lib, cuda_device):
    rng = np.random.default_rng(4)
    base = rng.normal(size=(3000, 3))
    dup = np.concatenate([base, np.repeat(base[:50], 5, axis=0)])[rng.permutation(3250)]
    keep = _check_statistical(cuda_device, dup, 6, 1.0)
    assert keep.sum() > 0
    _check_statistical(cuda_device, dup, 5, 1.0)
    far = rng.normal(size=(5000, 3)) * 0.01 + np.array([1e6, -1e6, 1e6])
    _check_statistical(cuda_device, far, 20, 2.0)
    same = np.tile([[1.5, -2.0, 3.0]], (2000, 1))
    assert not _check_statistical(cuda_device, same, 20, 2.0).any()


def test_statistical_removes_floaters(gsb_lib, cuda_device):
    rng = np.random.default_rng(9)
    v = rng.normal(size=(60000, 3))
    surface = v / np.linalg.norm(v, axis=1, keepdims=True)
    floaters = rng.uniform(-2, 2, size=(300, 3))
    floaters = floaters[np.abs(np.linalg.norm(floaters, axis=1) - 1) > 0.2]
    pts = np.concatenate([surface, floaters])
    keep = _check_statistical(cuda_device, pts, 20, 2.0, colors=False, normals=False)
    assert not keep[len(surface):].any()
    assert keep[:len(surface)].mean() > 0.97
    rkeep = _check_radius(cuda_device, pts, 5, 0.05)
    assert not rkeep[len(surface):].any() and rkeep[:len(surface)].mean() > 0.97


# ----------------------------------------------------------------------------------------------------------- radius
def test_radius_lattice_boundaries(gsb_lib, cuda_device):
    lat = _lattice(8)
    assert not _check_radius(cuda_device, lat, 1, 1.0).any()  # the face neighbours lie at exactly 1: excluded
    r = float(np.nextafter(1.0, 2.0))
    counts = po.radius_counts(lat, r)
    assert counts.max() == 7
    keep = _check_radius(cuda_device, lat, 7, r)  # count == nb_points: dropped
    assert not keep.any()
    keep = _check_radius(cuda_device, lat, 6, r)  # count == nb_points + 1: kept
    assert np.array_equal(keep, counts == 7)
    _check_radius(cuda_device, lat * 0.37 + 1e6, 4, 0.37 * r)


def test_radius_dense_clusters_and_large_radius(gsb_lib, cuda_device):
    rng = np.random.default_rng(6)
    pts = np.concatenate([rng.normal(size=(3000, 3)) * 1e-3, rng.uniform(-1, 1, size=(5000, 3)),
                          np.repeat(rng.uniform(-1, 1, size=(4, 3)), 50, axis=0)])[rng.permutation(8200)]
    for nb, r in ((3, 0.01), (10, 0.05), (200, 0.1), (60, 0.002)):
        _check_radius(cuda_device, pts, nb, r)
    small = rng.normal(size=(500, 3))
    assert _check_radius(cuda_device, small, 499, 100.0).all()  # every point sees all 500
    assert not _check_radius(cuda_device, small, 500, 100.0).any()
    same = np.tile([[0.25, 0.5, -1.0]], (300, 1))
    assert _check_radius(cuda_device, same, 299, 1e-3).all()


# ---------------------------------------------------------------------------------------------------------- the rest
def test_voxel_down_sample_attributes(gsb_lib, cuda_device):
    import torch

    from gs2mesh_b200 import tnt

    rng = np.random.default_rng(7)
    pts = np.round(rng.uniform(-1, 1, size=(200000, 3)) * 64) / 64
    col = rng.uniform(size=(200000, 3))
    nrm = rng.normal(size=(200000, 3))
    nrm[rng.integers(0, 200000, 500), rng.integers(0, 3, 500)] = np.nan
    for colors, normals in ((col, nrm), (None, None), (col, None), (None, nrm)):
        pcd = PointCloud(pts, colors, normals, device=cuda_device)
        for s in (0.05, 1.0 / 64, 3.0):
            out = pcd.voxel_down_sample(s)
            ref = tnt.voxel_down_sample(torch.as_tensor(pts, device=cuda_device), s).cpu().numpy()
            _same(out.points, ref)
            op, oc, on = po.voxel_down_sample(pts, s, colors, normals)
            _same(out.points, op)
            assert (out.colors is None) == (colors is None) and (out.normals is None) == (normals is None)
            if colors is not None:
                _same(out.colors, oc)
            if normals is not None:
                _same(out.normals, on)
            again = pcd.voxel_down_sample(s)
            for a in ("points", "colors", "normals"):
                x, y = getattr(out, a), getattr(again, a)
                assert (x is None and y is None) or x.tobytes() == y.tobytes()
    with pytest.raises(RuntimeError, match=r"^voxel_size is too small\.$"):
        PointCloud(np.array([[0.0, 0, 0], [1e3, 0, 0]]), device=cuda_device).voxel_down_sample(1e-7)
    assert len(PointCloud(np.zeros((0, 3)), np.zeros((0, 3)), device=cuda_device).voxel_down_sample(0.1).colors) == 0


def test_select_uniform_and_distances(gsb_lib, cuda_device):
    rng = np.random.default_rng(8)
    pts = rng.normal(size=(5000, 3))
    pts[4000:4010] = pts[:10]  # exact duplicates: nearest distance 0
    pcd = _cloud(pts, rng)
    pcd.device = cuda_device
    idx = rng.permutation(5000)[:1200]
    idx = np.concatenate([idx, idx[:300]])[rng.permutation(1500)]
    for invert in (False, True):
        sel = po.select(5000, idx, invert)
        out = pcd.select_by_index(idx, invert=invert)
        _same(out.points, pts[sel])
        _same(out.colors, pcd.colors[sel])
        _same(out.normals, pcd.normals[sel])
    assert len(pcd.select_by_index([]).points) == 0
    assert len(pcd.select_by_index([], invert=True).points) == 5000
    with pytest.raises(ValueError):
        pcd.select_by_index([5000])
    with pytest.raises(ValueError):
        pcd.select_by_index([-1])
    for k in (1, 3, 4999, 5000, 7000):
        out = pcd.uniform_down_sample(k)
        _same(out.points, pts[::k])
        _same(out.normals, pcd.normals[::k])
    nn = pcd.compute_nearest_neighbor_distance()
    _same(nn, po.nearest_neighbor_distance(pts))
    assert (nn[4000:4010] == 0).all() and (nn[:10] == 0).all()
    _same(PointCloud(pts[:1], device=cuda_device).compute_nearest_neighbor_distance(), np.zeros(1))
    target = PointCloud(pts[::3] + 0.01)
    d = pcd.compute_point_cloud_distance(target)
    from tests.normals_oracle import knn

    _same(d, np.sqrt(knn(pts, target.points, 1)[0][:, 0]))
    _same(pcd.compute_point_cloud_distance(PointCloud(np.zeros((0, 3)))), np.zeros(5000))
    empty = PointCloud(np.zeros((0, 3)), device=cuda_device)
    for out, ind in (empty.remove_statistical_outlier(20, 2.0), empty.remove_radius_outlier(3, 0.1)):
        assert len(out.points) == 0 and ind.dtype == np.int64 and len(ind) == 0


def test_o3d_compat_chain_and_ply_round_trip(gsb_lib, cuda_device, tmp_path):
    """integrate -> extract_point_cloud -> remove_statistical_outlier(20, 2.0) -> voxel_down_sample ->
    write_point_cloud through the facade, read back."""
    import torch

    import gs2mesh_b200.o3d_compat as o3d
    from gs2mesh_b200.io import _read_vertex_table
    from tests.test_gpu_tsdf import CX, CY, FX, FY, TRUNC, VL, W, H, _views

    with torch.cuda.device(cuda_device):
        volume = o3d.pipelines.integration.ScalableTSDFVolume(voxel_length=VL, sdf_trunc=TRUNC,
                                                              color_type=o3d.pipelines.integration.TSDFVolumeColorType.RGB8,
                                                              window_resolution=128, device=cuda_device)
        for depth, rgb, w2c in _views(4):
            rgbd = o3d.geometry.RGBDImage.create_from_color_and_depth(o3d.geometry.Image(rgb), o3d.geometry.Image(depth),
                                                                       depth_scale=1.0, depth_trunc=4.0,
                                                                       convert_rgb_to_intensity=False)
            volume.integrate(rgbd, o3d.camera.PinholeCameraIntrinsic(W, H, FX, FY, CX, CY), w2c)
        pcd = volume.extract_point_cloud()
    assert len(pcd.points) > 1000 and pcd.has_colors() and pcd.has_normals()
    before = pcd.points.copy()
    clean, ind = pcd.remove_statistical_outlier(nb_neighbors=20, std_ratio=2.0)
    assert isinstance(clean, o3d.geometry.PointCloud) and clean.device == pcd.device
    _, keep, _ = po.statistical(pcd.points, 20, 2.0)
    _same(ind, np.nonzero(keep)[0].astype(np.int64))
    _same(clean.colors, pcd.colors[keep])
    thin = clean.voxel_down_sample(voxel_size=4 * VL)
    assert isinstance(thin, o3d.geometry.PointCloud) and thin.has_colors() and thin.has_normals()
    op, oc, on = po.voxel_down_sample(clean.points, 4 * VL, clean.colors, clean.normals)
    _same(thin.points, op)
    _same(thin.colors, oc)
    _same(thin.normals, on)
    _same(pcd.points, before)
    path = str(tmp_path / "thin.ply")
    assert o3d.io.write_point_cloud(path, thin)
    tab = _read_vertex_table(path)
    _same(np.stack([tab["x"], tab["y"], tab["z"]], 1).astype(np.float64), thin.points)
    _same(np.stack([tab["nx"], tab["ny"], tab["nz"]], 1).astype(np.float64), thin.normals)
    assert len(tab) == len(thin.points)
