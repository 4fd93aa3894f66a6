"""GPU density clustering (gs2mesh_b200.pointcloud.cluster_dbscan over gsb_pcd_dbscan) against the numpy restatement
(tests/dbscan_oracle.py), label for label: random clouds with noise, border points and many clusters, lattices with
distance ties exactly at eps, constructed cases confirmed against the literal Open3D loop first, degenerate inputs,
known answers at scale (one ball, a long shuffled chain, separated triplets), run-to-run and grid-cell invariance, and
the uses: floater blobs a radius test keeps, and the facade chain from integration to a written PLY."""
import ctypes as C

import numpy as np
import pytest

from gs2mesh_b200.mesh import PointCloud
from tests import dbscan_oracle as do

pytestmark = pytest.mark.gpu


def _same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


def _gpu(dev, pts, eps, mp):
    """(labels, n_clusters) through PointCloud.cluster_dbscan, checked against the device arrays of pointcloud.dbscan;
    the cloud is left unchanged."""
    from gs2mesh_b200 import pointcloud

    pcd = PointCloud(pts, device=dev)
    before = pcd.points.copy()
    got = pcd.cluster_dbscan(eps, mp)
    assert got.dtype == np.int32 and got.shape == (len(pts),)
    r = pointcloud.dbscan(pcd, eps, mp)
    nc = 0 if r is None else int(r[1].item())
    if r is not None:
        _same(r[0].cpu().numpy(), got)
    assert nc == (int(got.max()) + 1 if len(got) else 0)
    _same(pcd.points, before)
    return got, nc


def _check(dev, pts, eps, mp, pairs=None):
    """The GPU labels against the restatement; returns them."""
    got, nc = _gpu(dev, pts, eps, mp)
    ref, ref_nc = do.dbscan(pts, eps, mp, pairs)
    _same(got, ref)
    assert nc == ref_nc
    return got


def _lattice(m):
    return np.stack(np.meshgrid(*[np.arange(float(m))] * 3, indexing="ij"), -1).reshape(-1, 3)


# ------------------------------------------------------------------------------------------------------- random
def _eps(n, mp):
    """The eps at which n uniform points in the unit cube expect 0.8 * min_points others within eps: near the core
    threshold and near percolation of the core graph, so noise, border points and many clusters all occur."""
    return (0.8 * mp / (n * 4.0 / 3.0 * np.pi)) ** (1 / 3)


@pytest.mark.parametrize("mp", [4, 10])
@pytest.mark.parametrize("n", [1, 2, 1023, 1025, 100000, 1048577])
def test_random_clouds(gsb_lib, cuda_device, n, mp):
    rng = np.random.default_rng(n * 10 + mp)
    pts = rng.uniform(size=(n, 3))
    eps = _eps(n, mp) if n > 2 else 0.5
    pairs = do.within_pairs(pts, eps)
    labels = _check(cuda_device, pts, eps, mp, pairs)
    if n >= 1023:
        core = pairs[0] >= mp
        assert (labels == -1).any() and (labels[~core] >= 0).any() and core.any()  # noise, border and core points
        assert labels.max() >= 2  # several clusters


# ------------------------------------------------------------------------------------------------------ lattices
def test_lattice_ties_at_eps(gsb_lib, cuda_device):
    lat = _lattice(8)
    n = len(lat)
    _same(_check(cuda_device, lat, 1.0, 1), np.arange(n, dtype=np.int32))  # face neighbours at exactly 1: excluded
    assert (_check(cuda_device, lat, 1.0, 2) == -1).all()
    eps = float(np.nextafter(1.0, 2.0))
    interior = (lat.min(axis=1) > 0) & (lat.max(axis=1) < 7)  # 7 points within eps: itself and 6 faces
    labels = _check(cuda_device, lat, eps, 7)  # count == min_points: core
    assert (labels[interior] == 0).all()
    corner = (lat == 0).all(axis=1)
    assert labels[corner][0] == -1  # no core point within eps of a corner
    assert (_check(cuda_device, lat, eps, 8) == -1).all()  # count == min_points - 1: nothing is core
    assert (_check(cuda_device, lat, eps, 4) == 0).all()
    _check(cuda_device, lat * 0.37 + 1e6, 0.37 * eps, 6)
    _check(cuda_device, _lattice(13)[np.random.default_rng(1).permutation(13**3)], eps, 6)


# ---------------------------------------------------------------------------------------------- constructed cases
def _line(xs):
    return np.array([[x, 0.0, 0.0] for x in xs])


CASES = {
    # point 0 is within eps of both clusters (cores 3..6 and 7..10) and below every core index: the lower number
    "two_clusters_border_below_cores": (_line([5.0, 50.0, 7.5, 4.2, 3.9, 3.6, 3.3, 5.8, 6.1, 6.4, 6.7]), 1.0, 4,
                                        [0, -1, 1, 0, 0, 0, 0, 1, 1, 1, 1]),
    # noise at index 0
    "noise_first": (_line([-40.0, 3.0, 3.3, 3.6, 3.9, 20.0]), 1.0, 4, [-1, 0, 0, 0, 0, -1]),
    # cluster X (cores 5..8) has border points 0 and 9; cluster Y (cores 1..4) comes first by its smallest core index
    "numbered_by_core_not_border": (_line([10.7, 0.0, 0.3, 0.6, 0.9, 9.0, 9.3, 9.6, 9.9, 8.2]), 1.0, 4,
                                    [1, 0, 0, 0, 0, 1, 1, 1, 1, 1]),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_constructed_cases(gsb_lib, cuda_device, name):
    pts, eps, mp, expect = CASES[name]
    for seed in range(3):
        assert do.open3d_loop(pts, eps, mp, seed=seed)[0].tolist() == expect
    assert _check(cuda_device, pts, eps, mp).tolist() == expect


def test_exactly_at_eps_is_outside(gsb_lib, cuda_device):
    inside = float(np.nextafter(1.0, 0.0))
    pts = np.array([[0.0, 0, 0], [0, 0, 0.1], [0, 0, -0.1], [0, 0.1, 0], [1.0, 0, 0], [-inside, 0, 0]])
    expect = [0, 0, 0, 0, -1, 0]  # (1, 0, 0) lies at exactly eps from the origin; its nextafter twin just inside
    assert do.open3d_loop(pts, 1.0, 4)[0].tolist() == expect
    assert _check(cuda_device, pts, 1.0, 4).tolist() == expect
    assert _check(cuda_device, pts, float(np.nextafter(1.0, 2.0)), 4).tolist() == [0] * 6


# ------------------------------------------------------------------------------------------------ degenerate inputs
def test_degenerate_inputs(gsb_lib, cuda_device):
    rng = np.random.default_rng(5)
    pts = rng.uniform(size=(3000, 3))
    n = len(pts)
    _same(_check(cuda_device, pts, 0.0, 0), np.arange(n, dtype=np.int32))
    assert (_check(cuda_device, pts, 0.0, 1) == -1).all()
    _same(_check(cuda_device, pts, 0.03, 0), _check(cuda_device, pts, 0.03, 1))  # every point core either way
    assert (_check(cuda_device, pts, 10.0, n + 1) == -1).all()
    assert (_check(cuda_device, pts, 10.0, n) == 0).all()
    assert (_gpu(cuda_device, pts, 10.0, 2**62)[0] == -1).all()
    same = np.tile([[0.25, -0.5, 1.0]], (500, 1))
    assert (_check(cuda_device, same, 1e-3, 500) == 0).all()
    assert (_check(cuda_device, same, 1e-3, 501) == -1).all()
    _same(_check(cuda_device, same, 0.0, 0), np.arange(500, dtype=np.int32))
    dup = np.concatenate([pts[:1000], np.repeat(pts[:40], 6, axis=0)])[rng.permutation(1240)]
    for mp in (3, 7, 8):
        _check(cuda_device, dup, 1e-6, mp)  # only exact duplicates are within eps: groups of 7 are clusters at 7
    assert _gpu(cuda_device, dup, 1e-6, 7)[1] == 40
    far = rng.normal(size=(20000, 3)) * 0.01 + np.array([1e6, -1e6, 1e6])
    _check(cuda_device, far, 0.002, 5)
    out = PointCloud(np.zeros((0, 3)), device=cuda_device).cluster_dbscan(0.1, 3)
    assert out.dtype == np.int32 and out.shape == (0,)


# ------------------------------------------------------------------------------------------- known answers at scale
def test_ball_below_eps_is_one_cluster(gsb_lib, cuda_device):
    """Every pair within eps: 50,000 points each link with every lower core index (the link pass's worst case)."""
    rng = np.random.default_rng(6)
    v = rng.normal(size=(50000, 3))
    pts = v / np.linalg.norm(v, axis=1, keepdims=True) * 0.45 * rng.uniform(size=(50000, 1)) ** (1 / 3) + 3.0
    labels, nc = _gpu(cuda_device, pts, 1.0, 10)
    assert (labels == 0).all() and nc == 1


def test_shuffled_chain_is_one_cluster(gsb_lib, cuda_device):
    """1,000,000 points 0.9 eps apart along a line in shuffled index order: long union-find paths."""
    rng = np.random.default_rng(7)
    pts = np.zeros((1000000, 3))
    pts[:, 0] = 0.9 * np.arange(1000000.0)
    pts = pts[rng.permutation(1000000)]
    labels, nc = _gpu(cuda_device, pts, 1.0, 3)
    assert (labels == 0).all() and nc == 1
    labels, nc = _gpu(cuda_device, pts, 1.0, 4)  # count 3 at most: nothing is core
    assert (labels == -1).all() and nc == 0


def test_separated_triplets_numbered_by_smallest_index(gsb_lib, cuda_device):
    rng = np.random.default_rng(8)
    t = 300000
    centres = _lattice(67)[:t] * 10.0
    owner = np.repeat(np.arange(t), 3)[rng.permutation(3 * t)]  # the triplet of each index
    pts = centres[owner] + rng.uniform(-0.2, 0.2, size=(3 * t, 3))
    first = np.full(t, 3 * t)
    np.minimum.at(first, owner, np.arange(3 * t))
    expect = np.searchsorted(np.sort(first), first[owner]).astype(np.int32)
    labels, nc = _gpu(cuda_device, pts, 1.0, 3)
    _same(labels, expect)
    assert nc == t
    assert (_gpu(cuda_device, pts, 1.0, 4)[0] == -1).all()


# ------------------------------------------------------------------------------------------------------ invariance
def test_same_bytes_across_runs_and_grid_cells(gsb_lib, cuda_device):
    import torch

    from gs2mesh_b200 import _lib
    from gs2mesh_b200._lib import ptr
    from gs2mesh_b200.evaluate import PointGrid

    rng = np.random.default_rng(9)
    pts = rng.uniform(size=(200000, 3))
    eps, mp = _eps(200000, 6), 6
    first, nc = _gpu(cuda_device, pts, eps, mp)
    assert nc > 100
    for _ in range(2):
        _same(_gpu(cuda_device, pts, eps, mp)[0], first)
    L = _lib.lib()
    n = len(pts)
    with torch.cuda.device(cuda_device):
        p = torch.as_tensor(pts, device=cuda_device)
        for cell in (2 * eps, 5 * eps):
            grid = PointGrid(p, radius=eps, min_cell=cell)
            assert grid.cell >= cell
            work = torch.empty(int(L.gsb_pcd_dbscan_workspace_bytes(n)), dtype=torch.uint8, device=cuda_device)
            labels = torch.empty(n, dtype=torch.int32, device=cuda_device)
            count = torch.empty(1, dtype=torch.int32, device=cuda_device)
            _lib.check(L.gsb_pcd_dbscan(C.byref(grid.desc), eps, mp, ptr(work), work.numel(), ptr(labels), ptr(count),
                                        _lib.stream(cuda_device)))
            _same(labels.cpu().numpy(), first)
            assert int(count.item()) == nc


# ------------------------------------------------------------------------------------------------------------ use
def test_separates_floater_blobs_a_radius_test_keeps(gsb_lib, cuda_device):
    rng = np.random.default_rng(10)
    v = rng.normal(size=(60000, 3))
    sphere = v / np.linalg.norm(v, axis=1, keepdims=True)
    d = rng.normal(size=(5, 3))
    centres = d / np.linalg.norm(d, axis=1, keepdims=True) * 1.5
    blobs = np.concatenate([c + rng.normal(scale=0.01, size=(300, 3)) for c in centres])
    pts = np.concatenate([sphere, blobs])
    pcd = PointCloud(pts, device=cuda_device)
    _, kept = pcd.remove_radius_outlier(5, 0.05)
    assert np.isin(np.arange(60000, len(pts)), kept).mean() > 0.95  # the radius test keeps the blobs
    labels = _check(cuda_device, pts, 0.05, 5)
    assert (labels[:60000] == 0).all()
    for b in range(5):
        lb = labels[60000 + 300 * b:60000 + 300 * (b + 1)]
        assert (lb >= 0).mean() > 0.95 and len(np.unique(lb[lb >= 0])) == 1 and lb.max() == b + 1
    largest = np.bincount(labels[labels >= 0]).argmax()
    sel = pcd.select_by_index(np.nonzero(labels == largest)[0])
    _same(sel.points, sphere)


def test_o3d_compat_chain_and_ply_round_trip(gsb_lib, cuda_device, tmp_path):
    """integrate -> extract_point_cloud -> cluster_dbscan -> select the largest cluster -> write_point_cloud through the
    facade, read back."""
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
    labels = pcd.cluster_dbscan(eps=3 * VL, min_points=10)
    ref, _ = do.dbscan(pcd.points, 3 * VL, 10)
    _same(labels, ref)
    assert labels.max() >= 0
    _same(pcd.points, before)
    keep = np.nonzero(labels == np.bincount(labels[labels >= 0]).argmax())[0]
    big = pcd.select_by_index(keep)
    assert isinstance(big, o3d.geometry.PointCloud) and big.has_colors() and big.has_normals()
    _same(big.points, pcd.points[keep])
    _same(big.colors, pcd.colors[keep])
    path = str(tmp_path / "largest.ply")
    assert o3d.io.write_point_cloud(path, big)
    tab = _read_vertex_table(path)
    assert len(tab) == len(keep)
    _same(np.stack([tab["x"], tab["y"], tab["z"]], 1).astype(np.float64), big.points)
    _same(np.stack([tab["nx"], tab["ny"], tab["nz"]], 1).astype(np.float64), big.normals)
