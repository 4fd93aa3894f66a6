"""Cluster cleaning on the GPU (gsb_mesh_clusters / gsb_mesh_remove_small_clusters) against the numpy / scipy path the
same TriangleMesh takes when it was built from host arrays: labels and counts equal as arrays, cleaned meshes equal bit
for bit, cluster areas within 1e-12 relative and the same bits on every GPU run."""
import copy
import os
import sys

import numpy as np
import pytest

from tests.test_mesh_cpu import _random_mesh

pytestmark = pytest.mark.gpu

THRESHOLD = 50 / 0.3  # TSDF_cleaning_threshold / TSDF_scale: 166.67


def _pair(v, t, dev, colors=None, normals=None):
    from gs2mesh_b200.mesh import TriangleMesh

    return TriangleMesh(v, t, colors, normals), TriangleMesh(v, t, colors, normals, device=dev)


def _same_array(a, b):
    if a is None or b is None:
        assert a is None and b is None
        return
    assert a.dtype == b.dtype and a.shape == b.shape
    assert a.tobytes() == b.tobytes()


def _check_clusters(host, gpu):
    hl, hc, ha = host.cluster_connected_triangles()
    gl, gc, ga = gpu.cluster_connected_triangles()
    _same_array(gl, hl)
    _same_array(gc, hc)
    assert ga.dtype == np.float64 and ga.shape == ha.shape
    np.testing.assert_allclose(ga, ha, rtol=1e-12, atol=0)
    _, _, ga2 = gpu.cluster_connected_triangles()
    assert ga2.tobytes() == ga.tobytes()
    return gl, gc, ga


def _check_clean(host, gpu, threshold):
    want = host.remove_small_clusters(threshold)
    got = gpu.remove_small_clusters(threshold)
    assert got.device == gpu.device and want.device is None
    for name in ("vertices", "triangles", "vertex_colors", "vertex_normals"):
        _same_array(getattr(got, name), getattr(want, name))
    return got, want


@pytest.mark.parametrize("seed", range(8))
def test_adversarial_meshes_match_host(gsb_lib, cuda_device, seed):
    """Non-manifold edges, duplicate and degenerate triangles, fans of 166 and 167 triangles around 166.67, isolated
    vertices."""
    v, t, col = _random_mesh(np.random.default_rng(seed))
    host, gpu = _pair(v, t, cuda_device, col, -v)
    _, counts, _ = _check_clusters(host, gpu)
    assert 166 in counts and 167 in counts
    got, _ = _check_clean(host, gpu, THRESHOLD)
    assert 0 < len(got.triangles) < len(t) and len(got.vertices) < len(v)


def test_contact_kinds(gsb_lib, cuda_device):
    """A shared vertex does not join; a shared edge joins in either orientation, a degenerate edge (a,a) included."""
    v = np.random.default_rng(0).normal(size=(12, 3))
    t = np.array([[0, 1, 2], [2, 3, 4],  # only vertex 2 in common
                  [5, 5, 6], [5, 7, 5],  # the degenerate edge (5,5) in common
                  [8, 9, 10], [9, 8, 11]])  # edge (8,9), opposite orientations
    host, gpu = _pair(v, t, cuda_device)
    labels, counts, _ = _check_clusters(host, gpu)
    assert labels.tolist() == [0, 1, 2, 2, 3, 3] and counts.tolist() == [1, 1, 2, 2]
    got, _ = _check_clean(host, gpu, 2)
    assert got.triangles.tolist() == [[0, 0, 1], [0, 2, 0], [3, 4, 5], [4, 3, 6]]


def test_thresholds(gsb_lib, cuda_device, tmp_path):
    """The comparison is a strict `<` against a float: exactly a cluster's size keeps it; 0 and 1 keep everything; a
    non-integer falls between sizes; more than n_triangles empties the mesh, which still writes a valid PLY."""
    v, t, col = _random_mesh(np.random.default_rng(11))
    host, gpu = _pair(v, t, cuda_device, col, v * 2)
    _, counts, _ = _check_clusters(host, gpu)
    size = int(np.sort(counts)[len(counts) // 2])
    for thr in (size, size + 1, 0, 1, 2.5, THRESHOLD, float(len(t) + 1), len(t) + 1):
        got, _ = _check_clean(host, gpu, thr)
        if thr == size:
            assert (counts >= size).sum() > 0 and len(got.triangles) == counts[counts >= size].sum()
        if thr in (0, 1):
            assert len(got.triangles) == len(t)
    got, want = _check_clean(host, gpu, len(t) + 1)
    assert len(got.triangles) == 0 and len(got.vertices) == 0
    a = got.write_ply(str(tmp_path / "gpu.ply"))
    b = want.write_ply(str(tmp_path / "host.ply"))
    raw = open(a, "rb").read()
    assert raw == open(b, "rb").read()
    assert b"element vertex 0\n" in raw and b"element face 0\n" in raw and raw.endswith(b"end_header\n")


@pytest.mark.parametrize("attrs", ["colors", "normals", "neither"])
def test_vertex_attributes(gsb_lib, cuda_device, attrs):
    v, t, col = _random_mesh(np.random.default_rng(5))
    host, gpu = _pair(v, t, cuda_device, col if attrs == "colors" else None, v[:, ::-1].copy() if attrs == "normals" else None)
    _check_clean(host, gpu, THRESHOLD)


def test_empty_inputs_and_unreferenced_vertices(gsb_lib, cuda_device):
    from gs2mesh_b200.mesh import TriangleMesh

    host, gpu = _pair(np.zeros((0, 3)), np.zeros((0, 3), np.int64), cuda_device, np.zeros((0, 3)))
    _check_clusters(host, gpu)
    got, _ = _check_clean(host, gpu, THRESHOLD)
    assert len(got.vertices) == 0 and got.vertex_colors.shape == (0, 3)

    # vertices but no triangles: every vertex is unreferenced
    v = np.arange(30, dtype=np.float64).reshape(10, 3)
    host, gpu = _pair(v, np.zeros((0, 3), np.int64), cuda_device, None, v)
    got, _ = _check_clean(host, gpu, 0)
    assert got.vertices.shape == (0, 3) and got.vertex_normals.shape == (0, 3)

    # vertices only some triangles reference, at both ends of the vertex array
    t = np.array([[3, 4, 5], [5, 4, 6], [1, 2, 3]])
    host, gpu = _pair(v, t, cuda_device, v / 30)
    got, _ = _check_clean(host, gpu, 1)
    assert got.vertices.tolist() == v[1:7].tolist()

    with pytest.raises(ValueError, match="out of range"):
        TriangleMesh(v, np.array([[0, 1, 10]]), device=cuda_device).remove_small_clusters(1)
    with pytest.raises(ValueError, match="out of range"):
        TriangleMesh(v, np.array([[0, -1, 2]]), device=cuda_device).cluster_connected_triangles()


def _shuffled_grid(n, rng):
    """(n+1)^2 vertices, 2 n^2 triangles of one edge-connected sheet; vertex ids and triangle order shuffled, so the
    union-find sees long chains in no particular order."""
    g = np.arange((n + 1) * (n + 1)).reshape(n + 1, n + 1)
    a, b, c, d = g[:-1, :-1].ravel(), g[:-1, 1:].ravel(), g[1:, :-1].ravel(), g[1:, 1:].ravel()
    t = np.concatenate([np.stack([a, b, d], 1), np.stack([a, d, c], 1)])
    perm = rng.permutation(g.size)
    t = perm[t][rng.permutation(len(t))]
    xy = np.stack(np.meshgrid(np.arange(n + 1.0), np.arange(n + 1.0), indexing="ij"), -1).reshape(-1, 2) * 0.01
    v = np.empty((g.size, 3))
    v[perm] = np.concatenate([xy, np.sin(xy[:, :1] * 3) * 0.1], 1)
    return v, t


def test_shuffled_grid_over_1m_triangles_is_one_cluster(gsb_lib, cuda_device):
    rng = np.random.default_rng(3)
    v, t = _shuffled_grid(710, rng)
    assert len(t) >= 1_000_000
    host, gpu = _pair(v, t, cuda_device, rng.random(v.shape))
    labels, counts, _ = _check_clusters(host, gpu)
    assert counts.tolist() == [len(t)] and not labels.any()
    got, _ = _check_clean(host, gpu, len(t))
    assert len(got.triangles) == len(t)
    got, _ = _check_clean(host, gpu, len(t) + 0.5)
    assert len(got.triangles) == 0


def test_over_1m_disjoint_triangles(gsb_lib, cuda_device):
    """One cluster per triangle: the per-triangle areas are bit-identical to numpy's, so the one-term sums are too."""
    rng = np.random.default_rng(4)
    nt = 1_000_000
    v = rng.normal(size=(3 * nt + 5, 3)) * np.exp(rng.normal(size=(3 * nt + 5, 1)) * 3)
    t = rng.permutation(3 * nt + 5)[: 3 * nt].reshape(nt, 3)
    host, gpu = _pair(v, t, cuda_device, None, v)
    labels, counts, area = _check_clusters(host, gpu)
    assert labels.tolist() == list(range(nt)) and (counts == 1).all()
    _, _, want = host.cluster_connected_triangles()
    assert area.tobytes() == want.tobytes()
    assert len(_check_clean(host, gpu, 1)[0].triangles) == nt
    assert len(_check_clean(host, gpu, 1.5)[0].triangles) == 0


def _fused_stage(tmp_path, cuda_device, threshold):
    from gs2mesh_b200 import scene
    from gs2mesh_b200.renderer import Renderer
    from gs2mesh_b200.tsdf import TSDF
    from tests.test_gpu_pipeline import Args

    class A(Args):
        TSDF_skip = None
        TSDF_cleaning_threshold = threshold
        TSDF_use_occlusion_mask = False

    cloud = scene.make_gaussians(20000, seed=9)
    rigs, baseline = scene.make_stereo_cameras(6, 320, 240)
    r = Renderer.from_scene(rigs, baseline, cloud, output_dir_root=str(tmp_path), args=A(), device=str(cuda_device))
    r.prepare_renderer()
    r.keep_frames = True
    for i in range(len(r)):
        r.render_image_pair(i)
    return TSDF(r, None, A(), "unit", window_resolution=128)


def test_stage_clean_mesh_writes_the_host_ply_without_scipy(gsb_lib, cuda_device, tmp_path, monkeypatch):
    """TSDF.run() -> extract_mesh() -> clean_mesh() cleans on the volume's device; the PLY it writes equals, byte for
    byte, the one the host path writes for the same mesh."""
    from gs2mesh_b200.mesh import TriangleMesh

    stage = _fused_stage(tmp_path, cuda_device, 50)
    stage.run()
    mesh = stage.extract_mesh()
    assert mesh.device == cuda_device and len(mesh.triangles) > 1000
    for name in ("scipy", "scipy.sparse", "scipy.sparse.csgraph"):
        monkeypatch.setitem(sys.modules, name, None)  # importing scipy now fails
    path = stage.clean_mesh()
    monkeypatch.undo()
    assert os.path.basename(path) == "unit_cleaned_mesh.ply" and stage.cleaned_mesh.device == cuda_device
    host = TriangleMesh(mesh.vertices, mesh.triangles, mesh.vertex_colors, mesh.vertex_normals)
    want = host.remove_small_clusters(50.0).write_ply(str(tmp_path / "host_cleaned.ply"))
    assert open(path, "rb").read() == open(want, "rb").read()


def test_o3d_compat_call_sequence_matches_host(gsb_lib, cuda_device):
    """tsdf_utils.py:130-140 through the Open3D facade on an extracted mesh, against the host path on a deep copy."""
    import torch

    import gs2mesh_b200.o3d_compat as o3d
    from tests.test_gpu_tsdf import CX, CY, FX, FY, TRUNC, VL, W, H, _views

    with torch.cuda.device(cuda_device):
        volume = o3d.pipelines.integration.ScalableTSDFVolume(voxel_length=VL, sdf_trunc=TRUNC,
                                                              color_type=o3d.pipelines.integration.TSDFVolumeColorType.RGB8,
                                                              window_resolution=128, device=cuda_device)
        for depth, rgb, w2c in _views(4):
            depth = depth.copy()
            depth[depth < 0.5] = 0
            rgbd = o3d.geometry.RGBDImage.create_from_color_and_depth(o3d.geometry.Image(rgb), o3d.geometry.Image(depth),
                                                                       depth_scale=1.0, depth_trunc=4.0,
                                                                       convert_rgb_to_intensity=False)
            volume.integrate(rgbd, o3d.camera.PinholeCameraIntrinsic(W, H, FX, FY, CX, CY), w2c)
        mesh = volume.extract_triangle_mesh()
        mesh.scale(0.5, (0, 0, 0))
        mesh.compute_vertex_normals()
    assert mesh.device == cuda_device and len(mesh.triangles) > 1000

    def clean(m):
        tri_clusters, n_tri, area = m.cluster_connected_triangles()
        tri_clusters, n_tri = np.asarray(tri_clusters), np.asarray(n_tri)
        m.remove_triangles_by_mask(n_tri[tri_clusters] < 100)
        m.remove_unreferenced_vertices()
        return tri_clusters, n_tri, area

    gpu = copy.deepcopy(mesh)
    host = copy.deepcopy(mesh)
    assert gpu.device == cuda_device
    host.device = None
    gl, gc, ga = clean(gpu)
    hl, hc, ha = clean(host)
    _same_array(gl, hl)
    _same_array(gc, hc)
    np.testing.assert_allclose(ga, ha, rtol=1e-12, atol=0)
    assert 0 < len(gpu.triangles) <= len(mesh.triangles)
    for name in ("vertices", "triangles", "vertex_colors", "vertex_normals"):
        _same_array(getattr(gpu, name), getattr(host, name))
