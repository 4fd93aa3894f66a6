"""GPU marching cubes / mesh post-processing vs the CPU restatement of Open3D's ExtractTriangleMesh
(oracle.extract_mesh_from_bricks) on the same fused volume."""
import os

import numpy as np
import pytest

from tests.test_gpu_tsdf import B0, CX, CY, FX, FY, H, NB, TRUNC, VL, W, _gpu_volume, _views
from tests.test_oracle_mesh import canonical_triangle_order

pytestmark = pytest.mark.gpu


def _rekey(mesh, b0, nb):
    """mesh.edge_keys index voxels inside mesh.key_window (the bounding box of the open bricks); re-express them inside the
    window (b0, nb) the oracle mesh was extracted from."""
    (k0, kn) = mesh.key_window
    key = mesh.edge_keys.astype(np.int64)
    axis = key % 3
    lin = key // 3
    ny, nz = kn[1] * 16, kn[2] * 16
    gz = lin % nz
    gy = (lin // nz) % ny
    gx = lin // (nz * ny)
    gx, gy, gz = gx + (k0[0] - b0[0]) * 16, gy + (k0[1] - b0[1]) * 16, gz + (k0[2] - b0[2]) * 16
    return ((gx * (nb[1] * 16) + gy) * (nb[2] * 16) + gz) * 3 + axis


def test_mesh_matches_open3d_restatement(oracle, gsb_lib, cuda_device):
    import torch

    from gs2mesh_b200.mesh import extract_triangle_mesh
    from tests.test_gpu_mesh_volumes import open3d_vertex_normals

    gvol = _gpu_volume(cuda_device, with_color=True)
    for depth, rgb, w2c in _views(5):
        gvol.integrate(gvol.prepare_depth(depth, W, H, depth_trunc=4.0), rgb, W, H, FX, FY, CX, CY, w2c)
    torch.cuda.synchronize()
    mesh = extract_triangle_mesh(gvol)
    tw = gvol.bricks().cpu().numpy()
    col = gvol.colors().cpu().numpy()
    ref = oracle.extract_mesh_from_bricks(tw, B0, NB, VL, color=col)
    assert len(ref["triangles"]) > 2000

    nx, ny, nz = (n * 16 for n in NB)
    ref_key = ((ref["keys"][:, 0] * ny + ref["keys"][:, 1]) * nz + ref["keys"][:, 2]) * 3 + ref["keys"][:, 3]
    order = np.argsort(ref_key)
    mine = _rekey(mesh, B0, NB)
    assert (np.diff(mine) > 0).all()  # both windows are row-major over (x, y, z): the vertex order is the same
    np.testing.assert_array_equal(mine, ref_key[order])  # same vertex set (sorted edge keys)
    np.testing.assert_allclose(mesh.vertices, ref["vertices"][order], rtol=0, atol=1e-12)
    np.testing.assert_allclose(mesh.vertex_colors, ref["colors"][order], atol=2e-6)
    rank = np.empty(len(order), np.int64)
    rank[order] = np.arange(len(order))
    want = rank[ref["triangles"][canonical_triangle_order(ref["cubes"])]]
    np.testing.assert_array_equal(mesh.triangles, want)  # the same triangles, windings and order

    # vertex normals: the float64 restatement on the oracle's vertices and triangles; area-weighted, unit length, pointing
    # away from the object centre
    mesh.compute_vertex_normals(cuda_device)
    n = mesh.vertex_normals
    np.testing.assert_array_equal(n, open3d_vertex_normals(ref["vertices"][order], want))
    np.testing.assert_allclose(np.linalg.norm(n, axis=1), 1.0, atol=1e-9)
    v, t = mesh.vertices, mesh.triangles
    fn = np.cross(v[t[:, 1]] - v[t[:, 0]], v[t[:, 2]] - v[t[:, 0]])
    acc = np.zeros_like(v)
    for k in range(3):
        np.add.at(acc, t[:, k], fn)
    acc /= np.linalg.norm(acc, axis=1, keepdims=True)
    np.testing.assert_allclose(n, acc, atol=1e-9)
    assert (np.einsum("ij,ij->i", n, v) > 0).mean() > 0.95


def test_cleaning_and_ply_roundtrip(gsb_lib, cuda_device, tmp_path):
    from gs2mesh_b200.mesh import TriangleMesh

    # two components: a tetrahedron (4 triangles) and a lone triangle
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1], [5, 5, 5], [6, 5, 5], [5, 6, 5]], float)
    t = np.array([[0, 2, 1], [0, 1, 3], [1, 2, 3], [0, 3, 2], [4, 5, 6]])
    m = TriangleMesh(v, t, vertex_colors=np.linspace(0, 1, 21).reshape(7, 3))
    labels, counts, area = m.cluster_connected_triangles()
    assert sorted(counts.tolist()) == [1, 4] and len(set(labels[:4])) == 1 and labels[4] != labels[0]
    assert area[labels[4]] == pytest.approx(0.5)
    clean = m.remove_small_clusters(2)
    assert len(clean.triangles) == 4 and len(clean.vertices) == 4 and clean.vertex_colors.shape == (4, 3)
    clean.compute_vertex_normals(cuda_device)
    path = clean.write_ply(str(tmp_path / "m.ply"))
    raw = open(path, "rb").read()
    head, body = raw.split(b"end_header\n")
    assert b"element vertex 4" in head and b"element face 4" in head and b"property double nx" in head and b"uchar red" in head
    assert len(body) == 4 * (6 * 8 + 3) + 4 * (1 + 12)
    np.testing.assert_allclose(np.frombuffer(body[:24], "<f8"), clean.vertices[0])


def test_stage_class_extract_save_clean(gsb_lib, cuda_device, tmp_path):
    """TSDF.run() -> extract_mesh() -> save_mesh() -> clean_mesh(): the calls of run_single.py:161-174."""
    from gs2mesh_b200 import scene
    from gs2mesh_b200.renderer import Renderer
    from gs2mesh_b200.tsdf import TSDF
    from tests.test_gpu_pipeline import Args

    class A(Args):
        TSDF_skip = None
        TSDF_cleaning_threshold = 50
        TSDF_use_occlusion_mask = False

    cloud = scene.make_gaussians(20000, seed=9)
    rigs, baseline = scene.make_stereo_cameras(6, 320, 240)
    r = Renderer.from_scene(rigs, baseline, cloud, output_dir_root=str(tmp_path), args=A(), device=str(cuda_device))
    r.prepare_renderer()
    r.keep_frames = True
    for i in range(len(r)):
        r.render_image_pair(i)
    stage = TSDF(r, None, A(), "unit", window_resolution=128)
    stage.run()
    mesh = stage.extract_mesh()
    assert len(mesh.triangles) > 1000 and mesh.vertex_normals.shape == mesh.vertices.shape
    rad = np.linalg.norm(mesh.vertices, axis=1)
    assert 0.5 < np.median(rad) < 1.0  # the synthetic object has radius ~0.8
    p1 = stage.save_mesh()
    p2 = stage.clean_mesh()
    assert os.path.basename(p1) == "unit_mesh.ply" and os.path.basename(p2) == "unit_cleaned_mesh.ply"
    assert 0 < len(stage.cleaned_mesh.triangles) <= len(mesh.triangles)
    assert os.path.getsize(p2) <= os.path.getsize(p1)
