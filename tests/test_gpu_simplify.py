"""Vertex-clustering simplification on the GPU (gsb_mesh_simplify through TriangleMesh.simplify_vertex_clustering)
against the numpy restatement in tests/simplify_oracle.py: vertices, colours, normals and triangles equal bit for bit,
the same count of cells that took the quadric solve, and the same bytes on every run."""
import numpy as np
import pytest

from tests import simplify_oracle as so

pytestmark = pytest.mark.gpu

MODES = [so.AVERAGE, so.QUADRIC]


def _same(a, b):
    if a is None or b is None:
        assert a is None and b is None
        return
    assert a.dtype == b.dtype and a.shape == b.shape
    assert a.tobytes() == b.tobytes()


def _check(dev, v, t, s, mode, colors=None, normals=None):
    from gs2mesh_b200.mesh import SimplificationContraction, TriangleMesh

    mesh = TriangleMesh(v, t, colors, normals, device=dev)
    got = mesh.simplify_vertex_clustering(s, SimplificationContraction(mode))
    wv, wt, wc, wn, wq = so.simplify(v, t, s, mode, colors, normals)
    assert type(got) is TriangleMesh and got.device == dev
    _same(got.vertices, wv)
    _same(got.triangles, wt)
    _same(got.vertex_colors, wc)
    _same(got.vertex_normals, wn)
    assert mesh.last_simplify_stats == {"vertices": len(wv), "triangles": len(wt), "quadric_cells": wq}
    return got, wq


def _adversarial(rng, nv=4000, nt=8000, scale=1.0):
    """Normal-distributed vertices with repeated positions and 64 unreferenced ones; random triangles with degenerate
    ones, rotated and oppositely wound copies and exact repeats, in shuffled order."""
    v = rng.normal(size=(nv, 3)) * scale
    rep = rng.random(nv) < 0.1
    v[rep] = v[rng.integers(0, nv, size=rep.sum())]
    t = rng.integers(0, nv - 64, size=(nt, 3))
    k = nt // 20
    t[:k, 1] = t[:k, 0]
    t[k:2 * k, 2] = t[k:2 * k, 1]
    t[2 * k:2 * k + 10] = t[2 * k:2 * k + 10, :1]
    d = t[rng.integers(0, nt, size=nt // 8)]
    t = np.concatenate([t, d[:, [1, 2, 0]], d[:, [2, 0, 1]], d[:, [0, 2, 1]], d])
    return v, t[rng.permutation(len(t))]


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("mode", MODES)
def test_adversarial_meshes(gsb_lib, cuda_device, seed, mode):
    rng = np.random.default_rng(seed)
    v, t = _adversarial(rng, scale=1.0 + seed)
    colors = rng.random(v.shape) if seed % 2 == 0 else None
    normals = rng.normal(size=v.shape) if seed % 3 != 2 else None
    for s in (0.3 * (1 + seed), 1.7 * (1 + seed)):
        got, nq = _check(cuda_device, v, t, s, mode, colors, normals)
        assert len(got.triangles) > 0 and len(got.vertices) < len(v)
        if mode == so.QUADRIC and s > 1:
            assert nq > 0  # large triangles at unit scale: many cells take the solve


@pytest.mark.parametrize("mode", MODES)
def test_boundary_exact_and_negative_coordinates(gsb_lib, cuda_device, mode):
    """Dyadic coordinates on the cell boundaries of a dyadic voxel (v - m and the division are exact), around 0."""
    rng = np.random.default_rng(11)
    s = 0.125
    v = rng.integers(-40, 40, size=(5000, 3)) * (s / 2) - 1.0
    v[:10] = v.min(axis=0)
    t = rng.integers(0, len(v), size=(12000, 3))
    _, c, _ = so.cells(v, s)
    assert len(np.unique(c, axis=0)) > 100
    _check(cuda_device, v, t, s, mode, rng.random(v.shape), None)
    _check(cuda_device, v, t, 3 * s / 4, mode, None, rng.normal(size=v.shape))


@pytest.mark.parametrize("mode", MODES)
def test_far_from_the_origin(gsb_lib, cuda_device, mode):
    rng = np.random.default_rng(12)
    v, t = _adversarial(rng, nv=3000, nt=6000, scale=0.05)
    for offset in ((1e6, -3e6, 2.5e5), (-1.25e9, 7e8, 1e3)):
        _check(cuda_device, v + offset, t, 0.013, mode, rng.random(v.shape), rng.normal(size=v.shape))


@pytest.mark.parametrize("mode", MODES)
def test_one_cell_holds_over_1m_vertices(gsb_lib, cuda_device, mode):
    rng = np.random.default_rng(13)
    nv = 1_100_000
    v = rng.random((nv, 3))
    t = rng.integers(0, nv, size=(300_000, 3))
    got, nq = _check(cuda_device, v, t, 10.0, mode, rng.random(v.shape), rng.normal(size=v.shape))
    assert len(got.vertices) == 1 and len(got.triangles) == 0 and nq == (mode == so.QUADRIC)


@pytest.mark.parametrize("mode", MODES)
def test_shuffled_grid_over_1m_triangles(gsb_lib, cuda_device, mode):
    from tests.test_gpu_mesh_clean import _shuffled_grid

    rng = np.random.default_rng(14)
    v, t = _shuffled_grid(710, rng)  # spacing 0.01
    assert len(t) >= 1_000_000
    for s in (0.02, 0.04):
        got, _ = _check(cuda_device, v, t, s, mode, rng.random(v.shape), None)
        assert 0 < len(got.triangles) < len(t) // 3


def test_fused_scene(gsb_lib, cuda_device, tmp_path):
    """The mesh of a fused scene (TSDF.run -> extract_mesh -> clean_mesh) at several voxel sizes, both contractions."""
    from tests.test_gpu_mesh_clean import _fused_stage

    stage = _fused_stage(tmp_path, cuda_device, 50)
    stage.run()
    stage.extract_mesh()
    stage.clean_mesh()
    mesh = stage.cleaned_mesh
    assert mesh.device == cuda_device and len(mesh.triangles) > 1000
    extent = float(np.max(mesh.vertices.max(axis=0) - mesh.vertices.min(axis=0)))
    for frac in (1 / 200, 1 / 80, 1 / 20):
        for mode in MODES:
            got, _ = _check(cuda_device, mesh.vertices, mesh.triangles, extent * frac, mode, mesh.vertex_colors,
                            mesh.vertex_normals)
            assert 0 < len(got.triangles) < len(mesh.triangles)


@pytest.mark.parametrize("mode", MODES)
def test_empty_and_triangle_free_inputs(gsb_lib, cuda_device, mode):
    got, _ = _check(cuda_device, np.zeros((0, 3)), np.zeros((0, 3), np.int64), 0.1, mode, np.zeros((0, 3)), None)
    assert got.vertices.shape == (0, 3) and got.triangles.shape == (0, 3) and got.vertex_colors.shape == (0, 3)
    v = np.random.default_rng(15).normal(size=(500, 3))
    got, nq = _check(cuda_device, v, np.zeros((0, 3), np.int64), 0.5, mode, None, v)
    assert 0 < len(got.vertices) < 500 and got.triangles.shape == (0, 3) and nq == 0


def test_errors(gsb_lib, cuda_device):
    from gs2mesh_b200.mesh import TriangleMesh

    v = np.random.default_rng(16).normal(size=(10, 3))
    mesh = TriangleMesh(v, np.array([[0, 1, 2]]), device=cuda_device)
    for s in (0.0, -2.0, float("nan")):
        with pytest.raises(RuntimeError, match=r"^voxel_size <= 0\.0$"):
            mesh.simplify_vertex_clustering(s)
    with pytest.raises(RuntimeError, match=r"^voxel_size is too small\.$"):
        TriangleMesh([[0, 0, 0], [1e7, 0, 0]], np.zeros((0, 3)), device=cuda_device).simplify_vertex_clustering(1e-3)
    with pytest.raises(ValueError, match="63 bits"):
        TriangleMesh([[0, 0, 0], [1e7, 1e7, 1e7]], np.zeros((0, 3)), device=cuda_device).simplify_vertex_clustering(1.0)
    with pytest.raises(ValueError, match="not finite"):
        TriangleMesh([[0, 0, 0], [np.nan, 0, 0]], np.zeros((0, 3)), device=cuda_device).simplify_vertex_clustering(1.0)
    with pytest.raises(ValueError, match="not finite"):
        mesh.simplify_vertex_clustering(float("inf"))
    with pytest.raises(ValueError, match="out of range"):
        TriangleMesh(v, np.array([[0, 1, 10]]), device=cuda_device).simplify_vertex_clustering(1.0)
    # the largest cell box that still packs: 2^21 x 2^21 x 2^21 cells
    w = np.array([[0.0, 0, 0], [2**21 - 1.0, 2**21 - 1.0, 2**21 - 1.0]])
    got = TriangleMesh(w, np.zeros((0, 3)), device=cuda_device).simplify_vertex_clustering(1.0)
    assert got.vertices.tolist() == w.tolist()


@pytest.mark.parametrize("mode", MODES)
def test_two_runs_give_the_same_bytes(gsb_lib, cuda_device, mode):
    from gs2mesh_b200.mesh import TriangleMesh

    rng = np.random.default_rng(17)
    v, t = _adversarial(rng, nv=200_000, nt=400_000)
    mesh = TriangleMesh(v, t, rng.random(v.shape), rng.normal(size=v.shape), device=cuda_device)
    a = mesh.simplify_vertex_clustering(0.6, mode)
    b = mesh.simplify_vertex_clustering(0.6, mode)
    for name in ("vertices", "triangles", "vertex_colors", "vertex_normals"):
        _same(getattr(a, name), getattr(b, name))


def test_host_mesh_runs_on_the_current_device(gsb_lib, cuda_device):
    import torch

    from gs2mesh_b200.mesh import TriangleMesh

    v, t = _adversarial(np.random.default_rng(18), nv=1000, nt=2000)
    with torch.cuda.device(cuda_device):
        got = TriangleMesh(v, t).simplify_vertex_clustering(0.5)
    assert got.device == cuda_device
    _same(got.vertices, so.simplify(v, t, 0.5)[0])


def test_o3d_compat_call_sequence_and_ply_round_trip(gsb_lib, cuda_device, tmp_path):
    """extract_triangle_mesh -> simplify_vertex_clustering -> write_triangle_mesh through the facade, read back."""
    import torch

    import gs2mesh_b200.o3d_compat as o3d
    from gs2mesh_b200.io import read_triangle_mesh_ply
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
        mesh = volume.extract_triangle_mesh()
        mesh.compute_vertex_normals()
    for mode in (o3d.geometry.SimplificationContraction.Average, o3d.geometry.SimplificationContraction.Quadric):
        small = mesh.simplify_vertex_clustering(4 * VL, mode)
        assert isinstance(small, o3d.geometry.TriangleMesh) and small.device == cuda_device
        wv, wt, wc, wn, _ = so.simplify(mesh.vertices, mesh.triangles, 4 * VL, int(mode), mesh.vertex_colors,
                                        mesh.vertex_normals)
        for got, want in ((small.vertices, wv), (small.triangles, wt), (small.vertex_colors, wc), (small.vertex_normals, wn)):
            _same(got, want)
        assert 0 < len(small.triangles) < len(mesh.triangles)
        path = str(tmp_path / f"small_{int(mode)}.ply")
        assert o3d.io.write_triangle_mesh(path, small)
        xyz, tris, rgb = read_triangle_mesh_ply(path, with_colors=True)
        assert xyz.tobytes() == small.vertices.tobytes() and (tris == small.triangles).all()
        from gs2mesh_b200.io import color_to_uint8

        assert (rgb == color_to_uint8(small.vertex_colors) / 255.0).all()
