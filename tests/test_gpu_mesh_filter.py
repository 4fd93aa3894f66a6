"""Smoothing and sharpening on the GPU (gsb_mesh_filter through TriangleMesh.filter_smooth_simple / _laplacian / _taubin
and filter_sharpen) against the numpy restatement in tests/filter_oracle.py: positions, colours and normals equal bit for
bit, the same bytes on every run, and the input mesh left as it was."""
import numpy as np
import pytest

from tests import filter_oracle as fo
from tests.test_gpu_simplify import _adversarial

pytestmark = pytest.mark.gpu

KINDS = [fo.SIMPLE, fo.LAPLACIAN, fo.TAUBIN, fo.SHARPEN]
SCOPES = [fo.ALL, fo.COLOR, fo.NORMAL, fo.VERTEX]
PARAMS = {fo.SIMPLE: (0.0, 0.0), fo.LAPLACIAN: (0.5, 0.0), fo.TAUBIN: (0.5, -0.53), fo.SHARPEN: (0.25, 0.0)}


def _same(a, b):
    if a is None or b is None:
        assert a is None and b is None
        return
    assert a.dtype == b.dtype and a.shape == b.shape
    assert a.tobytes() == b.tobytes()


def _run(mesh, kind, iterations, scope, params=None):
    from gs2mesh_b200.mesh import FilterScope

    p0, p1 = PARAMS[kind] if params is None else params
    scope = FilterScope(scope)
    if kind == fo.SIMPLE:
        return mesh.filter_smooth_simple(iterations, scope)
    if kind == fo.LAPLACIAN:
        return mesh.filter_smooth_laplacian(iterations, p0, scope)
    if kind == fo.TAUBIN:
        return mesh.filter_smooth_taubin(iterations, p0, p1, scope)
    return mesh.filter_sharpen(iterations, p0, scope)


def _check(dev, kind, v, t, iterations, scope, colors=None, normals=None, params=None):
    from gs2mesh_b200.mesh import TriangleMesh

    mesh = TriangleMesh(v, t, colors, normals, device=dev)
    got = _run(mesh, kind, iterations, scope, params)
    p0, p1 = PARAMS[kind] if params is None else params
    wv, wc, wn = fo.filter_mesh(kind, v, t, iterations, p0, p1, scope, colors, normals)
    assert type(got) is TriangleMesh and got.device == dev
    _same(got.vertices, wv)
    _same(got.vertex_colors, wc)
    _same(got.vertex_normals, wn)
    _same(got.triangles, mesh.triangles)
    assert got.triangles is not mesh.triangles
    return got


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("seed", range(4))
def test_adversarial_meshes(gsb_lib, cuda_device, seed, kind):
    """Shuffled ids, repeated positions, degenerate, duplicate, rotated and reversed triangles, unreferenced vertices;
    colours and normals on and off; every scope; 1, 2 and 3 iterations (both ping-pong parities), Taubin at 1 and 2."""
    rng = np.random.default_rng(100 + seed)
    v, t = _adversarial(rng, nv=2000, nt=4000, scale=1.0 + seed)
    colors = rng.random(v.shape) if seed % 2 == 0 else None
    normals = rng.normal(size=v.shape) if seed in (0, 1) else None
    for scope in SCOPES:
        for iterations in ((1, 2) if kind == fo.TAUBIN else (1, 2, 3)):
            _check(cuda_device, kind, v, t, iterations, scope, colors, normals)


def test_one_vertex_with_over_100k_neighbours(gsb_lib, cuda_device):
    """A closed fan: vertex 0 joined to 120 000 rim vertices, which one thread walks in one serial run."""
    rng = np.random.default_rng(21)
    rim = 120_000
    ang = 2 * np.pi * np.arange(rim) / rim
    v = np.concatenate([[[0.0, 0.0, 0.5]], np.stack([np.cos(ang), np.sin(ang), 0.01 * rng.normal(size=rim)], 1)])
    i = np.arange(1, rim + 1)
    t = np.stack([np.zeros(rim, np.int64), i, i % rim + 1], 1)
    t = t[rng.permutation(rim)]
    offsets, _ = fo.adjacency(t, len(v))
    assert offsets[1] - offsets[0] == rim
    col, nrm = rng.random(v.shape), rng.normal(size=v.shape)
    for kind in KINDS:
        _check(cuda_device, kind, v, t, 2 if kind != fo.TAUBIN else 1, fo.ALL, col, nrm)


def test_shuffled_grid_over_1m_triangles(gsb_lib, cuda_device):
    from tests.test_gpu_mesh_clean import _shuffled_grid

    rng = np.random.default_rng(22)
    v, t = _shuffled_grid(710, rng)  # spacing 0.01
    assert len(t) >= 1_000_000
    v = v + 0.002 * rng.normal(size=v.shape)
    got = _check(cuda_device, fo.TAUBIN, v, t, 1, fo.ALL, rng.random(v.shape), None)
    assert np.abs(got.vertices - v).max() > 1e-4
    _check(cuda_device, fo.SHARPEN, v, t, 1, fo.VERTEX, None, rng.normal(size=v.shape))


def test_fused_scene(gsb_lib, cuda_device, tmp_path):
    """The extract_triangle_mesh() mesh of a fused scene (colours and vertex normals), every filter."""
    from tests.test_gpu_mesh_clean import _fused_stage

    stage = _fused_stage(tmp_path, cuda_device, 50)
    stage.run()
    mesh = stage.extract_mesh()
    assert mesh.device == cuda_device and len(mesh.triangles) > 1000
    assert mesh.vertex_colors is not None and mesh.vertex_normals is not None
    v, t, col, nrm = mesh.vertices, mesh.triangles, mesh.vertex_colors, mesh.vertex_normals
    for kind, iterations, scope in ((fo.TAUBIN, 3, fo.ALL), (fo.LAPLACIAN, 2, fo.NORMAL), (fo.SIMPLE, 3, fo.COLOR),
                                    (fo.SHARPEN, 1, fo.VERTEX)):
        _check(cuda_device, kind, v, t, iterations, scope, col, nrm)


def test_far_from_the_origin(gsb_lib, cuda_device):
    rng = np.random.default_rng(23)
    v, t = _adversarial(rng, nv=3000, nt=6000, scale=0.05)
    for offset in ((1e6, -3e6, 2.5e5), (-1.25e9, 7e8, 1e3)):
        for kind in KINDS:
            _check(cuda_device, kind, v + offset, t, 2, fo.ALL, rng.random(v.shape), rng.normal(size=v.shape))


def test_empty_and_triangle_free_inputs(gsb_lib, cuda_device):
    for kind in KINDS:
        got = _check(cuda_device, kind, np.zeros((0, 3)), np.zeros((0, 3), np.int64), 3, fo.ALL, np.zeros((0, 3)), None)
        assert got.vertices.shape == (0, 3) and got.vertex_colors.shape == (0, 3) and got.vertex_normals is None
        v = np.random.default_rng(24).normal(size=(500, 3))
        got = _check(cuda_device, kind, v, np.zeros((0, 3), np.int64), 2, fo.ALL, None, v)
        assert got.vertices.tolist() == v.tolist() and got.triangles.shape == (0, 3)


def test_zero_iterations_and_scopes_copy(gsb_lib, cuda_device):
    rng = np.random.default_rng(25)
    v, t = _adversarial(rng, nv=1000, nt=2000)
    col, nrm = rng.random(v.shape), rng.normal(size=v.shape)
    for kind in KINDS:
        for scope in SCOPES:
            got = _check(cuda_device, kind, v, t, 0, scope, col, nrm)
            _same(got.vertices, v)
            _same(got.vertex_colors, col)
            _same(got.vertex_normals, nrm)


def test_errors(gsb_lib, cuda_device):
    from gs2mesh_b200.mesh import TriangleMesh

    v = np.random.default_rng(26).normal(size=(10, 3))
    mesh = TriangleMesh(v, np.array([[0, 1, 2]]), device=cuda_device)
    with pytest.raises(ValueError, match="number_of_iterations"):
        mesh.filter_smooth_taubin(-1)
    with pytest.raises(ValueError, match="out of range"):
        TriangleMesh(v, np.array([[0, 1, 10]]), device=cuda_device).filter_smooth_simple()
    with pytest.raises(ValueError, match="out of range"):
        TriangleMesh(v, np.array([[0, -1, 2]]), device=cuda_device).filter_sharpen()
    with pytest.raises(ValueError, match="one row per vertex"):
        TriangleMesh(v, np.array([[0, 1, 2]]), np.zeros((9, 3)), device=cuda_device).filter_smooth_laplacian()
    with pytest.raises(ValueError, match="one row per vertex"):
        TriangleMesh(v, np.array([[0, 1, 2]]), None, np.zeros((11, 3)), device=cuda_device).filter_smooth_laplacian()
    with pytest.raises(ValueError):
        mesh.filter_smooth_simple(1, 7)  # not a FilterScope


def test_two_runs_give_the_same_bytes_and_leave_the_input(gsb_lib, cuda_device):
    from gs2mesh_b200.mesh import TriangleMesh

    rng = np.random.default_rng(27)
    v, t = _adversarial(rng, nv=200_000, nt=400_000)
    col, nrm = rng.random(v.shape), rng.normal(size=v.shape)
    mesh = TriangleMesh(v.copy(), t.copy(), col.copy(), nrm.copy(), device=cuda_device)
    for kind in KINDS:
        a = _run(mesh, kind, 3, fo.ALL)
        b = _run(mesh, kind, 3, fo.ALL)
        for name in ("vertices", "triangles", "vertex_colors", "vertex_normals"):
            _same(getattr(a, name), getattr(b, name))
        assert (a.vertices != v).any()
    for got, want in ((mesh.vertices, v), (mesh.triangles, t), (mesh.vertex_colors, col), (mesh.vertex_normals, nrm)):
        _same(got, want)


def test_host_mesh_runs_on_the_current_device(gsb_lib, cuda_device):
    import torch

    from gs2mesh_b200.mesh import TriangleMesh

    v, t = _adversarial(np.random.default_rng(28), nv=1000, nt=2000)
    with torch.cuda.device(cuda_device):
        got = TriangleMesh(v, t).filter_smooth_taubin(2)
    assert got.device == cuda_device
    _same(got.vertices, fo.filter_mesh(fo.TAUBIN, v, t, 2, 0.5, -0.53)[0])


def _noisy_sphere(rng, n_lat=60, n_lon=120, noise=0.02):
    """A latitude-longitude unit sphere (two poles, n_lat - 1 rings) with its radii scaled by 1 + noise * N(0, 1)."""
    th, ph = np.pi * np.arange(1, n_lat) / n_lat, 2 * np.pi * np.arange(n_lon) / n_lon
    T, Ph = np.meshgrid(th, ph, indexing="ij")
    ring = np.stack([np.sin(T) * np.cos(Ph), np.sin(T) * np.sin(Ph), np.cos(T)], -1).reshape(-1, 3)
    v = np.concatenate([[[0.0, 0.0, 1.0]], ring, [[0.0, 0.0, -1.0]]])
    idx = 1 + np.arange((n_lat - 1) * n_lon).reshape(n_lat - 1, n_lon)
    j, j1 = np.arange(n_lon), (np.arange(n_lon) + 1) % n_lon
    tris = [np.stack([np.zeros(n_lon, np.int64), idx[0, j], idx[0, j1]], 1)]
    for i in range(n_lat - 2):
        a, b, c, d = idx[i, j], idx[i, j1], idx[i + 1, j], idx[i + 1, j1]
        tris += [np.stack([a, c, d], 1), np.stack([a, d, b], 1)]
    tris.append(np.stack([np.full(n_lon, len(v) - 1), idx[-1, j1], idx[-1, j]], 1))
    return v * (1 + noise * rng.normal(size=(len(v), 1))), np.concatenate(tris)


def test_noisy_sphere_laplacian_shrinks_taubin_keeps_the_radius(gsb_lib, cuda_device):
    """10 iterations at lambda 0.5, mu -0.53 on a sphere with 2% radial noise: Laplacian pulls the mean radius in by more
    than 0.004; Taubin keeps it within 0.001 of the input's and at least halves the radial spread."""
    from gs2mesh_b200.mesh import TriangleMesh

    v, t = _noisy_sphere(np.random.default_rng(29))
    mesh = TriangleMesh(v, t, device=cuda_device)
    r = lambda x: np.linalg.norm(x, axis=1)
    lap = _check(cuda_device, fo.LAPLACIAN, v, t, 10, fo.ALL).vertices
    tau = mesh.filter_smooth_taubin(10).vertices
    _same(tau, fo.filter_mesh(fo.TAUBIN, v, t, 10, 0.5, -0.53)[0])
    assert r(lap).mean() < r(v).mean() - 0.004
    assert abs(r(tau).mean() - r(v).mean()) < 0.001
    assert r(tau).std() < 0.5 * r(v).std()


def test_o3d_compat_call_sequence_and_ply_round_trip(gsb_lib, cuda_device, tmp_path):
    """extract_triangle_mesh -> filter_smooth_taubin -> write_triangle_mesh through the facade, read back."""
    import torch

    import gs2mesh_b200.o3d_compat as o3d
    from gs2mesh_b200.io import read_triangle_mesh_ply
    from gs2mesh_b200.io import color_to_uint8
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
    assert len(mesh.triangles) > 1000
    before = mesh.vertices.copy()
    smooth = mesh.filter_smooth_taubin(10)
    assert isinstance(smooth, o3d.geometry.TriangleMesh) and smooth.device == cuda_device
    wv, wc, wn = fo.filter_mesh(fo.TAUBIN, mesh.vertices, mesh.triangles, 10, 0.5, -0.53, fo.ALL, mesh.vertex_colors,
                                mesh.vertex_normals)
    for got, want in ((smooth.vertices, wv), (smooth.vertex_colors, wc), (smooth.vertex_normals, wn)):
        _same(got, want)
    _same(mesh.vertices, before)
    normals_only = mesh.filter_smooth_laplacian(2, 0.5, o3d.geometry.FilterScope.Normal)
    _same(normals_only.vertices, mesh.vertices)
    _same(normals_only.vertex_normals, fo.filter_mesh(fo.LAPLACIAN, mesh.vertices, mesh.triangles, 2, 0.5, 0.0, fo.NORMAL,
                                                      None, mesh.vertex_normals)[2])
    path = str(tmp_path / "smooth.ply")
    assert o3d.io.write_triangle_mesh(path, smooth)
    xyz, tris, rgb = read_triangle_mesh_ply(path, with_colors=True)
    assert xyz.tobytes() == smooth.vertices.tobytes() and (tris == smooth.triangles).all()
    assert (rgb == color_to_uint8(smooth.vertex_colors) / 255.0).all()
