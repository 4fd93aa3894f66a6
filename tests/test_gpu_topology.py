"""The topology queries on the GPU (gsb_mesh_edge_topology, gsb_mesh_non_manifold_vertices, gsb_mesh_self_intersections
and gsb_mesh_area_volume through TriangleMesh) against the numpy restatement in tests/topology_oracle.py: edge, vertex
and pair lists equal exactly, booleans and the Euler characteristic equal, area and volume equal bit for bit."""
import math

import numpy as np
import pytest

from tests import topology_oracle as to
from tests.test_topology_cpu import cube, moebius, torus, uv_sphere

pytestmark = pytest.mark.gpu


def _same(got, want):
    got, want = np.asarray(got), np.asarray(want)
    assert got.dtype == want.dtype and got.shape == want.shape
    assert got.tobytes() == want.tobytes()


def _check(dev, v, t, intersections=True):
    """Every query against the restatement; returns the GPU mesh.  intersections=False skips the self-intersection
    comparison (for inputs where the restatement's one-axis sweep would visit billions of pairs)."""
    from gs2mesh_b200.mesh import TriangleMesh

    v, t = np.asarray(v, np.float64).reshape(-1, 3), np.asarray(t, np.int64).reshape(-1, 3)
    mesh = TriangleMesh(v.copy(), t.copy(), device=dev)
    nv = len(v)
    for allow in (True, False):
        want, e = to.edges(t, nv, allow)
        _same(mesh.get_non_manifold_edges(allow), want)
        assert mesh.is_edge_manifold(allow) is (len(want) == 0)
    assert mesh.euler_poincare_characteristic() == nv + len(t) - e
    nmv = to.non_manifold_vertices(t, nv)
    _same(mesh.get_non_manifold_vertices(), nmv)
    assert mesh.is_vertex_manifold() is (len(nmv) == 0)
    orientable = to.is_orientable(t, nv)
    assert mesh.is_orientable() is orientable
    area = to.surface_area(v, t)
    assert mesh.get_surface_area() == area and math.copysign(1, mesh.get_surface_area()) == math.copysign(1, area)
    if intersections:
        pairs = to.self_intersecting_triangles(v, t)
        _same(mesh.get_self_intersecting_triangles(), pairs)
        assert mesh.is_self_intersecting() is (len(pairs) > 0)
        watertight = len(to.edges(t, nv, False)[0]) == 0 and len(nmv) == 0 and len(pairs) == 0
        assert mesh.is_watertight() is watertight
        if not watertight:
            with pytest.raises(RuntimeError, match=r"^The mesh is not watertight, and the volume cannot be computed\.$"):
                mesh.get_volume()
        elif not orientable:
            with pytest.raises(RuntimeError, match=r"^The mesh is not orientable, and the volume cannot be computed\.$"):
                mesh.get_volume()
        else:
            assert mesh.get_volume() == abs(to.signed_volume(v, t))
    # the mesh is left unchanged
    assert mesh.vertices.tobytes() == v.tobytes() and mesh.triangles.tobytes() == t.tobytes()
    return mesh


def _stats(mesh):
    """(pairs, candidate pairs, registrations, grid level) of the last self-intersection pass."""
    from gs2mesh_b200.mesh import _Topology

    with _Topology(mesh) as q:
        q.self_intersections()
        return q.stats


@pytest.mark.parametrize("seed", range(2))
def test_adversarial_meshes(gsb_lib, cuda_device, seed):
    """Random large triangles with degenerate, repeated, rotated and reversed ones: tens of millions of candidate pairs."""
    from tests.test_gpu_simplify import _adversarial

    rng = np.random.default_rng(seed)
    v, t = _adversarial(rng, nv=2500, nt=4500, scale=1.0 + seed)
    mesh = _check(cuda_device, v, t)
    pairs, candidates, registrations, level = _stats(mesh)
    assert candidates > 10_000_000 and pairs > 1_000_000 and 0 < registrations <= 4 * len(t)
    assert len(mesh.get_non_manifold_edges()) > 0 and len(mesh.get_non_manifold_vertices()) > 0


def test_closed_meshes(gsb_lib, cuda_device):
    for (v, t), chi in ((uv_sphere(40, 60), 2), (torus(60, 40), 0), (cube(0.5), 2)):
        mesh = _check(cuda_device, v, t)
        assert mesh.is_watertight() and mesh.is_orientable() and mesh.euler_poincare_characteristic() == chi
    assert _check(cuda_device, *cube(0.5)).get_volume() == 0.125
    v, t = moebius()
    assert not _check(cuda_device, v, t).is_orientable()


def test_shuffled_grid_over_1m_triangles(gsb_lib, cuda_device):
    """A height-field sheet: manifold with a boundary, orientable, Euler 1, no self-intersections.  The restatement's
    sweep along x would visit about 4e9 pairs on it, so its pairs are checked by the known answer."""
    from tests.test_gpu_mesh_clean import _shuffled_grid

    v, t = _shuffled_grid(710, np.random.default_rng(14))
    assert len(t) >= 1_000_000
    mesh = _check(cuda_device, v, t, intersections=False)
    assert mesh.euler_poincare_characteristic() == 1 and mesh.is_orientable() and mesh.is_edge_manifold()
    assert mesh.get_self_intersecting_triangles().shape == (0, 2) and not mesh.is_watertight()
    pairs, candidates, registrations, _ = _stats(mesh)
    assert pairs == 0 and candidates > len(t) and registrations <= 4 * len(t)
    flipped = t.copy()
    flipped[::7] = flipped[::7, ::-1]  # inconsistently wound, still orientable
    assert _check(cuda_device, v, flipped, intersections=False).is_orientable()


def test_moebius_strip_of_1m_triangles(gsb_lib, cuda_device):
    v, t = moebius(500_000, 1e-3)
    t = t[np.random.default_rng(15).permutation(len(t))]
    mesh = _check(cuda_device, v, t, intersections=False)
    assert not mesh.is_orientable() and mesh.is_edge_manifold() and mesh.is_vertex_manifold()
    with pytest.raises(RuntimeError, match="not watertight"):
        mesh.get_volume()
    # an embedded strip: no pairs.  The restatement's sweep is too slow on the whole strip (slivers 2e-3 wide and 1.3e-5
    # long), so it checks the pairs on 100,000 of the shuffled triangles, scattered along the strip
    assert mesh.get_self_intersecting_triangles().shape == (0, 2)
    pairs, candidates, _, _ = _stats(mesh)
    assert pairs == 0 and candidates > len(t)
    assert not _check(cuda_device, v, t[:100_000]).is_self_intersecting()


def test_fused_scene_raw_simplified_sharpened(gsb_lib, cuda_device, tmp_path):
    from tests.test_gpu_mesh_clean import _fused_stage

    stage = _fused_stage(tmp_path, cuda_device, 50)
    stage.run()
    stage.extract_mesh()
    stage.clean_mesh()
    mesh = stage.cleaned_mesh
    assert len(mesh.triangles) > 1000
    extent = float(np.max(mesh.vertices.max(axis=0) - mesh.vertices.min(axis=0)))
    for m in (mesh, mesh.simplify_vertex_clustering(extent / 60), mesh.filter_sharpen(2, 0.5)):
        # the restatement's sweep visits about n^1.5 pairs on a surface: its pairs are compared on the first 20,000
        # triangles, every other query on the whole mesh
        _check(cuda_device, m.vertices, m.triangles, intersections=len(m.triangles) <= 20_000)
        _check(cuda_device, m.vertices, m.triangles[:20_000])


def test_one_triangle_overlapping_every_other(gsb_lib, cuda_device):
    rng = np.random.default_rng(20)
    n = 20_000
    c = rng.uniform(-1, 1, size=(n, 3)) * [1, 1, 0.2]
    v = (c[:, None, :] + rng.normal(scale=0.01, size=(n, 3, 3))).reshape(-1, 3)
    big = np.array([[-3, -3, 0.0], [6, -3, 0.0], [-3, 6, 0.0]])
    v = np.concatenate([v, big])
    t = np.concatenate([np.arange(3 * n).reshape(n, 3), [[3 * n, 3 * n + 1, 3 * n + 2]]])
    mesh = _check(cuda_device, v, t)
    hits = mesh.get_self_intersecting_triangles()
    assert (hits[:, 1] == n).sum() > 100


def test_thousands_of_triangles_through_one_point(gsb_lib, cuda_device):
    rng = np.random.default_rng(21)
    n = 3000
    d = rng.normal(size=(n, 2, 3))
    v = np.concatenate([-(d[:, 0] + d[:, 1]), d[:, 0], d[:, 1]], axis=1).reshape(-1, 3)  # centroid at the origin
    t = np.arange(3 * n).reshape(n, 3)
    mesh = _check(cuda_device, v, t)
    pairs, candidates, _, _ = _stats(mesh)
    assert pairs > n * (n - 1) // 4 and candidates >= n * (n - 1) // 2


def test_fan_of_120000_triangles(gsb_lib, cuda_device):
    """Every triangle holds the centre vertex, so every pair is skipped by the shared index and the known answer is no
    pairs (the restatement's sweep would visit all 7.2e9 pairs).  Every box holds the centre, so one grid cell holds every
    triangle: over 2^31 candidate pairs, beyond 32-bit pair offsets and in-cell indices.  The centre's link graph is one
    long path, two after a cut, a cycle when closed."""
    n = 120_000
    ang = np.linspace(0, 2 * np.pi, n + 1)[:-1]
    v = np.concatenate([[[0, 0, 0]], np.stack([np.cos(ang), np.sin(ang), 0.1 * np.sin(7 * ang)], 1)])
    t = np.stack([np.zeros(n - 1, np.int64), np.arange(1, n), np.arange(2, n + 1)], 1)
    cut = np.delete(t, n // 2, axis=0)
    closed = np.concatenate([t, [[0, n, 1]]])
    for tris in (t, cut, closed):
        mesh = _check(cuda_device, v, tris, intersections=False)
        assert mesh.get_self_intersecting_triangles().shape == (0, 2)
        assert mesh.get_non_manifold_vertices().tolist() == ([0] if tris is cut else [])
    pairs, candidates, registrations, _ = _stats(mesh)
    assert pairs == 0 and candidates >= n * (n - 1) // 2 > 2**31 and registrations <= 4 * n
    assert not mesh.is_self_intersecting()


def test_far_from_the_origin(gsb_lib, cuda_device):
    from tests.test_gpu_simplify import _adversarial

    rng = np.random.default_rng(22)
    v, t = _adversarial(rng, nv=800, nt=1500, scale=0.05)
    for offset in ((1e6, -3e6, 2.5e5), (-1.25e9, 7e8, 1e3)):
        _check(cuda_device, v + offset, t)
    s, st = uv_sphere(30, 40)
    _check(cuda_device, s * 0.01 + (3e5, -2e5, 1e5), st)


def test_empty_triangle_free_and_single_triangle(gsb_lib, cuda_device):
    from gs2mesh_b200.mesh import TriangleMesh

    for v, t in ((np.zeros((0, 3)), np.zeros((0, 3))), (np.random.default_rng(23).normal(size=(5, 3)), np.zeros((0, 3))),
                 (np.eye(3), [[0, 1, 2]]), (np.eye(3), [[0, 0, 1]])):
        _check(cuda_device, v, t)
    empty = TriangleMesh(np.zeros((0, 3)), np.zeros((0, 3)), device=cuda_device)
    assert empty.is_watertight() and empty.get_volume() == 0.0 and empty.euler_poincare_characteristic() == 0
    assert TriangleMesh(np.eye(3), np.zeros((0, 3)), device=cuda_device).euler_poincare_characteristic() == 3


def test_noisy_sphere_folded_by_sharpening(gsb_lib, cuda_device):
    from gs2mesh_b200.mesh import TriangleMesh

    v, t = uv_sphere(30, 40)
    smooth = TriangleMesh(v, t, device=cuda_device)
    assert not _check(cuda_device, v, t).is_self_intersecting()
    noisy = v + np.random.default_rng(24).normal(scale=0.002, size=v.shape)
    assert not _check(cuda_device, noisy, t).is_self_intersecting()  # the unfolded twin
    folded = TriangleMesh(noisy, t, device=cuda_device).filter_sharpen(2, 1.0)
    got = _check(cuda_device, folded.vertices, folded.triangles)
    assert got.is_self_intersecting() and not got.is_watertight()
    assert smooth.is_watertight() and abs(smooth.get_volume() - 4 / 3 * math.pi) < 0.15


def test_two_runs_give_the_same_bytes(gsb_lib, cuda_device):
    from gs2mesh_b200.mesh import TriangleMesh
    from tests.test_gpu_simplify import _adversarial

    v, t = _adversarial(np.random.default_rng(25), nv=3000, nt=6000, scale=1.0)
    mesh = TriangleMesh(v, t, device=cuda_device)
    for name in ("get_self_intersecting_triangles", "get_non_manifold_vertices", "get_non_manifold_edges"):
        a, b = getattr(mesh, name)(), getattr(mesh, name)()
        _same(a, b)
    assert mesh.get_surface_area() == mesh.get_surface_area()
    assert mesh.vertices.tobytes() == v.tobytes() and mesh.triangles.tobytes() == t.tobytes()


def test_host_mesh_runs_on_the_current_device(gsb_lib, cuda_device):
    import torch

    from gs2mesh_b200.mesh import TriangleMesh

    v, t = uv_sphere()
    with torch.cuda.device(cuda_device):
        mesh = TriangleMesh(v, t)
        assert mesh.device is None
        assert mesh.is_watertight() and mesh.get_surface_area() == to.surface_area(v, t)
        assert mesh.get_volume() == abs(to.signed_volume(v, t))


def test_errors(gsb_lib, cuda_device):
    from gs2mesh_b200.mesh import TriangleMesh

    v = np.random.default_rng(26).normal(size=(10, 3))
    with pytest.raises(ValueError, match="out of range"):
        TriangleMesh(v, [[0, 1, 10]], device=cuda_device).is_watertight()
    with pytest.raises(ValueError, match="out of range"):
        TriangleMesh(v, [[0, -1, 2]], device=cuda_device).get_non_manifold_edges()
    bad = v.copy()
    bad[3, 1] = np.nan
    for name in ("get_self_intersecting_triangles", "get_surface_area", "is_orientable"):
        with pytest.raises(ValueError, match="not finite"):
            getattr(TriangleMesh(bad, [[0, 1, 2]], device=cuda_device), name)()


def test_o3d_compat_extract_then_query(gsb_lib, cuda_device):
    """extract_triangle_mesh -> is_watertight / get_surface_area through the facade."""
    import torch

    import gs2mesh_b200.o3d_compat as o3d
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
    assert isinstance(mesh, o3d.geometry.TriangleMesh) and len(mesh.triangles) > 100
    got = _check(cuda_device, mesh.vertices, mesh.triangles)
    assert mesh.is_watertight() == got.is_watertight()
    assert mesh.get_surface_area() == to.surface_area(mesh.vertices, mesh.triangles) > 0
