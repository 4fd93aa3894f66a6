"""Host-side mesh post-processing against independent restatements (PLY colour rounding, cluster cleaning), and a
compile-time guard that the mesh kernels keep one rounding per fp64 operation.  No GPU needed."""
import os
import re
import shutil
import subprocess
from decimal import ROUND_HALF_UP, Decimal

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_write_ply_rounds_colour_halves_away_from_zero(tmp_path):
    """Open3D's PLY writer stores utility::ColorToUint8(c) = uint8(std::round(min(1, max(0, c)) * 255)): clamp first, then
    round half away from zero.  np.rint would round the exact halves to even.  Meshes and point clouds write the same
    vertex records."""
    from gs2mesh_b200.io import color_to_uint8, write_point_cloud_ply
    from gs2mesh_b200.mesh import PointCloud, TriangleMesh

    halves = np.array([(k + 0.5) / 255.0 for k in range(255)])
    halves = halves[halves * 255.0 == np.arange(255)[: len(halves)] + 0.5]  # products that are exactly k + 0.5
    assert len(halves) > 100
    c = np.concatenate([halves, [-1.0, -0.0, 0.0, 1e-300, 0.5 / 255, 1.0, 1.0 + 1e-12, 7.0, np.nan, np.inf, -np.inf],
                        np.random.default_rng(0).uniform(-0.1, 1.1, 300)])
    c = np.concatenate([c, np.zeros((-len(c)) % 3)]).reshape(-1, 3)

    def std_round(x):  # uint8(std::round(std::min(1., std::max(0., x)) * 255.)), exactly
        x = float(x)
        x = x if x > 0.0 else 0.0  # std::max(0., x) returns 0. unless 0. < x (so NaN -> 0)
        x = x if x < 1.0 else 1.0
        return int(Decimal(x * 255.0).quantize(Decimal(1), rounding=ROUND_HALF_UP))

    want = np.array([std_round(x) for x in c.reshape(-1)], np.uint8).reshape(c.shape)
    assert (want[: len(halves) // 3] != np.rint(halves[: len(halves) // 3 * 3] * 255.0).reshape(-1, 3)).any()
    np.testing.assert_array_equal(color_to_uint8(c), want)

    v = np.arange(len(c) * 3, dtype=np.float64).reshape(-1, 3)
    path = TriangleMesh(v, np.zeros((0, 3), np.int64), vertex_colors=c).write_ply(str(tmp_path / "m.ply"))
    body = open(path, "rb").read().split(b"end_header\n")[1]
    rec = np.frombuffer(body, dtype=[("xyz", "<f8", (3,)), ("rgb", "u1", (3,))])
    np.testing.assert_array_equal(rec["xyz"], v)
    np.testing.assert_array_equal(rec["rgb"], want)
    for cloud in (PointCloud(v, c).write_ply(str(tmp_path / "p.ply")), write_point_cloud_ply(str(tmp_path / "q.ply"), v, c)):
        assert open(cloud, "rb").read().split(b"end_header\n")[1] == body


def _clean_by_union_find(v, t, colors, threshold):
    """tsdf_utils.py:130-140 in plain Python: triangles sharing an edge (either orientation) are in one cluster, clusters
    with fewer than `threshold` triangles go, then unreferenced vertices go, both keeping order."""
    parent = list(range(len(t)))

    def find(i):
        while parent[i] != i:
            parent[i] = parent[parent[i]]
            i = parent[i]
        return i

    first = {}
    for i, (a, b, c) in enumerate(t.tolist()):
        for e in ((a, b), (b, c), (c, a)):
            e = (min(e), max(e))
            if e in first:
                parent[find(i)] = find(first[e])
            else:
                first[e] = i
    size = {}
    for i in range(len(t)):
        size[find(i)] = size.get(find(i), 0) + 1
    kept = [tri for i, tri in enumerate(t.tolist()) if not size[find(i)] < threshold]
    used = sorted({k for tri in kept for k in tri})
    new = {old: i for i, old in enumerate(used)}
    return v[used], np.array([[new[k] for k in tri] for tri in kept], np.int64).reshape(-1, 3), colors[used]


def _random_mesh(rng):
    """Components of random sizes around the cleaning threshold, fans of exactly 166 and 167 triangles, non-manifold
    edges, duplicate and degenerate triangles, isolated vertices; shuffled."""
    nv = 4000
    ids = rng.permutation(nv)
    tris, at = [], 0
    for n_tri in list(rng.integers(1, 400, 25)) + [1, 1, 2, 3]:
        g = ids[at:at + int(rng.integers(3, 40))]
        at += len(g)
        tris.append(rng.choice(g, (int(n_tri), 3)))  # random triples of a small vertex set: non-manifold, degenerate
    t = np.concatenate(tris)
    tris = [t, t[rng.integers(0, len(t), 40)]]  # duplicate triangles
    for n_tri in (166, 167):
        g = ids[at:at + n_tri + 2]
        at += len(g)
        tris.append(np.column_stack([np.full(n_tri, g[0]), g[1:-1], g[2:]]))  # a fan: consecutive triangles share an edge
    t = np.concatenate(tris)
    t = t[rng.permutation(len(t))]  # ids[at:] are never used: isolated vertices
    return rng.normal(size=(nv, 3)), t, rng.random((nv, 3))


@pytest.mark.parametrize("seed", range(4))
def test_remove_small_clusters_matches_union_find(seed):
    from gs2mesh_b200.mesh import TriangleMesh

    rng = np.random.default_rng(seed)
    v, t, col = _random_mesh(rng)
    threshold = 50 / 0.3  # TSDF_cleaning_threshold / TSDF_scale: 166.67, not an integer
    got = TriangleMesh(v, t, vertex_colors=col, vertex_normals=-v).remove_small_clusters(threshold)
    wv, wt, wc = _clean_by_union_find(v, t, col, threshold)
    assert 0 < len(wt) < len(t)
    np.testing.assert_array_equal(got.vertices, wv)
    np.testing.assert_array_equal(got.triangles, wt)
    np.testing.assert_array_equal(got.vertex_colors, wc)
    np.testing.assert_array_equal(got.vertex_normals, -wv)


def test_mesh_kernels_compile_without_fp64_fma(tmp_path):
    """Vertex positions, colours and normals equal Open3D's doubles only with one rounding per operation: nvcc would
    contract `a + b*c` into an fma.rn.f64, which rounds once instead of twice."""
    from gs2mesh_b200 import build

    nvcc = shutil.which(os.environ.get("NVCC", "nvcc"))
    if nvcc is None:
        pytest.skip("nvcc is not on PATH")
    flags = [f for f in build.NVCC_FLAGS if f not in ("-shared", "-ldl")]
    ptx = tmp_path / "gsb_mesh.ptx"
    subprocess.run([nvcc, *flags, "-ptx", "-o", str(ptx), os.path.join(build.CSRC, "gsb_mesh.cu")], check=True,
                   capture_output=True)
    text = ptx.read_text()
    entries = re.findall(r"\.entry\s+(\w+)\(", text)
    assert any("mc_vertices_kernel" in e for e in entries) and any("mesh_vertex_normals_kernel" in e for e in entries)
    assert "fma.rn.f64" not in text
