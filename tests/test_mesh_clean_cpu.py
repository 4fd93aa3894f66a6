"""Cluster-cleaning entry points refuse bad arguments before anything is enqueued (no GPU needed), and the two numpy /
scipy properties the GPU path's equality with the host path rests on."""
import ctypes as C

import numpy as np
import pytest

from gs2mesh_b200 import _lib
from tests.test_mesh_cpu import _random_mesh

P = 256  # any non-NULL pointer: validation only checks pointers for NULL and dereferences none of them


def test_workspace_bytes(gsb_lib):
    assert gsb_lib.gsb_mesh_cluster_workspace_bytes(-1, 10) == 0
    assert gsb_lib.gsb_mesh_cluster_workspace_bytes(10, -1) == 0
    assert gsb_lib.gsb_mesh_cluster_workspace_bytes(2**31, 10) == 0
    assert gsb_lib.gsb_mesh_cluster_workspace_bytes(10, 2**31) == 0
    assert gsb_lib.gsb_mesh_cluster_workspace_bytes(10, 0) == 0  # triangles need vertices
    small = gsb_lib.gsb_mesh_cluster_workspace_bytes(1000, 600)
    big = gsb_lib.gsb_mesh_cluster_workspace_bytes(1_000_000, 600_000)
    # three (8 B key, 4 B triangle) pairs per triangle, double-buffered, + parent / root flag / rank
    assert 0 < small < big and big >= 1_000_000 * (3 * 2 * 12 + 3 * 4)


def test_argument_validation_without_gpu(gsb_lib):
    launches = gsb_lib.gsb_kernel_launch_count()
    ws = gsb_lib.gsb_mesh_cluster_workspace_bytes(100, 50)

    def clusters(nt=100, nv=50, tri=P, xyz=None, work=P, labels=P, counts=P, n=P, area=None):
        return gsb_lib.gsb_mesh_clusters(tri, nt, nv, xyz, work, ws, labels, counts, n, area, None)

    def remove(nt=100, nv=50, tri=P, labels=P, counts=P, work=P, out=P, ids=P, sizes=P):
        return gsb_lib.gsb_mesh_remove_small_clusters(tri, nt, nv, labels, counts, 166.67, work, ws, out, ids, sizes, None)

    bad = [dict(tri=None), dict(work=None), dict(labels=None), dict(counts=None), dict(n=None), dict(area=P),
           dict(nt=-1), dict(nv=-1), dict(nt=2**31), dict(nt=2**40), dict(nv=2**31), dict(nv=0)]
    for kw in bad:
        assert clusters(**kw) == _lib.GSB_ERR_INVALID, kw
        assert gsb_lib.gsb_last_error().startswith(b"mesh_clusters: ")
    assert clusters(nt=2**31) == _lib.GSB_ERR_INVALID and b"32-bit" in gsb_lib.gsb_last_error()
    assert clusters(nt=-1) == _lib.GSB_ERR_INVALID and b"negative" in gsb_lib.gsb_last_error()
    assert clusters(nv=0) == _lib.GSB_ERR_INVALID and b"no vertices" in gsb_lib.gsb_last_error()
    assert gsb_lib.gsb_mesh_clusters(P, 100, 50, None, P, ws - 1, P, P, P, None, None) == _lib.GSB_ERR_WORKSPACE

    bad = [dict(tri=None), dict(labels=None), dict(counts=None), dict(work=None), dict(out=None), dict(ids=None),
           dict(sizes=None), dict(nt=-1), dict(nv=-5), dict(nt=2**31), dict(nv=2**31), dict(nv=0)]
    for kw in bad:
        assert remove(**kw) == _lib.GSB_ERR_INVALID, kw
        assert gsb_lib.gsb_last_error().startswith(b"mesh_remove_small_clusters: ")
    assert gsb_lib.gsb_mesh_remove_small_clusters(P, 100, 50, P, P, 1.0, P, ws - 1, P, P, P, None) == _lib.GSB_ERR_WORKSPACE
    assert gsb_lib.gsb_kernel_launch_count() == launches  # nothing was enqueued


def test_host_cluster_labels_follow_the_smallest_triangle():
    """scipy's connected_components numbers components in the order of their smallest node, which is Open3D's BFS order
    and what the GPU's exclusive scan over root flags (root = smallest triangle) produces."""
    from gs2mesh_b200.mesh import TriangleMesh

    for seed in range(4):
        v, t, _ = _random_mesh(np.random.default_rng(seed))
        labels, counts, _ = TriangleMesh(v, t).cluster_connected_triangles()
        first = np.unique(labels, return_index=True)[1]  # smallest triangle of each label
        assert (np.diff(first) > 0).all() and first[0] == 0
        np.testing.assert_array_equal(counts, np.bincount(labels))


@pytest.mark.parametrize("n", [1, 2, 3, 7, 8, 9, 1000, 8193])
def test_numpy_triangle_area_rounding(n):
    """np.linalg.norm(axis=1) of an [n,3] array is sqrt((x*x + y*y) + z*z) and np.cross is (a1*b2 - a2*b1, a2*b0 - a0*b2,
    a0*b1 - a1*b0), one rounding per operation: the order the GPU's per-triangle area restates."""
    rng = np.random.default_rng(n)
    a = rng.normal(size=(n, 3)) * np.exp(rng.normal(size=(n, 3)) * 4)
    b = rng.normal(size=(n, 3)) * np.exp(rng.normal(size=(n, 3)) * 4)
    c = np.cross(a, b)
    want = np.stack([a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1], a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2],
                     a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]], 1)
    assert c.tobytes() == want.tobytes()
    s = c * c
    assert np.linalg.norm(c, axis=1).tobytes() == np.sqrt((s[:, 0] + s[:, 1]) + s[:, 2]).tobytes()
