"""The topology kernels (csrc/gsb_topology.cu) at the edges of tests/topology_edge_cases.py: self-intersection pairs
equal to the restatement exactly and to the exact integer intersection on every separated and crossing pair (lattice
soups, branch families, tie families, epsilon pairs); the grid's level and registrations as each grid case states,
unchanged pairs under dyadic translation and power-of-two scaling; a stray unreferenced vertex that must not stretch the
grid; 2^31-vertex edge keys and 2^28-vertex link keys through the C ABI; union and atomic storms on one edge and one
vertex; and the area / volume sum at its block seams, bit for bit and within its error bound of an exact sum."""
import math

import numpy as np
import pytest

from tests import topology_edge_cases as ec
from tests import topology_oracle as to
from tests.test_topology_cpu import moebius, uv_sphere

pytestmark = pytest.mark.gpu


def _mesh(dev, v, t):
    from gs2mesh_b200.mesh import TriangleMesh

    return TriangleMesh(np.asarray(v, np.float64).reshape(-1, 3), np.asarray(t, np.int64).reshape(-1, 3), device=dev)


def _pairs_and_stats(dev, v, t):
    """(GPU pairs, (pairs, candidates, registrations, level)), the pairs checked against the restatement."""
    from gs2mesh_b200.mesh import _Topology

    mesh = _mesh(dev, v, t)
    with _Topology(mesh) as q:
        pairs, k = q.self_intersections(with_list=True)
        stats = q.stats
    want = to.self_intersecting_triangles(v, t)
    assert pairs.dtype == want.dtype and pairs.shape == want.shape and (pairs == want).all()
    assert stats[0] == k == len(want)
    return pairs, stats


def _check_exact(pairs, P, Q, offset):
    """Triangles 2k, 2k + 1 (+ offset) are the pair (P[k], Q[k]): the GPU's verdict equals the exact one wherever the
    pair is separated or crossing."""
    n = len(P)
    cls, exact = ec.robust_class(P, Q), ec.exact_tri_tri(P, Q)
    got = ec.pair_flags(pairs, offset + 2 * np.arange(n), offset + 2 * np.arange(n) + 1, 10 ** 9)
    robust = cls != ec.CONTACT
    assert (got[robust] == exact[robust]).all()
    return cls


def _spread(P, Q, step=600):
    """Pairs (P[k], Q[k]) as triangles 2k, 2k + 1, pair k moved by (step k, 0, 0): far apart, and the per-axis sums of
    the six corners move by multiples of 6, so the normalisation (and every tie) is unchanged."""
    off = (step * np.arange(len(P)))[:, None, None] * np.array([1, 0, 0])
    T = np.stack([P + off, Q + off], axis=1).reshape(-1, 3, 3)
    return T


@pytest.mark.parametrize("seed", range(2))
def test_lattice_soups(gsb_lib, cuda_device, seed):
    T = ec.lattice_soup(seed)
    v, t = ec.soup_mesh(T)
    pairs, _ = _pairs_and_stats(cuda_device, v, t)
    i, j = ec.box_pairs(T)
    cls, exact = ec.robust_class(T[i], T[j]), ec.exact_tri_tri(T[i], T[j])
    got = ec.pair_flags(pairs, i, j, len(T))
    robust = cls != ec.CONTACT
    assert (got[robust] == exact[robust]).all() and np.bincount(cls, minlength=3).min() >= 1000


def test_branch_tie_and_epsilon_families(gsb_lib, cuda_device):
    families = list(ec.branch_family_pairs().values()) + list(ec.tie_family_pairs().values())
    P = np.concatenate([f[0] for f in families])
    Q = np.concatenate([f[1] for f in families])
    T = _spread(P, Q)
    pairs, _ = _pairs_and_stats(cuda_device, *ec.soup_mesh(T))
    cls = _check_exact(pairs, P, Q, 0)
    assert np.bincount(cls, minlength=3).min() > 100
    # epsilon pairs on their own: the normalised distance is what is built
    for (Pe, Qe, d) in ec.epsilon_pairs():
        got, _ = _pairs_and_stats(cuda_device, *ec.soup_mesh(np.stack([Pe, Qe])))
        assert len(got) == (abs(d) < 1e-6)


def _grid_cases():
    for L in (0, 1, 5, 10, 15, 19, 20, 21):
        T, level, regs, crossing = ec.level_case(L)
        yield f"level{L}", T, level, regs, crossing
    for over in (False, True):
        yield f"threshold{int(over)}", *ec.threshold_case(over=over), None
    yield "boundary", *ec.boundary_case(), None
    for axes in (1, 2, 3):
        yield f"flat{axes}", *ec.flat_case(axes), None


@pytest.mark.parametrize("case", [c[0] for c in _grid_cases()])
def test_grid_cases(gsb_lib, cuda_device, case):
    """Level and registrations as stated.  After a dyadic translation and a power-of-two scale the grid computes the
    same cells, so the candidates, registrations and level are unchanged, and so is every pair that does not hinge on
    rounding: all of them on the level and threshold cases; on the boundary case every pair that changes is a contact
    (the normalisation's rounding moves with the coordinates); the flat cases' degenerate triangles are compared with
    the restatement alone."""
    name, T, level, regs, crossing = next(c for c in _grid_cases() if c[0] == case)
    v, t = ec.soup_mesh(T)
    pairs, stats = _pairs_and_stats(cuda_device, v, t)
    assert (stats[3], stats[2]) == (level, regs)
    if crossing:
        assert {tuple(p) for p in crossing} <= {tuple(p) for p in pairs.tolist()}
    for scale, shift in ((32.0, (3.0, -5.5, 0.75)), (2.0 ** -7, (-1024.0, 0.0, 2.0 ** 20))):
        moved, moved_stats = _pairs_and_stats(cuda_device, v * scale + np.array(shift), t)
        assert moved_stats[1:] == stats[1:]
        changed = np.array(sorted({tuple(p) for p in pairs.tolist()} ^ {tuple(p) for p in moved.tolist()}), np.int64)
        if name == "boundary":
            assert len(changed) == 0 or (ec.robust_class(T[changed[:, 0]], T[changed[:, 1]]) == ec.CONTACT).all()
        elif not name.startswith("flat"):
            assert len(changed) == 0


def test_stray_unreferenced_vertex_does_not_stretch_the_grid(gsb_lib, cuda_device):
    """One vertex no triangle uses, at (1e7, 0, 0): the same pairs and the same candidates, registrations and level."""
    from gs2mesh_b200.mesh import _Topology

    v, t = uv_sphere(101, 100)
    assert len(t) == 20_000
    stray = np.concatenate([v, [[1e7, 0, 0]]])
    out = []
    for verts in (v, stray):
        with _Topology(_mesh(cuda_device, verts, t)) as q:
            pairs, _ = q.self_intersections(with_list=True)
            out.append((pairs, q.stats))
    assert (out[0][0] == out[1][0]).all() and out[0][1] == out[1][1]
    assert out[0][1][1] < 100 * len(t)  # about 29 per triangle (the poles are 100-triangle fans); n(n - 1) / 2 = 10^4 n


def _c_edges(dev, t, nv, allow):
    import torch

    from gs2mesh_b200 import _lib
    from gs2mesh_b200._lib import ptr

    L = _lib.lib()
    tri = torch.as_tensor(t, dtype=torch.int64, device=dev).contiguous()
    nt = len(t)
    work = torch.empty(L.gsb_mesh_edge_topology_workspace_bytes(nt, nv), dtype=torch.uint8, device=dev)
    out = torch.empty(3 * nt, 2, dtype=torch.int64, device=dev)
    sizes = torch.empty(3, dtype=torch.int64, device=dev)
    _lib.check(L.gsb_mesh_edge_topology(ptr(tri), nt, nv, int(allow), ptr(work), work.numel(), ptr(out), ptr(sizes),
                                        _lib.stream(dev)))
    k, e, orientable = sizes.cpu().tolist()
    return out[:k].cpu().numpy(), e, bool(orientable), work.numel()


def _c_vertices(dev, t, nv):
    import torch

    from gs2mesh_b200 import _lib
    from gs2mesh_b200._lib import ptr

    L = _lib.lib()
    tri = torch.as_tensor(t, dtype=torch.int64, device=dev).contiguous()
    nt = len(t)
    work = torch.empty(L.gsb_mesh_vertex_topology_workspace_bytes(nt, nv), dtype=torch.uint8, device=dev)
    out = torch.empty(3 * nt, dtype=torch.int64, device=dev)  # at most every referenced vertex
    count = torch.empty(1, dtype=torch.int64, device=dev)
    _lib.check(L.gsb_mesh_non_manifold_vertices(ptr(tri), nt, nv, ptr(work), work.numel(), ptr(out), ptr(count),
                                                _lib.stream(dev)))
    k = int(count.item())
    res = out[:k].cpu().numpy()
    del work
    torch.cuda.empty_cache()
    return res


def _topology_zoo():
    """Small meshes with known topology, ids below 50 near 0 and ids from 50 on moved to the top of the id range by
    _high: two tetrahedra sharing a vertex, a fin (three triangles on one edge) low and high, a Moebius strip, two
    triangles sharing only a vertex, and a triangle with a repeated id."""
    tet = np.array([[0, 2, 1], [0, 1, 3], [0, 3, 2], [1, 2, 3]])
    fin = np.array([[20, 21, 22], [20, 21, 23], [21, 20, 24]])
    parts = [tet, np.where(tet == 0, 0, tet + 10), fin, fin + 60, moebius(8)[1] + 50, np.array([[70, 71, 72], [70, 73, 74]]),
             np.array([[30, 30, 31]])]
    return np.concatenate(parts)


def _high(t, nv):
    return np.where(t >= 50, nv - 1 - (t - 50), t)


@pytest.mark.parametrize("allow", [True, False])
def test_edge_keys_at_2_31_vertices(gsb_lib, cuda_device, allow):
    """n_vertices = 2^31 - 1: stride 2^31, keys near 2^62, a 62-bit sort; ids near 0 and near 2^31 - 2.  The workspace
    does not depend on n_vertices and no vertex array is read."""
    nv = 2 ** 31 - 1
    t = _high(_topology_zoo(), nv)  # ids 50.. -> 2^31 - 2, 2^31 - 3, ...
    assert t.max() == nv - 1 and t.min() == 0
    edges, e, orientable, work = _c_edges(cuda_device, t, nv, allow)
    want, want_e = to.edges(t, nv, allow)
    assert edges.tolist() == want.tolist() and e == want_e
    assert orientable == to.is_orientable(t, nv) is False
    assert work == _c_edges(cuda_device, t, 100, allow)[3]
    assert nv + len(t) - e == to.euler_poincare(t, nv)


def test_link_keys_at_2_28_vertices(gsb_lib, cuda_device):
    """n_vertices = 2^28: link keys v nv + x up to 2^56; the workspace (about 3 GB) is sized by n_vertices."""
    nv = 2 ** 28
    t = _high(_topology_zoo(), nv)
    assert t.max() == nv - 1
    got = _c_vertices(cuda_device, t, nv)
    want = to.non_manifold_vertices(t, nv)
    assert got.tolist() == want.tolist() and len(want) > 0 and want.max() > 2 ** 27


def test_book_of_200000_triangles_on_one_edge(gsb_lib, cuda_device):
    """200,000 randomly wound triangles on the edge (0, 1): one non-manifold edge, orientable (every constraint is
    against the same centre); with a Moebius strip beside it, not orientable."""
    rng = np.random.default_rng(40)
    n = 200_000
    t = np.stack([np.zeros(n, np.int64), np.ones(n, np.int64), np.arange(2, n + 2)], axis=1)
    flip = rng.random(n) < 0.5
    t[flip] = t[flip][:, [1, 0, 2]]
    nv = n + 2
    for tris, nverts, orientable in ((t, nv, True), (np.concatenate([t, moebius(30)[1] + nv]), nv + 60, False)):
        edges, e, got_orientable, _ = _c_edges(cuda_device, tris, nverts, True)
        want, want_e = to.edges(tris, nverts, True)
        assert edges.tolist() == want.tolist() == [[0, 1]] and e == want_e
        assert got_orientable is to.is_orientable(tris, nverts) is orientable


def test_one_vertex_in_50000_separate_fans(gsb_lib, cuda_device):
    """Vertex 0 in 50,000 two-triangle fans that share nothing else: its link graph has 50,000 components, every root
    counted on one atomic counter; it is the one non-manifold vertex."""
    n = 50_000
    a = 1 + 3 * np.arange(n)
    t = np.concatenate([np.stack([np.zeros(n, np.int64), a, a + 1], 1), np.stack([np.zeros(n, np.int64), a + 1, a + 2], 1)])
    t = t[np.random.default_rng(41).permutation(len(t))]
    nv = 1 + 3 * n
    got = _c_vertices(cuda_device, t, nv)
    assert got.tolist() == to.non_manifold_vertices(t, nv).tolist() == [0]


@pytest.mark.parametrize("n", [1, 255, 256, 257, 65_535, 65_536, 65_537, 3 * 65_536 + 1])
def test_area_volume_at_block_seams(gsb_lib, cuda_device, n):
    """Bit for bit with the two-stage sum's restatement, and within its error bound of math.fsum.

    The sum is a tree of depth 8 over each block of 256 terms, then in one block thread i adds the partials i, i + 256,
    ... (r = ceil(nb / 256) of them, the first added to 0.0 exactly), then a tree of depth 8.  Each term passes
    through at most k = 8 + r + 8 rounded additions, so by the standard bound for a summation of depth k,
    |computed - exact| <= gamma_k * sum |term|, gamma_k = k u / (1 - k u), u = 2^-53.  The terms themselves are the
    restatement's, bit for bit (the bit-for-bit sums above check that)."""
    from gs2mesh_b200.mesh import _Topology

    rng = np.random.default_rng(n)
    v = rng.normal(size=(3 * n, 3)) * rng.choice([1e-3, 1.0, 1e3], size=(3 * n, 1)) + 0.5
    t = np.arange(3 * n).reshape(n, 3)
    with _Topology(_mesh(cuda_device, v, t)) as q:
        area, vol = q.area_volume()
    ta, tv = to.triangle_terms(v, t)
    assert area == to.fixed_sum(ta) and vol == to.fixed_sum(tv)
    nb = -(-n // 256)
    k = 16 + -(-nb // 256)
    u = 2.0 ** -53
    gamma = k * u / (1 - k * u)
    for got, terms in ((area, ta), (vol, tv)):
        assert abs(got - math.fsum(terms)) <= gamma * math.fsum(np.abs(terms))
