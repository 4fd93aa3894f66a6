"""GPU marching cubes on constructed brick volumes vs the CPU restatement of Open3D's ExtractTriangleMesh
(oracle.extract_mesh_from_bricks), and GPU vertex normals vs a float64 restatement of TriangleMesh::ComputeVertexNormals.

The volumes are written brick by brick, so they reach what a fused sphere never does: every cube case, every seam between a
brick and its +1 neighbours, missing neighbours, weight-0 halo voxels, tsdf values of exactly 0, -0 and +-1, subnormals,
lattice indices far from the origin and at the ends of the 21-bit brick key, and voxel lengths that are not dyadic.  Bars:
edge keys, vertices, colours and normals bit for bit; triangles as sets."""
import numpy as np
import pytest

from tests.test_gpu_mesh import _canon, _rekey

pytestmark = pytest.mark.gpu

VOXEL_LENGTHS = (2.0 / 512, 0.3 / 512, 0.1 * 2.0 / 512)  # TSDF_voxel / 512 (tsdf_utils.py:51): 2 (default), 0.3, 0.2
TOP = (1 << 20) - 1  # the largest brick lattice index: its +1 neighbour cannot exist


# ----------------------------------------------------------------------------------------------------- volume fixture

def _brick(rng, tsdf=None, weight=None, with_color=True):
    """(tsdf_weight float32 [4096,2], colour float32 [4096,3] | None) from [16,16,16] arrays indexed [x,y,z]: the pool
    layout x*256 + y*16 + z (DESIGN.md section 4)."""
    t = rng.uniform(-1, 1, (16, 16, 16)) if tsdf is None else np.broadcast_to(tsdf, (16, 16, 16))
    w = rng.uniform(0.5, 4, (16, 16, 16)) if weight is None else np.broadcast_to(weight, (16, 16, 16))
    tw = np.stack([np.asarray(t, np.float32).reshape(4096), np.asarray(w, np.float32).reshape(4096)], -1)
    col = rng.uniform(0, 255, (4096, 3)).astype(np.float32) if with_color else None
    return tw, col


@pytest.fixture
def brick_volume(cuda_device):
    """units {(bx,by,bz): (tsdf_weight [4096,2], colour [4096,3] | None)} -> a TSDFVolume holding exactly those bricks:
    opened with find_bricks(insert=True), pool slots written at the returned slots."""
    import torch

    from gs2mesh_b200.tsdf import TSDFVolume

    def make(units, voxel_length, with_color):
        vol = TSDFVolume(voxel_length, 4 * voxel_length, (0, 0, 0), (1, 1, 1), with_color=with_color, device=cuda_device,
                         pool_bricks=max(64, len(units)))
        if units:
            slots = vol.find_bricks(np.array(list(units), np.int32), insert=True).long()
            assert (slots >= 0).all() and len(set(slots.tolist())) == len(units)
            vol.pool()[slots] = torch.from_numpy(np.stack([u[0] for u in units.values()])).to(cuda_device)
            if with_color:
                col = np.zeros((len(units), 4096, 4), np.float32)
                col[..., :3] = np.stack([u[1] for u in units.values()])
                vol.color.view(vol.pool_bricks, 4096, 4)[slots] = torch.from_numpy(col).to(cuda_device)
        assert vol.num_bricks() == len(units)
        torch.cuda.synchronize()
        return vol

    return make


def _dense(units, b0, nb):
    """The oracle's dense window over bricks [b0, b0 + nb): row-major over (bx,by,bz), missing bricks zero."""
    total = int(np.prod(nb))
    tw = np.zeros((total, 4096, 2), np.float32)
    col = np.zeros((total, 4096, 3), np.float32)
    for (bx, by, bz), (t, c) in units.items():
        r = (bx - b0[0], by - b0[1], bz - b0[2])
        if all(0 <= r[k] < nb[k] for k in range(3)):
            i = (r[0] * nb[1] + r[1]) * nb[2] + r[2]
            tw[i] = t
            if c is not None:
                col[i] = c
    return tw, col


def _window(units):
    """(b0, nb) of the bricks' bounding box plus the +1 layer their cubes reach into."""
    idx = np.array(list(units), np.int64)
    lo, hi = idx.min(0), idx.max(0)
    return tuple(int(v) for v in lo), tuple(int(v) for v in hi - lo + 2)


def _lattice(mesh):
    """Global lattice voxel (gx,gy,gz) of every vertex's edge key."""
    (k0, kn) = mesh.key_window
    lin = mesh.edge_keys.astype(np.int64) // 3
    ny, nz = kn[1] * 16, kn[2] * 16
    g = np.stack([lin // (nz * ny), (lin // nz) % ny, lin % nz], 1)
    return g + np.array(k0, np.int64) * 16


def _compare(oracle, mesh, units, vl, with_color, b0=None, nb=None):
    """The part of `mesh` inside window (b0, nb) (default: all of `units`) equals the oracle's mesh of that window.
    Returns the number of triangles compared."""
    if b0 is None:
        b0, nb = _window(units)
    tw, col = _dense(units, b0, nb)
    ref = oracle.extract_mesh_from_bricks(tw, b0, nb, vl, color=col if with_color else None)
    nx, ny, nz = (n * 16 for n in nb)
    ref_key = ((ref["keys"][:, 0] * ny + ref["keys"][:, 1]) * nz + ref["keys"][:, 2]) * 3 + ref["keys"][:, 3]
    order = np.argsort(ref_key)
    g = _lattice(mesh) - np.array(b0, np.int64) * 16
    sel = ((g >= 0) & (g < np.array([nx, ny, nz]))).all(1)
    mine = _rekey(mesh, b0, nb)[sel]
    np.testing.assert_array_equal(mine, ref_key[order])  # same edge keys = same vertex set, in the same order
    np.testing.assert_array_equal(mesh.vertices[sel], ref["vertices"][order])
    if with_color:
        assert mesh.vertex_colors.dtype == np.float64
        np.testing.assert_array_equal(mesh.vertex_colors[sel], ref["colors"][order])
    else:
        assert mesh.vertex_colors is None
    rank = np.empty(len(order), np.int64)
    rank[order] = np.arange(len(order))
    loc = np.full(len(sel), -1, np.int64)
    loc[sel] = np.arange(int(sel.sum()))
    t = loc[mesh.triangles]
    t = t[(t >= 0).all(1)]
    assert len(t) == len(ref["triangles"])
    want = _canon(map(tuple, rank[ref["triangles"]]))
    assert len(want) == len(ref["triangles"]) and _canon(map(tuple, t)) == want
    return len(t)


def _cube_cases(tw, nb):
    """(case, valid) of every cube of a dense window, with the oracle's rules: skip if any corner has weight 0 (outside
    the window counts as weight 0), inside <=> tsdf < 0."""
    from oracle.oracle import _mc_tables

    shift = _mc_tables()[0]
    nbx, nby, nbz = nb
    g = tw.reshape(nbx, nby, nbz, 16, 16, 16, 2).transpose(0, 3, 1, 4, 2, 5, 6).reshape(nbx * 16, nby * 16, nbz * 16, 2)
    fp, wp = (np.pad(g[..., k], ((0, 1),) * 3) for k in (0, 1))
    X, Y, Z = g.shape[:3]
    case = np.zeros((X, Y, Z), np.int32)
    valid = np.ones((X, Y, Z), bool)
    for i, (sx, sy, sz) in enumerate(shift):
        valid &= wp[sx:sx + X, sy:sy + Y, sz:sz + Z] != 0
        case |= (fp[sx:sx + X, sy:sy + Y, sz:sz + Z] < 0).astype(np.int32) << i
    return case, valid


def _extract(vol):
    from gs2mesh_b200.mesh import extract_triangle_mesh

    return extract_triangle_mesh(vol)


# ----------------------------------------------------------------------------------------------------- extraction

def test_every_cube_case_and_every_seam(oracle, gsb_lib, brick_volume):
    """Random-sign tsdf in a 3x3x3 block of bricks: all 254 non-trivial cube cases occur, and cubes straddling each of
    the 7 seam kinds (x, y, z, xy, xz, yz, xyz: the halo staged from the +1 neighbours) are active."""
    rng = np.random.default_rng(1)
    units = {(bx, by, bz): _brick(rng) for bx in (-1, 0, 1) for by in (-1, 0, 1) for bz in (-1, 0, 1)}
    b0, nb = _window(units)
    case, valid = _cube_cases(_dense(units, b0, nb)[0], nb)
    active = valid & (case != 0) & (case != 255)
    assert set(np.unique(case[active]).tolist()) == set(range(1, 255))
    x, y, z = np.nonzero(active)
    kinds = {(int(a), int(b), int(c)) for a, b, c in zip(x % 16 == 15, y % 16 == 15, z % 16 == 15)}
    assert kinds == {(a, b, c) for a in (0, 1) for b in (0, 1) for c in (0, 1)}  # the 7 seam kinds and the brick interior
    vl = 0.3 / 512
    n = _compare(oracle, _extract(brick_volume(units, vl, True)), units, vl, True)
    assert n > 200000


NEIGHBOURS = [(dx, dy, dz) for dx in (0, 1) for dy in (0, 1) for dz in (0, 1) if (dx, dy, dz) != (0, 0, 0)]


@pytest.mark.parametrize("absent", NEIGHBOURS, ids=lambda d: "absent_" + "".join("xyz"[k] for k in range(3) if d[k]))
def test_missing_neighbour_and_weight0_halo(oracle, gsb_lib, brick_volume, absent):
    """One +1 neighbour of brick (0,0,0) is a hash miss; on the halo planes the present neighbours hand to (0,0,0), a
    third of the voxels have weight 0."""
    rng = np.random.default_rng(10 + NEIGHBOURS.index(absent))
    units = {(0, 0, 0): _brick(rng)}
    for d in NEIGHBOURS:
        if d == absent:
            continue
        tw, col = _brick(rng)
        t = tw.reshape(16, 16, 16, 2)
        plane = np.ones((16, 16, 16), bool)
        for k in range(3):
            if d[k]:
                plane &= (np.arange(16) == 0).reshape([16 if j == k else 1 for j in range(3)])
        t[..., 1][plane & (rng.random((16, 16, 16)) < 1 / 3)] = 0.0
        units[d] = (tw, col)
    vl = 2.0 / 512
    assert _compare(oracle, _extract(brick_volume(units, vl, True)), units, vl, True) > 10000


SPECIAL = np.array([0.0, -0.0, 1.0, -1.0, 0.5, -0.5, 0.25, -0.25, 1e-45, -1e-45, 3e-39, -3e-39, 1.2e-38, -1.2e-38, 0.1, -0.7],
                   np.float32)


def _special_units(rng, with_color=True):
    """2x2x2 bricks of tsdf drawn from exact zeros of both signs, +-1, equal magnitudes and subnormals; 5% weight 0."""
    units = {}
    for b in [(bx, by, bz) for bx in (0, 1) for by in (-1, 0) for bz in (3, 4)]:
        t = SPECIAL[rng.integers(0, len(SPECIAL), (16, 16, 16))]
        w = np.where(rng.random((16, 16, 16)) < 0.05, 0.0, rng.integers(1, 4, (16, 16, 16))).astype(np.float32)
        units[b] = _brick(rng, t, w, with_color)
    return units


@pytest.mark.parametrize("with_color", [True, False], ids=["color", "nocolor"])
@pytest.mark.parametrize("vl", VOXEL_LENGTHS, ids=["vl2", "vl0.3", "vl0.2"])
def test_special_tsdf_values(oracle, gsb_lib, brick_volume, vl, with_color):
    rng = np.random.default_rng(20)
    units = _special_units(rng, with_color)
    assert _compare(oracle, _extract(brick_volume(units, vl, with_color)), units, vl, with_color) > 10000


CLUSTERS = {
    # negative indices near the origin + a cluster near (-70000, 3, 2^20 - 2) that reaches the last brick index on z
    "far": [[(bx, by, bz) for bx in (-2, -1) for by in (-1, 0) for bz in (-3, -2)],
            [(bx, by, bz) for bx in (-70000, -69999) for by in (3, 4) for bz in (TOP - 1, TOP)]],
    # both ends of the z lattice: the key window is 2^21 + 1 bricks long
    "lattice_ends": [[(7, -5, -(1 << 20)), (7, -5, -(1 << 20) + 1)], [(7, -5, TOP - 1), (8, -5, TOP)]],
}


@pytest.mark.parametrize("name", sorted(CLUSTERS))
def test_far_apart_clusters(oracle, gsb_lib, brick_volume, name):
    """Bricks far from the origin and at the ends of the brick key range; the mesh is compared cluster by cluster."""
    rng = np.random.default_rng(30)
    clusters = [{b: _brick(rng) for b in c} for c in CLUSTERS[name]]
    units = {k: v for c in clusters for k, v in c.items()}
    vl = 0.3 / 512
    mesh = _extract(brick_volume(units, vl, True))
    n = [_compare(oracle, mesh, units, vl, True, *_window(c)) for c in clusters]
    assert min(n) > 1000 and sum(n) == len(mesh.triangles)


@pytest.mark.parametrize("with_color", [True, False], ids=["color", "nocolor"])
@pytest.mark.parametrize("kind", ["no_bricks", "zero_weight", "all_inside", "all_outside", "signed_zeros"])
def test_empty_meshes(gsb_lib, brick_volume, cuda_device, kind, with_color):
    rng = np.random.default_rng(40)
    blocks = [(bx, by, bz) for bx in (0, 1) for by in (0, 1) for bz in (0, 1)]
    tsdf = {"zero_weight": None, "all_inside": -0.5, "all_outside": 0.5,
            "signed_zeros": np.where(rng.random((16, 16, 16)) < 0.5, np.float32(0.0), np.float32(-0.0))}
    units = {} if kind == "no_bricks" else {
        b: _brick(rng, tsdf[kind], 0.0 if kind == "zero_weight" else 1.0, with_color) for b in blocks}
    mesh = _extract(brick_volume(units, 2.0 / 512, with_color))
    assert mesh.vertices.shape == (0, 3) and mesh.vertices.dtype == np.float64
    assert mesh.triangles.shape == (0, 3) and mesh.triangles.dtype == np.int64
    if with_color:
        assert mesh.vertex_colors.shape == (0, 3)
    else:
        assert mesh.vertex_colors is None
    mesh.compute_vertex_normals(cuda_device)
    assert mesh.vertex_normals.shape == (0, 3)


def test_key_window_limit_is_a_clear_error(gsb_lib, brick_volume):
    """Edge keys index voxels of the open bricks' bounding box in 63 bits: bricks 2^17 apart on all three axes do not
    fit, and extraction says so instead of failing with a bare 'bad arguments'."""
    from gs2mesh_b200 import _lib

    rng = np.random.default_rng(50)
    units = {(0, 0, 0): _brick(rng), (1 << 17, 1 << 17, 1 << 17): _brick(rng)}
    with pytest.raises(_lib.GsbError, match=r"too large for 63-bit edge keys \(16\^3 \* nbx \* nby \* nbz \* 3 must be < 9e18\)"):
        _extract(brick_volume(units, 2.0 / 512, True))


# ----------------------------------------------------------------------------------------------------- vertex normals

def open3d_vertex_normals(v, t):
    """TriangleMesh::ComputeVertexNormals(normalized=true) of Open3D 0.17 in float64: triangle normals
    (v1-v0).cross(v2-v0) without contraction, added to vertices t0, t1, t2 of triangle 0, 1, 2, ... in that order, then
    MeshBase::NormalizeNormals(): Eigen's normalize() divides by sqrt((x*x + y*y) + z*z) only when that is > 0, and a
    normal whose x is NaN becomes (0,0,1).  A zero sum stays (0,0,0)."""
    v = np.asarray(v, np.float64)
    t = np.asarray(t, np.int64).reshape(-1, 3)
    a, b = v[t[:, 1]] - v[t[:, 0]], v[t[:, 2]] - v[t[:, 0]]
    n = np.stack([a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1], a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2],
                  a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]], 1)
    acc = np.zeros_like(v)
    np.add.at(acc, t.reshape(-1), np.repeat(n, 3, axis=0))  # ufunc.at applies the index list in order: triangle order
    sq = (acc[:, 0] * acc[:, 0] + acc[:, 1] * acc[:, 1]) + acc[:, 2] * acc[:, 2]
    pos = sq > 0
    acc[pos] /= np.sqrt(sq[pos])[:, None]
    acc[np.isnan(acc[:, 0])] = (0.0, 0.0, 1.0)
    return acc


def _normals_twice(mesh, dev):
    mesh.compute_vertex_normals(dev)
    first = mesh.vertex_normals.copy()
    mesh.compute_vertex_normals(dev)
    np.testing.assert_array_equal(mesh.vertex_normals, first)  # the same bits on every call
    return first


def test_normals_of_degenerate_meshes(gsb_lib, cuda_device):
    """Zero-area triangles, repeated indices, unreferenced vertices, coincident vertices and one vertex in 20000
    triangles (a summation order that atomics would scramble)."""
    from gs2mesh_b200.mesh import TriangleMesh

    rng = np.random.default_rng(60)
    v = rng.normal(size=(3000, 3)) * np.array([1.0, 1e-3, 1e3])
    v[100:110] = v[99]  # coincident vertices
    v[200:210] = v[200] + np.outer(np.arange(10), [0.3, -0.1, 0.7])  # collinear points
    # vertices 101-106, 201 and 209 are only in zero-area triangles, vertices >= 2500 in none
    pool = np.setdiff1d(np.arange(1, 2500), np.r_[99:111, 199:211])
    t = [rng.choice(pool, (20000, 3)),
         np.column_stack([np.zeros(20000, np.int64), rng.choice(pool, (20000, 2))]),  # a 20000-triangle fan around vertex 0
         [[101, 102, 103], [104, 104, 105], [106, 106, 106], [200, 203, 207], [201, 201, 209]]]
    mesh = TriangleMesh(v, np.concatenate([np.asarray(x, np.int64) for x in t]))
    got = _normals_twice(mesh, cuda_device)
    want = open3d_vertex_normals(mesh.vertices, mesh.triangles)
    np.testing.assert_array_equal(got, want)
    assert (got[[101, 102, 103, 104, 105, 106, 201, 209]] == 0).all() and (got[2500:] == 0).all()


def test_normals_of_extracted_meshes(gsb_lib, brick_volume, cuda_device):
    """Meshes of the special-value volume: corners with tsdf exactly 0 put vertices on top of each other, which makes
    zero-area triangles."""
    rng = np.random.default_rng(20)
    for vl in VOXEL_LENGTHS:
        mesh = _extract(brick_volume(_special_units(rng), vl, True))
        v, t = mesh.vertices, mesh.triangles
        area2 = np.cross(v[t[:, 1]] - v[t[:, 0]], v[t[:, 2]] - v[t[:, 0]])
        assert (area2 == 0).all(1).sum() > 100
        want = open3d_vertex_normals(v, t)
        assert (want == 0).all(1).sum() > 100  # vertices whose triangles all have zero area
        np.testing.assert_array_equal(_normals_twice(mesh, cuda_device), want)
