"""The read-outs of the brick TSDF volume -- the mesh, its vertex normals, clusters and cleaning, both point clouds, ray
casts, and the PLYs written from them -- depend on the voxels alone, not on how the volume holds them.

Two contents (a crossing-rich 3x3x3 block of bricks with weight-0 voxels and missing bricks, and a fused sphere) are each
built in several states whose voxels are bit-identical (checked with export_units()), but whose pool order, pool and hash
size, probe chains, dead keys (a key in the hash with no pool slot, which a lost race for the last slot leaves) or fusion
history differ.  Every read-out of every state must equal, byte for byte, that of the same bricks inserted in ascending
lattice order, and extracting twice must give the same bytes."""
import numpy as np
import pytest

from tests import tsdf_host as th
from tests.raycast_oracle import look_at
from tests.test_gpu_mesh_volumes import _brick
from tests.test_gpu_pointcloud import _crossing_rich
from tests.test_gpu_tsdf_frames import _frame, _look_at, _plant_dead_key, _raycast

pytestmark = pytest.mark.gpu

VL = 2.0 / 512
TRUNC = 4 * VL
BLOCK = [(bx, by, bz) for bx in (-1, 0, 1) for by in (-1, 0, 1) for bz in (-1, 0, 1)]
MISSING = [(0, 0, 0), (1, -1, 0), (-1, 1, 1)]
SPHERE_CAMS = [(0.0, -1.0, 0.3), (0.8, -0.7, 0.5), (-0.7, -0.8, 0.1)]  # the point-cloud and ray-cast tests' sphere
NEIGHBOURS = [(dx, dy, dz) for dx in (0, 1) for dy in (0, 1) for dz in (0, 1) if (dx, dy, dz) != (0, 0, 0)]

BRICK_STATES = ["ascending", "descending", "permuted_8x_pool", "dead_keys"]
CASES = ([("block", s) for s in BRICK_STATES + ["shared_homes_wrap"]] +
         [("sphere", s) for s in BRICK_STATES + ["fused", "fused_preopened_descending", "fused_grown"]])


# ----------------------------------------------------------------------------------------------------------- contents

def _block_offset(slots):
    """The first lattice offset (k, 0, 0) at which the block's keys, in a hash table of `slots` entries, share home slots
    and one of them probes past the last slot to the start of the table (tests/tsdf_host.py restates the hash)."""
    rel = [b for b in BLOCK if b not in MISSING]
    for k in range(1000):
        homes = np.array([th.brick_hash(th.brick_key((x + k, y, z)), slots - 1) for x, y, z in rel])
        pos = th.linear_probe_positions(homes, slots)
        if len(set(homes.tolist())) <= len(homes) - 2 and (pos < homes).any():
            return k
    raise AssertionError("no offset gives shared home slots and a wrapping probe chain")


def _block(dev):
    """24 crossing-rich bricks (5% weight 0) of the 3x3x3 block at an offset whose keys collide in a 64-slot table."""
    rng = np.random.default_rng(7)
    k = _block_offset(64)
    units = {}
    for b in BLOCK:
        if b in MISSING:
            continue
        w = np.where(rng.random((16, 16, 16)) < 0.05, 0.0, rng.uniform(0.5, 4, (16, 16, 16))).astype(np.float32)
        tw, col = _brick(rng, _crossing_rich(rng), w)
        c4 = np.zeros((4096, 4), np.float32)
        c4[:, :3] = col
        units[(b[0] + k, b[1], b[2])] = (tw, c4)
    centre = (np.array([k, 0, 0]) + 0.5) * 16 * VL
    cams = [(look_at(centre + 0.3 * np.asarray(d) + (0.004, -0.003, 0.002), centre, up=(0.3, 0.5, 0.8)), 0.0, 2.0,
             (48, 40, 55.0, 55.0, 23.5, 19.5)) for d in ((1, 0, 0), (0, -1, 0.3), (-0.5, 0.4, -1))]
    return units, cams


def _sphere_frames():
    W, H, f = 96, 80, 90.0
    frames = []
    for pos in SPHERE_CAMS:
        w2c = _look_at(np.array(pos), (0.0, 0.0, 0.0))
        frames.append(_frame(_raycast(W, H, f, f, W / 2, H / 2, w2c, (0.0, 0.0, 0.0), 0.25), W, H, f, f, W / 2, H / 2, w2c))
    return frames


def _fuse(vol, frames):
    for f in frames:
        vol.integrate(vol.prepare_depth(f["depth"], f["W"], f["H"]), f["rgb"], f["W"], f["H"], *f["K"], f["w2c"])


def _volume(dev, pool):
    from gs2mesh_b200.tsdf import TSDFVolume

    return TSDFVolume(VL, TRUNC, with_color=True, device=dev, pool_bricks=pool)


def _sphere(dev):
    vol = _volume(dev, 4096)
    _fuse(vol, _sphere_frames())
    assert vol.pool_stats()["dropped_total"] == 0
    cams = [(look_at(np.array(p), (0.0, 0.0, 0.0)), 0.05, 3.0, (96, 80, 90.0, 90.0, 48.0, 40.0))
            for p in SPHERE_CAMS[1:] + [(0.3, -0.9, -0.4)]]
    return vol.export_units(), cams


# ------------------------------------------------------------------------------------------------------------- states

def _inserted(dev, units, order, pool):
    """A volume holding `units`, opened by one find_bricks(insert=True) call per brick in `order`: slot = call order."""
    import torch

    vol = _volume(dev, pool)
    slots = [int(vol.find_bricks(np.array([b], np.int32), insert=True)[0].item()) for b in order]
    assert slots == list(range(len(order)))
    idx = torch.arange(len(order), device=dev)
    vol.pool()[idx] = torch.from_numpy(np.stack([units[b][0] for b in order])).to(dev)
    vol.color.view(pool, 4096, 4)[idx] = torch.from_numpy(np.stack([units[b][1] for b in order])).to(dev)
    return vol


def _plant_dead_keys(vol, units):
    """Dead keys at one lattice position inside the bricks' bounding box and at three +1 neighbours that cubes reach, none
    of them an open brick; each at its home slot (the first free ones in sorted order)."""
    idx = np.array(sorted(units))
    lo, hi = idx.min(0), idx.max(0)
    inner = [tuple(int(v) for v in p) for p in np.stack(np.meshgrid(*[np.arange(lo[k] + 1, hi[k]) for k in range(3)],
                                                                    indexing="ij"), -1).reshape(-1, 3)]
    outer = sorted({(b[0] + d[0], b[1] + d[1], b[2] + d[2]) for b in units for d in NEIGHBOURS})
    free = lambda b: b not in units and int(vol._hash_keys[th.brick_hash(th.brick_key(b), vol.hash_slots - 1)].item()) == -1
    planted = []
    for cands, want in ((inner, 1), (outer, 3)):
        for b in filter(free, cands):
            _plant_dead_key(vol, b)
            planted.append(b)
            want -= 1
            if want == 0:
                break
    assert len(planted) == 4, planted
    return planted


def _state(dev, state, units):
    n = len(units)
    pool = max(64, n)
    asc = sorted(units)
    if state == "ascending":
        return _inserted(dev, units, asc, pool)
    if state == "descending":
        return _inserted(dev, units, asc[::-1], pool)
    if state == "permuted_8x_pool":
        perm = np.random.default_rng(3).permutation(n)
        vol = _inserted(dev, units, [asc[i] for i in perm], 8 * pool)
        assert vol.hash_slots >= 8 * _volume(dev, pool).hash_slots
        return vol
    if state == "dead_keys":
        vol = _inserted(dev, units, asc[::-1], pool)
        _plant_dead_keys(vol, units)
        return vol
    if state == "shared_homes_wrap":
        vol = _inserted(dev, units, asc, n)
        assert vol.hash_slots == 64
        table = vol._hash_keys.cpu().numpy().view(np.uint64)
        at = {int(table[p]): p for p in np.nonzero(table != np.uint64(2 ** 64 - 1))[0]}
        homes = {th.brick_key(b): th.brick_hash(th.brick_key(b), 63) for b in units}
        assert len(set(homes.values())) <= n - 2 and any(at[k] < h for k, h in homes.items())
        return vol
    frames = _sphere_frames()
    if state == "fused":
        vol = _volume(dev, 4096)
    elif state == "fused_preopened_descending":
        vol = _inserted(dev, {b: (np.zeros((4096, 2), np.float32), np.zeros((4096, 4), np.float32)) for b in asc}, asc[::-1],
                        4096)
    else:  # fused_grown: a pool far too small, grown by ensure_capacity() and fused again, as TSDF.run() does
        vol = _volume(dev, n // 3)
        for _ in range(4):
            _fuse(vol, frames)
            if vol.ensure_capacity():
                break
            vol.reset()
        assert vol.pool_bricks > n and vol.pool_stats()["dropped_total"] == 0
        return vol
    _fuse(vol, frames)
    assert vol.num_bricks() == n and vol.pool_stats()["dropped_total"] == 0
    return vol


# ---------------------------------------------------------------------------------------------------------- read-outs

def _readouts(vol, cams, threshold, tmp):
    """{name: bytes} of every read-out of `vol`."""
    from types import SimpleNamespace

    from gs2mesh_b200.mesh import extract_point_cloud, extract_triangle_mesh, extract_voxel_point_cloud
    from gs2mesh_b200.tsdf import TSDF

    tmp.mkdir()
    read = lambda path: open(path, "rb").read()
    out = {}
    mesh = extract_triangle_mesh(vol)
    mesh.compute_vertex_normals(vol.device)
    for a in ("vertices", "triangles", "vertex_colors", "vertex_normals", "edge_keys"):
        out["mesh." + a] = getattr(mesh, a)
    out["mesh.key_window"] = np.array(mesh.key_window)
    out["clusters.labels"], out["clusters.counts"], out["clusters.area"] = mesh.cluster_connected_triangles()
    clean = mesh.remove_small_clusters(threshold)
    for a in ("vertices", "triangles", "vertex_colors", "vertex_normals"):
        out["cleaned." + a] = getattr(clean, a)
    out["mesh.ply"] = read(mesh.write_ply(str(tmp / "mesh.ply")))
    out["cleaned.ply"] = read(clean.write_ply(str(tmp / "cleaned.ply")))
    for name, pcd in (("cloud", extract_point_cloud(vol)), ("voxels", extract_voxel_point_cloud(vol))):
        for a in ("points", "colors", "normals", "keys"):
            out[f"{name}.{a}"] = getattr(pcd, a)
        out[f"{name}.ply"] = read(pcd.write_ply(str(tmp / f"{name}.ply")))
    for i, (w2c, zmin, zmax, size) in enumerate(cams):
        r = vol.raycast(*size, w2c, zmin, zmax)
        for a in ("depth", "normals", "colors"):
            out[f"raycast{i}.{a}"] = getattr(r, a).cpu().numpy()
    # the stage's extract_mesh() (scaled, with normals), save_mesh() and clean_mesh()
    stage = TSDF(SimpleNamespace(output_dir_root=str(tmp)), None,
                 SimpleNamespace(TSDF_scale=0.5, TSDF_cleaning_threshold=threshold * 0.5), "inv", device=vol.device)
    stage.volume = vol
    stage.extract_mesh()
    out["stage.mesh.ply"] = read(stage.save_mesh())
    out["stage.cleaned_mesh.ply"] = read(stage.clean_mesh())
    return {k: v if v is None or isinstance(v, bytes) else (v.dtype.str, v.shape, v.tobytes()) for k, v in out.items()}


def _assert_same(got, want, what):
    assert sorted(got) == sorted(want)
    differ = [k for k in want if got[k] != want[k]]
    assert not differ, f"{what}: {len(differ)} read-outs differ: {differ}"


@pytest.fixture(scope="module")
def reference(cuda_device, tmp_path_factory):
    """content -> (units, cameras, cleaning threshold, read-outs of the bricks inserted in ascending lattice order)."""
    cache = {}

    def get(content):
        if content not in cache:
            units, cams = (_block if content == "block" else _sphere)(cuda_device)
            vol = _state(cuda_device, "ascending", units)
            from gs2mesh_b200.mesh import extract_triangle_mesh

            mesh = extract_triangle_mesh(vol)
            _, counts, _ = mesh.cluster_connected_triangles()
            threshold = float(counts.max())  # keeps the largest cluster(s), removes the others
            assert len(mesh.triangles) > 5000 and (counts < threshold).sum() > 0
            cache[content] = units, cams, threshold, _readouts(vol, cams, threshold, tmp_path_factory.mktemp(content) / "ascending")
        return cache[content]

    return get


@pytest.mark.parametrize("content,state", CASES, ids=[f"{c}-{s}" for c, s in CASES])
def test_readouts_do_not_depend_on_how_the_volume_holds_its_bricks(gsb_lib, cuda_device, reference, tmp_path, content,
                                                                     state):
    units, cams, threshold, want = reference(content)
    vol = _state(cuda_device, state, units)
    got_units = vol.export_units()
    assert sorted(got_units) == sorted(units)
    for b, (tw, col) in units.items():  # bit-identical voxels
        assert got_units[b][0].tobytes() == tw.tobytes() and got_units[b][1].tobytes() == col.tobytes(), b
    first = _readouts(vol, cams, threshold, tmp_path / "first")
    _assert_same(_readouts(vol, cams, threshold, tmp_path / "second"), first, f"{state}, extracted twice")
    _assert_same(first, want, f"{state} vs ascending insertion")
