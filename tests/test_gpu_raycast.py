"""GPU ray casting of the TSDF volume (gsb_tsdf_raycast, TSDFVolume.raycast, TSDF.raycast) against the numpy restatement
(tests/raycast_oracle.py), bit for bit in depth, normals and colours.

Brick-built volumes cover rays meeting faces of all six orientations, missing neighbours and weight-0 corners, signed
zeros and subnormal tsdf values, both ends of the lattice with a depth range far beyond it, voxel lengths that are not
dyadic, axis-aligned cameras whose rays run along unit faces with zero direction components, and depth-range edges.
Fused scenes come from the point-cloud tests' sphere; there the ray cast is also checked against the mesh and against
the depth maps that were fused."""
import numpy as np
import pytest

from tests.raycast_oracle import look_at, raycast_units, window_of
from tests.test_gpu_mesh_volumes import _brick
from tests.test_gpu_pointcloud import SPECIAL, VOXEL_LENGTHS, _crossing_rich, _fused, brick_volume  # noqa: F401
from tests.test_raycast_oracle import corner_case

pytestmark = pytest.mark.gpu

W, H, F = 48, 40, 55.0
CX, CY = (W - 1) / 2, (H - 1) / 2


def _compare(vol, units, w2c, zmin, zmax, with_color, size=(W, H, F, F, CX, CY), window=None):
    """vol.raycast equals the restatement's images bit for bit; returns the number of hits."""
    w, h, fx, fy, cx, cy = size
    got = vol.raycast(w, h, fx, fy, cx, cy, w2c, zmin, zmax, colors=with_color)
    ref = raycast_units(units, vol.voxel_length, vol.sdf_trunc, w, h, fx, fy, cx, cy, w2c, zmin, zmax,
                        with_color=with_color, window=window)
    depth = got.depth.cpu().numpy()
    np.testing.assert_array_equal(depth, ref["depth"])
    np.testing.assert_array_equal(got.normals.cpu().numpy(), ref["normals"])
    if with_color:
        np.testing.assert_array_equal(got.colors.cpu().numpy(), ref["colors"])
    else:
        assert got.colors is None
    assert (np.signbit(depth) == False).all()  # noqa: E712  (no -0: a miss writes +0)
    return int((depth > 0).sum())


def _block(rng, vl, weight0=0.0, missing=(), values=None):
    units = {}
    for b in [(bx, by, bz) for bx in (-1, 0, 1) for by in (-1, 0, 1) for bz in (-1, 0, 1)]:
        if b in missing:
            continue
        t = _crossing_rich(rng) if values is None else values[rng.integers(0, len(values), (16, 16, 16))]
        w = np.where(rng.random((16, 16, 16)) < weight0, 0.0, rng.uniform(0.5, 4, (16, 16, 16))).astype(np.float32)
        units[b] = _brick(rng, t, w)
    return units


FACES = {"+x": (1, 0, 0), "-x": (-1, 0, 0), "+y": (0, 1, 0), "-y": (0, -1, 0), "+z": (0, 0, 1), "-z": (0, 0, -1)}


@pytest.mark.parametrize("face", sorted(FACES))
def test_six_face_orientations(gsb_lib, brick_volume, face):
    """Cameras on each side of a 3x3x3 block of random crossing-rich bricks: rays enter through faces of every
    orientation, from empty space into valid cubes."""
    rng = np.random.default_rng(100 + sorted(FACES).index(face))
    vl = 2.0 / 512
    units = _block(rng, vl)
    vol = brick_volume(units, vl, True)
    n = np.asarray(FACES[face], float)
    w2c = look_at(0.3 * n + (0.004, -0.003, 0.002), (0.001, 0.002, -0.001), up=(0.3, 0.5, 0.8))
    assert _compare(vol, units, w2c, 0.0, 2.0, True) > 500


@pytest.mark.parametrize("vl", VOXEL_LENGTHS, ids=["vl2", "vl0.3", "vl0.2"])
def test_missing_neighbours_and_weight0_corners(gsb_lib, brick_volume, vl):
    rng = np.random.default_rng(110)
    units = _block(rng, vl, weight0=0.05, missing=[(0, 0, 0), (1, -1, 0), (-1, 1, 1)])
    vol = brick_volume(units, vl, True)
    s = vl / (2.0 / 512)
    w2c = look_at(np.array([0.2, -0.25, 0.15]) * s, (0.0, 0.0, 0.0))
    assert _compare(vol, units, w2c, 0.0, 2.0 * s, True) > 300


@pytest.mark.parametrize("with_color", [True, False], ids=["color", "nocolor"])
def test_signed_zeros_and_subnormals(gsb_lib, brick_volume, with_color):
    """tsdf of +-0, +-subnormals, +-0.98 and equal magnitudes: f_prev > 0 >= f at -0, interpolation to exact zeros."""
    rng = np.random.default_rng(120)
    vl = 0.3 / 512
    units = _block(rng, vl, weight0=0.02, values=SPECIAL)
    if not with_color:
        units = {k: (v[0], None) for k, v in units.items()}
    vol = brick_volume(units, vl, with_color)
    w2c = look_at(np.array([0.03, 0.04, -0.035]), (0.0, 0.0, 0.0))
    assert _compare(vol, units, w2c, 0.0, 1.0, with_color) > 300


def test_axis_aligned_rays_along_unit_faces(gsb_lib, brick_volume):
    """Cameras looking along +-x, +-y, +-z from an origin on unit faces in the two other axes, with the principal
    point on a pixel: that pixel's ray has two zero direction components and runs inside a face plane."""
    rng = np.random.default_rng(130)
    vl = 2.0 / 512
    units = _block(rng, vl, weight0=0.02)
    vol = brick_volume(units, vl, True)
    face = 16 * vl + vl / 2
    hits = 0
    for axis in range(3):
        for sign in (1.0, -1.0):
            fwd = np.zeros(3)
            fwd[axis] = sign
            right = np.zeros(3)
            right[(axis + 1) % 3] = 1.0
            R = np.stack([right, np.cross(fwd, right), fwd])  # camera rows: x, y, z = forward
            pos = np.full(3, face)
            pos[axis] = -0.3 * sign
            w2c = np.eye(4)
            w2c[:3, :3] = R
            w2c[:3, 3] = -R @ pos
            hits += _compare(vol, units, w2c, 0.0, 1.0, True, size=(33, 31, 40.0, 40.0, 16.0, 15.0))
    assert hits > 500


def test_depth_range_edges(gsb_lib, brick_volume):
    """z_min inside the block (the march starts among valid cubes), z_max cutting it, a range of one voxel."""
    rng = np.random.default_rng(140)
    vl = 2.0 / 512
    units = _block(rng, vl, weight0=0.02)
    vol = brick_volume(units, vl, True)
    w2c = look_at((0.25, 0.2, -0.3), (0.0, 0.0, 0.0))
    for zmin, zmax in ((0.4, 0.45), (0.43, 0.5), (0.0, 0.42), (0.44, 0.44 + vl), (0.5, float(np.nextafter(0.5, 1.0)))):
        _compare(vol, units, w2c, zmin, zmax, True)


@pytest.mark.parametrize("vl", VOXEL_LENGTHS, ids=["vl2", "vl0.3", "vl0.2"])
@pytest.mark.parametrize("sign", [1, -1], ids=["top", "bottom"])
def test_lattice_ends_with_far_depth_range(gsb_lib, brick_volume, sign, vl):
    """Bricks at the +-2^20 corner of the lattice, z_max = 1e12: rays from outside the lattice box into it, out of it,
    and from inside out of it; the march stops where the ray leaves the box."""
    units, _, _, cams = corner_case(vl, sign)
    vol = brick_volume(units, vl, True)
    hits = [_compare(vol, units, cams[c], 0.0, 1e12, True, size=(9, 7, 60.0, 60.0, 4.0, 3.0)) for c in sorted(cams)]
    assert hits[sorted(cams).index("outside_in")] == 63 and sum(hits) == 63


# ------------------------------------------------------------------------------------------------------- fused scenes

CAMS = [(0.0, -1.0, 0.3), (0.8, -0.7, 0.5), (-0.7, -0.8, 0.1)]  # the views _fused integrates
FW, FH, FF = 96, 80, 90.0


@pytest.mark.parametrize("vl", [2.0 / 512, 0.3 / 512], ids=["vl2", "vl0.3"])
def test_fused_scene(gsb_lib, cuda_device, vl):
    vol = _fused(cuda_device, vl)
    units = vol.export_units()
    s = vl / (2.0 / 512)
    size = (FW, FH, FF, FF, FW / 2, FH / 2)
    for pos in CAMS + [(0.3, -0.9, -0.4)]:
        w2c = look_at(np.array(pos) * s, (0.0, 0.0, 0.0))
        assert _compare(vol, units, w2c, 0.05 * s, 3.0 * s, True, size=size) > 1000
    again = [vol.raycast(FW, FH, FF, FF, FW / 2, FH / 2, w2c, 0.05 * s, 3.0 * s) for _ in range(2)]
    for a in ("depth", "normals", "colors"):
        assert getattr(again[0], a).cpu().numpy().tobytes() == getattr(again[1], a).cpu().numpy().tobytes()


def test_fused_scene_agrees_with_mesh_and_input_depth(gsb_lib, cuda_device):
    """Every hit lies within 2 vl of a vertex of the extracted mesh: marching cubes puts a vertex on every crossed edge of
    each cube the zero set passes through, and a point of that cube is within the cube's diagonal sqrt(3) vl < 2 vl of
    one of them.  Cast from an integrated view, the depth reproduces that view's input depth where both exist: the input
    is an exact sphere, the three views agree on it, and the fused zero level differs from it by the interpolation of
    samples one voxel apart, so the median |dz| is at most one voxel."""
    from scipy.spatial import cKDTree

    from gs2mesh_b200.mesh import extract_triangle_mesh
    from tests.test_gpu_tsdf_frames import _raycast

    vl = 2.0 / 512
    vol = _fused(cuda_device, vl)
    mesh = extract_triangle_mesh(vol)
    tree = cKDTree(mesh.vertices)
    for pos in CAMS:
        w2c = look_at(np.array(pos), (0.0, 0.0, 0.0))
        r = vol.raycast(FW, FH, FF, FF, FW / 2, FH / 2, w2c, 0.05, 3.0)
        depth = r.depth.cpu().numpy()
        hit = depth > 0
        assert hit.sum() > 1000
        c2w = np.linalg.inv(w2c)
        v, u = np.mgrid[0:FH, 0:FW]
        cam = np.stack([(u - FW / 2) / FF * depth, (v - FH / 2) / FF * depth, depth], -1)[hit]
        world = cam @ c2w[:3, :3].T + c2w[:3, 3]
        assert tree.query(world)[0].max() < 2 * vl
        truth = _raycast(FW, FH, FF, FF, FW / 2, FH / 2, w2c, (0.0, 0.0, 0.0), 0.25)
        both = hit & (truth > 0)
        assert both.sum() > 0.9 * hit.sum()
        assert np.median(np.abs(depth[both] - truth[both])) <= vl


def test_stage_raycast_is_the_volume_call_scaled(gsb_lib, cuda_device):
    from types import SimpleNamespace

    from gs2mesh_b200.tsdf import TSDF

    scale, baseline = 0.1, 0.02  # the default range, [4, 20] baselines / scale = [0.8, 4], holds the sphere
    vol = _fused(cuda_device, 2.0 / 512)
    args = SimpleNamespace(TSDF_scale=scale, TSDF_min_depth_baselines=4, TSDF_max_depth_baselines=20)
    stage = TSDF(SimpleNamespace(baseline=baseline), None, args, "scene", device=cuda_device)
    stage.volume = vol
    w2c_vol = look_at(np.array(CAMS[1]), (0.0, 0.0, 0.0))
    c2w = np.linalg.inv(w2c_vol)
    c2w[:3, 3] *= scale  # the camera in world units
    cam = dict(width=FW, height=FH, fx=FF, fy=FF, cx=FW / 2, cy=FH / 2, extrinsic=c2w)
    got = stage.raycast(cam)
    e = c2w.copy()
    e[:3, 3] /= scale
    ref = vol.raycast(FW, FH, FF, FF, FW / 2, FH / 2, np.linalg.inv(e), 4 * baseline / scale, 20 * baseline / scale)
    assert (ref.depth > 0).sum() > 1000
    assert got.depth.cpu().numpy().tobytes() == (ref.depth * scale).cpu().numpy().tobytes()
    assert got.normals.cpu().numpy().tobytes() == ref.normals.cpu().numpy().tobytes()
    assert got.colors.cpu().numpy().tobytes() == ref.colors.cpu().numpy().tobytes()
    near = stage.raycast(cam, depth_range=(0.01, 0.02))  # world units: the surface lies beyond 0.02
    assert (near.depth == 0).all()


def test_invalid_arguments_and_empty_volume(gsb_lib, brick_volume):
    import ctypes as C

    import torch

    from gs2mesh_b200 import _lib

    vl = 2.0 / 512
    L = _lib.lib()
    plain = brick_volume({(0, 0, 0): _brick(np.random.default_rng(150))}, vl, False)
    e = (C.c_double * 16)(*np.eye(4).reshape(-1))
    out = torch.zeros(4, 4, 3, device=plain.device)
    d, c = _lib.ptr(out), _lib.ptr(out)
    ok = dict(w=4, h=4, fx=10.0, fy=10.0, cx=2.0, cy=2.0, e=e, zmin=0.0, zmax=1.0, depth=d, colors=None)

    def call(**kw):
        a = {**ok, **kw}
        return L.gsb_tsdf_raycast(plain._h, a["w"], a["h"], a["fx"], a["fy"], a["cx"], a["cy"], a["e"], a["zmin"], a["zmax"],
                                  a["depth"], None, a["colors"], None)

    assert call() == _lib.GSB_OK
    torch.cuda.synchronize()
    bad_e = (C.c_double * 16)(*np.eye(4).reshape(-1))
    bad_e[5] = float("nan")
    for kw in (dict(w=0), dict(h=-1), dict(w=(1 << 16) + 1), dict(h=(1 << 15) + 1), dict(fx=0.0), dict(fy=-1.0),
               dict(cx=float("inf")), dict(cy=float("nan")), dict(e=bad_e), dict(e=None), dict(zmin=-1e-9),
               dict(zmin=1.0), dict(zmax=float("inf")), dict(depth=None), dict(colors=c)):
        assert call(**kw) == _lib.GSB_ERR_INVALID, kw
    with pytest.raises(ValueError, match="without colour"):
        plain.raycast(4, 4, 10.0, 10.0, 2.0, 2.0, np.eye(4), 0.0, 1.0, colors=True)
    empty = brick_volume({}, vl, True)
    r = empty.raycast(16, 12, 10.0, 10.0, 8.0, 6.0, look_at((0.1, 0.2, 0.3), (0.0, 0.0, 0.0)), 0.0, 5.0)
    for t in r:
        assert t.abs().sum().item() == 0 and not torch.signbit(t).any()
