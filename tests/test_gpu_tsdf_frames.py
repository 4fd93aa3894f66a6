"""TSDF integration on adversarial frames, at its frame-size and lattice limits and with a brick pool that runs out.

Every case fuses the same frames into a gs2mesh_b200 TSDFVolume and the CPU oracle (Open3D ScalableTSDFVolume
restatement) and requires the same unit set with bit-identical (tsdf, weight) (tests/volume_compare.py).  Each case also
checks, with a host restatement of the kernel's arithmetic (tests/tsdf_host.py), that its frames reach the edge it is
named for, so a case that stops reaching it fails instead of passing vacuously.
"""
import numpy as np
import pytest

from tests import tsdf_host as th
from tests.volume_compare import assert_units_equal

pytestmark = pytest.mark.gpu

F32 = np.float32


def _look_at(pos, target, up=(0.0, 0.0, 1.0)):
    """world->camera 4x4 (OpenCV axes) of a camera at `pos` looking at `target`."""
    pos = np.asarray(pos, float)
    f = np.asarray(target, float) - pos
    f /= np.linalg.norm(f)
    r = np.cross(f, up)
    r /= np.linalg.norm(r)
    d = np.cross(f, r)
    c2w = np.eye(4)
    c2w[:3, :3] = np.stack([r, d, f], axis=1)
    c2w[:3, 3] = pos
    return np.linalg.inv(c2w)


def _raycast(W, H, fx, fy, cx, cy, w2c, centre, radius, plane_z=None):
    """z-depth of a sphere (and optionally the plane z = plane_z behind it) seen by the camera; 0 where nothing is hit."""
    c2w = np.linalg.inv(w2c)
    ys, xs = np.mgrid[0:H, 0:W]
    dirs = np.stack([(xs - cx) / fx, (ys - cy) / fy, np.ones((H, W))], -1)
    dw = dirs @ c2w[:3, :3].T
    o = c2w[:3, 3] - np.asarray(centre, float)
    a = (dw * dw).sum(-1)
    b = 2 * (dw @ o)
    c = o @ o - radius ** 2
    disc = b * b - 4 * a * c
    t = np.where(disc > 0, (-b - np.sqrt(np.maximum(disc, 0))) / (2 * a), np.inf)
    t = np.where(t > 0, t, np.inf)
    if plane_z is not None:
        with np.errstate(divide="ignore", invalid="ignore"):
            tp = (plane_z - c2w[2, 3]) / dw[..., 2]
        t = np.minimum(t, np.where(tp > 0, tp, np.inf))
    return np.where(np.isfinite(t), t, 0.0).astype(F32)


def _rgb(W, H, seed=0):
    """R, G and B distinct per pixel and from each other, so a wrong pixel or channel order changes the colour."""
    rng = np.random.default_rng(seed)
    return rng.integers(0, 256, (H, W, 3), dtype=np.uint8)


def _frame(depth, W, H, fx, fy, cx, cy, w2c, rgb=None):
    return dict(depth=np.ascontiguousarray(depth, F32).reshape(H, W), W=W, H=H, K=(fx, fy, cx, cy),
                w2c=np.asarray(w2c, np.float64), rgb=_rgb(W, H) if rgb is None else rgb)


def _volume(dev, vl, trunc, pool=4096, color=True):
    from gs2mesh_b200.tsdf import TSDFVolume

    return TSDFVolume(vl, trunc, with_color=color, device=dev, pool_bricks=pool)


def _integrate(vol, f, prepare=True, exact=False):
    import torch

    W, H = f["W"], f["H"]
    if prepare:
        d = vol.prepare_depth(f["depth"], W, H)
    else:  # the frame's values as they are, straight into integrate
        d = torch.as_tensor(f["depth"]).to(vol.device)
    rgb = f["rgb"] if vol.color is not None else None
    (vol.integrate_exact if exact else vol.integrate)(d, rgb, W, H, *f["K"], f["w2c"])


def _fuse(oracle, dev, frames, vl, trunc, *, pool=4096, color=True, prepare=True, threads=8, compare=True):
    """Fuse `frames` into both volumes, checking per frame that the GPU touched the oracle's units and lost none."""
    vol = _volume(dev, vl, trunc, pool, color)
    ovol = oracle.OracleTSDFVolume(vl, trunc, with_color=color)
    for f in frames:
        n = ovol.integrate(f["depth"], f["rgb"] if color else None, f["W"], f["H"], *f["K"], f["w2c"], threads=threads)
        _integrate(vol, f, prepare)
        st = vol.pool_stats()
        assert st["dropped"] == 0 and st["out_of_range"] == 0 and st["touched"] == n, (st, n)
    if compare:
        assert assert_units_equal(vol, ovol) == vol.num_bricks()
    return vol, ovol


def _samples(oracle, ovol, f, vl, trunc):
    """The host restatement of what frame `f` does to every voxel of the oracle's units."""
    W, H = f["W"], f["H"]
    mult = oracle.depth_multiplier(W, H, *f["K"])
    return th.sample_units(ovol.unit_indices(), vl, trunc, f["depth"], W, H, *f["K"], f["w2c"], mult)


def _axis_w2c(R=np.eye(3), t=(0.0, 0.0, 0.0)):
    e = np.eye(4)
    e[:3, :3] = R
    e[:3, 3] = t
    return e


# ------------------------------------------------------------------------------------------------------------ frame sizes

SIZES = [(1, 1), (2, 3), (3, 5), (5, 2), (41, 43), (43, 41), (1, 97), (97, 1), (4 * 37 + 1, 4 * 9 + 3), (4 * 9 + 3, 4 * 37 + 1)]


@pytest.mark.parametrize("W,H", SIZES, ids=[f"{w}x{h}" for w, h in SIZES])
def test_frame_sizes(oracle, gsb_lib, cuda_device, W, H):
    """Stride-4 sampling with partial groups, a partial last CTA, one-pixel rows and columns."""
    fx = fy = 1.2 * max(W, H)
    cx, cy = W / 2, H / 2
    frames = []
    for k, pos in enumerate([(0.3, -2.0, 0.4), (-1.6, -1.2, -0.5), (0.2, 0.3, 2.1)]):
        w2c = _look_at(pos, (0.05, 0.02, 0.0), up=(0.0, 1.0, 0.0) if k == 2 else (0.0, 0.0, 1.0))
        frames.append(_frame(_raycast(W, H, fx, fy, cx, cy, w2c, (0, 0, 0), 0.6, plane_z=-0.9), W, H, fx, fy, cx, cy, w2c,
                             rgb=_rgb(W, H, k)))
    vol, ovol = _fuse(oracle, cuda_device, frames, 2.0 / 256, 0.03)
    last_u = last_v = False
    for f in frames:  # voxels read pixels of the last, possibly partial, stride-4 group of columns and of rows
        s = _samples(oracle, ovol, f, 2.0 / 256, 0.03)
        up = s["updated"]
        last_u |= bool((s["u"][up].astype(int) >= 4 * ((W - 1) // 4)).any())
        last_v |= bool((s["v"][up].astype(int) >= 4 * ((H - 1) // 4)).any())
    assert last_u and last_v


def _long_strip(W, H):
    """A fronto-parallel wall seen by an axis-aligned camera along a W x 4 or 4 x H strip.  Voxel length 1/256: on the
    layer z = 513/512 the long axis projects EXACTLY onto (2i+1)*64 + 63 + 0.5, so voxel column 511 lands on the last
    pixel, 65535.5 (W = 65536) / 32767.5 (H = 32768 with column 255)."""
    long_f, short_f = 64.125 * 512, 4.0
    fx, fy, cx, cy = (long_f, short_f, 63.0, 1.5) if W > H else (short_f, long_f, 1.5, 63.0)
    depth = np.full((H, W), F32(515.0 / 512))
    return _frame(depth, W, H, fx, fy, cx, cy, _axis_w2c())


@pytest.mark.parametrize("W,H", [(65536, 4), (4, 32768)], ids=["65536x4", "4x32768"])
def test_largest_frames(oracle, gsb_lib, cuda_device, W, H):
    """The packed pixel index holds u < 65536 and v < 32768: the largest frames are bit-exact, and voxels are updated from
    the last column / row."""
    f = _long_strip(W, H)
    vl, trunc = 1.0 / 256, 0.02
    vol, ovol = _fuse(oracle, cuda_device, [f], vl, trunc, pool=8192)
    s = _samples(oracle, ovol, f, vl, trunc)
    up = s["updated"]
    if W > H:
        assert (s["u"][up] == F32(65535.5)).any()
    else:
        assert (s["v"][up] == F32(32767.5)).any()


@pytest.mark.parametrize("W,H", [(65537, 4), (4, 32769)], ids=["65537x4", "4x32769"])
def test_frames_beyond_the_packed_pixel_index_are_refused(gsb_lib, cuda_device, W, H):
    from gs2mesh_b200 import _lib

    f = _long_strip(W, H)
    vol = _volume(cuda_device, 2.0 / 512, 0.02, pool=64)
    with pytest.raises(_lib.GsbError, match="65536x32768"):
        _integrate(vol, f)
    with pytest.raises(_lib.GsbError, match="65536x32768"):
        _integrate(vol, f, exact=True)  # gsb_tsdf_touch
    assert vol.num_bricks() == 0


# ---------------------------------------------------------------------------------------------- pixel and border edges

VL_EDGE = 1.0 / 64  # voxel centres at (2i+1)/128: with fx = 40.5 the layer z = 81/128 projects onto exact half pixels
TRUNC_EDGE = 1.0 / 16


def _edge_depth(W, H, base=81.0 / 128 + 3.0 / 128):
    """A fronto-parallel wall just behind the voxel layer z = 81/128, with a ripple so neighbouring pixels differ."""
    ys, xs = np.mgrid[0:H, 0:W]
    return (base + ((xs * 7 + ys * 3) % 5) / 1024.0).astype(F32)


@pytest.mark.parametrize("cx,cy", [(16.0, 12.0), (15.5, 11.5), (-3.5, 30.0), (40.0, -6.5)],
                         ids=["integer", "half-integer", "left-of-image", "below-image"])
def test_exact_half_pixels_and_principal_points(oracle, gsb_lib, cuda_device, cx, cy):
    """An axis-aligned camera at the origin: every voxel of the layer z = 81/128 projects EXACTLY onto u_f = i + 0.5 + cx + 0.5
    -- an integer pixel boundary for integer cx, k + 0.5 for half-integer cx -- so the int truncation alone picks the pixel.
    Principal points off the image move the frame off-centre."""
    W, H, fx = 32, 24, 40.5
    f = _frame(_edge_depth(W, H), W, H, fx, fx, cx, cy, _axis_w2c())
    vol, ovol = _fuse(oracle, cuda_device, [f], VL_EDGE, TRUNC_EDGE)
    s = _samples(oracle, ovol, f, VL_EDGE, TRUNC_EDGE)
    up = s["updated"]
    u, v = s["u"][up], s["v"][up]
    fu, fv = (0.0 if float(c).is_integer() else 0.5 for c in (cx, cy))
    assert ((u - np.floor(u)) == fu).sum() > 20 and ((v - np.floor(v)) == fv).sum() > 20


def test_image_border_band(oracle, gsb_lib, cuda_device):
    """Voxels landing in [0, 0.0001) and in [W - 0.0001, W): both lie outside Open3D's `safe` image window."""
    W, H, fx = 32, 24, 40.5
    eps = 2.0 ** -14  # < 0.0001
    # layer z = 81/128: u_f = (i + 0.5) + cx + 0.5; i = 4 -> cx = -5 + eps gives u_f = eps exactly
    # v_f = (j + 0.5) + cy + 0.5; j = -7 -> cy = H + 6 - 2^-15 ... gives v_f = H - 2^-15, inside [H - 0.0001, H)
    cx, cy = -5.0 + eps, H + 6.0 - 2.0 ** -15
    f = _frame(_edge_depth(W, H), W, H, fx, fx, cx, cy, _axis_w2c())
    f2 = _frame(_edge_depth(W, H), W, H, fx, fx, W + 6.0 - 2.0 ** -15, -5.0 + eps, _axis_w2c())
    vol, ovol = _fuse(oracle, cuda_device, [f, f2], VL_EDGE, TRUNC_EDGE)
    s, s2 = (_samples(oracle, ovol, g, VL_EDGE, TRUNC_EDGE) for g in (f, f2))
    lo = lambda a: (a >= 0) & (a < F32(0.0001))  # noqa: E731
    hi = lambda a, n: (a >= F32(n) - F32(0.0001)) & (a < n)  # noqa: E731
    assert (lo(s["u"]) & (s["pcz"] > 0)).any() and (hi(s["v"], H) & (s["pcz"] > 0)).any()
    assert (lo(s2["v"]) & (s2["pcz"] > 0)).any() and (hi(s2["u"], W) & (s2["pcz"] > 0)).any()


def test_exact_quarter_turn_rotations(oracle, gsb_lib, cuda_device):
    """Rotations by exact multiples of 90 degrees: every extrinsic entry is +-0 or +-1."""
    W, H, fx, fy, cx, cy = 48, 40, 50.0, 50.0, 23.5, 20.0
    rots = [
        np.array([[1.0, -0.0, 0.0], [0.0, 0.0, -1.0], [-0.0, 1.0, 0.0]]),
        np.array([[0.0, 0.0, 1.0], [-0.0, 1.0, 0.0], [-1.0, 0.0, -0.0]]),
        np.array([[0.0, -1.0, 0.0], [1.0, 0.0, -0.0], [0.0, 0.0, 1.0]]),
        np.array([[-1.0, 0.0, 0.0], [0.0, -1.0, 0.0], [0.0, -0.0, 1.0]]),
    ]
    frames = []
    for k, R in enumerate(rots):
        c = np.array([0.11, -0.07, 0.05])
        t = -R @ (c - 1.5 * R.T @ np.array([0.0, 0.0, 1.0]))  # camera 1.5 in front of the sphere centre, looking at it
        w2c = _axis_w2c(R, t)
        frames.append(_frame(_raycast(W, H, fx, fy, cx, cy, w2c, c, 0.5), W, H, fx, fy, cx, cy, w2c, rgb=_rgb(W, H, k)))
    _fuse(oracle, cuda_device, frames, 2.0 / 256, 0.04)
    for f in frames:
        e = f["w2c"][:3, :3]
        assert set(np.unique(e)) <= {-1.0, 0.0, 1.0} and (np.signbit(e) & (e == 0)).any()


# ------------------------------------------------------------------------------------------------------------- depth values

def _special_depth_frame():
    W, H, fx = 33, 25, 40.5
    cx, cy = 16.0, 12.0
    depth = _edge_depth(W, H)
    # mult == 1 exactly at (cx, cy); voxel column x = y = -1/128 hits it, its layer z = 81/128 exactly at u_f = 16.0
    zc = F32(81.0 / 128)
    depth[12, 16] = zc - F32(TRUNC_EDGE)       # sdf == -trunc exactly: NOT updated (strict >)
    depth[12, 17] = zc                         # voxel x = +1/128 of the layer: sdf == 0
    depth[13, 16] = zc + F32(TRUNC_EDGE)       # sdf * (1/trunc) >= 1: clamped
    specials = [0.0, -0.0, -0.25, np.nan, 1e-42, np.finfo(F32).tiny / 4, -1e-40, 1e-3]
    for k, val in enumerate(specials):
        depth[2 + 2 * k, 3:6] = F32(val)
        depth[0:2, 4 * k] = F32(val)  # on stride-4 sample pixels too
    return _frame(depth, W, H, fx, fx, cx, cy, _axis_w2c())


@pytest.mark.parametrize("prepare", [True, False], ids=["prepare_depth", "direct"])
def test_depth_values(oracle, gsb_lib, cuda_device, prepare):
    """0, -0, negative, NaN and subnormal depths, sdf exactly 0 and exactly -trunc, and the clamp at 1.  A depth of 1e-3 or a
    subnormal one on a sample pixel opens bricks around the camera, whose voxels lie behind it (pcz <= 0)."""
    f = _special_depth_frame()
    f2 = dict(f, depth=f["depth"].copy())
    f2["depth"][12, 16] = F32(81.0 / 128) + F32(TRUNC_EDGE)  # the mult == 1 voxel at exactly sdf == +trunc: t == 1.0
    vol, ovol = _fuse(oracle, cuda_device, [f, f2], VL_EDGE, TRUNC_EDGE, prepare=prepare)
    s, s2 = (_samples(oracle, ovol, g, VL_EDGE, TRUNC_EDGE) for g in (f, f2))
    trunc, inv = F32(TRUNC_EDGE), F32(1) / F32(TRUNC_EDGE)
    ins = s["inside"] & (s["d"] > 0)
    assert (ins & (s["sdf"] == -trunc)).any()             # the strict > rejects it
    assert (ins & (s["sdf"] == 0)).any()
    assert (s["updated"] & (s["sdf"] * inv > 1)).any()
    assert (s2["updated"] & (s2["sdf"] * inv == 1)).any()
    assert (s["inside"] & np.isnan(s["d"])).any()
    assert (s["inside"] & (s["d"] < 0)).any()
    assert (s["pcz"] <= 0).any()                          # bricks around the camera


def test_steps_and_grazing_planes(oracle, gsb_lib, cuda_device):
    """Depth steps between neighbouring pixels and a plane seen at a grazing angle (large multiplier, boxes elongated)."""
    W, H, fx, fy, cx, cy = 64, 48, 25.0, 25.0, 31.5, 23.5
    ys, xs = np.mgrid[0:H, 0:W]
    step = np.where((xs // 3 + ys // 5) % 2 == 0, 0.8, 1.7).astype(F32)
    w2c = _look_at((0.0, -1.5, 0.08), (0.0, 0.0, 0.0))
    graze = _raycast(W, H, fx, fy, cx, cy, w2c, (0, 0, -100.0), 99.97)  # a huge sphere = a nearly flat floor, grazed
    frames = [_frame(step, W, H, fx, fy, cx, cy, _axis_w2c()), _frame(graze, W, H, fx, fy, cx, cy, w2c)]
    vol, ovol = _fuse(oracle, cuda_device, frames, 2.0 / 256, 0.04)
    mult = oracle.depth_multiplier(W, H, fx, fy, cx, cy)
    assert mult.max() > 1.8
    g = frames[1]["depth"]
    assert (g > 0).mean() > 0.2 and np.nanmax(np.abs(np.diff(g, axis=0))) > 0.5  # far-reaching depth jumps on the floor


def test_camera_inside_the_volume(oracle, gsb_lib, cuda_device):
    """A camera in the middle of the fused surface (voxels behind it), and an extrinsic that squeezes camera z to ~1e-37 so
    the projection of the touched voxels overflows to +-inf."""
    W, H, fx, fy, cx, cy = 40, 30, 35.0, 35.0, 19.5, 14.5
    outer = _look_at((1.6, 0.3, 0.2), (0, 0, 0))
    f1 = _frame(_raycast(W, H, fx, fy, cx, cy, outer, (0, 0, 0), 0.5), W, H, fx, fy, cx, cy, outer)
    inner = _look_at((0.02, 0.0, 0.01), (0.0, 1.0, 0.0))  # inside a small sphere, looking at its far wall
    c2w = np.linalg.inv(inner)
    ys, xs = np.mgrid[0:H, 0:W]
    dirs = np.stack([(xs - cx) / fx, (ys - cy) / fy, np.ones((H, W))], -1) @ c2w[:3, :3].T
    o = c2w[:3, 3]
    a, b, c = (dirs * dirs).sum(-1), 2 * (dirs @ o), o @ o - 0.12 ** 2
    d = ((-b + np.sqrt(b * b - 4 * a * c)) / (2 * a)).astype(F32)  # the far intersection: the camera is inside
    f2 = _frame(d, W, H, fx, fy, cx, cy, inner)
    squeeze = np.diag([1.0, 1.0, 1e-38, 1.0])  # camera z = 1e-38 * world z: subnormal in fp32
    f3 = _frame(np.full((H, W), F32(0.6e-38)), W, H, fx, fy, cx, cy, squeeze)  # back-projects to world z ~ 0.6
    vol, ovol = _fuse(oracle, cuda_device, [f1, f2, f3], 2.0 / 256, 0.04)
    s2 = _samples(oracle, ovol, f2, 2.0 / 256, 0.04)
    only3 = oracle.OracleTSDFVolume(2.0 / 256, 0.04, with_color=False)  # the bricks frame 3 touches
    only3.integrate(f3["depth"], None, W, H, *f3["K"], f3["w2c"])
    s3 = _samples(oracle, only3, f3, 2.0 / 256, 0.04)
    assert (s2["pcz"] <= 0).any() and s2["updated"].any()
    assert np.isinf(s3["u"]).any() and (s3["pcz"] > 0).all() and (s3["pcz"] < 1e-36).all()


# ------------------------------------------------------------------------------------------ truncation against brick size

def test_truncation_below_one_voxel(oracle, gsb_lib, cuda_device):
    W, H, fx, fy, cx, cy = 64, 48, 60.0, 60.0, 31.7, 24.2
    vl = 2.0 / 256
    frames = []
    for k, pos in enumerate([(1.5, 0.4, 0.3), (-0.4, 1.6, -0.2), (0.2, -0.3, 1.7)]):
        w2c = _look_at(pos, (0, 0, 0))
        frames.append(_frame(_raycast(W, H, fx, fy, cx, cy, w2c, (0, 0, 0), 0.55), W, H, fx, fy, cx, cy, w2c, rgb=_rgb(W, H, k)))
    vol, ovol = _fuse(oracle, cuda_device, frames, vl, 0.7 * vl)
    assert sum(int((ovol.unit_data(i)[1] > 0).sum()) for i in range(ovol.num_units)) > 2000


def test_truncation_of_several_bricks_overflows_the_cta_buffer(oracle, gsb_lib, cuda_device):
    """trunc = 2.4 brick lengths: each sample's box spans 5^3..6^3 bricks.  The frame's only samples are the 256 of its
    first sample row, i.e. of ONE mark_bricks CTA, with depths that vary per sample, so that CTA must queue more bricks
    than its 1024-entry shared buffer holds and append the rest straight to the work list."""
    W, H = 1024, 4
    fx = fy = 600.0
    cx, cy = 511.5, 1.5
    rng = np.random.default_rng(7)
    depth = np.repeat(rng.uniform(0.9, 1.6, (1, W)).astype(F32), H, axis=0)
    vl = 1.0 / 128
    trunc = 2.4 * 16 * vl
    f = _frame(depth, W, H, fx, fy, cx, cy, _axis_w2c())
    s, lo, hi = th.mark_boxes(f["depth"], W, H, fx, fy, cx, cy, f["w2c"], trunc, 16 * vl)
    assert (s < 256).all() and len(s) == 256  # one CTA of 256 threads
    span = hi - lo + 1
    assert span.min() >= 5 and (span.prod(1) > 3 ** 3).all()
    cells = {(x, y, z) for a, b in zip(lo, hi) for x in range(a[0], b[0] + 1) for y in range(a[1], b[1] + 1)
             for z in range(a[2], b[2] + 1)}
    assert len(cells) > 1024
    vol, ovol = _fuse(oracle, cuda_device, [f], vl, trunc, pool=1 << 14, color=False)
    assert ovol.num_units == len(cells)


# ----------------------------------------------------------------------------------------- voxel lengths, rigs, many frames

@pytest.mark.parametrize("voxel", [0.3, 0.2])
def test_non_dyadic_voxel_lengths_away_from_the_origin(oracle, gsb_lib, cuda_device, voxel):
    vl = voxel / 512
    centre = np.array([37.3, -12.1, 5.7])
    W, H, fx, fy, cx, cy = 64, 48, 70.0, 70.0, 32.3, 23.9
    frames = []
    for k, off in enumerate([(0.09, 0.01, 0.02), (-0.03, 0.08, -0.02), (0.01, -0.05, 0.08)]):
        w2c = _look_at(centre + np.array(off), centre)
        frames.append(_frame(_raycast(W, H, fx, fy, cx, cy, w2c, centre, 0.03), W, H, fx, fy, cx, cy, w2c, rgb=_rgb(W, H, k)))
    vol, ovol = _fuse(oracle, cuda_device, frames, vl, 5 * vl)
    assert ovol.num_units > 30 and (np.abs(ovol.unit_indices()) > 1000).any()


def test_many_frames_and_fp32_colour(oracle, gsb_lib, cuda_device):
    """36 frames, repeated and varied, so the running means' rounding builds up.  (tsdf, weight) bit-exact; colour bit-identical
    to the oracle's fp32-colour variant (the kernel's (c*w + rgb)/(w + 1)) and within tests/volume_compare.py's tolerance of
    the fp64 colour Open3D keeps."""
    W, H, fx, fy, cx, cy = 48, 36, 45.0, 45.0, 23.6, 17.8
    vl, trunc = 2.0 / 256, 0.05
    rng = np.random.default_rng(3)
    base = []
    for k in range(12):
        az, el = 2 * np.pi * k / 12, rng.uniform(-0.4, 0.4)
        w2c = _look_at(1.7 * np.array([np.cos(az) * np.cos(el), np.sin(az) * np.cos(el), np.sin(el)]), (0, 0, 0))
        base.append(_frame(_raycast(W, H, fx, fy, cx, cy, w2c, (0, 0, 0), 0.5), W, H, fx, fy, cx, cy, w2c, rgb=_rgb(W, H, k)))
    frames = base + base[::-1] + [dict(f, rgb=_rgb(W, H, 100 + i)) for i, f in enumerate(base)]
    assert len(frames) >= 32
    oracle.tsdf_set_variant(8)
    try:
        vol, o32 = _fuse(oracle, cuda_device, frames, vl, trunc)
    finally:
        oracle.tsdf_set_variant(0)
    o64 = oracle.OracleTSDFVolume(vl, trunc, with_color=True)
    for f in frames:
        o64.integrate(f["depth"], f["rgb"], W, H, *f["K"], f["w2c"], threads=8)
    got = vol.export_units()
    idx = o32.unit_indices()
    top = 0
    for i, k in enumerate(idx):
        _, w, c32 = o32.unit_data(i)
        col = got[tuple(int(v) for v in k)][1][:, :3].astype(np.float64)
        np.testing.assert_array_equal(col, c32, err_msg=f"colour of unit {tuple(k)}")
        top = max(top, int(w.max()))
    assert top >= 12  # voxels seen by a third of the frames or more
    assert_units_equal(vol, o64)  # colour within the documented tolerance of the fp64 colour
    diff = max(np.abs(o32.unit_data(i)[2] - o64.unit_data(i)[2]).max() for i in range(len(idx)))
    assert 0 < diff < 1e-3  # the two colour roundings really differ, and only by rounding


# ------------------------------------------------------------------------------------------------------ pool and hash edges

def _pool_frame():
    W, H, fx, fy, cx, cy = 64, 48, 55.0, 55.0, 31.5, 23.5
    w2c = _look_at((1.4, -0.6, 0.5), (0, 0, 0))
    return _frame(_raycast(W, H, fx, fy, cx, cy, w2c, (0, 0, 0), 0.5), W, H, fx, fy, cx, cy, w2c)


VL_POOL, TRUNC_POOL = 2.0 / 256, 0.04


def test_pool_of_exactly_the_unit_count(oracle, gsb_lib, cuda_device):
    f = _pool_frame()
    ovol = oracle.OracleTSDFVolume(VL_POOL, TRUNC_POOL)
    n = ovol.integrate(f["depth"], f["rgb"], f["W"], f["H"], *f["K"], f["w2c"])
    vol, _ = _fuse(oracle, cuda_device, [f], VL_POOL, TRUNC_POOL, pool=n)
    assert vol.num_bricks() == vol.pool_bricks == n and vol.ensure_capacity()
    # one short: counted, the pool grows, and the repeat is bit-exact
    small = _volume(cuda_device, VL_POOL, TRUNC_POOL, pool=n - 1)
    _integrate(small, f)
    st = small.pool_stats()
    assert st["dropped"] >= 1 and st["dropped_total"] >= 1 and st["bricks"] == n - 1 and st["out_of_range"] == 0
    assert small.ensure_capacity() is False and small.pool_bricks == 2 * (n - 1)
    small.reset()
    _integrate(small, f)
    assert small.pool_stats()["dropped"] == 0 and small.ensure_capacity()
    assert assert_units_equal(small, ovol) == n


def test_first_frame_drops_are_all_counted(oracle, gsb_lib, cuda_device):
    """For pools 1 .. 64 bricks short of the frame's unit count: the oracle units without a GPU slot never outnumber the
    drops the frame reports, whichever threads won the race for the last slots."""
    f = _pool_frame()
    ovol = oracle.OracleTSDFVolume(VL_POOL, TRUNC_POOL, with_color=False)
    n = ovol.integrate(f["depth"], None, f["W"], f["H"], *f["K"], f["w2c"])
    want = {tuple(int(v) for v in k) for k in ovol.unit_indices()}
    assert n > 64
    for pool in range(n - 1, n - 65, -1):
        vol = _volume(cuda_device, VL_POOL, TRUNC_POOL, pool=pool, color=False)
        _integrate(vol, f)
        st = vol.pool_stats()
        missing = len(want - set(vol.export_units()))
        assert missing == n - pool and st["dropped"] >= missing and st["dropped_total"] == st["dropped"], (pool, st, missing)


def test_probe_chain_wraps_past_the_last_slot(oracle, gsb_lib, cuda_device):
    """A table small enough that, by the host restatement of brick_hash, some key's probe chain wraps from the last slot to
    slot 0; the GPU's table holds the keys exactly where linear probing puts them, and the volume is bit-exact."""
    W, H, fx = 9, 7, 12.0
    for k in range(200):
        w2c = _look_at((1.3 + 0.01 * k, 0.3, 0.2), (0, 0, 0))
        f = _frame(_raycast(W, H, fx, fx, 4.2, 3.1, w2c, (0, 0, 0), 0.5), W, H, fx, fx, 4.2, 3.1, w2c)
        o = oracle.OracleTSDFVolume(VL_POOL, TRUNC_POOL)
        n = o.integrate(f["depth"], f["rgb"], W, H, *f["K"], f["w2c"])
        slots = 1 << max(4, (2 * n - 1).bit_length())
        keys = [th.brick_key(u) for u in o.unit_indices()]
        homes = [th.brick_hash(key, slots - 1) for key in keys]
        pos = th.linear_probe_positions(homes, slots)
        if (pos < np.array(homes)).any():
            break
    else:
        pytest.fail("no frame with a wrapping probe chain")
    vol, ovol = _fuse(oracle, cuda_device, [f], VL_POOL, TRUNC_POOL, pool=n)
    assert vol.hash_slots == slots
    table = vol._hash_keys.cpu().numpy().view(np.uint64)
    got = {int(table[p]): p for p in np.nonzero(table != np.uint64(2 ** 64 - 1))[0]}
    assert set(got) == set(keys) and sorted(got.values()) == sorted(pos.tolist())
    assert any(got[key] < h for key, h in zip(keys, homes))


def _plant_dead_key(vol, brick):
    """The state a lost race for the last pool slot leaves: the brick's key at its home slot, no pool slot (0xFFFFFFFF)."""
    key = th.brick_key(brick)
    h = th.brick_hash(key, vol.hash_slots - 1)
    assert int(vol._hash_keys[h].item()) == -1
    vol._hash_keys[h] = key - (1 << 64) if key >= 1 << 63 else key
    vol._hash_vals[h] = -1


@pytest.mark.parametrize("path", ["integrate", "touch", "find_bricks"])
def test_dead_key_is_counted_as_dropped(oracle, gsb_lib, cuda_device, path):
    """A key without a pool slot is a brick the volume does not hold.  The frame (or find_bricks call) that touches it counts
    it as dropped, ensure_capacity() grows the pool, and the volume fused again is bit-exact."""
    import torch

    f = _pool_frame()
    ovol = oracle.OracleTSDFVolume(VL_POOL, TRUNC_POOL)
    ovol.integrate(f["depth"], f["rgb"], f["W"], f["H"], *f["K"], f["w2c"])
    brick = ovol.unit_indices()[ovol.num_units // 2]
    vol = _volume(cuda_device, VL_POOL, TRUNC_POOL, pool=1024)
    _plant_dead_key(vol, brick)
    if path == "integrate":
        _integrate(vol, f)
    elif path == "touch":
        from gs2mesh_b200 import _lib

        d = vol.prepare_depth(f["depth"], f["W"], f["H"])
        e = np.ascontiguousarray(f["w2c"].reshape(16))
        _lib.check(vol._L.gsb_tsdf_touch(vol._h, _lib.ptr(d), f["W"], f["H"], *[float(v) for v in f["K"]],
                                         e.ctypes.data_as(_lib.C.POINTER(_lib.C.c_double)), vol._stream()))
    else:
        slots = vol.find_bricks(torch.as_tensor(np.asarray(brick).reshape(1, 3)), insert=True)
        assert int(slots[0].item()) == -1
    st = vol.pool_stats()
    assert st["dropped"] == 1 and st["dropped_total"] == 1 and st["out_of_range"] == 0, st
    assert vol.ensure_capacity() is False and vol.pool_bricks == 2048
    vol.reset()
    _integrate(vol, f)
    assert assert_units_equal(vol, ovol) == ovol.num_units
    # the Open3D-shaped path: integrate_exact() meets the dead key in gsb_tsdf_touch, grows, then fuses everything
    vol2 = _volume(cuda_device, VL_POOL, TRUNC_POOL, pool=1024)
    _plant_dead_key(vol2, brick)
    _integrate(vol2, f, exact=True)
    assert vol2.pool_bricks == 2048 and vol2.pool_stats()["dropped"] == 0
    assert assert_units_equal(vol2, ovol) == ovol.num_units


# -------------------------------------------------------------------------------------------------------------- lattice range

VL_LAT = 2.0 ** -10  # unit length 2^-6: brick index 2^20 starts at world x = 2^14, where fp32 resolves 2 voxels


def _lattice_frames(sign):
    W, H, fx, fy, cx, cy = 40, 32, 40.0, 40.0, 19.5, 15.5
    edge = sign * 2.0 ** 14
    frames = []
    for k, dx in enumerate([0.0, 0.013]):
        w2c = _axis_w2c(t=(-(edge + dx), 0.0, 0.0))  # camera at x = edge + dx, looking down +z
        ys, xs = np.mgrid[0:H, 0:W]
        depth = (0.25 + 0.01 * np.sin(xs * 0.3) + 0.004 * ys / H).astype(F32)
        frames.append(_frame(depth, W, H, fx, fy, cx, cy, w2c, rgb=_rgb(W, H, k)))
    return frames


def _assert_in_range_units_equal(vol, ovol):
    got = vol.export_units()
    idx = ovol.unit_indices()
    inside = (idx >= -th.BIAS).all(1) & (idx < th.BIAS).all(1)
    assert inside.any() and (~inside).any()
    assert set(got) == {tuple(int(v) for v in k) for k in idx[inside]}
    for i in np.nonzero(inside)[0]:
        t, w, _ = ovol.unit_data(int(i))
        tw = got[tuple(int(v) for v in idx[i])][0]
        np.testing.assert_array_equal(tw[:, 1], w)
        np.testing.assert_array_equal(tw[:, 0], t)
    return int(inside.sum())


@pytest.mark.parametrize("sign", [1, -1], ids=["plus", "minus"])
def test_lattice_range_edges(oracle, gsb_lib, cuda_device, sign):
    """Frames straddling brick index +2^20 / -2^20: bricks inside the lattice are bit-exact with the oracle (which has no
    range), those outside are counted as out of range -- not as pool drops, so ensure_capacity() does not grow the pool but
    raises, and so do integrate_exact() and TSDF.run()."""
    frames = _lattice_frames(sign)
    trunc = 0.02
    vol = _volume(cuda_device, VL_LAT, trunc, pool=1024)
    ovol = oracle.OracleTSDFVolume(VL_LAT, trunc)
    for f in frames:
        ovol.integrate(f["depth"], f["rgb"], f["W"], f["H"], *f["K"], f["w2c"], threads=8)
        _integrate(vol, f)
        st = vol.pool_stats()
        assert st["out_of_range"] > 0 and st["dropped"] == 0 and st["dropped_total"] == 0, st
    assert st["out_of_range_total"] >= st["out_of_range"]
    n = _assert_in_range_units_equal(vol, ovol)
    assert n > 10 and sum(int((ovol.unit_data(i)[1] > 0).sum()) for i in range(ovol.num_units)) > 0
    with pytest.raises(RuntimeError, match=r"\[-2\^20, 2\^20\)"):
        vol.ensure_capacity()
    assert vol.pool_bricks == 1024
    v2 = _volume(cuda_device, VL_LAT, trunc, pool=1024)
    with pytest.raises(RuntimeError, match=r"\[-2\^20, 2\^20\)"):
        _integrate(v2, frames[0], exact=True)
    assert v2.pool_bricks == 1024


def test_stage_run_raises_on_the_lattice_range(gsb_lib, cuda_device):
    from gs2mesh_b200.tsdf import TSDF

    frames = _lattice_frames(1)

    class Renderer:
        baseline = 0.05  # depths kept in [4, 20) baselines = [0.2, 1.0) (TSDF_min/max_depth_baselines)
        device = cuda_device
        left_cameras = [dict(width=f["W"], height=f["H"], fx=f["K"][0], fy=f["K"][1], cx=f["K"][2], cy=f["K"][3],
                             extrinsic=np.linalg.inv(f["w2c"])) for f in frames]

        def get_frame(self, n):
            return dict(left_u8=frames[n]["rgb"], depth=frames[n]["depth"])

        def render_folder_name(self, n):
            return f"/nonexistent/{n}"

    class Args:
        TSDF_voxel = VL_LAT * 512
        TSDF_sdf_trunc = 0.02

    stage = TSDF(Renderer(), None, Args(), "lattice", pool_bricks=1024, device=cuda_device)
    with pytest.raises(RuntimeError, match=r"\[-2\^20, 2\^20\)"):
        stage.run()
    assert stage.volume.pool_bricks == 1024
