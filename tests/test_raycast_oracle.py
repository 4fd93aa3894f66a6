"""The numpy restatement of the TSDF ray cast (tests/raycast_oracle.py) against closed-form answers, on brick volumes that
hold analytic signed distance fields: planes on every axis and an oblique one, a sphere, and no-hit cases (a weight-0
hole, a missing brick, a surface outside the depth range, a ray that starts behind the surface).  And the skipping
march against a dense one.  CPU only; the GPU kernel is compared with this restatement bit for bit in
tests/test_gpu_raycast.py."""
import numpy as np
import pytest

from tests.raycast_oracle import analytic_units, look_at, raycast_units, rays

VL = 2.0 / 512
W, H, FX, FY = 40, 32, 50.0, 50.0
CX, CY = (W - 1) / 2, (H - 1) / 2
BLOCK = [(bx, by, bz) for bx in range(-2, 2) for by in range(-2, 2) for bz in range(-2, 2)]  # [-0.125, 0.125)^3
# tau larger than any distance inside the block: the stored field is the SDF itself, never clipped
TAU_WIDE = 0.5
EPS32 = 2.0 ** -24


def _cast(units, w2c, zmin=0.0, zmax=10.0, tau=TAU_WIDE, **kw):
    return raycast_units(units, VL, tau, W, H, FX, FY, CX, CY, w2c, zmin, zmax, **kw)


def _angle(a, b):
    a = a / np.linalg.norm(a, axis=-1, keepdims=True)
    return np.arccos(np.clip((a * b).sum(-1), -1, 1))


PLANES = {"+x": (1, 0, 0), "-x": (-1, 0, 0), "+y": (0, 1, 0), "-y": (0, -1, 0), "+z": (0, 0, 1), "-z": (0, 0, -1),
          "oblique": (1, 2, 3)}


@pytest.mark.parametrize("name", sorted(PLANES))
def test_plane_known_answer(name):
    """Plane n.p = c, sdf = n.p - c (positive on the camera's side), never clipped.  A linear field is reproduced exactly
    by trilinear interpolation and by the linear interpolation between the two samples, so the only error is the
    float32 storage of f (relative 2^-24, |f| <= 1): the interpolated root lies where |f_true| <= 2^-24, i.e.
    |n.p* - c| <= 2^-24 tau, plus double rounding.  Normals: central differences of a linear field are exact up to the
    same storage error over a 2 * 0.99 vl baseline; within 1e-5 rad."""
    n = np.asarray(PLANES[name], float)
    n /= np.linalg.norm(n)
    c = 0.01
    units = analytic_units(lambda p: p @ n - c, BLOCK, VL, TAU_WIDE)
    w2c = look_at(0.4 * n + (0.003, -0.002, 0.001), (0.0, 0.0, 0.0), up=(0.3, 0.5, 0.8))
    r = _cast(units, w2c)
    o, d, dn = rays(W, H, FX, FY, CX, CY, w2c)
    t = (c - o @ n) / (d @ n)
    pt = o + t[:, None] * d
    inside = (np.abs(pt) < 0.125 - 3 * VL).all(1)  # the analytic hit lies well inside the block
    hit = ~np.isnan(r["z"])
    assert inside.sum() > 200 and hit[inside].all()
    ps = o + r["z"][hit, None] * d[hit]
    assert np.abs(ps @ n - c).max() <= EPS32 * TAU_WIDE + 1e-12
    assert np.array_equal(r["depth"].reshape(-1)[hit], r["z"][hit].astype(np.float32))
    # (at the block's faces the normal samples reach unopened units, which read 0)
    assert _angle(r["normals"].reshape(-1, 3)[inside].astype(np.float64), n).max() < 1e-5
    col = r["colors"].reshape(-1, 3)[hit]
    assert (col >= 0).all() and (col <= 1).all() and (col > 0).any()


def test_sphere_known_answer():
    """Sphere |p - m| = R, sdf = |p - m| - R, never clipped.  The sdf's Hessian has trace 2/|p - m| and no negative
    eigenvalue, so trilinear interpolation over a cube whose corners lie >= r_min = R - 2 vl from m is off by at most
    e_tri = vl^2/8 * 2/r_min; the linear interpolation between the two samples z_prev, z_next (ray length D apart) adds
    at most D^2/(8 r_min); storage adds 2^-24 tau.  The sdf at the hit is bounded by their sum e, and along a ray meeting
    the sphere at cos(theta) >= 0.3 the hit lies within 2 e / cos(theta) of the analytic intersection.  Normals: the
    central differences over 2 * 0.99 vl carry at most 2 e_tri / (1.98 vl) per component, under vl / r_min in angle."""
    m = np.array([0.01, -0.02, 0.015])
    R = 0.09
    units = analytic_units(lambda p: np.linalg.norm(p - m, axis=-1) - R, BLOCK, VL, TAU_WIDE)
    w2c = look_at(m + 0.45 * np.array([0.6, -0.7, 0.4]) / np.linalg.norm([0.6, -0.7, 0.4]), m)
    r = _cast(units, w2c)
    o, d, dn = rays(W, H, FX, FY, CX, CY, w2c)
    u = d / dn[:, None]
    oc = o - m
    b = u @ oc
    disc = b * b - (oc @ oc - R * R)
    t = -b - np.sqrt(np.maximum(disc, 0))  # ray length to the first intersection
    hit = ~np.isnan(r["z"])
    assert np.array_equal(hit, disc > 0) or (hit == (disc > 0)).mean() > 0.99
    nrm = (o + t[:, None] * u - m) / R
    cos = -(nrm * u).sum(1)
    sel = hit & (disc > 0) & (cos >= 0.3)  # the sphere lies inside the block, so normal samples stay in open units
    assert sel.sum() > 100
    r_min = R - 2 * VL
    e_tri = VL * VL / 8 * 2 / r_min
    D = (r["z_next"] - r["z_prev"]) * dn
    e = e_tri + D * D / (8 * r_min) + EPS32 * TAU_WIDE
    err = np.abs(r["z"] * dn - t)
    assert (err[sel] <= 2 * e[sel] / cos[sel]).all()
    assert err[sel].max() < 0.05 * VL
    ang = _angle(r["normals"].reshape(-1, 3)[sel].astype(np.float64), nrm[sel])
    assert ang.max() < VL / r_min


# ------------------------------------------------------------------------------------------------------------ no hits

def _plane_z(c=8 * VL, weight=None, bricks=BLOCK):
    """The plane z = c facing +z, and a camera above the centre of brick (0,0,0) looking straight down."""
    units = analytic_units(lambda p: p[..., 2] - c, bricks, VL, TAU_WIDE, weight=weight)
    w2c = look_at((8 * VL + 0.0011, 8 * VL - 0.0007, 0.3), (8 * VL + 0.0011, 8 * VL - 0.0007, 0.0), up=(0.0, 1.0, 0.0))
    return units, w2c


CENTRE = (H // 2, W // 2)


def test_no_hit_through_a_weight0_hole():
    target = np.array([8 * VL, 8 * VL, 8 * VL])
    units, w2c = _plane_z(weight=lambda p: np.linalg.norm(p - target, axis=-1) > 4 * VL)
    full, _ = _plane_z()
    r, ref = _cast(units, w2c), _cast(full, w2c)
    assert ref["depth"][CENTRE] > 0 and r["depth"][CENTRE] == 0
    assert (r["normals"][CENTRE] == 0).all() and (r["colors"][CENTRE] == 0).all()
    assert (r["depth"] > 0).sum() > 0.8 * (ref["depth"] > 0).sum()  # away from the hole the plane is still there


def test_no_hit_through_a_missing_brick():
    units, w2c = _plane_z(bricks=[b for b in BLOCK if b != (0, 0, 0)])
    r = _cast(units, w2c)
    assert r["depth"][CENTRE] == 0 and (r["depth"] > 0).sum() > 100


def test_no_hit_outside_the_depth_range():
    units, w2c = _plane_z()
    ref = _cast(units, w2c)
    z = ref["z"].reshape(H, W)[CENTRE]
    assert abs(z - (0.3 - 8 * VL)) < 1e-9
    assert (_cast(units, w2c, zmax=z - 2 * VL)["depth"] == 0).all()  # the surface lies beyond z_max
    assert (_cast(units, w2c, zmin=0.2, zmax=z - 1e-3)["depth"] == 0).all()
    # the sample after the crossing must lie in range too: with one voxel of margin past the surface it does
    assert _cast(units, w2c, zmin=0.2, zmax=z + 1.01 * VL)["depth"][CENTRE] > 0


def test_no_hit_for_a_ray_starting_behind_the_surface():
    """From behind the plane f is negative all along: entering from f <= 0 is not a hit, and back faces give none."""
    units, w2c = _plane_z()
    z = _cast(units, w2c)["z"].reshape(H, W)[CENTRE]
    assert (_cast(units, w2c, zmin=z + 2 * VL)["depth"] == 0).all()
    back = look_at((8 * VL, 8 * VL, -0.3), (8 * VL, 8 * VL, 0.0), up=(0.0, 1.0, 0.0))  # below the plane looking up
    assert (_cast(units, back)["depth"] == 0).all()


def test_zero_direction_components():
    """Axis-aligned rays (zero direction components) whose origin lies on unit faces."""
    units, _ = _plane_z()
    face = 16 * VL + VL / 2  # a unit face: p - vl/2 = U
    w2c = np.eye(4)
    w2c[:3, :3] = np.diag([1.0, -1.0, -1.0])  # looking down -z
    w2c[:3, 3] = -w2c[:3, :3] @ np.array([face, face, 0.3])
    r = raycast_units(units, VL, TAU_WIDE, 5, 5, 50.0, 50.0, 2.0, 2.0, w2c, 0.0, 10.0)
    assert r["depth"][2, 2] == np.float32(0.3 - 8 * VL) and (r["depth"] > 0).all()


TOP = (1 << 20) - 1


def corner_case(vl, sign=1):
    """A plane n.(p - c0) = 0, n = sign (1,1,1)/sqrt3, across the 2x2x2 bricks at the +sign corner of the lattice, and
    cameras: from outside the lattice box looking in at it, from outside looking away, from inside looking out (distances
    scale with vl, so every voxel length sees the same picture)."""
    hi = TOP if sign > 0 else -(1 << 20)
    lo = hi - sign
    bricks = [(x, y, z) for x in (lo, hi) for y in (lo, hi) for z in (lo, hi)]
    U = 16 * vl
    c0 = np.full(3, (max(lo, hi) * U) + vl / 2)  # the shared corner of the eight bricks
    n = sign * np.ones(3) / np.sqrt(3)
    units = analytic_units(lambda p: (p - c0) @ n, bricks, vl, TAU_WIDE)
    s = vl / VL
    outside_in = look_at(c0 + 0.3 * s * n, c0)
    outside_out = look_at(c0 + 0.3 * s * n, c0 + 1.0 * s * n)
    inside_out = look_at(c0 - 0.01 * s * n, c0 + 1.0 * s * n)
    return units, c0, n, dict(outside_in=outside_in, outside_out=outside_out, inside_out=inside_out)


@pytest.mark.parametrize("sign", [1, -1], ids=["top", "bottom"])
def test_lattice_ends_and_far_depth_range(sign):
    """At both ends of the lattice, with z_max far beyond it: the march stops where the ray leaves the lattice box."""
    units, c0, n, cams = corner_case(VL, sign)
    r = raycast_units(units, VL, TAU_WIDE, 5, 5, 50.0, 50.0, 2.0, 2.0, cams["outside_in"], 0.0, 1e12)
    assert (r["depth"] > 0).all()
    o, d, dn = rays(5, 5, 50.0, 50.0, 2.0, 2.0, cams["outside_in"])
    assert np.abs((o + r["z"][:, None] * d - c0) @ n).max() < 1e-9
    for cam in ("outside_out", "inside_out"):
        assert (raycast_units(units, VL, TAU_WIDE, 5, 5, 50.0, 50.0, 2.0, 2.0, cams[cam], 0.0, 1e12)["depth"] == 0).all()


# ---------------------------------------------------------------------------------------------- skipping vs dense march

def _thin_slabs(p):
    """Two slabs 3 vl thick, one oblique: as thin as the negative band a fused surface leaves behind it (tau = 4 vl deep
    along the viewing ray, less across it).  Thinner features can fall between two one-voxel steps."""
    a = np.abs(p[..., 2] - 0.02) - 1.5 * VL
    n = np.array([0.3, -0.2, 0.93]) / np.linalg.norm([0.3, -0.2, 0.93])
    b = np.abs(p @ n + 0.05) - 1.5 * VL
    return np.minimum(a, b)


@pytest.mark.parametrize("shape", ["sphere", "thin_slabs"])
def test_skipping_finds_what_dense_marching_finds(shape):
    """Truncated at tau = 4 vl like a fused volume.  Every ray on which a march of fixed vl/4 steps finds a crossing away
    from holes (all samples within tau along the ray on both sides VALID; the block's faces border unopened bricks) is
    hit by the skipping march too, within one voxel along the ray."""
    from tests.raycast_oracle import _Grid, dense_units, window_of

    m = np.array([0.0, 0.01, -0.005])
    sdf = (lambda p: np.linalg.norm(p - m, axis=-1) - 0.08) if shape == "sphere" else _thin_slabs
    units = analytic_units(sdf, BLOCK, VL, 4 * VL)
    w2c = look_at((0.25, -0.3, 0.35), (0.0, 0.0, 0.0))
    skip = _cast(units, w2c, tau=4 * VL)
    dense = _cast(units, w2c, tau=4 * VL, fixed_step=VL / 4, with_normals=False, with_color=False)
    o, d, dn = rays(W, H, FX, FY, CX, CY, w2c)
    b0, nb = window_of(units)
    tw, _, alloc = dense_units(units, b0, nb)
    grid = _Grid(tw, b0, nb, VL, None, alloc)
    want = np.nonzero(~np.isnan(dense["z"]))[0]
    zs = dense["z"][want, None] + (np.arange(-16, 17) * (VL / 4))[None, :] / dn[want, None]
    state, _ = grid.classify((o + zs[..., None] * d[want, None, :]).reshape(-1, 3))
    want = want[(state.reshape(len(want), -1) == 2).all(1)]
    assert len(want) > 100
    got = ~np.isnan(skip["z"])
    assert got[want].all()
    assert (np.abs(skip["z"] - dense["z"])[want] * dn[want]).max() <= VL
