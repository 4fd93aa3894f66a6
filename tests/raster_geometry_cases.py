"""Rasterizer inputs aimed at the per-Gaussian geometry of gsb_raster.cu's preprocess_kernel wherever its result hangs on
one comparison or one rounding, and the float32 host restatements that show each input reaches its edge
(tests/test_raster_geometry_host.py checks them on the CPU, tests/test_gpu_raster_geometry.py renders them):

  near_plane / near_plane_rotated   view depths at 0.2f and a few ulp either side; with a rotated camera also points where
                                    the FMA-contracted and the plainly rounded depth dot product fall on different sides
  guard_band                        centres just inside / outside 1.3 tan(fov) whose footprints still reach the frame
  tile_edge_centres                 centres where ndc2Pix in float32 and in float64 give different tile rectangles
  degenerate_cov                    cov3D_precomp with a negative 2-D determinant, and with a determinant of exactly 0
  needles                           conics with k = ac/det just below, at and above 1000 (shrink_rect's cut-off) and >= 1e4
  huge_footprints                   radii from the frame size up to ~1e5 px, centred inside, outside and far outside
  opacity_edges                     opacities 0, just below / at 1/255, 1 - ulp and 1
  quaternions                       norms 0.5 and 2, the zero quaternion, sign-flipped pairs
  sh_clamp_d0..3 / colors_precomp   colours driven far below 0 and above 1, along directions where basis functions vanish
  toed_in_pair                      a convergent rig: Gaussians one eye culls at the near plane or off-screen, the other not

Cameras come from camera.view_transforms with general rotations, or from raster_cases.identity_view where an exact float
value is needed (there the view depth of a Gaussian is its world z, bit for bit)."""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Optional

import numpy as np

from gs2mesh_b200 import camera as cam
from gs2mesh_b200.scene import GaussianCloud
from tests.raster_cases import SH_C0, Case, exact_rects, identity_view, place, tile_rects  # noqa: F401  (re-exported)

F = np.float32
F64 = np.float64
NEAR = F(0.2)
W0, H0, FOCAL0 = 320, 240, 300.0  # the small frame most cases use: tan_fovx != tan_fovy, so limx != limy


@dataclass
class GeoCase(Case):
    """A Case with the rest of the rasterizer's per-Gaussian inputs.  `features` of the cloud is [P, (D+1)^2, 3]."""
    sh_degree: int = 0
    cov3D: Optional[np.ndarray] = None  # [P, 6]: replaces scales / rotations
    colors: Optional[np.ndarray] = None  # [P, 3]: replaces the SH features
    scale_modifier: float = 1.0


def preprocess(oracle, case, fma=False, vt=None, scale_modifier=None):
    """The CPU oracle's per-Gaussian stage on `case` (seen from `vt`, default its own camera)."""
    g, vt = case.cloud, case.vt if vt is None else vt
    kw = dict(colors_precomp=case.colors) if case.colors is not None else dict(shs=g.features)
    kw.update(cov3D_precomp=case.cov3D) if case.cov3D is not None else kw.update(scales=g.scaling, rotations=g.rotation)
    return oracle.preprocess(g.xyz, g.opacity, vt.world_view, vt.full_proj, vt.cam_center, vt.width, vt.height, vt.tan_fovx,
                             vt.tan_fovy, sh_degree=case.sh_degree, fma=fma,
                             scale_modifier=case.scale_modifier if scale_modifier is None else scale_modifier, **kw)


def forward(oracle, case, bg, fma=False):
    g, vt = case.cloud, case.vt
    kw = dict(colors_precomp=case.colors) if case.colors is not None else dict(shs=g.features)
    kw.update(cov3D_precomp=case.cov3D) if case.cov3D is not None else kw.update(scales=g.scaling, rotations=g.rotation)
    return oracle.forward(g.xyz, g.opacity, vt.world_view, vt.full_proj, vt.cam_center, vt.width, vt.height, vt.tan_fovx,
                          vt.tan_fovy, bg=bg, sh_degree=case.sh_degree, scale_modifier=case.scale_modifier, fma=fma, **kw)


# ---------------------------------------------------------------------------------------------------- float32 restatements

def fma32(a, b, c):
    """Correctly rounded float32 fma(a, b, c), vectorised: the product is exact in float64, the sum's rounding error is
    recovered (TwoSum) and decides the one case where rounding twice goes wrong, a float64 sum on a float32 midpoint."""
    a, b, c = (np.asarray(v, F).astype(F64) for v in (a, b, c))
    p = a * b
    s = p + c
    bb = s - p
    e = (p - (s - bb)) + (c - bb)
    r = s.astype(F)
    lo = np.where(r.astype(F64) <= s, r, np.nextafter(r, F(-np.inf)))
    hi = np.nextafter(lo, F(np.inf))
    tie = (s == (lo.astype(F64) + hi.astype(F64)) / 2) & (e != 0)
    return np.where(tie, np.where(e > 0, hi, lo), r).astype(F)


def view_depths(xyz, vm):
    """z_view = vm[2] x + vm[6] y + vm[10] z + vm[14] (auxiliary.h transformPoint4x3) three ways: plainly rounded left to
    right, and with each of the two contractions a compiler may form (the later product fused onto the rounded earlier one,
    or the reverse; the third product is then fused and vm[14] added).  Returns (plain, fused_late, fused_early)."""
    x, y, z = (np.asarray(xyz, F)[:, k] for k in range(3))
    m = np.asarray(vm, F).reshape(16)
    plain = ((m[2] * x + m[6] * y) + m[10] * z) + m[14]
    late = fma32(m[10], z, fma32(m[6], y, m[2] * x)) + m[14]
    early = fma32(m[10], z, fma32(m[2], x, m[6] * y)) + m[14]
    return plain.astype(F), late.astype(F), early.astype(F)


def lim(vt):
    """The guard band 1.3 tan(fov) per axis, as the kernel rounds it."""
    return F(F(1.3) * F(vt.tan_fovx)), F(F(1.3) * F(vt.tan_fovy))


def focal(vt):
    """rasterizer_impl.cu: focal = size / (2 tan(fov / 2)), float32."""
    return F(F(vt.width) / (F(2) * F(vt.tan_fovx))), F(F(vt.height) / (F(2) * F(vt.tan_fovy)))


def ndc2pix(proj, size):
    """ndc2Pix three ways: in double (what the reference computes), in float32 plainly rounded, and in float32 with the
    multiply-subtract contracted."""
    proj = np.asarray(proj, F)
    dbl = (((proj.astype(F64) + 1.0) * size - 1.0) * 0.5).astype(F)
    s = proj + F(1)
    plain = ((s * F(size)) - F(1)) * F(0.5)
    fused = fma32(s, F(size), F(-1)) * F(0.5)
    return dbl, plain.astype(F), fused.astype(F)


def identity_proj(xyz, vt):
    """(projx, projy) of Gaussians seen by an identity_view camera at the origin: every other term of the projection's dot
    products is an exact zero, so these float32 restatements hold bit for bit whatever the contraction."""
    xyz = np.asarray(xyz, F)
    pm = np.asarray(vt.full_proj, F).reshape(16)
    p_w = F(1) / (xyz[:, 2] + F(1e-7))
    return (pm[0] * xyz[:, 0]) * p_w, (pm[5] * xyz[:, 1]) * p_w


def conic_k(conic):
    """shrink_rect's elongation k = ac / (ac - b^2), float32."""
    a, b, c = (np.asarray(conic, F)[:, i] for i in range(3))
    ac = a * c
    return (ac / (ac - b * b)).astype(F)


def sh_basis_count(deg):
    return (deg + 1) ** 2


# ---------------------------------------------------------------------------------------------------- builders

def gcloud(xyz, scales, rot, opacity, features, sh_degree=0) -> GaussianCloud:
    P = len(xyz)
    c = lambda a, *s: np.ascontiguousarray(np.asarray(a, F).reshape(P, *s))
    return GaussianCloud(c(xyz, 3), c(features, -1, 3), c(opacity, 1), c(scales, 3), c(rot, 4), sh_degree=sh_degree)


def dc_features(rgb):
    """Degree-0 SH coefficients whose colour is `rgb`."""
    return ((np.asarray(rgb, F64) - 0.5) / SH_C0).reshape(-1, 1, 3).astype(F)


def unit_quats(rng, n):
    q = rng.normal(size=(n, 4))
    return (q / np.linalg.norm(q, axis=1, keepdims=True)).astype(F)


def rotated_view(W, H, focal_px, angles_deg, t):
    """A camera with a general rotation (no axis-aligned row): c2w = Euler(angles), world->view translation t."""
    fov_x, fov_y = 2 * math.atan(W / (2 * focal_px)), 2 * math.atan(H / (2 * focal_px))
    return cam.view_transforms(cam.euler_deg_to_matrix(angles_deg), np.asarray(t, F64), fov_x, fov_y, W, H)


def to_world(vt, pv):
    """World points whose (float64) view coordinates are pv."""
    inv = np.linalg.inv(np.asarray(vt.world_view, F64))
    pv = np.asarray(pv, F64)
    return (np.c_[pv, np.ones(len(pv))] @ inv)[:, :3]


def _ulps(x, k):
    """x moved by k float32 steps (away from zero for k > 0), elementwise."""
    x = np.asarray(x, F)
    return (x.view(np.int32) + np.asarray(k, np.int32)).view(F)


def _spheres(rng, n, sigma_world):
    return np.repeat(np.asarray(sigma_world, F64).reshape(-1, 1), 3, 1) * rng.uniform(0.7, 1.3, (n, 3)), unit_quats(rng, n)


def _geo(name, vt, xyz, scales, rot, opacity, rgb=None, features=None, sh_degree=0, focal_px=FOCAL0, **info):
    P = len(xyz)
    feats = dc_features(rgb) if features is None else features
    return GeoCase(name, gcloud(xyz, scales, rot, opacity, feats, sh_degree), vt, float(focal_px), 0.0, dict(info),
                   sh_degree=sh_degree)


# ---------------------------------------------------------------------------------------------------- near plane

NEAR_OFFSETS = np.r_[-64, -16, -8:9, 16, 64]  # ulps from 0.2f


def near_plane(seed=20):
    """Identity camera: world z = view depth.  Three small Gaussians at each depth 0.2f + k ulp for k in NEAR_OFFSETS, spread
    over the frame, then eight that cover the whole frame at 0.2f + 1..4 ulp and two at 0.2f itself."""
    rng = np.random.default_rng(seed)
    W, H = W0, H0
    k = np.repeat(NEAR_OFFSETS, 3)
    kb = np.r_[1, 1, 2, 2, 3, 3, 4, 4, 0, 0]
    z = _ulps(np.full(len(k) + len(kb), NEAR), np.r_[k, kb])
    n = len(z)
    u = np.r_[rng.uniform(8, W - 8, len(k)), rng.uniform(0.3 * W, 0.7 * W, len(kb))]
    v = np.r_[rng.uniform(8, H - 8, len(k)), rng.uniform(0.3 * H, 0.7 * H, len(kb))]
    xyz = place(u, v, np.ones(n), W, H, FOCAL0, 0.0) * z.astype(F64)[:, None]
    xyz[:, 2] = z
    sig_px = np.r_[rng.uniform(2, 6, len(k)), rng.uniform(250, 400, len(kb))]
    scales, rot = _spheres(rng, n, sig_px * 0.2 / FOCAL0)
    op = np.r_[rng.uniform(0.3, 0.9, len(k)), rng.uniform(0.05, 0.15, len(kb))]
    return _geo("near_plane", identity_view(W, H, FOCAL0), xyz.astype(F), scales, rot, op, rng.uniform(0.05, 0.95, (n, 3)),
                ulps=np.r_[k, kb], covers_frame=np.arange(len(k), n))


NEAR_ANGLES = (23.0, -37.0, 61.0)
NEAR_T = (0.021, -0.013, 0.017)  # camera near the world origin: one ulp of a world coordinate moves the depth < 1 ulp


def near_plane_rotated(seed=21):
    """A rotated camera.  Seeded search over world points near the plane (each base point scanned over +-6 ulp per coordinate):
    the plainly rounded and both contracted depth dot products agree at 0.2f exactly and at 1..4 ulp either side (four
    Gaussians per offset), then up to 16 points where both contractions fall on the other side of 0.2 from the plainly
    rounded sum, then six frame-covering Gaussians 1..3 ulp in front of the plane."""
    rng = np.random.default_rng(seed)
    W, H = W0, H0
    vt = rotated_view(W, H, FOCAL0, NEAR_ANGLES, NEAR_T)
    nb = 400
    u, v = rng.uniform(10, W - 10, nb), rng.uniform(10, H - 10, nb)
    pv = np.c_[(u - (W - 1) / 2) * 0.2 / FOCAL0, (v - (H - 1) / 2) * 0.2 / FOCAL0, np.full(nb, 0.2)]
    base = to_world(vt, pv).astype(F)
    g = np.arange(-6, 7)
    steps = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3).astype(np.int32)  # +-6 ulp per coordinate
    cand = _ulps(np.repeat(base, len(steps), 0), np.tile(steps, (nb, 1)))
    plain, late, early = view_depths(cand, vt.world_view)
    origin = np.repeat(np.arange(nb), len(steps))
    used = np.zeros(nb, bool)
    pick, offs = [], []

    def take(mask, k, off):
        got = 0
        for i in np.flatnonzero(mask):
            if got == k:
                break
            if not used[origin[i]]:
                used[origin[i]] = True
                pick.append(i)
                offs.append(off)
                got += 1

    agree = (plain == late) & (late == early)
    bits = plain.view(np.int32) - NEAR.view(np.int32)
    for off in range(-4, 5):
        take(agree & (bits == off), 4, off)
    split = ((late > NEAR) == (early > NEAR)) & ((late > NEAR) != (plain > NEAR))
    take(split & (late > NEAR), 8, 99)  # both directions of the split
    take(split & (late <= NEAR), 8, 99)
    cover = agree & (bits >= 1) & (bits <= 3)
    take(cover, 6, 100)
    pick, offs = np.asarray(pick), np.asarray(offs)
    xyz = cand[pick]
    n = len(xyz)
    big = offs == 100
    sig_px = np.where(big, rng.uniform(250, 400, n), rng.uniform(2, 6, n))
    scales, rot = _spheres(rng, n, sig_px * 0.2 / FOCAL0)
    op = np.where(big, 0.1, rng.uniform(0.3, 0.9, n))
    return _geo("near_plane_rotated", vt, xyz, scales, rot, op, rng.uniform(0.05, 0.95, (n, 3)), ulps=offs,
                split=np.flatnonzero(offs == 99), covers_frame=np.flatnonzero(big))


# ---------------------------------------------------------------------------------------------------- guard band

GUARD_RATIOS = [1 - 1e-3, 1 - 2 ** -18, 1 + 2 ** -18, 1 + 1e-3, 1.05, 1.2]


def guard_band(seed=22):
    """Identity camera, 320 x 240.  Centres with |t.x/t.z| (left / right edge), |t.y/t.z| (top / bottom edge) or both
    (corners) at GUARD_RATIOS x 1.3 tan(fov), two of each, the other coordinate inside the frame; near-spherical Gaussians
    (so the clamped third column of J matters) large enough that their footprints reach into the frame."""
    rng = np.random.default_rng(seed)
    W, H = W0, H0
    vt = identity_view(W, H, FOCAL0)
    lx, ly = lim(vt)
    rows = []
    for r in GUARD_RATIOS:
        for sx, sy in ((1, 0), (-1, 0), (0, 1), (0, -1), (1, 1), (-1, -1), (1, -1), (-1, 1)):
            for _ in range(2):
                tx = sx * r * float(lx) if sx else rng.uniform(-0.6, 0.6) * float(lx) / 1.3
                ty = sy * r * float(ly) if sy else rng.uniform(-0.6, 0.6) * float(ly) / 1.3
                rows.append((tx, ty))
    rows = np.asarray(rows)
    n = len(rows)
    z = rng.uniform(1.5, 3.0, n).astype(F)
    xyz = np.c_[rows * z[:, None].astype(F64), z].astype(F)
    scales, rot = _spheres(rng, n, rng.uniform(45, 70, n) * z / FOCAL0)
    return _geo("guard_band", vt, xyz, scales, rot, rng.uniform(0.3, 0.9, n), rng.uniform(0.05, 0.95, (n, 3)))


# ---------------------------------------------------------------------------------------------------- tile-edge centres

def _tile_edge_search(rng, vt, axis, n_targets, r):
    """World positions (identity camera) whose pixel coordinate on `axis` is within an ulp of a tile edge of a radius-r
    rectangle, where ndc2Pix in float32 (either form) lands on the other side of it than ndc2Pix in double."""
    W, H = vt.width, vt.height
    size = W if axis == 0 else H
    pm = np.asarray(vt.full_proj, F).reshape(16)
    p = pm[0] if axis == 0 else pm[5]
    out = []
    for _ in range(n_targets * 6):
        if len(out) == n_targets:
            break
        z = F(rng.uniform(2.0, 6.0))
        lo_edge = rng.integers(0, 2) == 0
        kt = rng.integers(2, size // 16 - 2)
        N = 16 * kt + r if lo_edge else 16 * kt - r - 15  # (px - r)/16 or (px + r + 15)/16 is an integer here
        if not 4 <= N <= size - 5:
            continue
        proj = (2 * N + 1) / size - 1
        x0 = F(proj * float(z) / float(p))
        xs = _ulps(np.full(801, x0), (np.arange(-400, 401) * (1 if x0 >= 0 else -1)).astype(np.int32))
        pw = F(1) / (z + F(1e-7))
        pj = (p * xs) * pw
        dbl, plain, fused = ndc2pix(pj, size)
        hit = ((dbl >= N) != (plain >= N)) & ((dbl >= N) != (fused >= N))
        if hit.any():
            i = np.flatnonzero(hit)[rng.integers(0, hit.sum())]
            out.append((xs[i], z))
    return out


def tile_edge_centres(seed=23, r=10, n_per_axis=24):
    """Identity camera, 320 x 240; round discs of radius r px facing the camera.  Seeded search for centres whose getRect
    rectangle changes by one tile when ndc2Pix is evaluated in float32 instead of double: n_per_axis on each axis (x0 / x1
    and y0 / y1 edges mixed), the other coordinate in the middle of a tile."""
    rng = np.random.default_rng(seed)
    W, H = W0, H0
    vt = identity_view(W, H, FOCAL0)
    sig_px = math.sqrt(((r - 0.5) / 3) ** 2 - 0.3 - math.sqrt(0.1))  # 3 sqrt(lambda) = r - 0.5: radius r
    xyz = []
    for axis in (0, 1):
        for c, z in _tile_edge_search(rng, vt, axis, n_per_axis, r):
            other = (16 * rng.integers(1, (H if axis == 0 else W) // 16 - 1) + 8.0 - ((H if axis == 0 else W) - 1) / 2)
            o = F(other * float(z) / FOCAL0)
            xyz.append((c, o, z) if axis == 0 else (o, c, z))
    xyz = np.asarray(xyz, F)
    n = len(xyz)
    s = np.repeat((sig_px * xyz[:, 2].astype(F64) / FOCAL0)[:, None], 3, 1) * np.array([1.0, 1.0, 0.01])
    rot = np.zeros((n, 4), F)
    rot[:, 0] = 1
    return _geo("tile_edge_centres", vt, xyz, s, rot, rng.uniform(0.3, 0.9, n), rng.uniform(0.05, 0.95, (n, 3)), radius=r)


# ---------------------------------------------------------------------------------------------------- covariances

DET0_TARGETS = [0.5, 0.75, 1.0, 1.25, 1.5, 2.0, 3.0, 4.5]  # few significant bits: a * a is exact in float32


def _hit(f, start, target, span=4000):
    """The float32 v nearest `start` (scanning +-span ulp) with f(v) == target, or None."""
    vs = _ulps(np.full(2 * span + 1, F(start)), np.arange(-span, span + 1, dtype=np.int32))
    ok = np.flatnonzero(f(vs) == F(target))
    return None if ok.size == 0 else vs[ok[np.argmin(np.abs(ok - span))]]


def det0_cov(vt, z, a):
    """cov3D_precomp of a Gaussian on the optical axis (identity camera) at depth z whose 2-D covariance after the +0.3
    low-pass is exactly [[a, a], [a, a]]: every product of the EWA projection has a single non-zero term there, so
    cxx = fl(fl(jx V00) jx + 0.3), cyy = fl(fl(jy V11) jy + 0.3), cxy = fl(fl(jy V01) jx) hold bit for bit, and
    cxx cyy - cxy^2 = a^2 - a^2 = 0 exactly under any contraction."""
    fx, fy = focal(vt)
    jx, jy = F(fx / F(z)), F(fy / F(z))
    v00 = _hit(lambda v: (v * jx) * jx + F(0.3), (a - 0.3) / float(jx) ** 2, a)
    v11 = _hit(lambda v: (v * jy) * jy + F(0.3), (a - 0.3) / float(jy) ** 2, a)
    v01 = _hit(lambda v: (v * jy) * jx, a / (float(jx) * float(jy)), a)
    if v00 is None or v11 is None or v01 is None:
        return None
    return np.array([v00, v01, F(0.1) * v00, v11, F(-0.05) * v11, F(0.2) * v00], F)


def degenerate_cov(seed=24, scale_modifier=1.0):
    """cov3D_precomp path, identity camera, 320 x 240:
      * 64 indefinite matrices R diag(s1^2, -s2^2, s3^2) R^T whose projected 2-D covariance is indefinite (negative
        determinant: exact culling must keep their whole rectangle), spread over the frame;
      * DET0_TARGETS: matrices whose float32 2-D determinant is exactly 0 (the Gaussian is culled), on the optical axis at
        depths where the projection's scale jx < 1 (so the seeded search reaches every float32 2-D covariance);
      * 16 ordinary positive-definite ones;
      * 16 indefinite ones whose 2-D diagonal is negative: conic a, c > 0 with ac - b^2 < 0 and k = ac / (ac - b^2) < -2e4,
        so only the determinant test keeps make_footprint from treating them as ellipses (with tau < 0: nothing drawn).
    scale_modifier is passed through: the cov3D_precomp path must ignore it."""
    rng = np.random.default_rng(seed)
    W, H = W0, H0
    vt = identity_view(W, H, FOCAL0)
    n_ind, n_pd = 64, 16
    u, v = rng.uniform(20, W - 20, n_ind + n_pd), rng.uniform(20, H - 20, n_ind + n_pd)
    z = rng.uniform(2.0, 5.0, n_ind + n_pd)
    xyz = place(u, v, z, W, H, FOCAL0, 0.0)
    s = rng.uniform(8, 30, (n_ind + n_pd, 3)) * z[:, None] / FOCAL0
    sign = np.ones((n_ind + n_pd, 3))
    sign[:n_ind, 1] = -1
    q = unit_quats(rng, n_ind + n_pd).astype(F64)
    covs = []
    for i in range(n_ind + n_pd):
        R = _quat_to_mat(q[i])
        Vm = R @ np.diag(sign[i] * s[i] ** 2) @ R.T
        covs.append(Vm[[0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]])
    covs = np.asarray(covs, F)
    d0_xyz, d0_cov = [], []
    for a in DET0_TARGETS:
        zz = F(rng.uniform(1.4, 1.9) * FOCAL0)
        c = det0_cov(vt, zz, a)
        if c is not None:
            d0_xyz.append((0.0, 0.0, zz))
            d0_cov.append(c)
    # 2-D covariance [[-s, +-s(1 + e)], [+-s(1 + e), -s]] after the low-pass: conic a, c > 0 but ac - b^2 < 0, and
    # k = cxx cyy / det = -1 / (2e) < -2e4, so a footprint that trusted a and c alone would get tau < 0 (nothing blended)
    n_neg = 16
    zn = rng.uniform(2.0, 5.0, n_neg)
    fx, fy = (float(f) for f in focal(vt))
    sn, en = rng.uniform(5e4, 2e5, n_neg), rng.uniform(1e-5, 2e-5, n_neg)
    jx, jy = fx / zn, fy / zn
    neg = np.zeros((n_neg, 6))
    neg[:, 0] = (-sn - 0.3) / jx ** 2
    neg[:, 3] = (-sn - 0.3) / jy ** 2
    neg[:, 1] = np.where(np.arange(n_neg) % 2, -1, 1) * sn * (1 + en) / (jx * jy)
    xyz = np.r_[xyz, np.asarray(d0_xyz, F), place(rng.uniform(20, W - 20, n_neg), rng.uniform(20, H - 20, n_neg), zn, W, H,
                                                  FOCAL0, 0.0)]
    cov = np.r_[covs, np.asarray(d0_cov, F), neg.astype(F)]
    n = len(xyz)
    n_d0 = len(d0_xyz)
    case = _geo("degenerate_cov" if scale_modifier == 1.0 else f"degenerate_cov_sm{scale_modifier}", vt, xyz,
                np.ones((n, 3)), np.tile([1.0, 0, 0, 0], (n, 1)), rng.uniform(0.3, 0.9, n), rng.uniform(0.05, 0.95, (n, 3)),
                indefinite=np.r_[np.arange(n_ind), np.arange(n - n_neg, n)], det0=np.arange(n_ind + n_pd, n_ind + n_pd + n_d0),
                det0_target=np.asarray(DET0_TARGETS, F), tau_negative=np.arange(n - n_neg, n))
    case.cov3D = cov
    case.scale_modifier = float(scale_modifier)
    return case


def _quat_to_mat(q):
    r, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y)],
                     [2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x)],
                     [2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)]])


# ---------------------------------------------------------------------------------------------------- needles

def _needle_cloud(rng, n, W, H, z, theta, sl_px, ss_px):
    u, v = rng.uniform(0.25 * W, 0.75 * W, n), rng.uniform(0.25 * H, 0.75 * H, n)
    xyz = place(u, v, z, W, H, FOCAL0, 0.0)
    s = np.c_[sl_px * z / FOCAL0, ss_px * z / FOCAL0, np.full(n, 1e-4) * z]
    rot = np.c_[np.cos(theta / 2), np.zeros(n), np.zeros(n), np.sin(theta / 2)]
    return xyz, s, rot


def needles(oracle, seed=25):
    """Identity camera, 320 x 240; thin discs facing the camera, rotated in the image plane.  Seeded search (CPU oracle
    conics, float32 k as shrink_rect computes it): eight Gaussians each with k exactly 1000, 1..3 ulp below and above it,
    within 0.5 % below and above it, and eight with k >= 1e4."""
    rng = np.random.default_rng(seed)
    W, H = W0, H0
    vt = identity_view(W, H, FOCAL0)
    nb, span = 256, 300
    z = rng.uniform(3.0, 6.0, nb)
    theta = rng.uniform(np.pi / 6, np.pi / 3, nb) * rng.choice([-1, 1], nb)
    sl = rng.uniform(40, 80, nb)
    # long / short axis variances in px^2 (+0.3 low-pass): k = (l1 + l2)^2 / (4 l1 l2) at theta = 45 deg, roughly; solve
    # for the short axis in float64 at the actual angle, then scan it over +-span ulp
    ss = np.empty(nb)
    for i in range(nb):
        lo, hi = 1e-4, sl[i]
        for _ in range(80):
            mid = 0.5 * (lo + hi)
            lo, hi = (mid, hi) if _k64(sl[i], mid, theta[i]) > 1000 else (lo, mid)
        ss[i] = 0.5 * (lo + hi)
    xyz, s, rot = _needle_cloud(rng, nb, W, H, z, theta, sl, ss)
    steps = np.arange(-span, span + 1)
    cx = np.repeat(xyz, len(steps), 0)
    cs = np.repeat(s, len(steps), 0).astype(F)
    cs[:, 1] = _ulps(cs[:, 1], np.tile(steps, nb).astype(np.int32))
    cr = np.repeat(rot, len(steps), 0)
    cand = _geo("cand", vt, cx, cs, cr, np.full(len(cx), 0.6), np.full((len(cx), 3), 0.5))
    pre = preprocess(oracle, cand)
    k = conic_k(pre["conic_opacity"])
    kb = k.view(np.int32) - F(1000).view(np.int32)
    origin = np.repeat(np.arange(nb), len(steps))
    used = np.zeros(nb, bool)
    pick, tag = [], []
    for name, mask in (("at", kb == 0), ("below_ulp", (kb < 0) & (kb >= -3)), ("above_ulp", (kb > 0) & (kb <= 3)),
                       ("below", (k < 1000) & (k > 995)), ("above", (k > 1000) & (k < 1005))):
        got = 0
        for i in np.flatnonzero(mask & (pre["radii"] > 0)):
            if got == 8:
                break
            if not used[origin[i]] or name != "at":
                used[origin[i]] = True
                pick.append(i)
                tag.append(name)
                got += 1
    pick = np.asarray(pick)
    m = 8
    zf = rng.uniform(3.0, 6.0, m)
    fx, fs, fr = _needle_cloud(rng, m, W, H, zf, rng.uniform(0.6, 1.0, m), rng.uniform(140, 200, m), np.full(m, 0.05))
    xyz = np.r_[cx[pick], fx].astype(F)
    s = np.r_[cs[pick], fs].astype(F)
    rot = np.r_[cr[pick], fr].astype(F)
    tag = np.asarray(tag + ["huge_k"] * m)
    n = len(xyz)
    return _geo("needles", vt, xyz, s, rot, rng.uniform(0.3, 0.9, n), rng.uniform(0.05, 0.95, (n, 3)), tag=tag)


def _k64(sl, ss, theta):
    c, s_ = math.cos(theta), math.sin(theta)
    cxx = sl ** 2 * c * c + ss ** 2 * s_ * s_ + 0.3
    cyy = sl ** 2 * s_ * s_ + ss ** 2 * c * c + 0.3
    cxy = (sl ** 2 - ss ** 2) * c * s_
    return cxx * cyy / (cxx * cyy - cxy * cxy)


# ---------------------------------------------------------------------------------------------------- huge footprints

HUGE_W, HUGE_H = 1600, 1200


def huge_footprints(seed=26, n=96):
    """1600 x 1200, identity camera; round discs facing the camera with radii log-spread from the frame size to 1e5 px,
    a third centred inside the frame, a third just outside it (the rectangle still reaches in), a third far outside (up
    to 0.8 radius away from the frame).  At most n * 7500 instances."""
    rng = np.random.default_rng(seed)
    W, H, f = HUGE_W, HUGE_H, 0.9 * HUGE_W
    r = np.exp(rng.uniform(np.log(max(W, H)), np.log(1e5), n))
    where = np.arange(n) % 3
    u, v = rng.uniform(0, W, n), rng.uniform(0, H, n)
    ang = rng.uniform(0, 2 * np.pi, n)
    out = np.where(where == 1, rng.uniform(0.05, 0.3, n), rng.uniform(0.3, 0.8, n)) * r
    u = np.where(where == 0, u, W / 2 + np.cos(ang) * (W / 2 + out))
    v = np.where(where == 0, v, H / 2 + np.sin(ang) * (H / 2 + out))
    z = rng.uniform(2.0, 10.0, n)
    sig = np.sqrt(np.maximum((r / 3) ** 2 - 0.3 - math.sqrt(0.1), 0.01))
    xyz = place(u, v, z, W, H, f, 0.0)
    s = np.c_[sig * z / f, sig * z / f, 0.01 * sig * z / f]
    rot = np.tile([1.0, 0, 0, 0], (n, 1))
    return _geo("huge_footprints", identity_view(W, H, f), xyz, s, rot, rng.uniform(0.02, 0.2, n), rng.uniform(0.05, 0.95, (n, 3)),
                focal_px=f, where=where)


# ---------------------------------------------------------------------------------------------------- opacity

ALPHA_MIN = F(1) / F(255)
OPACITY_EDGES = np.array([0.0, np.nextafter(ALPHA_MIN, F(0)), ALPHA_MIN, np.nextafter(F(1), F(0)), 1.0], F)


def opacity_edges(seed=27, per=8):
    """320 x 240, identity camera: `per` large overlapping Gaussians (radius 60..150 px) at each of OPACITY_EDGES."""
    rng = np.random.default_rng(seed)
    W, H = W0, H0
    n = per * len(OPACITY_EDGES)
    op = np.tile(OPACITY_EDGES, per)
    z = rng.uniform(2.0, 6.0, n)
    xyz = place(rng.uniform(0, W, n), rng.uniform(0, H, n), z, W, H, FOCAL0, 0.0)
    scales, rot = _spheres(rng, n, rng.uniform(20, 50, n) * z / FOCAL0)
    return _geo("opacity_edges", identity_view(W, H, FOCAL0), xyz, scales, rot, op, rng.uniform(0.05, 0.95, (n, 3)))


# ---------------------------------------------------------------------------------------------------- quaternions

def quaternions(seed=28, per=12):
    """320 x 240, rotated camera; anisotropic Gaussians whose quaternions have norm 0.5 (`per`), norm 2 (`per`), are zero
    (`per`: R = I) or come in sign-flipped pairs q, -q of random norm (`per` pairs, adjacent)."""
    rng = np.random.default_rng(seed)
    W, H = W0, H0
    vt = rotated_view(W, H, FOCAL0, (12.0, 31.0, -17.0), (0.05, -0.1, 0.0))
    q_half = 0.5 * unit_quats(rng, per)
    q_two = 2.0 * unit_quats(rng, per)
    q_zero = np.zeros((per, 4))
    q_pair = unit_quats(rng, per) * rng.uniform(0.3, 3.0, (per, 1))
    q_pairs = np.empty((2 * per, 4))
    q_pairs[0::2], q_pairs[1::2] = q_pair, -q_pair
    rot = np.r_[q_half, q_two, q_zero, q_pairs].astype(F)
    n = len(rot)
    z = rng.uniform(2.0, 5.0, n)
    xyz = to_world(vt, np.c_[(rng.uniform(30, W - 30, n) - (W - 1) / 2) * z / FOCAL0,
                             (rng.uniform(30, H - 30, n) - (H - 1) / 2) * z / FOCAL0, z])
    s = rng.uniform(3, 20, (n, 3)) * z[:, None] / FOCAL0
    s[:, rng.integers(0, 3)] *= 0.2
    s[3 * per + 1::2] = s[3 * per::2]  # a pair shares its scales: only the quaternion's sign differs
    kind = np.repeat(["half", "two", "zero", "pair"], [per, per, per, 2 * per])
    return _geo("quaternions", vt, xyz, s, rot, rng.uniform(0.3, 0.9, n), rng.uniform(0.05, 0.95, (n, 3)), kind=kind)


# ---------------------------------------------------------------------------------------------------- SH colour clamp

SH_DEGREES = [0, 1, 2, 3]


def sh_clamp(deg, seed=29, n=64):
    """320 x 240, identity camera at the origin.  Degree-`deg` SH whose colours land far below 0 and above 1: DC terms
    from {-2.5, -0.8, 0.4, 1.3, 2.5} / C0 per channel, higher orders N(0, 1).  A quarter of the Gaussians sit on the optical
    axis (view direction (0, 0, 1) exactly: every basis function with an x or y factor vanishes), a quarter in the plane
    x = 0 and a quarter in y = 0 (the x resp. y terms vanish), the rest anywhere."""
    rng = np.random.default_rng(seed + deg)
    W, H = W0, H0
    z = rng.uniform(2.0, 6.0, n).astype(F)
    u, v = rng.uniform(20, W - 20, n), rng.uniform(20, H - 20, n)
    xyz = place(u, v, z, W, H, FOCAL0, 0.0)
    q = n // 4
    xyz[:q, :2] = 0
    xyz[q:2 * q, 0] = 0
    xyz[2 * q:3 * q, 1] = 0
    xyz[:, 2] = z
    feats = rng.normal(0, 1.0, (n, sh_basis_count(deg), 3))
    feats[:, 0, :] = rng.choice([-2.5, -0.8, 0.4, 1.3, 2.5], (n, 3)) / SH_C0
    scales, rot = _spheres(rng, n, rng.uniform(4, 12, n) * z / FOCAL0)
    return _geo(f"sh_clamp_d{deg}", identity_view(W, H, FOCAL0), xyz.astype(F), scales, rot, rng.uniform(0.3, 0.9, n),
                features=feats.astype(F), sh_degree=deg, on_axis=np.arange(q))


def colors_precomp(seed=30, n=64):
    """colors_precomp in [-0.5, 1.5] per channel: passed through unclamped."""
    rng = np.random.default_rng(seed)
    case = sh_clamp(0, seed=seed, n=n)
    case.name = "colors_precomp"
    case.colors = rng.uniform(-0.5, 1.5, (n, 3)).astype(F)
    return case


# ---------------------------------------------------------------------------------------------------- toed-in pair

TOE_DEG, TOE_BASELINE = 8.0, 0.12


def toed_in_views(W=W0, H=H0, focal_px=FOCAL0):
    """Two cameras TOE_BASELINE apart along world x, each turned TOE_DEG towards the other, with a common pitch and roll:
    their view matrices share no row."""
    fov_x, fov_y = 2 * math.atan(W / (2 * focal_px)), 2 * math.atan(H / (2 * focal_px))
    out = []
    for side in (-1, 1):
        R = cam.euler_deg_to_matrix((7.0, -side * TOE_DEG, 3.0))
        C = np.array([side * TOE_BASELINE / 2, 0.0, 0.0])
        out.append(cam.view_transforms(R, -R.T @ C, fov_x, fov_y, W, H))
    return out


def toed_in_pair(oracle, seed=31):
    """Degree-3 Gaussians around the near plane of the rig and around the outer frame edges of each eye, seeded and then
    picked with the CPU oracle: 24 each that only the left / only the right eye culls at the near plane (the other eye
    renders them), 24 each that only one eye culls off-screen, and 96 both eyes render."""
    rng = np.random.default_rng(seed)
    W, H = W0, H0
    vl, vr = toed_in_views()
    m = 6000
    z = rng.uniform(0.1, 0.5, m)
    xyz = np.c_[rng.uniform(-0.9, 0.9, m) * z, rng.uniform(-0.5, 0.5, m) * z, z]
    feats = rng.normal(0, 0.3, (m, 16, 3))
    scales, rot = _spheres(rng, m, rng.uniform(2, 6, m) * z / FOCAL0)
    cand = _geo("cand", vl, xyz.astype(F), scales, rot, rng.uniform(0.3, 0.9, m), features=feats.astype(F), sh_degree=3)
    pre = [preprocess(oracle, cand, vt=v) for v in (vl, vr)]
    dep = [view_depths(cand.cloud.xyz, v.world_view) for v in (vl, vr)]
    front = [(d[0] > NEAR * F(1.001)) & (d[1] > NEAR * F(1.001)) for d in dep]
    behind = [(d[0] < NEAR * F(0.999)) & (d[1] < NEAR * F(0.999)) for d in dep]
    vis = [p["radii"] > 0 for p in pre]
    groups = dict(near_left=vis[1] & behind[0], near_right=vis[0] & behind[1], off_left=vis[1] & front[0] & ~vis[0],
                  off_right=vis[0] & front[1] & ~vis[1], both=vis[0] & vis[1])
    pick, tag = [], []
    for name, mask in groups.items():
        k = 96 if name == "both" else 24
        idx = np.flatnonzero(mask)
        assert len(idx) >= k, (name, len(idx))
        pick.append(rng.choice(idx, k, replace=False))
        tag += [name] * k
    pick = np.concatenate(pick)
    perm = rng.permutation(len(pick))  # mixed across warps
    pick, tag = pick[perm], np.asarray(tag)[perm]
    g = cand.cloud
    case = _geo("toed_in_pair", vl, g.xyz[pick], g.scaling[pick], g.rotation[pick], g.opacity[pick], features=g.features[pick],
                sh_degree=3, tag=tag)
    case.info["right"] = vr
    return case


# ---------------------------------------------------------------------------------------------------- registry

def build(name, oracle=None):
    if name.startswith("sh_clamp_d"):
        return sh_clamp(int(name[-1]))
    if name in ("needles", "toed_in_pair"):
        return globals()[name](oracle)
    if name == "degenerate_cov_sm0.5":
        return degenerate_cov(scale_modifier=0.5)
    return globals()[name]()


SINGLE_CASES = ["near_plane", "near_plane_rotated", "guard_band", "tile_edge_centres", "degenerate_cov", "needles",
                "huge_footprints", "opacity_edges", "quaternions"] + [f"sh_clamp_d{d}" for d in SH_DEGREES] + ["colors_precomp"]


def blend64(pre, W, H, bg):
    """forward.cu's blend restated in float64 from the oracle's per-Gaussian records (pre: preprocess output): every pixel
    takes the Gaussians whose tile rectangle covers its tile, in (depth, index) order, alpha = min(0.99, o exp(power)),
    skipped below 1/255, stopping before T drops under 1e-4.  Returns (colour [3, H, W], final_T [H, W])."""
    vis = np.flatnonzero(pre["radii"] > 0)
    order = vis[np.lexsort((vis, pre["depths"][vis]))]
    rects = tile_rects(pre["xy"], pre["radii"], W, H)
    ys, xs = np.mgrid[0:H, 0:W].astype(F64)
    tx, ty = (xs // 16).astype(np.int64), (ys // 16).astype(np.int64)
    T = np.ones((H, W))
    C = np.zeros((3, H, W))
    live = np.ones((H, W), bool)
    for i in order:
        x0, y0, x1, y1 = rects[i]
        a, b, c, op = (float(v) for v in pre["conic_opacity"][i])
        dx, dy = float(pre["xy"][i, 0]) - xs, float(pre["xy"][i, 1]) - ys
        power = -0.5 * (a * dx * dx + c * dy * dy) - b * dx * dy
        alpha = np.minimum(0.99, op * np.exp(np.minimum(power, 0.0)))
        use = live & (tx >= x0) & (tx < x1) & (ty >= y0) & (ty < y1) & (power <= 0) & (alpha >= 1 / 255)
        test_T = T * (1 - alpha)
        stop = use & (test_T < 1e-4)
        live &= ~stop
        use &= ~stop
        C += np.where(use, alpha * T, 0.0) * pre["rgb"][i].astype(F64)[:, None, None]
        T = np.where(use, test_T, T)
    return C + T * np.asarray(bg, F64)[:, None, None], T
