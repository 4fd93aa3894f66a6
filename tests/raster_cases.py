"""Rasterizer inputs aimed at the code paths of gsb_raster.cu / gsb_radix.cuh that change with size or shape, and host
restatements that show each input reaches its edge (tests/test_raster_cases_host.py checks them on the CPU,
tests/test_gpu_raster_limits.py renders them).

Every constructor is seeded and returns a Case.  The cameras are built directly: identity rotation, looking down +z,
translation t, so a Gaussian at world z has view depth fl(z + t_z) -- the same float for every Gaussian at one world z --
and lands on pixel (W-1)/2 + f x/z_view, (H-1)/2 + f y/z_view.  Gaussians are flat discs facing the camera (scales
s, s, s/100, identity rotation), so their screen footprint stays round away from the optical axis: sigma_px = f s / z_view
and radius = ceil(3 sqrt(sigma_px^2 + 0.3 + sqrt(0.1))).  Colours are degree-0 SH equal to the given rgb."""
from __future__ import annotations

import math
from dataclasses import dataclass, field

import numpy as np

from gs2mesh_b200 import camera as cam
from gs2mesh_b200.scene import GaussianCloud

F = np.float32
TILE = 16
SIDE_LIMIT = 8191 * TILE  # validate_frame: packed rectangles hold 13-bit tile coordinates
SMALL_SORT = 1 << 22  # kRdxSmallSort: sorts of up to this many items run radix_pass_kernel<8>, larger ones <16>
DEPTH_SORT_BLOCK = 256 * 8  # items per CTA of the 8-item (depth) sort
SCAN_BLOCK = 1024 * 8  # kScanBlock: items per CTA of scan_tiles_kernel
SCAN_WINDOW = 32  # predecessors one look-back round of scan_tiles_kernel inspects
SH_C0 = 0.28209479177387814
ALPHA_MIN = F(1.0) / F(255.0)
T_MIN = F(0.0001)


@dataclass
class Case:
    name: str
    cloud: GaussianCloud
    vt: cam.ViewTransforms
    focal: float
    tz: float
    info: dict = field(default_factory=dict)  # what the constructor aimed at (indices of special Gaussians, ...)

    @property
    def W(self):
        return self.vt.width

    @property
    def H(self):
        return self.vt.height

    @property
    def P(self):
        return self.cloud.num_points

    def right_eye(self, baseline):
        """The other eye of a rig: shifted along the camera x axis, same z row of the view matrix (shared view depth)."""
        return identity_view(self.W, self.H, self.focal, (-baseline, 0.0, self.tz))


def identity_view(W, H, focal, t=(0.0, 0.0, 0.0)) -> cam.ViewTransforms:
    fov_x, fov_y = 2 * math.atan(W / (2 * focal)), 2 * math.atan(H / (2 * focal))
    wv = np.eye(4, dtype=F)
    wv[3, :3] = np.asarray(t, F)  # row-vector convention: view = [x y z 1] @ wv
    proj = cam.projection_matrix(cam.ZNEAR, cam.ZFAR, fov_x, fov_y).T
    full = (wv @ proj).astype(F)
    return cam.ViewTransforms(world_view=wv, full_proj=np.ascontiguousarray(full), cam_center=-np.asarray(t, F),
                              tan_fovx=math.tan(fov_x * 0.5), tan_fovy=math.tan(fov_y * 0.5), width=int(W), height=int(H))


def place(u, v, zv, W, H, focal, tz):
    """World positions of Gaussians that land near pixel (u, v) at view depth zv."""
    zv = np.asarray(zv, np.float64)
    x = (np.asarray(u, np.float64) - (W - 1) / 2) * zv / focal
    y = (np.asarray(v, np.float64) - (H - 1) / 2) * zv / focal
    return np.stack([x, y, zv - tz], -1).astype(F)


def cloud(xyz, sigma_world, opacity, rgb) -> GaussianCloud:
    P = len(xyz)
    s = np.asarray(sigma_world, np.float64).reshape(-1, 1) * np.array([[1.0, 1.0, 0.01]])
    s = np.broadcast_to(s, (P, 3))
    feats = ((np.asarray(rgb, np.float64).reshape(P, 1, 3) - 0.5) / SH_C0).astype(F)
    rot = np.zeros((P, 4), F)
    rot[:, 0] = 1
    return GaussianCloud(np.ascontiguousarray(xyz, F), np.ascontiguousarray(feats), np.asarray(opacity, F).reshape(P, 1).copy(),
                         np.ascontiguousarray(s, F), rot, sh_degree=0)


def sigma_world(sigma_px, zv, focal):
    return np.asarray(sigma_px, np.float64) * np.asarray(zv, np.float64) / focal


def sigma_for_radius(r):
    """sigma_px of a disc whose rectangle radius is ~r px."""
    return np.sqrt(np.maximum((np.asarray(r, np.float64) / 3) ** 2 - 0.3 - math.sqrt(0.1), 0.01))


def _make(name, W, H, focal, tz, u, v, zv, sig_px, opacity, rgb, **info):
    xyz = place(u, v, zv, W, H, focal, tz)
    return Case(name, cloud(xyz, sigma_world(sig_px, zv, focal), opacity, rgb), identity_view(W, H, focal, (0.0, 0.0, tz)),
                float(focal), float(tz), info)


# ---------------------------------------------------------------------------------------------------- host restatements

def higher_msb(n: int) -> int:
    """rasterizer_impl.cu's binary search for the most significant bit (tile-id bits of the tile sort)."""
    msb = step = 16
    while step > 1:
        step //= 2
        msb = msb + step if n >> msb else msb - step
    return msb + 1 if n >> msb else msb


def tile_sort_shape(ntiles: int):
    """(key bits, passes, bits per digit) of the tile sort."""
    bits = higher_msb(ntiles)
    passes = (bits + 7) // 8
    return bits, passes, (bits + passes - 1) // passes


def grid(W, H):
    return (W + TILE - 1) // TILE, (H + TILE - 1) // TILE


def tile_rects(xy, radii, W, H):
    """getRect (auxiliary.h) as tile_rect evaluates it, float32, vectorised: int[P, 4] = x0, y0, x1, y1."""
    gx, gy = grid(W, H)
    px, py = np.asarray(xy, F)[:, 0], np.asarray(xy, F)[:, 1]
    r = np.asarray(radii).astype(F)
    t = F(TILE)

    def cv(a, g):  # (uint32) min(g, max(0, (int)a))
        return np.minimum(g, np.maximum(0, np.trunc(a).astype(np.int64)))

    return np.stack([cv((px - r) / t, gx), cv((py - r) / t, gy), cv((px + r + F(TILE - 1)) / t, gx),
                     cv((py + r + F(TILE - 1)) / t, gy)], -1)


def exact_rects(pre, W, H, idx=None):
    """The candidate rectangle under GSB_RASTER_EXACT_TILE_CULL: shrink_rect of the reference rectangle (float32
    restatement of tests/test_exact_cull_math.py), for the Gaussians `idx` (default: all)."""
    from tests.test_exact_cull_math import make_footprint, shrink_rect

    ref = tile_rects(pre["xy"], pre["radii"], W, H)
    out = ref.copy()
    idx = np.arange(len(ref)) if idx is None else np.asarray(idx)
    for i in idx[pre["radii"][idx] > 0]:
        a, b, c, op = (F(v) for v in pre["conic_opacity"][i])
        f = make_footprint(a, b, c, F(2.0) * F(np.log(F(255.0) * op)))
        out[i] = shrink_rect(tuple(int(v) for v in ref[i]), F(pre["xy"][i, 0]), F(pre["xy"][i, 1]), f)
    return out


def rect_shape(rects):
    """(w, h) per rectangle."""
    return np.stack([rects[:, 2] - rects[:, 0], rects[:, 3] - rects[:, 1]], -1)


def rect_margin(xy, radii):
    """Distance, in tiles, of getRect's four quotients from the nearest integer: a rectangle with a margin well above the
    host/GPU rounding difference of the projected centre (~1e-5 relative) is the same rectangle on both."""
    px, py = np.asarray(xy, np.float64)[:, 0], np.asarray(xy, np.float64)[:, 1]
    r = np.asarray(radii, np.float64)
    q = np.stack([(px - r) / TILE, (py - r) / TILE, (px + r + TILE - 1) / TILE, (py + r + TILE - 1) / TILE], -1)
    return np.abs(q - np.round(q)).min(-1)


def preprocess(oracle, case):
    g = case.cloud
    return oracle.preprocess(g.xyz, g.opacity, case.vt.world_view, case.vt.full_proj, case.vt.cam_center, case.W, case.H,
                             case.vt.tan_fovx, case.vt.tan_fovy, shs=g.features, scales=g.scaling, rotations=g.rotation,
                             sh_degree=0)


def tile_hits(rects, W, H):
    """Reference instances per tile: how many rectangles cover each tile (int[ntiles])."""
    gx, gy = grid(W, H)
    acc = np.zeros((gy + 1, gx + 1), np.int64)
    for x0, y0, x1, y1 in rects:
        if x1 > x0 and y1 > y0:
            acc[y0, x0] += 1
            acc[y0, x1] -= 1
            acc[y1, x0] -= 1
            acc[y1, x1] += 1
    return acc.cumsum(0).cumsum(1)[:gy, :gx].reshape(-1)


def blend_pixel(alphas):
    """forward.cu's blend loop for one pixel, float32: (final T, 1-based hit at which the pixel saturated or None)."""
    T = F(1.0)
    for k, a in enumerate(alphas, 1):
        a = min(F(0.99), F(a))
        if a < ALPHA_MIN:
            continue
        test_T = F(T * F(F(1.0) - a))
        if test_T < T_MIN:
            return T, k
        T = test_T
    return T, None


# ---------------------------------------------------------------------------------------------------- constructors

def random_frame(name, P, W, H, seed, focal=None, tz=0.0, zrange=(2.0, 8.0), sigma_px=(0.3, 2.5), margin=20):
    """P small Gaussians spread over the whole frame at random depths (the sort-size cases)."""
    rng = np.random.default_rng(seed)
    focal = 0.9 * W if focal is None else focal
    u = rng.uniform(-margin, W + margin, P)
    v = rng.uniform(-margin, H + margin, P)
    zv = rng.uniform(*zrange, P)
    return _make(name, W, H, focal, tz, u, v, zv, rng.uniform(*sigma_px, P), rng.uniform(0.1, 1.0, P), rng.uniform(0.05, 0.95, (P, 3)))


def sort_size(P, seed=0):
    """P Gaussians on a C1-sized (1600x1200) frame: the depth sort's item count is P."""
    return random_frame(f"P{P}", P, 1600, 1200, seed)


SORT_SIZES = [SMALL_SORT, SMALL_SORT + 1, SCAN_BLOCK * (SCAN_WINDOW + 2) + 1, 3 * DEPTH_SORT_BLOCK - 1, 3 * DEPTH_SORT_BLOCK + 1,
              3 * SCAN_BLOCK - 1, 3 * SCAN_BLOCK + 1]


def depth_ties(n=320, seed=1):
    """n overlapping Gaussians at one world z (bitwise-equal view depth 3.0), distinct colours, opacity ~0.5: their blend
    order is the index order, and any other order changes pixel bits."""
    rng = np.random.default_rng(seed)
    W, H, f = 97, 81, 120.0
    u = rng.uniform(24, 72, n)
    v = rng.uniform(20, 60, n)
    return _make("depth_ties", W, H, f, 3.0, u, v, np.full(n, 3.0), rng.uniform(3, 10, n), rng.uniform(0.45, 0.55, n),
                 rng.uniform(0.05, 0.95, (n, 3)))


def _from_depth_bits(name, bits, seed, W=320, H=240):
    rng = np.random.default_rng(seed)
    zv = np.asarray(bits, np.uint32).view(F).astype(np.float64)
    P = len(zv)
    c = _make(name, W, H, 0.9 * W, 0.0, rng.uniform(0, W, P), rng.uniform(0, H, P), zv, rng.uniform(1, 4, P),
              rng.uniform(0.2, 0.9, P), rng.uniform(0.05, 0.95, (P, 3)))
    c.cloud.xyz[:, 2] = zv.astype(F)  # t_z = 0: view depth = world z, bit for bit
    return c


def keys_shared_upper(seed=2):
    """Depth keys 3.0f + k ulp, k < 256: all keys share their upper three bytes (every full warp takes the histogram's
    match-all path in passes 1..3, one bin per pass); the first 16 warps have one key each (match-all in every pass)."""
    rng = np.random.default_rng(seed)
    base = np.uint32(np.float32(3.0).view(np.uint32))
    low = rng.integers(0, 256, 8192).astype(np.uint32)
    low[:512] = np.repeat(rng.integers(0, 256, 16), 32)
    return _from_depth_bits("keys_shared_upper", base + low, seed)


def keys_spread(seed=3, P=20000):
    """Depth keys spread over all 256 bins of the three low passes and over the top byte as far as view depths in
    (0.2, 100) allow."""
    rng = np.random.default_rng(seed)
    zv = np.exp(rng.uniform(np.log(0.21), np.log(99.0), P)).astype(F)
    return _from_depth_bits("keys_spread", zv.view(np.uint32), seed)


# (W, H) -> tile count: 1, 1, 2, 255, 256, 257, 8191, 8192, 8193, 65535, 65536, 65792 (17 bits), 1056639 (21 bits)
TILE_FRAMES = [(1, 1), (16, 16), (32, 16), (4080, 16), (4096, 16), (4112, 16), (SIDE_LIMIT, 16), (2048, 1024), (43696, 48),
               (4080, 4112), (4096, 4096), (4112, 4096), (SIDE_LIMIT, 2064), (16, SIDE_LIMIT)]


def tile_frame(W, H, seed=4):
    """Gaussians over the whole frame -- one per tile up to 70k tiles, one per 4 tiles above, plus one in the first and
    one in the last tile.  On the 131056 x 2064 frame also Gaussians centred right of the frame whose rectangle is the
    last tile column (x0 = 8190) and 64 tiles tall: a full 64-bit mask at the largest packed x0."""
    rng = np.random.default_rng(seed)
    gx, gy = grid(W, H)
    n = gx * gy if gx * gy <= 70_000 else gx * gy // 4
    focal = max(W, H) / 2.0
    t = np.arange(n) if n == gx * gy else rng.integers(0, gx * gy, n)
    u = (t % gx) * TILE + rng.uniform(0, TILE, n)
    v = (t // gx) * TILE + rng.uniform(0, TILE, n)
    u = np.r_[u, 0.5, W - 0.5]
    v = np.r_[v, 0.5, H - 0.5]
    m = len(u)
    zv = rng.uniform(4.0, 8.0, m)
    sig = rng.uniform(0.5, 4.0, m)
    info = {}
    if (W, H) == (SIDE_LIMIT, 2064):
        k = 64  # two full warps of x0 = 8190 rectangles: radius ~508, centre 508 - 8 px right of the frame
        u = np.r_[u, np.full(k, W - 8 + 508.0) + rng.uniform(-0.2, 0.2, k)]
        v = np.r_[v, rng.uniform(600, 1000, k)]  # 64 or 65 tile rows
        zv = np.r_[zv, rng.uniform(4.0, 8.0, k)]
        sig = np.r_[sig, np.full(k, sigma_for_radius(507.5))]
        info["x0_last"] = np.arange(m, m + k)
    P = len(u)
    op = rng.uniform(0.3, 0.9, P)
    if "x0_last" in info:
        op[info["x0_last"]] = 0.95  # opaque enough that exact culling keeps the whole column
    return _make(f"tiles_{W}x{H}", W, H, focal, 0.0, u, v, zv, sig, op, rng.uniform(0.05, 0.95, (P, 3)), **info)


RECT_W = RECT_H = 1024  # 64 x 64 tiles: rectangles up to 64 tiles wide and tall


def _rect_candidates(oracle, rng, n, r_lo, r_hi, opacity, edge_only=False, keep=None):
    """n candidate Gaussians of radius ~[r_lo, r_hi] px, most of them (all with edge_only) centred just outside a frame
    edge (clamped rectangles); returns dict(u, v, zv, sig, op, rect = shape in rectangle mode, exact = shape under exact
    culling (computed where keep(rect shapes) holds), margin, radii)."""
    W, H, f = RECT_W, RECT_H, 1000.0
    r = np.exp(rng.uniform(np.log(r_lo), np.log(r_hi), n))
    sig = sigma_for_radius(r)
    u, v = rng.uniform(0, W, n), rng.uniform(0, H, n)
    edge = rng.integers(1 if edge_only else 0, 5, n)  # 0: interior, 1..4: centre outside the left / right / top / bottom edge
    d = rng.uniform(0, 6 * TILE, n)
    u = np.where(edge == 1, -r + d, np.where(edge == 2, W + r - d, u))
    v = np.where(edge == 3, -r + d, np.where(edge == 4, H + r - d, v))
    zv = rng.uniform(5.0, 15.0, n)
    op = np.full(n, opacity) if np.isscalar(opacity) else opacity
    c = _make("cand", W, H, f, 0.0, u, v, zv, sig, op, np.full((n, 3), 0.5))
    pre = preprocess(oracle, c)
    rect = rect_shape(tile_rects(pre["xy"], pre["radii"], W, H))
    idx = np.arange(n) if keep is None else np.flatnonzero(keep(rect))
    return dict(u=u, v=v, zv=zv, sig=sig, op=op, rect=rect, exact=rect_shape(exact_rects(pre, W, H, idx)),
                margin=rect_margin(pre["xy"], pre["radii"]), radii=pre["radii"])


def _wanted(rect):
    w, h = rect[:, 0], rect[:, 1]
    want = ((w == 8) & (h == 8)) | ((w * h > 64) & (np.arange(len(w)) % 16 == 0))
    for a, b in RECT_SHAPES:
        want |= (w == a) & (h == b)
    return want


RECT_SHAPES = [(64, 1), (1, 64), (2, 32), (32, 2), (7, 9), (9, 7), (63, 1), (1, 63), (5, 13), (13, 5)]


def rects(oracle, seed=5):
    """Packed-rectangle binning on a 1024 x 1024 frame, every Gaussian's rectangle the same in both culling modes:
      warp 0: 32 rectangles of exactly 8 x 8 = 64 tiles (full masks);
      warp 1: rectangles above 64 tiles (cooperative re-test) alternating with rectangles of at most 4 tiles;
      warps 2..: 1x64, 64x1, 2x32, 32x2 and 63- and 65-tile shapes (RECT_SHAPES), then Gaussians below 1/255 opacity
      whose rectangle exact culling shrinks to nothing, mixed with small ones."""
    rng = np.random.default_rng(seed)
    pool = [_rect_candidates(oracle, rng, 40000, 24, 560, rng.uniform(0.6, 0.9, 40000), keep=_wanted),
            _rect_candidates(oracle, rng, 40000, 40, 560, rng.uniform(0.6, 0.9, 40000), edge_only=True, keep=_wanted)]
    small = _rect_candidates(oracle, rng, 4000, 3, 12, 0.5)
    faint = _rect_candidates(oracle, rng, 64, 10, 80, 0.002)
    cand = {k: np.concatenate([p[k] for p in pool]) for k in pool[0]}
    same = _wanted(cand["rect"]) & (cand["rect"] == cand["exact"]).all(1) & (cand["margin"] > 1e-3) & (cand["radii"] > 0)
    pick = []

    def take(mask, k):
        idx = np.flatnonzero(mask & same)
        assert len(idx) >= k, ("not enough candidates", k, len(idx))
        chosen = rng.choice(idx, k, replace=False)
        same[chosen] = False
        return chosen

    w, h = cand["rect"][:, 0], cand["rect"][:, 1]
    pick.append(take((w == 8) & (h == 8), 32))
    big = take(w * h > 64, 16)
    sm_ok = (small["margin"] > 1e-3) & (small["radii"] > 0) & (small["rect"].prod(1) <= 4) & (small["rect"].prod(1) > 0)
    sm = rng.choice(np.flatnonzero(sm_ok), 48, replace=False)
    shapes = np.concatenate([take((w == a) & (h == b), 2) for a, b in RECT_SHAPES])
    fields = ("u", "v", "zv", "sig", "op")
    parts = [{k: cand[k][pick[0]] for k in fields}]
    inter = {k: np.empty(32) for k in fields}
    for k in fields:
        inter[k][0::2] = cand[k][big]
        inter[k][1::2] = small[k][sm[:16]]
    parts.append(inter)
    parts.append({k: cand[k][shapes] for k in fields})
    mixed = {k: np.empty(32) for k in fields}  # faint ones at even slots, small ones at odd
    for k in fields:
        mixed[k][0::2] = faint[k][:16]
        mixed[k][1::2] = small[k][sm[16:32]]
    parts.append(mixed)
    allp = {k: np.concatenate([p[k] for p in parts]) for k in fields}
    n = len(allp["u"])
    return _make("rects", RECT_W, RECT_H, 1000.0, 0.0, allp["u"], allp["v"], allp["zv"], allp["sig"], allp["op"],
                 rng.uniform(0.05, 0.95, (n, 3)), full_masks=np.arange(32), mixed_large=np.arange(32, 64, 2),
                 shapes=np.arange(64, 64 + len(shapes)), faint=np.arange(64 + len(shapes), n, 2))


HIT_COUNTS = [0, 1, 2, 31, 32, 33, 63, 64, 65]
HIT_FRAMES = [(161, 9), (168, 15), (169, 1), (175, 8)]  # W, H = 1, 8, 9, 15 (mod 16)


def tile_hit_counts(W, H, seed=6):
    """Tiles 0..8 of the first tile row hold exactly HIT_COUNTS[k] Gaussians each; 33 more sit in the ragged last tile (10),
    spilling into the empty tile 9.  Each Gaussian of tiles 0..8 covers that tile alone and all four 8x8 blocks of it;
    opacity ~0.06, so no pixel saturates."""
    rng = np.random.default_rng(seed)
    nk = len(HIT_COUNTS)
    tiles = np.repeat(np.r_[np.arange(nk), nk + 1], HIT_COUNTS + [33])
    n = len(tiles)
    last_w = W - TILE * (nk + 1)
    cx = np.where(tiles < nk, tiles * TILE + 7.5, TILE * (nk + 1) + (last_w - 1) / 2)
    u = cx + rng.uniform(-0.4, 0.4, n)
    v = np.full(n, (H - 1) / 2) + rng.uniform(-0.4, 0.4, n)
    return _make(f"hits_{W}x{H}", W, H, 200.0, 0.0, u, v, rng.uniform(2.0, 6.0, n), np.full(n, 1.7), rng.uniform(0.04, 0.08, n),
                 rng.uniform(0.05, 0.95, (n, 3)), tile_of=tiles)


STACK_W = STACK_H = 17  # the centre pixel (8, 8) sits exactly on x = y = 0


def _stack(name, opacities, seed):
    """Gaussians at world (0, 0, 0) -- all on the centre pixel, power 0 there, so alpha = opacity exactly -- with equal
    view depth (blended in index order) and distinct colours."""
    rng = np.random.default_rng(seed)
    n = len(opacities)
    c = _make(name, STACK_W, STACK_H, 20.0, 2.0, np.full(n, 8.0), np.full(n, 8.0), np.full(n, 2.0), rng.uniform(2.5, 4.0, n),
              np.asarray(opacities, F), rng.uniform(0.05, 0.95, (n, 3)))
    c.cloud.xyz[:] = 0
    return c


def alpha_threshold(seed=7):
    """Three Gaussians on the centre pixel with opacity just below, at and just above 1/255 (float32)."""
    ops = [np.nextafter(ALPHA_MIN, F(0)), ALPHA_MIN, np.nextafter(ALPHA_MIN, F(1))]
    c = _stack("alpha_threshold", ops, seed)
    c.info["centre_alphas"] = np.asarray(ops, F)
    return c


SATURATE_AT = [2, 32, 33, 64]


def saturate_at(k, seed=8):
    """k + 8 Gaussians on the centre pixel whose transmittance crosses 1e-4 exactly at hit k (T_{k-1} >= 1e-4 > T_k,
    float32).  Opacity 1.0 for k = 2 (alpha clamped to 0.99; one hit can never take T below 1e-4, so 2 is the first hit
    where a pixel can saturate), otherwise the opacity whose k-th power puts 1e-4 halfway between T_{k-1} and T_k."""
    a = 1.0 if k == 2 else 1.0 - 1e-4 ** (1.0 / (k - 0.5))
    ops = np.full(k + 8, a, F)
    c = _stack(f"saturate_at_{k}", ops, seed + k)
    c.info["centre_alphas"] = ops
    c.info["k"] = k
    return c


def blend_cases():
    return [tile_hit_counts(W, H) for W, H in HIT_FRAMES] + [alpha_threshold()] + [saturate_at(k) for k in SATURATE_AT]
