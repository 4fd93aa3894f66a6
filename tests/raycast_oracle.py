"""TEST INFRASTRUCTURE ONLY -- numpy restatement of the TSDF ray cast (gsb_tsdf_raycast, gs2mesh_b200/csrc/gsb_raycast.cu;
DESIGN.md section 7, "Ray casting") on the dense brick window of tests/pointcloud_oracle.py, vectorised over rays with a
loop over march steps.  The product package never imports it.
"""
import numpy as np

from tests.pointcloud_oracle import _allocated, _dense_window, _tsdf_at

# Semantics (ours: Open3D's ScalableTSDFVolume has no ray cast).  vl = voxel length, U = 16 vl, tau = sdf_trunc; every
# array is float64 and every operation rounds once in the order written (numpy never contracts a*b + c).
#
# Ray of pixel (u, v), integers: a = ((u - cx)/fx, (v - cy)/fy, 1); with world->camera [R|t]:
#   o_k = -((R[0,k] t0 + R[1,k] t1) + R[2,k] t2),  d_k = (R[0,k] a_x + R[1,k] a_y) + R[2,k],  p(z) = o + z d,
#   |d| = sqrt((dx dx + dy dy) + dz dz).  z is the camera-frame depth.  Integration's project_voxel assigns a camera point
#   to pixel (int)(x fx / z + cx + 0.5), so pixel u collects x fx / z + cx in [u - 0.5, u + 0.5): the ray through u is
#   the centre of the points that pixel's depth came from.
# Sample at p: q = p - vl/2, fl = floor(q / U) (compared in double before any integer conversion),
#   EMPTY   if fl lies outside [-2^20, 2^20) or the unit fl is not open;
#   INVALID if any corner of GetTSDFAt's cube (g = (q - fl U)/vl, c = clamp(floor(g), 0, 15), corners c + kMcShift, past
#           15 in the +1 units) has weight 0, a corner in an unopened unit counting as weight 0;
#   VALID   otherwise, f = GetTSDFAt(p) (pointcloud_oracle._tsdf_at, the same bits).
# March: lattice box lo = -2^20 U + vl/2, hi = 2^20 U + vl/2; per axis with d_k != 0, t = (lo - o_k)/d_k and
#   (hi - o_k)/d_k, z_in = max of the nearer, z_out = min of the farther; an axis with d_k == 0 whose o_k is not in
#   [lo, hi) misses the box (no hit).  z = max(z_min, z_in); while z <= min(z_max, z_out):
#   EMPTY   z' = the unit box's exit min_k (((fl_k + 1) if d_k > 0 else fl_k) U + vl/2 - o_k)/d_k over d_k != 0, or
#           z + vl/|d| if that is not > z; breaks the chain of valid samples
#   INVALID z' = z + vl/|d|; breaks the chain
#   VALID   previous sample VALID with f_prev > 0 and f <= 0: hit, z* = z_prev + (z - z_prev) (f_prev / (f_prev - f));
#           otherwise z' = z + max(f tau, vl)/|d| if f > 0, z + vl/|d| if not
#   a step with z' not > z ends the ray without a hit.
# Hit: p* = o + z* d; depth = (float)z*; normal = GetNormalAt(p*) normalized (the surface point cloud's formula: central
#   differences of GetTSDFAt at +-0.99 vl, divided by sqrt((x x + y y) + z z) when that is > 0); colour channel k =
#   the GetTSDFAt interpolation of the stored colour over the cube of p* / 255.  Each rounded once to float32.
# No hit: depth, normal and colour 0.

LATTICE = 1 << 20
SHIFT = np.array(((0, 0, 0), (1, 0, 0), (1, 1, 0), (0, 1, 0), (0, 0, 1), (1, 0, 1), (1, 1, 1), (0, 1, 1)), np.int64)


def rays(width, height, fx, fy, cx, cy, w2c):
    """(o [3], d [H*W,3], |d| [H*W]) of every pixel, row-major."""
    E = np.asarray(w2c, np.float64).reshape(4, 4)
    v, u = np.mgrid[0:height, 0:width]
    ax = (u.reshape(-1).astype(np.float64) - np.float64(cx)) / np.float64(fx)
    ay = (v.reshape(-1).astype(np.float64) - np.float64(cy)) / np.float64(fy)
    o = -((E[0, :3] * E[0, 3] + E[1, :3] * E[1, 3]) + E[2, :3] * E[2, 3])
    d = np.stack([(E[0, k] * ax + E[1, k] * ay) + E[2, k] for k in range(3)], 1)
    dn = np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])
    return o, d, dn


def _lattice_interval(o, d, U, half):
    lo = np.float64(-LATTICE) * U + half
    hi = np.float64(LATTICE) * U + half
    z_in = np.full(len(d), -np.inf)
    z_out = np.full(len(d), np.inf)
    ok = np.ones(len(d), bool)
    for k in range(3):
        nz = d[:, k] != 0
        if not (o[k] >= lo and o[k] < hi):
            ok &= nz
        with np.errstate(divide="ignore", invalid="ignore"):
            t1 = (lo - o[k]) / d[:, k]
            t2 = (hi - o[k]) / d[:, k]
        z_in = np.where(nz, np.maximum(z_in, np.minimum(t1, t2)), z_in)
        z_out = np.where(nz, np.minimum(z_out, np.maximum(t1, t2)), z_out)
    return ok, z_in, z_out


class _Grid:
    """The dense window and the per-sample classification."""

    def __init__(self, tw, brick_origin, brick_count, vl, color, allocated):
        self.f, self.w, self.col = _dense_window(tw, brick_count, color)
        self.alloc = _allocated(tw, brick_count, allocated)
        self.wp = np.pad(self.w, ((0, 1),) * 3)  # the +1 layer past the window: missing units, weight 0
        self.b0 = np.asarray(brick_origin, np.int64)
        self.nb = np.asarray(brick_count, np.int64)
        self.vl = np.float64(vl)
        self.U = self.vl * np.float64(16)
        self.half = self.vl * np.float64(0.5)

    def tsdf_at(self, p, field=None):
        return _tsdf_at(self.f if field is None else field, self.alloc, self.b0, self.nb, self.vl, p)

    def classify(self, p):
        """(state 0 EMPTY / 1 INVALID / 2 VALID, fl) of the samples p [N,3]."""
        q = p - self.half
        fl = np.floor(q / self.U)
        inr = ((fl >= -LATTICE) & (fl < LATTICE)).all(1)
        rel = np.where(inr[:, None], fl, 0).astype(np.int64) - self.b0
        inside = inr & ((rel >= 0) & (rel < self.nb)).all(1)
        relc = np.clip(rel, 0, self.nb - 1)
        present = inside & self.alloc[relc[:, 0], relc[:, 1], relc[:, 2]]
        g = (q - fl * self.U) / self.vl
        c = np.clip(np.floor(np.where(present[:, None], g, 0)), 0, 15).astype(np.int64)
        base = relc * 16 + c
        wk = np.stack([self.wp[base[:, 0] + sx, base[:, 1] + sy, base[:, 2] + sz] for sx, sy, sz in SHIFT], 1)
        valid = present & (wk != np.float32(0)).all(1)
        return np.where(present, np.where(valid, 2, 1), 0), fl


def raycast_from_bricks(tw, brick_origin, brick_count, voxel_length, sdf_trunc, width, height, fx, fy, cx, cy, w2c,
                        depth_min, depth_max, color=None, allocated=None, with_normals=True, fixed_step=None):
    """CPU restatement of gsb_tsdf_raycast on a dense brick window (tw [n_bricks,4096,2] row-major over the window,
    `allocated` its per-brick flags, colour [n_bricks,4096,>=3]); bricks outside the window count as not open.
    fixed_step (test use only): advance every sample by fixed_step/|d| instead, a dense reference march.
    Returns dict(depth [H,W] f32, normals [H,W,3] f32 | None, colors [H,W,3] f32 | None, z [H*W] f64 hit (nan: none),
    z_prev / z_next [H*W] f64 the two valid samples the hit lies between)."""
    grid = _Grid(tw, brick_origin, brick_count, voxel_length, color, allocated)
    vl, U, half, tau = grid.vl, grid.U, grid.half, np.float64(sdf_trunc)
    o, d, dn = rays(width, height, fx, fy, cx, cy, w2c)
    n = len(d)
    step_vl = vl / dn if fixed_step is None else np.float64(fixed_step) / dn
    ok, z_in, z_out = _lattice_interval(o, d, U, half)
    ok &= dn > 0
    z = np.maximum(np.float64(depth_min), z_in)
    z_end = np.minimum(np.float64(depth_max), z_out)
    prev_valid = np.zeros(n, bool)
    f_prev = np.zeros(n)
    z_prev = np.zeros(n)
    hit = np.full(n, np.nan)
    hit_prev = np.full(n, np.nan)
    hit_next = np.full(n, np.nan)
    active = ok & (z <= z_end)
    while active.any():
        idx = np.nonzero(active)[0]
        zi, di = z[idx], d[idx]
        p = o + zi[:, None] * di
        state, fl = grid.classify(p)
        z_next = zi + step_vl[idx]
        # EMPTY: the exit from the unit's box
        e = state == 0
        if fixed_step is None and e.any():
            exit_ = np.full(e.sum(), np.inf)
            for k in range(3):
                dk = di[e, k]
                face = np.where(dk > 0, fl[e, k] + np.float64(1), fl[e, k]) * U + half
                with np.errstate(divide="ignore", invalid="ignore"):
                    t = (face - o[k]) / dk
                exit_ = np.where(dk != 0, np.minimum(exit_, t), exit_)
            z_next[e] = np.where(exit_ > zi[e], exit_, z_next[e])
        v = state == 2
        f = np.zeros(len(idx))
        if v.any():
            f[v] = grid.tsdf_at(p[v])
        is_hit = v & prev_valid[idx] & (f_prev[idx] > 0) & (f <= 0)
        if is_hit.any():
            h = idx[is_hit]
            fp, zp = f_prev[h], z_prev[h]
            hit[h] = zp + (zi[is_hit] - zp) * (fp / (fp - f[is_hit]))
            hit_prev[h] = zp
            hit_next[h] = zi[is_hit]
        go = v & ~is_hit & (f > 0)
        if fixed_step is None:
            z_next[go] = zi[go] + np.maximum(f[go] * tau, vl) / dn[idx[go]]
        prev_valid[idx] = v
        f_prev[idx] = np.where(v, f, f_prev[idx])
        z_prev[idx] = np.where(v, zi, z_prev[idx])
        stop = is_hit | ~(z_next > zi)
        z[idx] = z_next
        active[idx] = ~stop & (z_next <= z_end[idx])
    found = ~np.isnan(hit)
    depth = np.where(found, hit, 0).astype(np.float32)
    pstar = o + np.where(found, hit, 0)[:, None] * d
    normals = colors = None
    if with_normals:
        nrm = np.zeros((n, 3))
        if found.any():
            ps = pstar[found]
            h = np.float64(0.99) * vl
            m = np.empty_like(ps)
            for j in range(3):
                pp, pm = ps.copy(), ps.copy()
                pm[:, j] -= h
                pp[:, j] += h
                m[:, j] = grid.tsdf_at(pp) - grid.tsdf_at(pm)
            sq = (m[:, 0] * m[:, 0] + m[:, 1] * m[:, 1]) + m[:, 2] * m[:, 2]
            pos = sq > 0
            m[pos] /= np.sqrt(sq[pos])[:, None]
            nrm[found] = m
        normals = nrm.astype(np.float32).reshape(height, width, 3)
    if color is not None:
        col = np.zeros((n, 3))
        if found.any():
            for k in range(3):
                col[found, k] = grid.tsdf_at(pstar[found], grid.col[..., k]) / np.float64(255)
        colors = col.astype(np.float32).reshape(height, width, 3)
    return dict(depth=depth.reshape(height, width), normals=normals, colors=colors, z=hit, z_prev=hit_prev, z_next=hit_next)


def window_of(units):
    """(brick_origin, brick_count) of the bounding box of `units` plus the +1 brick each cube may reach."""
    idx = np.array(list(units), np.int64)
    lo, hi = idx.min(0), idx.max(0)
    return tuple(int(v) for v in lo), tuple(int(v) for v in hi - lo + 2)


def dense_units(units, b0, nb):
    """(tsdf_weight, colour, allocated) of the window [b0, b0 + nb) from {(bx,by,bz): (tw [4096,2], colour | None)}."""
    total = int(np.prod(nb))
    tw = np.zeros((total, 4096, 2), np.float32)
    col = np.zeros((total, 4096, 3), np.float32)
    alloc = np.zeros(total, bool)
    for (bx, by, bz), (t, c) in units.items():
        r = (bx - b0[0], by - b0[1], bz - b0[2])
        if all(0 <= r[k] < nb[k] for k in range(3)):
            i = (r[0] * nb[1] + r[1]) * nb[2] + r[2]
            tw[i], alloc[i] = t, True
            if c is not None:
                col[i] = np.asarray(c)[:, :3]
    return tw, col, alloc


def raycast_units(units, vl, tau, width, height, fx, fy, cx, cy, w2c, depth_min, depth_max, with_color=True,
                  window=None, **kw):
    """raycast_from_bricks on the window of `units` (default: their bounding box + 1)."""
    b0, nb = window_of(units) if window is None else window
    tw, col, alloc = dense_units(units, b0, nb)
    return raycast_from_bricks(tw, b0, nb, vl, tau, width, height, fx, fy, cx, cy, w2c, depth_min, depth_max,
                               color=col if with_color else None, allocated=alloc, **kw)


def voxel_centres(b, vl):
    """[16,16,16,3] centres vl/2 + vl x + b U of the voxels of brick b, indexed [x,y,z]."""
    x = np.arange(16, dtype=np.float64)
    g = np.stack(np.meshgrid(x, x, x, indexing="ij"), -1)
    return (np.float64(vl) * 0.5 + np.float64(vl) * g) + np.asarray(b, np.float64) * (np.float64(vl) * 16)


def analytic_units(sdf, bricks, vl, tau, weight=None, seed=0):
    """Bricks holding the truncated SDF clip(sdf(p) / tau, -1, 1) at the voxel centres, weight 1 (or weight(p)), random
    colours: {(bx,by,bz): (tw [4096,2], colour [4096,3])}."""
    rng = np.random.default_rng(seed)
    units = {}
    for b in bricks:
        p = voxel_centres(b, vl)
        t = np.clip(sdf(p) / tau, -1, 1).astype(np.float32).reshape(4096)
        w = np.ones(4096, np.float32) if weight is None else np.asarray(weight(p), np.float32).reshape(4096)
        units[tuple(int(v) for v in b)] = (np.stack([t, w], -1), rng.uniform(0, 255, (4096, 3)).astype(np.float32))
    return units


def look_at(pos, target, up=(0.0, 0.0, 1.0)):
    """world->camera 4x4 (OpenCV axes: x right, y down, z forward) of a camera at `pos` looking at `target`."""
    pos = np.asarray(pos, float)
    f = np.asarray(target, float) - pos
    f /= np.linalg.norm(f)
    r = np.cross(f, up)
    if np.linalg.norm(r) < 1e-9:
        r = np.cross(f, (0.0, 1.0, 0.0))
    r /= np.linalg.norm(r)
    c2w = np.eye(4)
    c2w[:3, :3] = np.stack([r, np.cross(f, r), f], axis=1)
    c2w[:3, 3] = pos
    return np.linalg.inv(c2w)
