"""TEST INFRASTRUCTURE ONLY -- numpy restatement of Open3D 0.17.0 ScalableTSDFVolume::ExtractPointCloud and
::ExtractVoxelPointCloud on the dense brick window of extract_mesh_from_bricks (oracle/oracle.py), for the tests of the
CUDA point-cloud extraction (gs2mesh_b200/csrc/gsb_pointcloud.cu).  The product package never imports it.
"""
import numpy as np

# Restated from Open3D 0.17.0 ScalableTSDFVolume (names are Open3D's; vl = voxel_length_, U = volume_unit_length_ =
# 16 vl, index0 = lattice index of the unit, (x,y,z) = voxel inside it).  Every array below carries an explicit dtype, so
# each float32 and float64 operation rounds once, in the order written (numpy never contracts a*b + c).
#
# ExtractPointCloud: for every voxel with w0 != 0 && f0 < 0.98f && f0 >= -0.98f and every axis i, the +1 neighbour on
# axis i (in the +1 unit when the step leaves this one; a missing unit gives w1 = f1 = 0); if w1 != 0 && f1 < 0.98f &&
# f1 >= -0.98f && f0 * f1 < 0 (a float product: two tiny values of opposite sign underflow to -0 and emit nothing):
#   r0 = |f0|, r1 = |f1| (float)
#   p0 = Vector3d(vl/2 + vl x, vl/2 + vl y, vl/2 + vl z) + index0.cast<double>() * U   (per unit: not the
#        vl/2 + vl (16 b + x) of the mesh vertices, which differs in the last bits far from the origin)
#   p1 = p0; p1(i) += vl
#   point = (p0 * r1 + p1 * r0) / (r0 + r1)
#     DOUBT: Eigen promotes r0, r1 to double for the two products, while r0 + r1 is summed in float and then widened.
#   colour = ((c0 * r1 + c1 * r0) / (r0 + r1) / 255.0f).cast<double>(), in float (Open3D casts its voxel colour to float
#     first; ours is float already).
#     DOUBT: that the host compiler does not contract c0 * r1 + c1 * r0 into an FMA (x86-64 without -mfma cannot).
#   normal = GetNormalAt(point): n(j) = GetTSDFAt(point + h e_j) - GetTSDFAt(point - h e_j), h = 0.99 vl, then
#     n.normalized(): Eigen divides by sqrt((x*x + y*y) + z*z) when that is > 0 and returns a zero vector unchanged.
#     DOUBT: the factor 0.99 of the half gap.
#     DOUBT: the summation order of squaredNorm() (Eigen's redux of a Vector3d; the one the mesh normals use, DESIGN.md section 7).
# GetTSDFAt(p), in double: q = p - Vector3d(0.5, 0.5, 0.5) * vl; index0 = floor(q / U) per component
#   (LocateVolumeUnit); a missing unit returns 0.0; g = (q - index0 * U) / vl; idx0 = clamp(floor(g), 0, 15);
#   r = g - idx0; the eight corners idx0 + kMcShift[k] (past 15: the +1 unit(s), 0.0f when missing; weights are not
#   consulted) and
#   (1-r0)((1-r1)((1-r2)f0 + r2 f4) + r1((1-r2)f3 + r2 f7)) + r0((1-r1)((1-r2)f1 + r2 f5) + r1((1-r2)f2 + r2 f6)).
#   A never-observed voxel of an open unit has tsdf 0 (Open3D's default TSDFVoxel).
# ExtractVoxelPointCloud: for every voxel with w != 0 && f < 0.98f && f >= -0.98f: point = p0 of that voxel, colour =
#   c = ((double)f + 1.0) * 0.5 three times.
#     DOUBT: that f + 1.0 is a double sum (a double literal) rather than a float one.
# Order: Open3D's follows its unordered_map.  Ours, and the CUDA path's: surface points by ascending edge key
# (window voxel index * 3 + axis), voxel points by ascending window voxel index, the window being (brick_origin,
# brick_count) as in extract_mesh_from_bricks; bricks outside it count as missing.

def _dense_window(tw, brick_count, color=None):
    nbx, nby, nbz = (int(v) for v in brick_count)
    perm = (0, 3, 1, 4, 2, 5, 6)
    g = np.asarray(tw, np.float32).reshape(nbx, nby, nbz, 16, 16, 16, 2).transpose(perm).reshape(nbx * 16, nby * 16,
                                                                                                  nbz * 16, 2)
    col = None
    if color is not None:
        col = np.asarray(color, np.float32).reshape(nbx, nby, nbz, 16, 16, 16, -1).transpose(perm).reshape(
            nbx * 16, nby * 16, nbz * 16, -1)[..., :3]
    return g[..., 0], g[..., 1], col


def _near_surface(f, w):
    return (w != np.float32(0)) & (f < np.float32(0.98)) & (f >= np.float32(-0.98))


def _unit_points(gv, brick_origin, vl):
    """p0 of window voxels gv [N,3] (int64): (vl/2 + vl*x) + index0*U per component, float64."""
    vl = np.float64(vl)
    half, U = vl * np.float64(0.5), vl * np.float64(16)
    index0 = np.asarray(brick_origin, np.int64) + (gv >> 4)
    return (half + vl * (gv & 15).astype(np.float64)) + index0.astype(np.float64) * U


def _tsdf_at(f, allocated, brick_origin, brick_count, vl, p):
    """GetTSDFAt of the points p [N,3] (float64) on the dense window f; allocated [nbx,nby,nbz] bool."""
    vl = np.float64(vl)
    U = vl * np.float64(16)
    b0 = np.asarray(brick_origin, np.int64)
    nb = np.asarray(brick_count, np.int64)
    q = p - vl * np.float64(0.5)
    index0 = np.floor(q / U).astype(np.int64)
    rel = index0 - b0
    inside = ((rel >= 0) & (rel < nb)).all(1)
    relc = np.clip(rel, 0, nb - 1)
    present = inside & allocated[relc[:, 0], relc[:, 1], relc[:, 2]]
    g = (q - index0.astype(np.float64) * U) / vl
    c = np.clip(np.floor(g), 0, 15).astype(np.int64)
    r = g - c.astype(np.float64)
    fp = np.pad(f, ((0, 1),) * 3)  # the +1 layer past the window: missing units
    base = relc * 16 + c
    shift = ((0, 0, 0), (1, 0, 0), (1, 1, 0), (0, 1, 0), (0, 0, 1), (1, 0, 1), (1, 1, 1), (0, 1, 1))
    fk = [fp[base[:, 0] + sx, base[:, 1] + sy, base[:, 2] + sz].astype(np.float64) for sx, sy, sz in shift]
    one = np.float64(1)
    a0, a1, a2 = one - r[:, 0], one - r[:, 1], one - r[:, 2]
    r0, r1, r2 = r[:, 0], r[:, 1], r[:, 2]
    lo = a1 * (a2 * fk[0] + r2 * fk[4]) + r1 * (a2 * fk[3] + r2 * fk[7])
    hi = a1 * (a2 * fk[1] + r2 * fk[5]) + r1 * (a2 * fk[2] + r2 * fk[6])
    return np.where(present, a0 * lo + r0 * hi, np.float64(0))


def _allocated(tw, brick_count, allocated):
    nb = tuple(int(v) for v in brick_count)
    if allocated is None:  # a brick with any observed voxel; pass the real mask for bricks opened but never observed
        allocated = (np.asarray(tw, np.float32).reshape(-1, 4096, 2)[..., 1] != 0).any(1)
    return np.asarray(allocated, bool).reshape(nb)


def extract_point_cloud_from_bricks(tw, brick_origin, brick_count, voxel_length, color=None, allocated=None,
                                    with_normals=True):
    """CPU restatement of ScalableTSDFVolume::ExtractPointCloud on a dense brick window (tw: [n_bricks,4096,2] as
    returned by OracleTSDFVolume.export_bricks, `allocated` its per-brick flags; colour [n_bricks,4096,>=3] float32).
    Returns dict(keys, points, colors, normals) in ascending key = window voxel index * 3 + axis."""
    f, w, col = _dense_window(tw, brick_count, color)
    ok = _near_surface(f, w)
    X, Y, Z = f.shape
    fp, okp = np.pad(f, ((0, 1),) * 3), np.pad(ok, ((0, 1),) * 3)
    lin = np.arange(X * Y * Z, dtype=np.int64).reshape(X, Y, Z)
    keys = []
    for i in range(3):
        s = tuple(slice(1, None) if k == i else slice(0, n) for k, n in enumerate((X, Y, Z)))
        f1, ok1 = fp[s][:X, :Y, :Z], okp[s][:X, :Y, :Z]
        hit = ok & ok1 & (f * f1 < np.float32(0))  # float32 product
        keys.append(lin[hit] * 3 + i)
    keys = np.sort(np.concatenate(keys))
    axis = keys % 3
    v = keys // 3
    gv = np.stack([v // (Y * Z), (v // Z) % Y, v % Z], 1)
    step = np.eye(3, dtype=np.int64)[axis]
    gn = gv + step
    f0 = f[gv[:, 0], gv[:, 1], gv[:, 2]]
    f1 = fp[gn[:, 0], gn[:, 1], gn[:, 2]]
    r0, r1 = np.abs(f0), np.abs(f1)
    rs = r0 + r1  # float32
    p0 = _unit_points(gv, brick_origin, voxel_length)
    p1 = p0.copy()
    p1[np.arange(len(keys)), axis] += np.float64(voxel_length)
    pts = (p0 * r1.astype(np.float64)[:, None] + p1 * r0.astype(np.float64)[:, None]) / rs.astype(np.float64)[:, None]
    colors = None
    if col is not None:
        cp = np.pad(col, ((0, 1),) * 3 + ((0, 0),))
        c0, c1 = cp[gv[:, 0], gv[:, 1], gv[:, 2]], cp[gn[:, 0], gn[:, 1], gn[:, 2]]
        colors = ((c0 * r1[:, None] + c1 * r0[:, None]) / rs[:, None] / np.float32(255)).astype(np.float64)
    normals = None
    if with_normals:
        alloc = _allocated(tw, brick_count, allocated)
        h = np.float64(0.99) * np.float64(voxel_length)
        n = np.empty_like(pts)
        for j in range(3):
            pp, pm = pts.copy(), pts.copy()
            pm[:, j] -= h
            pp[:, j] += h
            n[:, j] = _tsdf_at(f, alloc, brick_origin, brick_count, voxel_length, pp) - \
                _tsdf_at(f, alloc, brick_origin, brick_count, voxel_length, pm)
        sq = (n[:, 0] * n[:, 0] + n[:, 1] * n[:, 1]) + n[:, 2] * n[:, 2]
        pos = sq > 0
        n[pos] /= np.sqrt(sq[pos])[:, None]
        normals = n
    return dict(keys=keys, points=pts.reshape(-1, 3), colors=colors, normals=normals)


def extract_voxel_point_cloud_from_bricks(tw, brick_origin, brick_count, voxel_length):
    """CPU restatement of ScalableTSDFVolume::ExtractVoxelPointCloud on a dense brick window.  Returns dict(keys, points,
    colors) in ascending key = window voxel index."""
    f, w, _ = _dense_window(tw, brick_count)
    X, Y, Z = f.shape
    gv = np.argwhere(_near_surface(f, w)).astype(np.int64)  # C order: ascending window voxel index
    keys = (gv[:, 0] * Y + gv[:, 1]) * Z + gv[:, 2]
    grey = (f[gv[:, 0], gv[:, 1], gv[:, 2]].astype(np.float64) + np.float64(1)) * np.float64(0.5)
    return dict(keys=keys, points=_unit_points(gv, brick_origin, voxel_length).reshape(-1, 3),
                colors=np.repeat(grey[:, None], 3, 1))
