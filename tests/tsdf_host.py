"""Host restatements of the TSDF volume's addressing (gs2mesh_b200/csrc/gsb_common.h) and of its per-voxel projection
(gsb_tsdf.cu integrate_kernel), used by the tests to construct and recognise edge cases."""
import numpy as np

BIAS = 1 << 20  # lattice indices in [-2^20, 2^20)
_M64 = (1 << 64) - 1


def brick_key(b):
    """(bx, by, bz) -> the 64-bit packed key (three 21-bit biased indices), as a Python int."""
    bx, by, bz = (int(v) for v in b)
    return ((bx + BIAS) << 42) | ((by + BIAS) << 21) | (bz + BIAS)


def brick_hash(key, mask):
    """splitmix64 finaliser of the key, masked: the home slot of a brick in a table of mask + 1 slots."""
    k = int(key) & _M64
    k ^= k >> 33
    k = (k * 0xFF51AFD7ED558CCD) & _M64
    k ^= k >> 33
    k = (k * 0xC4CEB9FE1A85EC53) & _M64
    k ^= k >> 33
    return k & 0xFFFFFFFF & int(mask)


def brick_hash_np(keys, mask):
    """Vectorised brick_hash on uint64 arrays (numpy wraps uint64 products mod 2^64)."""
    k = np.asarray(keys, dtype=np.uint64).copy()
    with np.errstate(over="ignore"):
        k ^= k >> np.uint64(33)
        k *= np.uint64(0xFF51AFD7ED558CCD)
        k ^= k >> np.uint64(33)
        k *= np.uint64(0xC4CEB9FE1A85EC53)
        k ^= k >> np.uint64(33)
    return (k & np.uint64(mask)).astype(np.int64)


def linear_probe_positions(homes, slots):
    """Positions linear probing gives keys with these home slots in a table of `slots` entries.  The SET of occupied
    positions does not depend on the insertion order, nor does whether some key wrapped past the last slot."""
    taken = np.zeros(slots, bool)
    pos = []
    for h in homes:
        p = int(h)
        while taken[p]:
            p = (p + 1) % slots
        taken[p] = True
        pos.append(p)
    return np.array(pos, np.int64)


def project_units(units, vl, fx, fy, cx, cy, w2c):
    """integrate_kernel's projection of every voxel of the given bricks, in its fp32 operation order:
    returns (u_f, v_f, pcz), float32 [n, 16, 16, 16] in x*256 + y*16 + z order."""
    f32 = np.float32
    units = np.asarray(units, np.int64).reshape(-1, 3)
    E = np.asarray(w2c, np.float64).reshape(16).astype(f32)
    vlf = f32(vl)
    half = vlf * f32(0.5)
    ul = float(vl) * 16
    loc = (half + vlf * np.arange(16, dtype=f32)).astype(np.float64)  # float(half + vl*i), then + origin in double
    origin = units.astype(np.float64) * ul
    px = (loc[None, :] + origin[:, 0:1]).astype(f32)[:, :, None]
    py = (loc[None, :] + origin[:, 1:2]).astype(f32)[:, None, :]
    pz = (np.float64(half) + origin[:, 2]).astype(f32)[:, None, None]
    out = []
    for r in range(3):
        out.append(((E[4 * r] * px + E[4 * r + 1] * py) + E[4 * r + 2] * pz) + E[4 * r + 3])
    step = [E[2] * vlf, E[6] * vlf, E[10] * vlf]
    cam = np.empty((3, len(units), 16, 16, 16), f32)
    for z in range(16):
        for r in range(3):
            cam[r, :, :, :, z] = out[r]
            out[r] = out[r] + step[r]
    with np.errstate(all="ignore"):
        u = ((cam[0] * f32(fx)) / cam[2] + f32(cx)) + f32(0.5)
        v = ((cam[1] * f32(fy)) / cam[2] + f32(cy)) + f32(0.5)
    return u, v, cam[2]


def sample_units(units, vl, trunc, depth, W, H, fx, fy, cx, cy, w2c, mult):
    """What the frame does to every voxel of the bricks: dict(u, v, pcz, inside, d, sdf, updated), float32 where the
    kernel computes in float32.  `inside`: projects into the image; `updated`: the frame changes the voxel."""
    f32 = np.float32
    u, v, pcz = project_units(units, vl, fx, fy, cx, cy, w2c)
    inside = (pcz > 0) & (u >= f32(0.0001)) & (u < f32(W) - f32(0.0001)) & (v >= f32(0.0001)) & (v < f32(H) - f32(0.0001))
    ui = np.where(inside, u, 0).astype(np.int64)
    vi = np.where(inside, v, 0).astype(np.int64)
    d = np.where(inside, depth.reshape(H, W)[vi, ui], f32(0)).astype(f32)
    m = mult.reshape(H, W)[vi, ui]
    with np.errstate(all="ignore"):
        sdf = ((d - pcz) * m).astype(f32)
        updated = inside & (d > 0) & (sdf > -f32(trunc))
    return dict(u=u, v=v, pcz=pcz, inside=inside, d=d, sdf=sdf, updated=updated)


def mark_boxes(depth, W, H, fx, fy, cx, cy, w2c, trunc, unit_length):
    """mark_bricks_kernel's brick box of every stride-4 sample with depth > 0, in fp64: (sample index s, lo[3], hi[3])."""
    pose = np.linalg.inv(np.asarray(w2c, np.float64).reshape(4, 4))
    nsx = (W + 3) // 4
    ii, jj = np.mgrid[0:H:4, 0:W:4]
    s = (ii // 4) * nsx + jj // 4
    z = depth.reshape(H, W)[ii, jj].astype(np.float64)
    ok = z > 0
    s, ii, jj, z = s[ok], ii[ok], jj[ok], z[ok]
    x = ((jj - cx) * z) / fx
    y = ((ii - cy) * z) / fy
    w = [((pose[r, 0] * x + pose[r, 1] * y) + pose[r, 2] * z) + pose[r, 3] for r in range(3)]
    lo = np.stack([np.floor((c - trunc) / unit_length) for c in w], -1).astype(np.int64)
    hi = np.stack([np.floor((c + trunc) / unit_length) for c in w], -1).astype(np.int64)
    return s, lo, hi
