"""Inputs for the MobileBrick evaluation tests (host only): point clouds for the Poisson-disk elimination, meshes for the
uniform sampler, and a synthetic MobileBrick scan written to a directory the way the benchmark lays it out
(visibility_mask.npy as a pickled dict, mesh/gt_mesh.ply, and a vertex-coloured predicted mesh)."""
from __future__ import annotations

import os

import numpy as np

from oracle import mobilebrick_oracle as mo


# ------------------------------------------------------------------------------------------- elimination clouds
def elimination_clouds(n_random=200):
    """{name: (points [M,3], N, r_max, r_min)}: random clouds plus the tie, boundary, clamping, isolation, gradient and
    size-edge cases the round-based elimination must get right."""
    cases = {}
    for s in range(n_random):
        rng = np.random.default_rng(1000 + s)
        M = int(rng.integers(20, 400))
        kind = s % 5
        if kind == 0:  # uniform in a box
            p = rng.uniform(0, 1, (M, 3))
        elif kind == 1:  # on a plane, quantised: many exact distance ties
            p = np.concatenate([rng.integers(0, 12, (M, 2)) * 0.125, np.zeros((M, 1))], 1)
        elif kind == 2:  # mirror-symmetric pairs about x = 0.5 (equal weights)
            h = rng.uniform(0, 1, (M // 2, 3))
            m = h.copy()
            m[:, 0] = 1.0 - h[:, 0]
            p = np.concatenate([h, m])
        elif kind == 3:  # duplicates at d2 = 0
            base = rng.uniform(0, 1, (max(M // 3, 2), 3))
            p = base[rng.integers(0, len(base), M)]
        else:  # density gradient along x: long chains of decreasing keys, many rounds
            x = rng.uniform(0, 1, M) ** 3
            p = np.stack([x, rng.uniform(0, 0.2, M), rng.uniform(0, 0.2, M)], 1)
        M = len(p)
        N = int(rng.integers(1, M + 1))
        r_max = float(rng.uniform(0.05, 0.4))
        r_min = r_max * 0.5 * (1 - (N / M) ** 1.5)
        cases[f"random_{s:03d}"] = (p, N, r_max, r_min)
    # points at exactly r_max (excluded) next to points just inside it
    g = np.arange(8, dtype=np.float64) * 0.25
    line = np.stack([g, np.zeros(8), np.zeros(8)], 1)
    cases["at_r_max"] = (np.concatenate([line, line + [0.0, 0.25 * (1 - 2 ** -40), 0.0]]), 6, 0.25, 0.05)
    # r_min clamping: every neighbour closer than r_min (equal terms)
    cases["r_min_clamp"] = (np.random.default_rng(7).uniform(0, 0.01, (60, 3)), 20, 0.5, 0.2)
    # isolated points of weight 0 among a clump
    rng = np.random.default_rng(8)
    cases["isolated"] = (np.concatenate([rng.uniform(0, 0.1, (40, 3)), np.arange(10)[:, None] * [1.0, 0, 0] + 5.0]), 25,
                         0.08, 0.02)
    # a long 1-D gradient: the round count grows with the chain length
    x = np.cumsum(np.linspace(0.001, 0.05, 300))
    cases["gradient_chain"] = (np.stack([x, np.zeros(300), np.zeros(300)], 1), 100, 0.2, 0.01)
    p = np.random.default_rng(9).uniform(0, 1, (120, 3))
    cases["n_is_m_minus_1"] = (p, 119, 0.3, 0.01)
    cases["n_is_m"] = (p, 120, 0.3, 0.0)
    return cases


def oracle_elimination(points, N, r_max, r_min, heap=True):
    nbr, d2 = mo.neighbour_lists(points, r_max)
    term = mo.weight_term(d2, r_min, r_max)
    if heap:
        return mo.eliminate_heap(nbr, term, N)[0]
    return mo.eliminate_rounds(nbr, term, N)


# ------------------------------------------------------------------------------------------------------ meshes
def grid_mesh(nx, ny, size=0.2, amp=0.01, seed=0):
    """A heightfield of nx*ny vertices over [0, size]^2, two triangles per cell."""
    rng = np.random.default_rng(seed)
    x, y = np.meshgrid(np.linspace(0, size, nx), np.linspace(0, size, ny), indexing="ij")
    z = amp * np.sin(31.0 * x) * np.cos(23.0 * y) + rng.uniform(0, amp * 0.05, x.shape)
    v = np.stack([x.ravel(), y.ravel(), z.ravel()], 1)
    i = np.arange(nx - 1)[:, None] * ny + np.arange(ny - 1)[None, :]
    i = i.ravel()
    t = np.concatenate([np.stack([i, i + ny, i + 1], 1), np.stack([i + 1, i + ny, i + ny + 1], 1)])
    return v, t.astype(np.int64)


def half_round_mesh():
    """Triangles whose CDF times M lands on x.5 (std::round goes up) and a zero-area triangle (no samples)."""
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [1, 1, 0], [2, 0, 0], [2, 1, 0], [3, 0, 0]], np.float64)
    # areas 0.5, 0.5, 0 (collinear), 0.5, 0.5 -> CDF 0.25, 0.5, 0.5, 0.75, 1; with M = 10: 2.5 -> 3, 5, 5, 7.5 -> 8, 10
    t = np.array([[0, 1, 2], [1, 3, 2], [0, 1, 4], [1, 4, 5], [4, 6, 5]], np.int64)
    return v, t


def rigid(angle_deg, axis, t):
    a = np.deg2rad(angle_deg)
    k = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    K = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    T = np.eye(4)
    T[:3, :3] = np.eye(3) + np.sin(a) * K + (1 - np.cos(a)) * K @ K
    T[:3, 3] = t
    return T


def write_scan(root, nx=60, ny=60, no_triangles=False, colored=True, seed=0):
    """A synthetic MobileBrick scan under root: root/gt/{visibility_mask.npy, mesh/gt_mesh.ply}, root/pred.ply (the GT
    moved by a small rigid motion, with vertex colours and one vertex no triangle uses) and root/exp.  With no_triangles
    only the voxels of a checkerboard of the vertices are visible (use a coarse grid), so the crop keeps no triangle.
    Returns (gt_dir, pred_path, exp_path, info)."""
    from gs2mesh_b200.mesh import TriangleMesh

    gt_dir = os.path.join(root, "gt")
    exp = os.path.join(root, "exp")
    os.makedirs(os.path.join(gt_dir, "mesh"), exist_ok=True)
    os.makedirs(exp, exist_ok=True)
    v, t = grid_mesh(nx, ny, seed=seed)
    TriangleMesh(v, t).write_ply(os.path.join(gt_dir, "mesh", "gt_mesh.ply"))
    from oracle import tnt_oracle as to

    T = rigid(0.4, [0.3, -0.5, 1.0], [0.0015, -0.001, 0.0008])
    pv = to.transform(v, T)
    pv = np.concatenate([pv, pv[-1:] - 0.001])  # one vertex no triangle uses: the crop must keep it
    rng = np.random.default_rng(seed + 1)
    colors = rng.integers(0, 256, (len(pv), 3)) / 255.0 if colored else None
    TriangleMesh(pv, t, colors).write_ply(os.path.join(root, "pred.ply"))
    # visibility: a 32 x 24 x 16 volume over the GT's box, visible in a slab that cuts off one corner of the surface
    res = np.array([32, 24, 16])
    min_pts = v.min(0) - 0.005
    voxel_size = float((v.max(0) - min_pts).max() / 20.0)
    mask = np.zeros(tuple(res), bool)
    if no_triangles:
        i, j = np.divmod(np.arange(len(v)), ny)
        idx = mo.visibility_index(v[(i + j) % 2 == 0], min_pts, res, voxel_size)
        mask[idx[:, 0], idx[:, 1], idx[:, 2]] = True
    else:
        mask[:16, :14, :] = True
        mask[16:, :, :] = True
    np.save(os.path.join(gt_dir, "visibility_mask.npy"),
            {"mask": mask.reshape(-1), "resolutions": res, "voxel_size": voxel_size, "min_pts": min_pts}, allow_pickle=True)
    return gt_dir, os.path.join(root, "pred.ply"), exp, {"T": T, "colors": colors}


def load_scan(gt_dir, pred_path):
    from gs2mesh_b200.io import read_triangle_mesh_ply

    d = np.load(os.path.join(gt_dir, "visibility_mask.npy"), allow_pickle=True).item()
    gv, gt = read_triangle_mesh_ply(os.path.join(gt_dir, "mesh", "gt_mesh.ply"))
    pv, pt, pc = read_triangle_mesh_ply(pred_path, with_colors=True)
    return gv, gt, pv, pt, pc, d
