"""CPU restatement of the DTU mask cull (test infrastructure only; numpy + scipy, no trimesh, no scikit-image).

Written from the reference's behaviour (file:line in the gs2mesh sources):
  evaluation/DTU/eval_code/evaluate_single_scene.py:57-75   fp32 projection M @ [x,y,z,1], pixel / grid coordinates
  evaluation/DTU/eval_code/evaluate_single_scene.py:79-80   channel-0 masks dilated by skimage's disk(24)
  evaluation/DTU/eval_code/evaluate_single_scene.py:92-99   nearest grid_sample (align_corners=True) and keep decision
  evaluation/DTU/eval_code/evaluate_single_scene.py:100-114 order-preserving compaction, float64 world transform
"""
from __future__ import annotations

import numpy as np


def disk(radius):
    """skimage.morphology.disk(radius) with strict_radius=True: x*x + y*y <= radius*radius on a (2r+1)^2 window."""
    L = np.arange(-radius, radius + 1)
    X, Y = np.meshgrid(L, L)
    return (X * X + Y * Y) <= radius * radius


def dilate_masks(masks, radius):
    """Nonzero pixels of each [H,W] mask dilated by disk(radius), pixels outside the image unset -> bool [V,H,W]."""
    from scipy.ndimage import binary_dilation

    masks = np.asarray(masks) != 0
    fp = disk(radius)
    return np.array([binary_dilation(m, structure=fp, border_value=0) for m in masks], np.bool_).reshape(masks.shape)


def fma32(a, b, c):
    """Correctly rounded float32 fma(a, b, c): a*b is exact in float64, TwoSum gives the exact sum s + e, and when s is a
    float32 tie (the only case where rounding s differs from rounding s + e) e decides the direction."""
    a, b, c = (np.asarray(t, np.float32).astype(np.float64) for t in (a, b, c))
    p = a * b
    s = p + c
    bb = s - p
    e = (p - (s - bb)) + (c - bb)
    r = np.asarray(s.astype(np.float32))
    tie = ((s.view(np.uint64) & np.uint64((1 << 29) - 1)) == np.uint64(1 << 28)) & (e != 0)
    if tie.any():
        r[tie] = np.nextafter(s[tie], np.copysign(np.inf, e[tie])).astype(np.float32)
    return r


def camera_points(vertices, matrices):
    """Rows 0..2 of M @ [x, y, z, 1] (float32 [V,3,N]) for the fp32-rounded vertices, in the order cuBLAS computes
    evaluate_single_scene.py:70 on the GPU for large N: fma(M[r][3], 1, fma(M[r][2], z, fma(M[r][1], y, M[r][0] * x)))."""
    v = np.asarray(vertices, np.float64).reshape(-1, 3).astype(np.float32)
    x, y, z = v[:, 0], v[:, 1], v[:, 2]
    one = np.ones_like(x)
    out = []
    for M in np.asarray(matrices, np.float32).reshape(-1, 4, 4):
        cam = []
        for r in range(3):
            acc = np.zeros_like(x)
            for m, t in zip(M[r], (x, y, z, one)):
                acc = fma32(m, t, acc)
            cam.append(acc)
        out.append(np.stack(cam))
    return np.stack(out) if out else np.zeros((0, 3, len(v)), np.float32)


def grid_coords(cam, image_size=(1600, 1200)):
    """evaluate_single_scene.py:71-75 for cam [V,3,N] -> g float32 [V,N,2], one rounding per operation; the scalar
    division by W-1 / H-1 is a multiplication by the fp32 reciprocal, as torch does it for a CUDA tensor."""
    W, H = image_size
    inv_w, inv_h = np.float32(1) / np.float32(W - 1), np.float32(1) / np.float32(H - 1)
    cam = np.asarray(cam, np.float32)
    with np.errstate(all="ignore"):
        den = cam[:, 2] + np.float32(1e-6)
        px, py = cam[:, 0] / den * inv_w, cam[:, 1] / den * inv_h
        return np.stack([(px - np.float32(0.5)) * np.float32(2), (py - np.float32(0.5)) * np.float32(2)], -1)


def project(vertices, matrices, image_size=(1600, 1200)):
    """Grid coordinates g (float32 [V,N,2]) of evaluate_single_scene.py:57-75 as torch computes them on the GPU."""
    return grid_coords(camera_points(vertices, matrices), image_size)


def sample_nearest(mask, g):
    """F.grid_sample(mask, g, mode='nearest', padding_mode='zeros', align_corners=True) of one [h,w] mask at g [N,2]:
    index nearbyint(((g + 1) / 2) * (size - 1)) in float32 (round half to even), 0 outside."""
    h, w = mask.shape
    with np.errstate(all="ignore"):
        fx = ((g[:, 0] + np.float32(1)) / np.float32(2)) * np.float32(w - 1)
        fy = ((g[:, 1] + np.float32(1)) / np.float32(2)) * np.float32(h - 1)
    ok = np.isfinite(fx) & np.isfinite(fy)
    ix = np.where(ok, np.rint(np.where(ok, fx, 0)), -1).astype(np.int64)
    iy = np.where(ok, np.rint(np.where(ok, fy, 0)), -1).astype(np.int64)
    inb = (ix >= 0) & (ix < w) & (iy >= 0) & (iy < h)
    s = np.zeros(len(g), np.float32)
    s[inb] = mask[iy[inb], ix[inb]]
    return s


def keep_vertices(g, dilated):
    """evaluate_single_scene.py:76, 92-99: kept iff every view has sample + (1 - valid) > 0, valid = -1 < g < 1 on both
    axes."""
    keep = np.ones(g.shape[1], np.bool_)
    for gv, m in zip(g, dilated):
        valid = ((gv > -1) & (gv < 1)).all(-1)
        keep &= sample_nearest(m, gv) + (1 - valid.astype(np.float32)) > 0
    return keep


def cull_scan_mesh(vertices, triangles, matrices, masks, scale_mat, image_size=(1600, 1200), radius=24):
    """cull_scan's result for vertices in the normalised frame: (keep, world vertices, remapped faces).  Faces whose three
    vertices are kept survive in order; the kept vertices go through v * scale_mat[0,0] + scale_mat[:3,3] in float64."""
    vertices = np.asarray(vertices, np.float64).reshape(-1, 3)
    triangles = np.asarray(triangles, np.int64).reshape(-1, 3)
    keep = keep_vertices(project(vertices, matrices, image_size), dilate_masks(masks, radius))
    face_keep = keep[triangles].all(axis=1)
    remap = np.cumsum(keep) - 1
    scale_mat = np.asarray(scale_mat, np.float32)
    return keep, vertices[keep] * scale_mat[0, 0] + scale_mat[:3, 3][None], remap[triangles[face_keep]]
