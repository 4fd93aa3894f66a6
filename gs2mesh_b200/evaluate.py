"""Mesh-quality metrics on the GPU, without Open3D or sklearn.

Restated (file:line in the gs2mesh sources):
  evaluation/DTU/eval_code/eval.py:48-71          surface sampling of a triangle mesh (`data_pcd`)
  evaluation/DTU/eval_code/eval.py:119-120,132-133 nearest-neighbour distances (sklearn kd_tree kneighbors)
  evaluation/DTU/eval_code/eval.py:80-94          greedy radius downsampling of the shuffled samples
  evaluation/DTU/eval_code/eval.py:96-134         ObsMask / bounding-box / ground-plane masking, d2s and s2d means
  evaluation/DTU/eval_code/eval.py:136-166        visualisation clouds, the printed line, results.json
  evaluation/MobileBrick/eval_code/evaluate.py:46-63  Chamfer distance, precision, recall, F1

The hot path is gsb_eval_* of include/gs2mesh_b200.h (gs2mesh_b200/csrc/gsb_eval.cu): fp64 kernels with explicit
roundings, so sample coordinates and distances equal numpy's float64 results bit for bit.  There is no CPU fallback.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import math
import os

import numpy as np
import torch

from . import _lib
from ._lib import ptr


def _stream(dev):
    return C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def _points(x, dev=None):
    t = torch.as_tensor(x)
    if dev is not None:
        t = t.to(dev)
    if t.device.type != "cuda":
        raise ValueError("gs2mesh_b200.evaluate needs CUDA tensors (or arrays with a device given)")
    return t.to(torch.float64).reshape(-1, 3).contiguous()


def sample_mesh_points(vertices, triangles, density=0.2):
    """`data_pcd` of eval.py:48-71: [mesh vertices ; grid samples of every non-degenerate triangle, in triangle order],
    fp64 [N,3] on the vertices' device.  density = eval.py's --downsample_density (`thresh`)."""
    v = _points(vertices)
    dev = v.device
    t = torch.as_tensor(triangles).to(dev).to(torch.int64).reshape(-1, 3).contiguous()
    nv, nt = v.shape[0], t.shape[0]
    if nt and (int(t.min().item()) < 0 or int(t.max().item()) >= nv):
        raise IndexError(f"sample_mesh_points: triangle vertex indices outside [0, {nv})")
    L = _lib.lib()
    with torch.cuda.device(dev):
        s = _stream(dev)
        counts = torch.empty(nt, dtype=torch.int64, device=dev)
        _lib.check(L.gsb_eval_sample_count(ptr(v), nv, ptr(t), nt, float(density), ptr(counts), s))
        ends = torch.cumsum(counts, 0)
        ns = int(ends[-1].item()) if nt else 0  # the one host read: the size of the output
        out = torch.empty(nv + ns, 3, dtype=torch.float64, device=dev)
        out[:nv] = v
        if ns:
            starts = ends - counts
            _lib.check(L.gsb_eval_sample_emit(ptr(v), nv, ptr(t), nt, float(density), ptr(starts), ptr(out[nv:]), s))
    return out


class PointGrid:
    """Reference points bucketed into a uniform grid (gsb_eval_grid_build), reusable for many nearest() queries.

    The cell size comes from the point spacing inside the 1%..99% quantile box of each axis (so a few far floaters do not
    stretch the cells over the whole object), never below min_cell; the grid then covers every point, and the cell grows
    only when that would need more than max_cells cells."""

    def __init__(self, reference, cells_per_point=4.0, min_cell=0.0, max_cells=1 << 26):
        self.points = _points(reference)
        dev = self.points.device
        n = self.points.shape[0]
        if n == 0:
            raise ValueError("PointGrid: no reference points")
        lo = self.points.min(dim=0).values.cpu().numpy()
        hi = self.points.max(dim=0).values.cpu().numpy()
        if not (np.isfinite(lo).all() and np.isfinite(hi).all()):
            raise ValueError("PointGrid: reference points must be finite")
        sub = self.points[:: max(1, n // (1 << 20))]
        srt = sub.sort(dim=0).values
        m = srt.shape[0]
        core = (srt[min(m - 1, int(0.99 * m))] - srt[int(0.01 * m)]).cpu().numpy()
        big = float(core.max())
        cell = (float(np.prod(np.maximum(core, big * 1e-3))) / (cells_per_point * n)) ** (1.0 / 3.0) if big > 0 else 0.0
        cell = max(cell, float(min_cell), float((hi - lo).max()) * 1e-6, 1e-300)
        ext = hi - lo
        while True:
            dims = [int(e // cell) + 1 for e in ext]
            if dims[0] * dims[1] * dims[2] <= max_cells:
                break
            cell *= 1.25
        self.origin, self.cell, self.dims = lo, cell, dims
        cells = dims[0] * dims[1] * dims[2]
        self.cell_start = torch.empty(cells + 1, dtype=torch.int64, device=dev)
        self.ids = torch.empty(n, dtype=torch.int64, device=dev)
        self.desc = _lib.GsbPointGrid((C.c_double * 3)(*[float(x) for x in lo]), cell, (C.c_int32 * 3)(*dims),
                                      ptr(self.points), n, ptr(self.cell_start), ptr(self.ids))
        L = _lib.lib()
        ws = torch.empty(int(L.gsb_eval_grid_workspace_bytes(n, cells)), dtype=torch.uint8, device=dev)
        with torch.cuda.device(dev):
            _lib.check(L.gsb_eval_grid_build(C.byref(self.desc), ptr(ws), ws.numel(), _stream(dev)))

    def nearest(self, queries, max_dist=math.inf):
        q = _points(queries, self.points.device)
        dev = q.device
        n = q.shape[0]
        dist = torch.empty(n, dtype=torch.float64, device=dev)
        idx = torch.empty(n, dtype=torch.int64, device=dev)
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().gsb_eval_nearest(C.byref(self.desc), ptr(q), n, float(max_dist), ptr(dist), ptr(idx),
                                                   _stream(dev)))
        return dist, idx


def nearest(queries, reference, max_dist=math.inf):
    """Exact 1-NN of every query among `reference` -> (dist fp64 [N], idx int64 [N]) on the device.  dist equals sklearn's
    kd_tree kneighbors distance sqrt(((dx*dx)+dy*dy)+dz*dz) bit for bit; among equal squared distances the lowest index
    wins.  Queries with nothing closer than max_dist get (+inf, -1)."""
    return PointGrid(reference).nearest(queries, max_dist)


def precision_recall_f1(pred_points, gt_points, threshold):
    """MobileBrick `evaluate()` (evaluate.py:46-63) with exact GPU nearest neighbours; same keys, the means taken in numpy
    over the same arrays."""
    pred = _points(pred_points)
    gt = _points(gt_points, pred.device)
    d = nearest(pred, gt)[0].cpu().numpy()
    pred_gt_dist = np.mean(d)
    precision = np.sum(d < threshold) / len(d)
    d = nearest(gt, pred)[0].cpu().numpy()
    gt_pred_dist = np.mean(d)
    recall = np.sum(d < threshold) / len(d)
    F1 = 2 * precision * recall / (precision + recall)
    chamfer = pred_gt_dist + gt_pred_dist
    return {"pred_gt": pred_gt_dist, "accuracy": precision, "gt_pred": gt_pred_dist, "recall": recall, "chamfer": chamfer,
            "F1": F1}


def radius_downsample(points, radius, seed=0, order=None):
    """eval.py:80-94: shuffle, then keep a point iff no earlier kept point lies within `radius` (inclusive, on
    ((dx*dx)+dy*dy)+dz*dz <= radius*radius like sklearn's radius_neighbors).  The order is the permutation `order` (int
    [N]) or np.random.default_rng(seed).permutation(N), which indexes like eval.py's default_rng(seed).shuffle.
    Returns (shuffled points, keep mask) as device tensors; shuffled[keep] is eval.py's `data_down`."""
    p = _points(points)
    dev = p.device
    n = p.shape[0]
    if order is None:
        order = np.random.default_rng(seed).permutation(n)
    order = torch.as_tensor(np.asarray(order, dtype=np.int64)).to(dev)
    if order.shape != (n,):
        raise ValueError("radius_downsample: order must be a permutation of the points")
    shuffled = p[order].contiguous()
    keep = torch.zeros(n, dtype=torch.uint8, device=dev)
    if n:
        grid = PointGrid(shuffled, min_cell=float(radius) * 1.001)
        counters = torch.empty(4, dtype=torch.int32, device=dev)
        host = torch.empty(1, dtype=torch.int32).pin_memory()
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().gsb_eval_radius_downsample(C.byref(grid.desc), float(radius), ptr(keep), ptr(counters),
                                                             ptr(host), None, _stream(dev)))
    return shuffled, keep.bool()


def dtu_chamfer(data, stl_points, obs_mask, bb, res, plane, *, mode="mesh", downsample_density=0.2, patch_size=60,
                max_dist=20, seed=0, device=None):
    """eval.py:43-134 on the GPU.  data = (vertices, triangles) for mode "mesh", points for mode "pcd"; stl_points the
    reference scan; obs_mask / bb / res the ObsMask .mat fields, plane its Plane .mat field P.  Returns mean_d2s,
    mean_s2d, overall (numpy float64, bit-identical to eval.py run with np.random.default_rng(seed)) and the per-point
    arrays the visualisation needs."""
    dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
    thresh = downsample_density
    if mode == "mesh":
        vertices, triangles = data
        data_pcd = sample_mesh_points(torch.as_tensor(np.asarray(vertices, np.float64)).to(dev),
                                      torch.as_tensor(np.asarray(triangles, np.int64)).to(dev), thresh)
    elif mode == "pcd":
        data_pcd = _points(np.asarray(data, np.float64), dev)
    else:
        raise ValueError(f"dtu_chamfer: mode must be 'mesh' or 'pcd', not {mode!r}")
    shuffled, keep = radius_downsample(data_pcd, thresh, seed=seed)
    data_down = shuffled[keep]

    # eval.py:99-110: BB in float32, the margins computed in float32 like numpy does, compared in float64
    BB = np.asarray(bb).astype(np.float32)
    patch = patch_size
    lo = torch.as_tensor((BB[:1] - patch).astype(np.float64), device=dev)
    hi = torch.as_tensor((BB[1:] + patch * 2).astype(np.float64), device=dev)
    inbound = ((data_down >= lo) & (data_down < hi)).sum(dim=-1) == 3
    data_in = data_down[inbound]
    res_t = torch.as_tensor(np.asarray(res, dtype=np.float64).reshape(-1)[:1], device=dev)
    bb0 = torch.as_tensor(BB[:1].astype(np.float64), device=dev)
    data_grid = torch.round((data_in - bb0) / res_t).to(torch.int32)  # np.around: round half to even
    obs = torch.as_tensor(np.ascontiguousarray(np.asarray(obs_mask)).astype(np.bool_), device=dev)
    shape = torch.as_tensor(list(obs.shape), dtype=torch.int32, device=dev)
    grid_inbound = ((data_grid >= 0) & (data_grid < shape)).sum(dim=-1) == 3
    g = data_grid[grid_inbound].long()
    in_obs = obs[g[:, 0], g[:, 1], g[:, 2]]
    data_in_obs = data_in[grid_inbound][in_obs]

    stl = _points(np.asarray(stl_points, np.float64), dev)
    dist_d2s = PointGrid(stl).nearest(data_in_obs, max_dist)[0].cpu().numpy()
    mean_d2s = dist_d2s[dist_d2s < max_dist].mean()

    # eval.py:126-130: ((P0*x + P1*y) + P2*z) + P3*1 > 0
    P = np.asarray(plane, dtype=np.float64).reshape(4)
    above = ((stl[:, 0] * P[0] + stl[:, 1] * P[1]) + stl[:, 2] * P[2]) + P[3] > 0
    stl_above = stl[above]
    dist_s2d = PointGrid(data_in).nearest(stl_above, max_dist)[0].cpu().numpy()
    mean_s2d = dist_s2d[dist_s2d < max_dist].mean()
    over_all = (mean_d2s + mean_s2d) / 2

    inb = inbound.nonzero()[:, 0]
    d2s_index = inb[grid_inbound][in_obs].cpu().numpy()
    return {"mean_d2s": mean_d2s, "mean_s2d": mean_s2d, "overall": over_all, "data_down": data_down.cpu().numpy(),
            "stl": stl.cpu().numpy(), "dist_d2s": dist_d2s, "d2s_index": d2s_index, "dist_s2d": dist_s2d,
            "s2d_index": above.nonzero()[:, 0].cpu().numpy()}


def vis_colors(n, index, dist, visualize_threshold=10, max_dist=20):
    """eval.py:138-152: blue everywhere, red-to-white by distance (clipped at visualize_threshold) on the evaluated points,
    green where the distance is >= max_dist (+inf here)."""
    R = np.array([[1, 0, 0]], dtype=np.float64)
    G = np.array([[0, 1, 0]], dtype=np.float64)
    B = np.array([[0, 0, 1]], dtype=np.float64)
    W = np.array([[1, 1, 1]], dtype=np.float64)
    color = np.tile(B, (n, 1))
    alpha = dist.reshape(-1, 1).clip(max=visualize_threshold) / visualize_threshold
    color[index] = R * alpha + W * (1 - alpha)
    color[index[dist >= max_dist]] = G
    return color


def report(result, vis_out_dir):
    """eval.py:157-166: the stdout line run_and_evaluate_dtu.py parses, and results.json."""
    print(result["mean_d2s"], result["mean_s2d"], result["overall"])
    with open(os.path.join(vis_out_dir, "results.json"), "w") as fp:
        json.dump({"mean_d2s": result["mean_d2s"], "mean_s2d": result["mean_s2d"], "overall": result["overall"]}, fp,
                  indent=True)


def build_parser():
    """eval.py:30-40's flags and defaults, plus --seed (eval.py shuffles with an unseeded generator)."""
    parser = argparse.ArgumentParser(description="DTU Chamfer evaluation of a mesh or point cloud on the GPU")
    parser.add_argument("--data", type=str, default="data_in.ply")
    parser.add_argument("--scan", type=int, default=1)
    parser.add_argument("--mode", type=str, default="mesh", choices=["mesh", "pcd"])
    parser.add_argument("--dataset_dir", type=str, default=".")
    parser.add_argument("--vis_out_dir", type=str, default=".")
    parser.add_argument("--downsample_density", type=float, default=0.2)
    parser.add_argument("--patch_size", type=float, default=60)
    parser.add_argument("--max_dist", type=float, default=20)
    parser.add_argument("--visualize_threshold", type=float, default=10)
    parser.add_argument("--seed", type=int, default=0)
    return parser


def main(argv=None):
    from scipy.io import loadmat

    from .io import read_point_cloud_ply, read_triangle_mesh_ply, write_point_cloud_ply

    args = build_parser().parse_args(argv)
    data = read_triangle_mesh_ply(args.data) if args.mode == "mesh" else read_point_cloud_ply(args.data)
    m = loadmat(f"{args.dataset_dir}/ObsMask/ObsMask{args.scan}_10.mat")
    stl = read_point_cloud_ply(f"{args.dataset_dir}/Points/stl/stl{args.scan:03}_total.ply")
    plane = loadmat(f"{args.dataset_dir}/ObsMask/Plane{args.scan}.mat")["P"]
    r = dtu_chamfer(data, stl, m["ObsMask"], m["BB"], m["Res"], plane, mode=args.mode,
                    downsample_density=args.downsample_density, patch_size=args.patch_size, max_dist=args.max_dist,
                    seed=args.seed)
    write_point_cloud_ply(f"{args.vis_out_dir}/vis_{args.scan:03}_d2s.ply", r["data_down"],
                          vis_colors(len(r["data_down"]), r["d2s_index"], r["dist_d2s"], args.visualize_threshold,
                                     args.max_dist))
    write_point_cloud_ply(f"{args.vis_out_dir}/vis_{args.scan:03}_s2d.ply", r["stl"],
                          vis_colors(len(r["stl"]), r["s2d_index"], r["dist_s2d"], args.visualize_threshold,
                                     args.max_dist))
    report(r, args.vis_out_dir)


if __name__ == "__main__":
    main()
