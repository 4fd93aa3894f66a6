"""MobileBrick evaluation on the GPU, without Open3D: `evaluate_single` of evaluation/MobileBrick/eval_code/evaluate.py.

Restated (file:line under evaluation/MobileBrick/eval_code):
  evaluate.py:34-44   visibility_test: the voxel visibility crop, RemoveVerticesByMask, compute_vertex_normals
  evaluate.py:46-63   evaluate (gs2mesh_b200.evaluate.precision_recall_f1)
  evaluate.py:65-66   sample_surface_points: TriangleMesh.sample_points_poisson_disk(n)
  evaluate.py:72-108  evaluate_single: ICP alignment, crop, sampling, the written cropped mesh, the seven numbers

The Open3D 0.17 operations underneath (GetSurfaceArea, SamplePointsUniformlyImpl, SamplePointsPoissonDisk) are gsb_eval_*
kernels of include/gs2mesh_b200.h (gs2mesh_b200/csrc/gsb_mobilebrick.cu); DESIGN.md section 7e gives their operation
orders and the argument that the round-based elimination keeps the points Open3D's heap loop keeps.  Random draws come
from one std::mt19937 stream per evaluate_single call, generated on the host: seeded, so the numbers are reproducible
(the reference never seeds, so its own are not).  There is no CPU fallback.
"""
from __future__ import annotations

import argparse
import ctypes as C
import os

import numpy as np
import torch

from . import _lib
from ._lib import ptr
from .evaluate import PointGrid, _points, precision_recall_f1
from .mesh import TriangleMesh, remove_vertices_by_mask

ALPHA, BETA, GAMMA = 8.0, 0.5, 1.5  # Yuksel's constants as Open3D sets them
# csv_headers['MobileBrick'] of gs2mesh_utils/eval_utils.py:14 after 'Scan Name': the order evaluate_single returns
CSV_HEADER = ["Chamfer Distance", "Accuracy (2.5mm)", "Recall (2.5mm)", "F1 Score (2.5mm)", "Accuracy (5mm)", "Recall (5mm)",
              "F1 Score (5mm)"]


class Mt19937Stream:
    """std::mt19937(seed) read in turn by every sampling call given it.  uniform(n) returns n doubles of
    std::uniform_real_distribution<double>(0, 1) under libstdc++: generate_canonical<double, 53> over two 32-bit outputs,
    (u0 + u1 * 2^32) / 2^64, and nextafter(1, 0) for a result >= 1.  numpy's legacy MT19937 seeding is init_genrand, the
    seeding of std::mt19937(seed)."""

    def __init__(self, seed=0):
        self.seed = int(seed)
        self._bg = np.random.RandomState(self.seed & 0xFFFFFFFF)._bit_generator
        self.drawn = 0  # 32-bit outputs taken so far

    def outputs(self, n):
        self.drawn += int(n)
        return np.asarray(self._bg.random_raw(int(n)), dtype=np.uint64)

    def uniform(self, n):
        u = self.outputs(2 * int(n)).reshape(-1, 2)
        r = (u[:, 0].astype(np.float64) + u[:, 1].astype(np.float64) * 4294967296.0) / 18446744073709551616.0
        return np.where(r >= 1.0, np.nextafter(1.0, 0.0), r)


def _mesh(vertices, triangles, device=None):
    v = _points(vertices, _lib.device(device, vertices))
    t = torch.as_tensor(triangles).to(v.device).to(torch.int64).reshape(-1, 3).contiguous()
    nv = v.shape[0]
    if t.shape[0] and (int(t.min().item()) < 0 or int(t.max().item()) >= nv):
        raise IndexError(f"triangle vertex indices outside [0, {nv})")
    return v, t


def _areas(v, t):
    a = torch.empty(t.shape[0], dtype=torch.float64, device=v.device)
    with torch.cuda.device(v.device):
        _lib.check(_lib.lib().gsb_eval_triangle_areas(ptr(v), v.shape[0], ptr(t), t.shape[0], ptr(a), _lib.stream(v.device)))
    return a.cpu().numpy()


def _uniform(v, t, n_samples, stream):
    """SamplePointsUniformlyImpl -> (device samples [n,3], surface area)."""
    if t.shape[0] == 0:
        raise ValueError("Input mesh has no triangles.")
    areas = _areas(v, t)
    S = float(np.cumsum(areas)[-1])  # GetSurfaceArea: added in triangle order
    if not S > 0.0:
        raise ValueError(f"Invalid surface area {S}, it must be > 0.")
    x = np.cumsum(areas / S) * float(n_samples)  # the CDF: a[i] = area[i] / S + a[i-1], sequentially
    lo = np.floor(x)
    n = np.minimum(lo + (x - lo >= 0.5), float(n_samples))  # std::round; Open3D would write past the end above M
    bounds = np.concatenate([np.zeros(1, np.int64), np.maximum.accumulate(n.astype(np.int64))])
    dev = v.device
    variates = torch.as_tensor(stream.uniform(2 * n_samples), device=dev)
    out = torch.empty(n_samples, 3, dtype=torch.float64, device=dev)
    b = torch.as_tensor(bounds, device=dev)
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().gsb_eval_sample_uniform(ptr(v), v.shape[0], ptr(t), t.shape[0], ptr(b), ptr(variates),
                                                      n_samples, ptr(out), _lib.stream(dev)))
    return out, S


def sample_points_uniformly(vertices, triangles, number_of_points, stream=None, device=None):
    """TriangleMesh.sample_points_uniformly(number_of_points) (Open3D 0.17, SamplePointsUniformlyImpl) -> device fp64
    [number_of_points, 3].  stream: a Mt19937Stream (Mt19937Stream(0) when None)."""
    if int(number_of_points) <= 0:
        raise ValueError("number_of_points <= 0")
    v, t = _mesh(vertices, triangles, device)
    return _uniform(v, t, int(number_of_points), Mt19937Stream(0) if stream is None else stream)[0]


def poisson_radii(surface_area, number_of_points, n_init):
    ratio = float(number_of_points) / float(n_init)
    r_max = 2 * np.sqrt((surface_area / number_of_points) / (2 * np.sqrt(3.0)))
    r_min = r_max * BETA * (1 - np.power(ratio, GAMMA))
    return float(r_max), float(r_min)


def eliminate(points, number_of_points, r_max, r_min, return_info=False):
    """Weighted sample elimination of `points` (device fp64 [M,3]) down to number_of_points: the indices Open3D's
    SamplePointsPoissonDisk loop keeps, ascending (device int64).  With return_info also a dict of the removal keys,
    each point's round, the round count and the neighbour count."""
    p = _points(points)
    dev = p.device
    M, N = p.shape[0], int(number_of_points)
    info = {"rounds": 0, "neighbours": 0}
    if N >= M or M == 0:
        kept = torch.arange(M, device=dev)
        return (kept, info) if return_info else kept
    L = _lib.lib()
    grid = PointGrid(p, r_max)
    counts = torch.empty(M, dtype=torch.int64, device=dev)
    with torch.cuda.device(dev):
        s = _lib.stream(dev)
        _lib.check(L.gsb_eval_poisson_neighbours(C.byref(grid.desc), r_max, r_min, ptr(counts), None, None, None, s))
        offsets = torch.zeros(M + 1, dtype=torch.int64, device=dev)
        torch.cumsum(counts, 0, out=offsets[1:])
        total = int(offsets[-1].item())
        nbr = torch.empty(max(total, 1), dtype=torch.int32, device=dev)
        terms = torch.empty(max(total, 1), dtype=torch.float64, device=dev)
        _lib.check(L.gsb_eval_poisson_neighbours(C.byref(grid.desc), r_max, r_min, None, ptr(offsets), ptr(nbr), ptr(terms),
                                                 s))
        weight = torch.empty(M, dtype=torch.float64, device=dev)
        round_of = torch.empty(M, dtype=torch.int32, device=dev)
        counters = torch.empty(4, dtype=torch.int32, device=dev)
        host = torch.empty(4, dtype=torch.int32).pin_memory()
        rounds = C.c_int32(0)
        _lib.check(L.gsb_eval_poisson_eliminate(ptr(offsets), ptr(nbr), ptr(terms), M, ptr(weight), ptr(round_of),
                                                ptr(counters), ptr(host), C.byref(rounds), s))
    # the N smallest removal keys (weight, index): a stable sort keeps equal weights in index order
    order = torch.sort(weight, stable=True).indices
    kept = torch.sort(order[:N]).values
    if return_info:
        info = {"rounds": int(rounds.value), "neighbours": total, "keys": weight, "round_of": round_of}
        return kept, info
    return kept


def sample_points_poisson_disk(vertices, triangles, number_of_points, init_factor=5, stream=None, device=None,
                               return_info=False):
    """TriangleMesh.sample_points_poisson_disk(number_of_points, init_factor) of Open3D 0.17 -> device fp64
    [number_of_points, 3]: init_factor * number_of_points uniform samples from `stream` (a Mt19937Stream, Mt19937Stream(0)
    when None), then weighted sample elimination; the kept points in their sampling order."""
    N = int(number_of_points)
    if N <= 0:
        raise ValueError("number_of_points <= 0")
    v, t = _mesh(vertices, triangles, device)
    M = int(init_factor * N)
    pts, S = _uniform(v, t, M, Mt19937Stream(0) if stream is None else stream)
    r_max, r_min = poisson_radii(S, N, M)
    kept, info = eliminate(pts, N, r_max, r_min, return_info=True)
    out = pts[kept]
    if return_info:
        info.update(samples=pts, kept=kept, r_max=r_max, r_min=r_min)
        return out, info
    return out


def visibility_test(vertices, volume, min_pts, resolution, voxel_size, device=None):
    """evaluate.py:34-41's visibility: device bool [N], True where the nearest voxel of `volume` (reshaped to
    `resolution`, read as D, H, W) is > 0 as a float32, False outside the volume.  Raises ValueError for a resolution
    below 2 on any axis, a voxel_size that is not finite and > 0, or a min_pts that is not finite."""
    v = _points(vertices, _lib.device(device, vertices))
    dev = v.device
    res = np.asarray(resolution).astype(np.int64).reshape(3)
    vol = np.asarray(volume).reshape(tuple(res)).astype(np.float32) > 0  # torch.from_numpy(volume).float() > 0
    vol_d = torch.as_tensor(np.ascontiguousarray(vol.astype(np.uint8)), device=dev)
    mins = np.asarray(min_pts).astype(np.float64).reshape(3)
    keep = torch.empty(v.shape[0], dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        rc = _lib.lib().gsb_eval_visibility(ptr(v), v.shape[0], (C.c_double * 3)(*mins.tolist()),
                                            float(np.float64(voxel_size)), (C.c_int32 * 3)(*[int(r) for r in res]),
                                            ptr(vol_d), ptr(keep), _lib.stream(dev))
    _lib.check(rc, invalid_is_value_error=True)
    return keep.bool()


def align_prediction(gt_vertices, pred_vertices):
    """evaluate.py:82-93: point-to-point ICP of the GT vertices onto the predicted ones (threshold 0.02, identity start,
    no scaling, 10 iterations); when its fitness is strictly above 0.99 the prediction moves by the inverse transform.
    Returns (predicted vertices, the ICP result)."""
    from .tnt import registration_icp, transform_points

    pred = _points(pred_vertices)
    reg = registration_icp(_points(gt_vertices, pred.device), pred, 0.02, np.eye(4), with_scaling=False, max_iteration=10)
    if reg.fitness > 0.99:
        pred = transform_points(pred, np.linalg.inv(reg.transformation))
    return pred, reg


def evaluate_single(gt_dir, pred_path, exp_path, scan_name, device="cuda", seed=0, number_of_points=100000):
    """evaluate.py:72-108: the list [chamfer@2.5mm, accuracy@2.5mm, recall@2.5mm, F1@2.5mm, accuracy@5mm, recall@5mm,
    F1@5mm]; writes <exp_path>/<scan_name>_cropped.ply.  One Mt19937Stream(seed) feeds both Poisson-disk samplings, the
    GT's first.  The no-triangle fallback permutes with np.random.RandomState(seed)."""
    from .io import read_triangle_mesh_ply

    dev = torch.device(device)
    if dev.type == "cuda" and dev.index is None:
        dev = torch.device("cuda", torch.cuda.current_device())
    visibility_mask = np.load(os.path.join(gt_dir, "visibility_mask.npy"), allow_pickle=True).item()
    resolution = visibility_mask["resolutions"]
    volume = np.asarray(visibility_mask["mask"]).reshape(resolution)
    voxel_size = visibility_mask["voxel_size"]
    min_pts = visibility_mask["min_pts"]
    gt_v, gt_t = read_triangle_mesh_ply(os.path.join(gt_dir, "mesh", "gt_mesh.ply"))
    stream = Mt19937Stream(seed)
    gt_vd, gt_td = _mesh(gt_v, gt_t, dev)
    gt_points = sample_points_poisson_disk(gt_vd, gt_td, number_of_points, stream=stream)
    pred_v, pred_t, pred_c = read_triangle_mesh_ply(pred_path, with_colors=True)
    pred_vd = _points(pred_v, dev)

    pred_vd, _ = align_prediction(gt_vd, pred_vd)
    keep = visibility_test(pred_vd, volume, min_pts, resolution, voxel_size)
    v, t, c, _ = remove_vertices_by_mask(pred_vd, pred_t, ~keep, pred_c)
    mesh = TriangleMesh(v.cpu().numpy(), t.cpu().numpy(), None if c is None else c.cpu().numpy())
    mesh.compute_vertex_normals(dev)
    if len(mesh.triangles) > 0:
        pred_points = sample_points_poisson_disk(v, t, number_of_points, stream=stream)
    else:
        pred_points = torch.as_tensor(np.random.RandomState(seed).permutation(mesh.vertices)[:number_of_points],
                                      device=dev)
    mesh.write_ply(os.path.join(exp_path, f"{scan_name}_cropped.ply"))

    out_2_5mm = precision_recall_f1(pred_points, gt_points, threshold=0.0025)
    out_5mm = precision_recall_f1(pred_points, gt_points, threshold=0.005)
    return [out_2_5mm["chamfer"], out_2_5mm["accuracy"], out_2_5mm["recall"], out_2_5mm["F1"], out_5mm["accuracy"],
            out_5mm["recall"], out_5mm["F1"]]


def build_parser():
    """evaluate_single's arguments, plus --seed (the random stream of both Poisson-disk samplings)."""
    parser = argparse.ArgumentParser(description="MobileBrick Chamfer / accuracy / recall / F1 of one scan on the GPU")
    parser.add_argument("--gt_dir", type=str, required=True, help="scan directory with visibility_mask.npy and mesh/")
    parser.add_argument("--pred_path", type=str, required=True, help="the predicted mesh (PLY)")
    parser.add_argument("--exp_path", type=str, required=True, help="where <scan_name>_cropped.ply is written")
    parser.add_argument("--scan_name", type=str, required=True)
    parser.add_argument("--device", type=str, default="cuda")
    parser.add_argument("--seed", type=int, default=0)
    return parser


def main(argv=None):
    args = build_parser().parse_args(argv)
    out = evaluate_single(args.gt_dir, args.pred_path, args.exp_path, args.scan_name, args.device, args.seed)
    for name, value in zip(CSV_HEADER, out):
        print(f"{name}: {value}")
    return out


if __name__ == "__main__":
    main()
