"""Tanks and Temples F-score on the GPU, without Open3D: the TnT toolbox's `run_evaluation` (evaluate_tnt.py:45).

Restated (file:line under evaluation/TNT/eval_code/python_toolbox/evaluation):
  run.py:55-148            run_evaluation: alignment, three ICP refinements, histograms, the printed block
  trajectory_io.py:23-35   read_trajectory
  registration.py:42-103   read_mapping, gen_sparse_trajectory, trajectory_alignment (RANSAC on correspondences)
  registration.py:106-199  crop_and_downsample, registration_unif, registration_vol_ds
  evaluation.py:60-205     EvaluateHisto, get_f1_score_histo2
  plot.py:40-109           plot_graph (only when matplotlib is installed)

The Open3D 0.17 operations underneath (PointCloud.Transform, CropInPolygon, VoxelDownSample, RegistrationICP with
TransformationEstimationPointToPoint, EstimateNormals) are gsb_eval_* kernels of include/gs2mesh_b200.h, and
gsb_pcd_voxel_downsample for VoxelDownSample (gs2mesh_b200/csrc/gsb_tnt.cu, gsb_eval.cu, gsb_normals.cu); DESIGN.md section 7d gives their operation orders.  Host work per ICP iteration is the 3x3 SVD and two
reads of 13 moments.  There is no CPU fallback.  The rough RANSAC alignment runs on the host over the camera centres
with a seeded generator: it is the one step that cannot equal Open3D's bits (its random sequence is not reproducible).
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import math
import os
from dataclasses import dataclass, field

import numpy as np
import torch

from . import _lib
from ._lib import ptr
from .evaluate import PointGrid, _points

# The benchmark's published thresholds (toolbox config.py) for the scenes gs2mesh evaluates.
SCENES_TAU = {"Barn": 0.01, "Caterpillar": 0.005, "Ignatius": 0.003, "Truck": 0.005}
MAX_POINT_NUMBER = 4e6
_AXES = {"x": 0, "y": 1, "z": 2}


# ----------------------------------------------------------------------------------------------------------- readers
class CameraPose:
    def __init__(self, meta, mat):
        self.metadata = meta
        self.pose = mat


def read_trajectory(filename):
    """trajectory_io.py:23-35: repeated [metadata line, 4 rows of 4 floats]."""
    traj = []
    with open(filename, "r") as f:
        metastr = f.readline()
        while metastr:
            meta = [int(x) for x in metastr.split()]
            mat = np.zeros((4, 4))
            for i in range(4):
                row = np.array(f.readline().split(), dtype=np.float64)
                if row.shape != (4,):
                    raise ValueError(f"{filename}: a pose row must hold 4 numbers")
                mat[i] = row
            traj.append(CameraPose(meta, mat))
            metastr = f.readline()
    return traj


def read_mapping(filename):
    """registration.py:42-54: [n_sampled_frames, n_total_frames, float array [n_sampled_frames, 2]]."""
    with open(filename, "r") as f:
        n_sampled_frames = int(f.readline())
        n_total_frames = int(f.readline())
        mapping = np.zeros(shape=(n_sampled_frames, 2))
        for i in range(n_sampled_frames):
            mapping[i, :] = [int(x) for x in f.readline().split()]
    return [n_sampled_frames, n_total_frames, mapping]


def gen_sparse_trajectory(mapping, f_trajectory):
    return [f_trajectory[int(m[1] - 1)] for m in mapping]


@dataclass
class SelectionPolygonVolume:
    """open3d.visualization.SelectionPolygonVolume: the prism over `bounding_polygon` between axis_min and axis_max."""
    orthogonal_axis: str
    axis_min: float
    axis_max: float
    bounding_polygon: np.ndarray

    def crop_point_cloud(self, points):
        return crop_point_cloud(points, self)


def read_selection_polygon_volume(filename):
    """o3d.visualization.read_selection_polygon_volume: the crop JSON (orthogonal_axis, axis_min, axis_max,
    bounding_polygon as a list of 3-vectors)."""
    with open(filename) as f:
        d = json.load(f)
    poly = np.asarray(d["bounding_polygon"], dtype=np.float64)
    if poly.ndim != 2 or poly.shape[1] != 3:
        raise ValueError(f"{filename}: bounding_polygon must be a list of 3-vectors")
    return SelectionPolygonVolume(str(d["orthogonal_axis"]), float(d["axis_min"]), float(d["axis_max"]), poly)


# -------------------------------------------------------------------------------------------------- point clouds
def transform_points(points, transformation):
    """PointCloud.transform(T) into a new device tensor."""
    p = _points(points)
    out = torch.empty_like(p)
    T = np.ascontiguousarray(np.asarray(transformation, dtype=np.float64).reshape(4, 4))
    with torch.cuda.device(p.device):
        _lib.check(_lib.lib().gsb_eval_transform_points(ptr(p), p.shape[0], T.ctypes.data_as(C.POINTER(C.c_double)),
                                                        ptr(out), _lib.stream(p.device)))
    return out


def crop_point_cloud(points, volume):
    """SelectionPolygonVolume.crop_point_cloud: the points inside the volume, in input order."""
    p = _points(points)
    axis = _AXES.get(volume.orthogonal_axis.lower()) if isinstance(volume.orthogonal_axis, str) else None
    poly = np.asarray(volume.bounding_polygon, dtype=np.float64).reshape(-1, 3)
    if axis is None:
        raise ValueError(f"crop_point_cloud: orthogonal_axis must be x, y or z, not {volume.orthogonal_axis!r}")
    if len(poly) < 3:
        raise ValueError("crop_point_cloud: the bounding polygon needs at least 3 vertices")
    if not np.isfinite(poly).all():
        raise ValueError("crop_point_cloud: the bounding polygon must be finite")
    dev = p.device
    n = p.shape[0]
    keep = torch.empty(n, dtype=torch.uint8, device=dev)
    counter = torch.empty(1, dtype=torch.int32, device=dev)
    host = torch.empty(1, dtype=torch.int32).pin_memory()
    poly_d = torch.as_tensor(poly, device=dev)
    with torch.cuda.device(dev):
        rc = _lib.lib().gsb_eval_crop_polygon(ptr(p), n, ptr(poly_d), len(poly), axis, float(volume.axis_min),
                                              float(volume.axis_max), ptr(keep), ptr(counter), ptr(host), _lib.stream(dev))
    _lib.check(rc, invalid_is_value_error=True)
    return p[keep.bool()]


def voxel_down_sample(points, voxel_size):
    """PointCloud.voxel_down_sample: the mean of each voxel's points (summed in input order).  Open3D emits the voxels
    in hash-map order; here they come in ascending (x, y, z) voxel order, the same set of points."""
    p = _points(points)
    if not float(voxel_size) > 0.0:
        raise ValueError("voxel_down_sample: voxel_size <= 0")
    if p.shape[0] == 0:
        return p.clone()
    return _voxel_downsample(p, None, None, float(voxel_size))[0]


def _voxel_downsample(xyz, rgb, nrm, voxel_size):
    """gsb_pcd_voxel_downsample of a non-empty cloud: device fp64 [n,3] points, colours or None and normals or None ->
    (points, colours, normals) of the voxels, None where none was given.  The library's refusals are ValueErrors."""
    dev = xyz.device
    n = xyz.shape[0]
    L = _lib.lib()
    dbl3 = C.c_double * 3
    with torch.cuda.device(dev):
        like = lambda t: None if t is None else torch.empty_like(t)
        out, out_c, out_n = like(xyz), like(rgb), like(nrm)
        ws = torch.empty(int(L.gsb_eval_voxel_workspace_bytes(n)), dtype=torch.uint8, device=dev)
        count = torch.empty(1, dtype=torch.int64, device=dev)
        rc = L.gsb_pcd_voxel_downsample(ptr(xyz), ptr(rgb), ptr(nrm), n, dbl3(*xyz.min(dim=0).values.tolist()),
                                        dbl3(*xyz.max(dim=0).values.tolist()), voxel_size, ptr(ws), ws.numel(), ptr(out),
                                        ptr(out_c), ptr(out_n), ptr(count), _lib.stream(dev))
        _lib.check(rc, invalid_is_value_error=True)
        m = int(count.item())
    head = lambda t: None if t is None else t[:m]
    return head(out), head(out_c), head(out_n)


def uniform_down_sample(points, every_k_points):
    """PointCloud.uniform_down_sample: points 0, k, 2k, ..."""
    if int(every_k_points) <= 0:
        raise ValueError("uniform_down_sample: every_k_points must be positive")
    return _points(points)[::int(every_k_points)].contiguous()


def estimate_normals(points, knn=20):
    """PointCloud.estimate_normals(KDTreeSearchParamKNN(knn)) for a cloud without normals (Open3D 0.17, with
    fast_normal_computation): per point, the covariance of its knn nearest points (itself included; the identity for
    fewer than 3), FastEigen3x3's eigenvector of the smallest eigenvalue, (0, 0, 1) where that is zero.  Not oriented.
    fp64 [N,3] on the points' device (gsb_eval_estimate_normals); knn is 1..32."""
    p = _points(points)
    knn = int(knn)
    if not 1 <= knn <= _lib.KNN_MAX_K:
        raise ValueError(f"estimate_normals: knn must be in 1..{_lib.KNN_MAX_K}, not {knn}")
    out = torch.empty_like(p)
    if p.shape[0] == 0:
        return out
    grid = PointGrid(p)
    with torch.cuda.device(p.device):
        _lib.check(_lib.lib().gsb_eval_estimate_normals(C.byref(grid.desc), ptr(p), p.shape[0], knn, ptr(out),
                                                        _lib.stream(p.device)))
    return out


def compute_point_cloud_distance(source, target):
    """PointCloud.compute_point_cloud_distance: exact 1-NN distance of every source point (0 when target is empty)."""
    s = _points(source)
    t = _points(target, s.device)
    if s.shape[0] == 0 or t.shape[0] == 0:
        return torch.zeros(s.shape[0], dtype=torch.float64, device=s.device)
    return PointGrid(t).nearest(s)[0]


# ------------------------------------------------------------------------------------------------------------- ICP
def umeyama(sums, means_count, second, with_scaling=True):
    """Eigen::umeyama from the ICP moments: means = sum * (1/n); sigma = S_dst_src * (1/n); src_var = ((Sxx + Syy) + Szz)
    * (1/n); SVD sigma = U D V^T, S = diag(1, 1, -1 if det U * det V < 0); R = U S V^T; c = 1/src_var * D.S;
    t = mu_dst - (c R) mu_src; returns the 4x4 [[c R, t], [0, 1]].  sums: pass-0 sums (7), second: pass-1 sums (12)."""
    n = means_count
    one_over_n = 1.0 / n
    mu_s = sums[1:4] * one_over_n
    mu_t = sums[4:7] * one_over_n
    sigma = second[:9].reshape(3, 3) * one_over_n
    U, D, Vt = np.linalg.svd(sigma)
    S = np.ones(3)
    if np.linalg.det(U) * np.linalg.det(Vt) < 0:
        S[2] = -1.0
    R = (U * S) @ Vt
    T = np.eye(4)
    if with_scaling:
        src_var = ((second[9] + second[10]) + second[11]) * one_over_n
        c = 1.0 / src_var * ((D[0] * S[0] + D[1] * S[1]) + D[2] * S[2])
        T[:3, 3] = mu_t - (c * R) @ mu_s
        T[:3, :3] = R * c
    else:
        T[:3, 3] = mu_t - R @ mu_s
        T[:3, :3] = R
    return T


@dataclass
class ICPResult:
    transformation: np.ndarray
    fitness: float
    inlier_rmse: float
    iterations: int
    transformations: list = field(default_factory=list)  # the cumulative transformation after each iteration


class _Moments:
    """gsb_eval_icp_moments with its buffers; each call reads back the 13 sums."""

    def __init__(self, dev):
        self.dev = dev
        self.ws = torch.empty(13 * 256, dtype=torch.float64, device=dev)
        self.out = torch.empty(13, dtype=torch.float64, device=dev)

    def __call__(self, src, idx, d2, tgt, pass_, means=None):
        m = None if means is None else (C.c_double * 6)(*[float(x) for x in means])
        with torch.cuda.device(self.dev):
            _lib.check(_lib.lib().gsb_eval_icp_moments(ptr(src), ptr(idx), ptr(d2), src.shape[0], ptr(tgt), pass_, m,
                                                       ptr(self.ws), ptr(self.out), _lib.stream(self.dev)))
        r = self.out.cpu().numpy()
        return r[:12], int(r[12])


def registration_icp(source, target, threshold, init=None, with_scaling=True, relative_fitness=1e-6, relative_rmse=1e-6,
                     max_iteration=30):
    """open3d.pipelines.registration.registration_icp with TransformationEstimationPointToPoint(with_scaling) and
    ICPConvergenceCriteria(relative_fitness, relative_rmse, max_iteration) (Open3D's defaults).  A correspondence is the
    nearest target point with squared distance < threshold^2; fitness = |corr| / |source|, inlier_rmse =
    sqrt(sum d^2 / |corr|).  Each iteration applies the Umeyama update to the current source points, and the loop stops
    once both |d fitness| < relative_fitness and |d rmse| < relative_rmse, or after max_iteration iterations."""
    if not float(threshold) > 0.0:
        raise ValueError("registration_icp: threshold must be positive")
    src = _points(source)
    dev = src.device
    tgt = _points(target, dev)
    init = np.eye(4) if init is None else np.asarray(init, dtype=np.float64).reshape(4, 4)
    T = init.copy()
    pcd = transform_points(src, init) if not np.array_equal(init, np.eye(4)) else src.clone()
    n = pcd.shape[0]
    grid = PointGrid(tgt) if tgt.shape[0] else None
    idx = torch.full((n,), -1, dtype=torch.int64, device=dev)
    d2 = torch.full((n,), math.inf, dtype=torch.float64, device=dev)
    moments = _Moments(dev)

    def result():
        if grid is None:  # an empty target: no correspondences, and no target rows for the moments to read
            return np.zeros(12), 0, 0.0, 0.0
        if n:
            with torch.cuda.device(dev):
                _lib.check(_lib.lib().gsb_eval_icp_correspond(C.byref(grid.desc), ptr(pcd), n, float(threshold), ptr(idx),
                                                              ptr(d2), _lib.stream(dev)))
        sums, cnt = moments(pcd, idx, d2, tgt, 0)
        if cnt == 0:
            return sums, cnt, 0.0, 0.0
        return sums, cnt, cnt / n, math.sqrt(sums[0] / cnt)

    sums, cnt, fitness, rmse = result()
    history = []
    it = 0
    for it in range(1, int(max_iteration) + 1):
        if cnt == 0:
            update = np.eye(4)
        else:
            mu = np.concatenate([sums[1:4], sums[4:7]]) * (1.0 / cnt)
            second, _ = moments(pcd, idx, d2, tgt, 1, mu)
            update = umeyama(sums, cnt, second, with_scaling)
        T = update @ T
        history.append(T.copy())
        pcd = transform_points(pcd, update)
        prev_fitness, prev_rmse = fitness, rmse
        sums, cnt, fitness, rmse = result()
        if abs(prev_fitness - fitness) < relative_fitness and abs(prev_rmse - rmse) < relative_rmse:
            break
    return ICPResult(T, fitness, rmse, it, history)


# ----------------------------------------------------------------------------------------------- rough alignment
def _umeyama_batch(src, dst):
    """Eigen::umeyama with scaling for a batch of point sets src, dst [B, k, 3] (host float64)."""
    one_over_n = 1.0 / src.shape[1]
    mu_s = src.sum(axis=1) * one_over_n
    mu_d = dst.sum(axis=1) * one_over_n
    sd = src - mu_s[:, None]
    dd = dst - mu_d[:, None]
    sigma = np.einsum("bnj,bnk->bjk", dd, sd) * one_over_n
    U, D, Vt = np.linalg.svd(sigma)
    S = np.ones((len(src), 3))
    S[np.linalg.det(U) * np.linalg.det(Vt) < 0, 2] = -1.0
    R = (U * S[:, None, :]) @ Vt
    src_var = (sd * sd).sum(axis=(1, 2)) * one_over_n
    with np.errstate(divide="ignore", invalid="ignore"):
        c = 1.0 / src_var * (D * S).sum(axis=1)
    T = np.tile(np.eye(4), (len(src), 1, 1))
    cR = R * c[:, None, None]
    T[:, :3, :3] = cR
    T[:, :3, 3] = mu_d - np.einsum("bjk,bk->bj", cR, mu_s)
    return T


def _host_transform(points, T):
    v = [((T[r, 0] * points[:, 0] + T[r, 1] * points[:, 1]) + T[r, 2] * points[:, 2]) + T[r, 3] for r in range(4)]
    return np.stack([v[0] / v[3], v[1] / v[3], v[2] / v[3]], axis=1)


def registration_ransac_based_on_correspondence(source, target, max_correspondence_distance, ransac_n=6,
                                                max_iteration=100000, confidence=0.999, seed=0, batch=256):
    """Open3D's RANSAC over the correspondences i <-> i with PointToPoint(with_scaling=True): hypotheses from ransac_n
    correspondences drawn with replacement (np.random.default_rng(seed)), each validated by the fitness (then the lower
    RMSE) of the nearest-neighbour matches within max_correspondence_distance; the run ends after max_iteration
    hypotheses or when Open3D's confidence bound log(1 - confidence) / log(1 - inlier_ratio^ransac_n) is reached.
    Hypotheses are drawn and solved in batches; the best one in hypothesis order wins."""
    src = np.asarray(source, dtype=np.float64).reshape(-1, 3)
    dst = np.asarray(target, dtype=np.float64).reshape(-1, 3)
    n = len(src)
    if len(dst) != n:
        raise ValueError("trajectory_alignment: the two trajectories must have the same number of cameras")
    if n < ransac_n or not max_correspondence_distance > 0.0:
        return np.eye(4)
    rng = np.random.default_rng(seed)
    r2 = max_correspondence_distance * max_correspondence_distance
    best, best_fit, best_rmse = np.eye(4), 0.0, 0.0
    exit_itr = max_iteration
    chunk = max(1, min(batch, (1 << 22) // (n * n)))
    for b0 in range(0, max_iteration, batch):
        if b0 >= exit_itr:
            break
        nb = min(batch, max_iteration - b0)
        pick = rng.integers(0, n, size=(nb, ransac_n))  # RandomInt(0, n - 1) per drawn correspondence
        Ts = _umeyama_batch(src[pick], dst[pick])
        for c0 in range(0, nb, chunk):
            if b0 + c0 >= exit_itr:
                break
            T = Ts[c0:c0 + chunk]
            v = [((T[:, r, 0, None] * src[:, 0] + T[:, r, 1, None] * src[:, 1]) + T[:, r, 2, None] * src[:, 2]) +
                 T[:, r, 3, None] for r in range(4)]
            with np.errstate(divide="ignore", invalid="ignore"):
                moved = np.stack([v[0] / v[3], v[1] / v[3], v[2] / v[3]], axis=2)  # [c, n, 3]
                diff = moved[:, :, None, :] - dst[None, None, :, :]
                nearest = ((diff[..., 0] * diff[..., 0] + diff[..., 1] * diff[..., 1]) + diff[..., 2] * diff[..., 2]).min(2)
                hit = nearest < r2
                cnt = hit.sum(axis=1)
                fit = cnt / n
                rmse = np.sqrt(np.where(hit, nearest, 0.0).sum(axis=1) / np.maximum(cnt, 1))
                pair = moved - dst[None]
                ratio = (((pair[..., 0] * pair[..., 0] + pair[..., 1] * pair[..., 1]) + pair[..., 2] * pair[..., 2]) <
                         r2).mean(axis=1)
            for k in range(len(T)):  # Open3D's IsBetterRANSACThan and exit bound, in hypothesis order
                if b0 + c0 + k >= exit_itr:
                    break
                if cnt[k] and (fit[k] > best_fit or (fit[k] == best_fit and rmse[k] < best_rmse)):
                    best, best_fit, best_rmse = T[k], float(fit[k]), float(rmse[k])
                    if ratio[k] > 0.0:
                        est = 0.0 if ratio[k] >= 1.0 else math.log(1.0 - confidence) / math.log(1.0 - ratio[k] ** ransac_n)
                        exit_itr = min(exit_itr, math.ceil(est))
    return best


def convert_trajectory_to_points(traj):
    return np.array([t.pose[:3, 3] for t in traj], dtype=np.float64).reshape(-1, 3)


def trajectory_alignment(map_file, traj_to_register, gt_traj_col, gt_trans, scene=None, seed=0):
    """registration.py:65-103: RANSAC alignment of the camera centres to the GT trajectory's centres mapped by gt_trans
    (correspondences i <-> i, max distance 0.2, ransac_n 6, 100000 iterations).  The toolbox's noise term
    (randomvar = 0) multiplies every coordinate by exactly 1 and is left out."""
    target = _host_transform(convert_trajectory_to_points(gt_traj_col), np.asarray(gt_trans, dtype=np.float64))
    if len(traj_to_register) > 1600:
        _, _, mapping = read_mapping(map_file)
        traj_to_register = gen_sparse_trajectory(mapping, traj_to_register)
    source = convert_trajectory_to_points(traj_to_register)
    return registration_ransac_based_on_correspondence(source, target, 0.2, 6, 100000, seed=seed)


def crop_and_downsample(points, crop_volume, down_sample_method="voxel", voxel_size=0.01, trans=None):
    """registration.py:106-125."""
    p = transform_points(points, np.eye(4) if trans is None else trans)
    p = crop_point_cloud(p, crop_volume)
    if down_sample_method == "voxel":
        return voxel_down_sample(p, voxel_size)
    if down_sample_method == "uniform":
        n_points = p.shape[0]
        if n_points > MAX_POINT_NUMBER:
            return uniform_down_sample(p, int(round(n_points / float(MAX_POINT_NUMBER))))  # round half to even
    return p


def registration_unif(source, gt_target, init_trans, crop_volume, threshold, max_itr, max_size=4 * MAX_POINT_NUMBER,
                      verbose=True):
    """registration.py:128-157.  ICPConvergenceCriteria(1e-6, max_itr) is positional: it sets relative_rmse = max_itr
    and leaves max_iteration at 30."""
    if verbose:
        print("[Registration] threshold: %f" % threshold)
    s = crop_and_downsample(source, crop_volume, down_sample_method="uniform", trans=init_trans)
    t = crop_and_downsample(gt_target, crop_volume, down_sample_method="uniform")
    reg = registration_icp(s, t, threshold, np.identity(4), True, 1e-6, max_itr)
    reg.transformation = np.matmul(reg.transformation, init_trans)
    return reg


def registration_vol_ds(source, gt_target, init_trans, crop_volume, voxel_size, threshold, max_itr, verbose=True):
    """registration.py:160-199, with the same positional ICPConvergenceCriteria(1e-6, max_itr)."""
    if verbose:
        print("[Registration] voxel_size: %f, threshold: %f" % (voxel_size, threshold))
    s = crop_and_downsample(source, crop_volume, down_sample_method="voxel", voxel_size=voxel_size, trans=init_trans)
    t = crop_and_downsample(gt_target, crop_volume, down_sample_method="voxel", voxel_size=voxel_size)
    reg = registration_icp(s, t, threshold, np.identity(4), True, 1e-6, max_itr)
    reg.transformation = np.matmul(reg.transformation, init_trans)
    return reg


# ------------------------------------------------------------------------------------------------------- metrics
def get_f1_score_histo2(threshold, filename_mvs, plot_stretch, distance1, distance2, verbose=True):
    """evaluation.py:163-205: precision / recall as Python floats, fscore = 2 r p / (r + p) (ZeroDivisionError when both
    are 0), cumulative histograms over np.arange(0, 5 tau, tau / 100); zeros when either list is empty."""
    d1 = np.asarray(distance1, dtype=np.float64)
    d2 = np.asarray(distance2, dtype=np.float64)
    if len(d1) and len(d2):
        recall = float(int(np.count_nonzero(d2 < threshold))) / float(len(d2))
        precision = float(int(np.count_nonzero(d1 < threshold))) / float(len(d1))
        fscore = 2 * recall * precision / (recall + precision)
        bins = np.arange(0, threshold * plot_stretch, threshold / 100)
        hist, edges_source = np.histogram(d1, bins)
        cum_source = np.cumsum(hist).astype(float) / len(d1)
        bins = np.arange(0, threshold * plot_stretch, threshold / 100)
        hist, edges_target = np.histogram(d2, bins)
        cum_target = np.cumsum(hist).astype(float) / len(d2)
    else:
        precision = recall = fscore = 0
        edges_source = cum_source = edges_target = cum_target = np.array([0])
    return [precision, recall, fscore, edges_source, cum_source, edges_target, cum_target]


def _matplotlib():
    try:
        import matplotlib

        matplotlib.use("Agg")
        import matplotlib.pyplot as plt
        return plt
    except ImportError:
        return None


def write_color_distances(path, points, distances, max_distance, normals=None):
    """evaluation.py:48-55: hot_r(min(d, max) / max), written with Open3D's ColorToUint8 rounding, and the normals (x y z
    nx ny nz red green blue) when given.  Needs matplotlib (returns None without it)."""
    plt = _matplotlib()
    if plt is None:
        return None
    from .io import write_point_cloud_ply

    colors = plt.get_cmap("hot_r")(np.minimum(np.asarray(distances), max_distance) / max_distance)[:, :3]
    return write_point_cloud_ply(path, points, colors, normals)


def plot_graph(scene, fscore, dist_threshold, edges_source, cum_source, edges_target, cum_target, plot_stretch,
               mvs_outpath):
    """plot.py:40-107: the precision / recall curves, PR_<scene>_@d_th_0_<tau*1e4>.png and .pdf.  Needs matplotlib."""
    plt = _matplotlib()
    if plt is None:
        return None
    f = plt.figure()
    ax = plt.subplot(111)
    ax.plot(edges_source[1::], cum_source * 100, c="red", label="precision", linewidth=2.0)
    ax.plot(edges_target[1::], cum_target * 100, c="blue", label="recall", linewidth=2.0)
    ax.grid(True)
    plt.title("Precision and Recall: " + scene + ", " + "%02.2f f-score" % (fscore * 100))
    plt.axvline(x=dist_threshold, c="black", ls="dashed", linewidth=2.0)
    plt.ylabel("# of points (%)", fontsize=15)
    plt.xlabel("Meters", fontsize=15)
    plt.axis([0, dist_threshold * plot_stretch, 0, 100])
    box = ax.get_position()
    ax.set_position([box.x0, box.y0, box.width * 0.8, box.height])
    ax.legend(loc="center left", bbox_to_anchor=(1, 0.5))
    stem = mvs_outpath + "/PR_{0}_@d_th_0_{1}".format(scene, "%04d" % (dist_threshold * 10000))
    f.savefig(stem + ".png", format="png", bbox_inches="tight")
    f.savefig(stem + ".pdf", format="pdf", bbox_inches="tight")
    plt.close(f)
    return stem


def evaluate_histo(source, target, trans, crop_volume, voxel_size, threshold, filename_mvs, plot_stretch, scene_name,
                   verbose=True):
    """evaluation.py:60-160 (EvaluateHisto).  Writes <scene>.recall.txt, .precision.txt and .prf_tau_plotstr.txt, and the
    coloured <scene>.precision.ply / .recall.ply with the toolbox's normals (estimate_normals, knn = 20) when matplotlib
    is installed."""
    s = voxel_down_sample(crop_point_cloud(transform_points(source, trans), crop_volume), voxel_size)
    t = voxel_down_sample(crop_point_cloud(_points(target, s.device), crop_volume), voxel_size)
    s_normals = estimate_normals(s, 20).cpu().numpy()
    t_normals = estimate_normals(t, 20).cpu().numpy()
    distance1 = compute_point_cloud_distance(s, t).cpu().numpy()
    distance2 = compute_point_cloud_distance(t, s).cpu().numpy()
    write_color_distances(filename_mvs + "/" + scene_name + ".precision.ply", s.cpu().numpy(), distance1, 3 * threshold,
                          s_normals)
    write_color_distances(filename_mvs + "/" + scene_name + ".recall.ply", t.cpu().numpy(), distance2, 3 * threshold,
                          t_normals)
    r = get_f1_score_histo2(threshold, filename_mvs, plot_stretch, distance1, distance2)
    precision, recall, fscore, _, cum_source, _, cum_target = r
    np.savetxt(filename_mvs + "/" + scene_name + ".recall.txt", cum_target)
    np.savetxt(filename_mvs + "/" + scene_name + ".precision.txt", cum_source)
    np.savetxt(filename_mvs + "/" + scene_name + ".prf_tau_plotstr.txt",
               np.array([precision, recall, fscore, threshold, plot_stretch]))
    return r


def scene_tau(scene, tau=None):
    if tau is not None:
        return float(tau)
    if scene not in SCENES_TAU:
        raise ValueError(f"invalid dataset-dir, not in the scene thresholds {sorted(SCENES_TAU)}: {scene} (pass tau)")
    return SCENES_TAU[scene]


def run_evaluation(dataset_dir, traj_path, ply_path, out_dir, seed=0, tau=None, device=None):
    """run.py:55-148 on the GPU: returns [precision, recall, fscore].  The dataset directory <scene>/ holds <scene>.ply,
    <scene>_trans.txt, <scene>.json, <scene>_COLMAP_SfM.log and (for trajectories over 1600 cameras)
    <scene>_mapping_reference.txt.  seed drives the RANSAC alignment; tau overrides the scene's threshold."""
    from .io import read_point_cloud_ply

    scene = os.path.basename(os.path.normpath(dataset_dir))
    dTau = scene_tau(scene, tau)
    print("")
    print("===========================")
    print("Evaluating %s" % scene)
    print("===========================")
    dev = _lib.device(device)
    colmap_ref_logfile = os.path.join(dataset_dir, scene + "_COLMAP_SfM.log")
    alignment = os.path.join(dataset_dir, scene + "_trans.txt")
    gt_filen = os.path.join(dataset_dir, scene + ".ply")
    cropfile = os.path.join(dataset_dir, scene + ".json")
    map_file = os.path.join(dataset_dir, scene + "_mapping_reference.txt")
    os.makedirs(out_dir, exist_ok=True)

    print(ply_path)
    pcd = _points(read_point_cloud_ply(ply_path), dev)
    print(gt_filen)
    gt_pcd = _points(read_point_cloud_ply(gt_filen), dev)
    gt_trans = np.loadtxt(alignment)
    traj_to_register = read_trajectory(traj_path)
    gt_traj_col = read_trajectory(colmap_ref_logfile)
    trajectory_transform = trajectory_alignment(map_file, traj_to_register, gt_traj_col, gt_trans, scene, seed=seed)

    vol = read_selection_polygon_volume(cropfile)
    r2 = registration_vol_ds(pcd, gt_pcd, trajectory_transform, vol, dTau, dTau * 80, 20)
    r3 = registration_vol_ds(pcd, gt_pcd, r2.transformation, vol, dTau / 2.0, dTau * 20, 20)
    r = registration_unif(pcd, gt_pcd, r3.transformation, vol, 2 * dTau, 20)

    plot_stretch = 5
    precision, recall, fscore, edges_source, cum_source, edges_target, cum_target = evaluate_histo(
        pcd, gt_pcd, r.transformation, vol, dTau / 2.0, dTau, out_dir, plot_stretch, scene)
    eva = [precision, recall, fscore]
    print("==============================")
    print("evaluation result : %s" % scene)
    print("==============================")
    print("distance tau : %.3f" % dTau)
    print("precision : %.4f" % eva[0])
    print("recall : %.4f" % eva[1])
    print("f-score : %.4f" % eva[2])
    print("==============================")
    plot_graph(scene, fscore, dTau, edges_source, cum_source, edges_target, cum_target, plot_stretch, out_dir)
    return eva


def build_parser():
    """run.py:151-183's flags, plus --seed (the RANSAC generator) and --tau (scenes outside the table)."""
    parser = argparse.ArgumentParser(description="Tanks and Temples precision / recall / F-score on the GPU")
    parser.add_argument("--dataset-dir", type=str, required=True,
                        help="path to a dataset/scene directory containing X.json, X.ply, ...")
    parser.add_argument("--traj-path", type=str, required=True, help="path to trajectory file")
    parser.add_argument("--ply-path", type=str, required=True, help="path to reconstruction ply file")
    parser.add_argument("--out-dir", type=str, default="",
                        help="output directory, default: an evaluation directory next to the ply file")
    parser.add_argument("--seed", type=int, default=0, help="seed of the RANSAC trajectory alignment")
    parser.add_argument("--tau", type=float, default=None, help="distance threshold for scenes without a published one")
    return parser


def main(argv=None):
    args = build_parser().parse_args(argv)
    if args.out_dir.strip() == "":
        args.out_dir = os.path.join(os.path.dirname(args.ply_path), "evaluation")
    return run_evaluation(args.dataset_dir, args.traj_path, args.ply_path, args.out_dir, seed=args.seed, tau=args.tau)


if __name__ == "__main__":
    main()
