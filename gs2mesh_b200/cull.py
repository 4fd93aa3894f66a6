"""Mesh culling by the DTU object masks on the GPU, without trimesh or scikit-image.

Restated (file:line in the gs2mesh sources):
  evaluation/DTU/eval_code/evaluate_single_scene.py:23-45   cameras.npz, image count, mask files
  evaluation/DTU/eval_code/render_utils.py:31-52           load_K_Rt_from_P (cv2.decomposeProjectionMatrix)
  evaluation/DTU/eval_code/evaluate_single_scene.py:57-99   projection, disk(24)-dilated masks, nearest grid_sample, keep
  evaluation/DTU/eval_code/evaluate_single_scene.py:100-115 compaction, transform to DTU world coordinates, export
  evaluation/DTU/eval_code/evaluate_single_scene.py:118-142 command line, then eval.py on the culled mesh

The hot path is gsb_eval_mask_dilate_disk and gsb_eval_cull_vertices_by_masks of include/gs2mesh_b200.h
(gs2mesh_b200/csrc/gsb_cull.cu): an exact integer disk dilation into bit-packed masks, then one thread per vertex in the
reference's fp32 operation order.  There is no CPU fallback.

Vertex order: the reference loads the mesh with trimesh's default processing, which merges duplicate vertices.  This
module keeps the vertices as they are in the file (meshes from this project have no duplicates), and refuses non-finite
coordinates, which trimesh would drop on load.
"""
from __future__ import annotations

import argparse
import ctypes as C
import glob
import os

import numpy as np
import torch

from . import _lib
from ._lib import ptr

IMAGE_SIZE = (1600, 1200)  # W, H of evaluate_single_scene.py:47: the frame pixel coordinates are normalised to
RADIUS = 24  # disk(24), evaluate_single_scene.py:80


def _device(device, x=None):
    """`device` if given, else the device of a CUDA tensor x, else the current CUDA device."""
    if device is not None:
        return torch.device(device)
    if isinstance(x, torch.Tensor) and x.is_cuda:
        return x.device
    return torch.device("cuda", torch.cuda.current_device())


def _stream(dev):
    return C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def _mask_stack(masks):
    """[V,H,W] uint8 tensor from a tensor / array / list of equally sized [H,W] masks (nonzero = set)."""
    if isinstance(masks, torch.Tensor):
        t = masks
    else:
        masks = [np.asarray(m) for m in masks]
        if len({m.shape for m in masks}) > 1:
            raise ValueError("masks must all have the same size")
        t = torch.from_numpy(np.stack(masks)) if masks else torch.zeros(0, 1, 1, dtype=torch.uint8)
    if t.dim() != 3:
        raise ValueError(f"masks must be [V,H,W], not {tuple(t.shape)}")
    return t if t.dtype == torch.uint8 else (t != 0).to(torch.uint8)


def _dilate_packed(masks, radius):
    """gsb_eval_mask_dilate_disk of a [V,H,W] uint8 device tensor -> int32 [V,H,ceil(W/32)] bit-packed rows."""
    V, H, W = masks.shape
    dev = masks.device
    packed = torch.empty(V, H, (W + 31) // 32, dtype=torch.int32, device=dev)
    work = torch.empty(V * H * W, dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().gsb_eval_mask_dilate_disk(ptr(masks), V, H, W, int(radius), ptr(packed), ptr(work),
                                                        _stream(dev)))
    return packed


def dilate_masks(masks, radius=RADIUS, device=None):
    """Each mask's set (nonzero) pixels dilated by skimage's disk(radius), x*x + y*y <= radius*radius, with pixels
    outside the image unset -> device bool [V,H,W]."""
    m = _mask_stack(masks).to(_device(device, masks)).contiguous()
    V, H, W = m.shape
    packed = _dilate_packed(m, radius)
    bits = torch.arange(32, dtype=torch.int32, device=m.device)
    return ((packed.unsqueeze(-1) >> bits) & 1).reshape(V, H, -1)[..., :W].bool()


def cull_vertices(vertices, matrices, masks, image_size=IMAGE_SIZE, radius=RADIUS, device=None):
    """Keep mask (device bool [N]) of evaluate_single_scene.py:57-99.  vertices: float64 [N,3] in the normalised frame;
    matrices: float32 [V,4,4], intrinsic @ w2c per view (dtu_cameras); masks: at least V equally sized [H,W] masks, view
    i using masks[i].  A vertex is culled iff some view projects it strictly inside the image_size frame onto an unset
    pixel of that view's mask dilated by disk(radius).  Raises ValueError for non-finite vertices, for fewer masks than
    views and for masks of different sizes."""
    v = torch.as_tensor(vertices).to(torch.float64).reshape(-1, 3)
    if not bool(torch.isfinite(v).all()):
        raise ValueError("cull_vertices: vertex coordinates must be finite")
    M = torch.as_tensor(matrices).to(torch.float32).reshape(-1, 4, 4)
    n_views = M.shape[0]
    if len(masks) < n_views:
        raise ValueError(f"cull_vertices: {len(masks)} masks for {n_views} views")
    m = _mask_stack(masks[:n_views])
    dev = _device(device, vertices)
    v, M, m = v.to(dev).contiguous(), M.to(dev).contiguous(), m.to(dev).contiguous()
    W, H = (int(s) for s in image_size)
    n = v.shape[0]
    keep = torch.ones(n, dtype=torch.uint8, device=dev)
    if n and n_views:
        packed = _dilate_packed(m, radius)
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().gsb_eval_cull_vertices_by_masks(ptr(v), n, ptr(M), n_views, W, H, m.shape[2], m.shape[1],
                                                                  ptr(packed), ptr(keep), _stream(dev)))
    return keep.bool()


def cull_mesh(vertices, triangles, matrices, masks, scale_mat, image_size=IMAGE_SIZE, radius=RADIUS, device=None):
    """evaluate_single_scene.py:57-114: the kept vertices in order, moved to DTU world coordinates with
    v * scale_mat[0,0] + scale_mat[:3,3] (float64), and the faces whose three vertices are kept, in order, remapped.
    Returns a TriangleMesh."""
    from .mesh import TriangleMesh

    keep = cull_vertices(vertices, matrices, masks, image_size, radius, device)
    dev = keep.device
    v = torch.as_tensor(vertices).to(dev).to(torch.float64).reshape(-1, 3)
    t = torch.as_tensor(np.asarray(triangles, np.int64)).to(dev).reshape(-1, 3)
    face_keep = keep[t].all(dim=1)
    remap = torch.cumsum(keep.to(torch.int64), 0) - 1
    s = np.asarray(scale_mat, np.float32)
    world = v[keep] * float(s[0, 0]) + torch.as_tensor(s[:3, 3].astype(np.float64), device=dev)
    return TriangleMesh(world.cpu().numpy(), remap[t[face_keep]].cpu().numpy())


def decompose_projection(P):
    """render_utils.load_K_Rt_from_P for a 3x4 P: (intrinsics float64 4x4 = K / K[2,2], pose float32 4x4 = [R^T | c])."""
    import cv2

    K, R, t = cv2.decomposeProjectionMatrix(P)[:3]
    K = K / K[2, 2]
    intrinsics = np.eye(4)
    intrinsics[:3, :3] = K
    pose = np.eye(4, dtype=np.float32)
    pose[:3, :3] = R.transpose()
    pose[:3, 3] = (t[:3] / t[3])[:, 0]
    return intrinsics, pose


def dtu_cameras(instance_dir, device=None):
    """evaluate_single_scene.py:24-38, 64-66 with the same library calls on the same dtypes: the projection matrices
    intrinsic.float() @ inverse(pose) (float32 [V,4,4] on the device, the inverse taken on the CPU) and scale_mat_i
    (float32 numpy) of the first V = len(images/*.png) views."""
    dev = _device(device)
    n_images = len(glob.glob(os.path.join(instance_dir, "images", "*.png")))
    camera_dict = np.load(os.path.join(instance_dir, "cameras.npz"))
    scale_mats = [camera_dict["scale_mat_%d" % i].astype(np.float32) for i in range(n_images)]
    world_mats = [camera_dict["world_mat_%d" % i].astype(np.float32) for i in range(n_images)]
    matrices = []
    for scale_mat, world_mat in zip(scale_mats, world_mats):
        intrinsics, pose = decompose_projection((world_mat @ scale_mat)[:3, :4])
        w2c = torch.inverse(torch.from_numpy(pose).float()).to(dev)
        matrices.append(torch.from_numpy(intrinsics).float().to(dev) @ w2c)
    M = torch.stack(matrices) if matrices else torch.zeros(0, 4, 4, dtype=torch.float32, device=dev)
    return M, scale_mats


def read_masks(instance_dir):
    """Channel 0 of cv2.imread of every mask/*.png in sorted order (evaluate_single_scene.py:40-45, 79)."""
    import cv2

    masks = []
    for p in sorted(glob.glob(os.path.join(instance_dir, "mask", "*.png"))):
        m = cv2.imread(p)
        if m is None:
            raise ValueError(f"{p}: unreadable mask")
        masks.append(m[:, :, 0])
    return masks


def cull_scan(scan, mesh_path, result_mesh_file, Offical_DTU_Dataset):
    """evaluate_single_scene.cull_scan: reads <DTU>/../../scan<scan>/{images,mask,cameras.npz} and the mesh, writes the
    culled mesh in DTU world coordinates to result_mesh_file (binary PLY, float64 vertices)."""
    from .io import read_triangle_mesh_ply

    instance_dir = os.path.abspath(os.path.join(Offical_DTU_Dataset, "..", "..", f"scan{scan}"))
    n_images = len(glob.glob(os.path.join(instance_dir, "images", "*.png")))
    if n_images == 0:
        raise ValueError(f"{instance_dir}/images: no *.png images")
    masks = read_masks(instance_dir)
    if len(masks) < n_images:
        raise ValueError(f"{instance_dir}/mask: {len(masks)} masks for {n_images} images")
    if len({m.shape for m in masks}) > 1:
        raise ValueError(f"{instance_dir}/mask: masks of different sizes")
    vertices, triangles = read_triangle_mesh_ply(mesh_path)
    if not np.isfinite(vertices).all():
        raise ValueError(f"{mesh_path}: non-finite vertex coordinates")
    matrices, scale_mats = dtu_cameras(instance_dir)
    mesh = cull_mesh(vertices, triangles, matrices, masks, scale_mats[0], device=matrices.device)
    mesh.write_ply(result_mesh_file)
    return mesh


def build_parser():
    """evaluate_single_scene.py:120-128's flags and defaults, plus --seed for eval.py's shuffle."""
    parser = argparse.ArgumentParser(description="Cull a mesh by the DTU masks on the GPU, then evaluate it")
    parser.add_argument("--input_mesh", type=str, help="path to the mesh to be evaluated")
    parser.add_argument("--scan_id", type=str, help="scan id of the input mesh")
    parser.add_argument("--output_dir", type=str, default="evaluation_results_single", help="path to the output folder")
    parser.add_argument("--DTU", type=str, default="Offical_DTU_Dataset", help="path to the GT DTU point clouds")
    parser.add_argument("--seed", type=int, default=0)
    return parser


def main(argv=None):
    from . import evaluate

    args = build_parser().parse_args(argv)
    os.makedirs(args.output_dir, exist_ok=True)
    result_mesh_file = os.path.join(args.output_dir, "culled_mesh.ply")
    cull_scan(args.scan_id, args.input_mesh, result_mesh_file, args.DTU)
    evaluate.main(["--data", result_mesh_file, "--scan", str(args.scan_id), "--mode", "mesh", "--dataset_dir", args.DTU,
                   "--vis_out_dir", args.output_dir, "--seed", str(args.seed)])


if __name__ == "__main__":
    main()
