"""ctypes binding of libgs2mesh_b200.so (the C ABI declared in include/gs2mesh_b200.h).

There is no CPU fallback: if the shared library is missing this module raises at first
use, and every compute call needs a CUDA device.
"""
from __future__ import annotations

import ctypes as C
import os

_PKG = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_PKG, "libgs2mesh_b200.so")

GSB_OK, GSB_ERR_INVALID, GSB_ERR_WORKSPACE, GSB_ERR_CUDA, GSB_ERR_ALIGNMENT = range(5)
GSB_PCD_SURFACE, GSB_PCD_VOXELS = 0, 1  # gsb_pcd_* mode
GSB_SIMPLIFY_AVERAGE, GSB_SIMPLIFY_QUADRIC = 0, 1  # gsb_mesh_simplify contraction
GSB_FILTER_SIMPLE, GSB_FILTER_LAPLACIAN, GSB_FILTER_TAUBIN, GSB_FILTER_SHARPEN = range(4)  # gsb_mesh_filter kind

RASTER_EXACT_TILE_CULL = 1
RASTER_NO_TMA = 2
RASTER_DEBUG_SYNC = 4
RASTER_CUB_SORT = 8
RASTER_ASYNC = 16
RASTER_FAST_EXP = 32
RASTER_PAIR_SHARED_DEPTH = 64

BRICK = 16
BRICK_VOXELS = 4096
KNN_MAX_K = 32  # GSB_KNN_MAX_K

_vp = C.c_void_p


class GsbRasterArgs(C.Structure):
    _fields_ = [
        ("P", C.c_int32), ("sh_degree", C.c_int32), ("sh_coeffs", C.c_int32), ("width", C.c_int32), ("height", C.c_int32),
        ("background", _vp), ("means3D", _vp), ("shs", _vp), ("colors_precomp", _vp), ("opacities", _vp), ("scales", _vp),
        ("rotations", _vp), ("cov3D_precomp", _vp), ("scale_modifier", C.c_float), ("viewmatrix", _vp), ("projmatrix", _vp),
        ("cam_pos", _vp), ("tan_fovx", C.c_float), ("tan_fovy", C.c_float), ("prefiltered", C.c_int32), ("flags", C.c_uint32),
        ("out_color", _vp), ("out_depth", _vp), ("out_final_T", _vp), ("radii", _vp), ("num_rendered", _vp),
        ("workspace", _vp), ("workspace_bytes", C.c_size_t), ("max_instances", C.c_int64),
    ]


class GsbVolumeDesc(C.Structure):
    _fields_ = [
        ("voxel_length", C.c_double), ("sdf_trunc", C.c_double), ("pool_bricks", C.c_uint32), ("hash_slots", C.c_uint32),
        ("tsdf_weight", _vp), ("color", _vp), ("brick_index", _vp), ("hash_keys", _vp), ("hash_vals", _vp), ("hash_stamp", _vp),
        ("brick_list", _vp), ("counters", _vp),
    ]


class GsbPointGrid(C.Structure):
    _fields_ = [
        ("origin", C.c_double * 3), ("cell", C.c_double), ("dims", C.c_int32 * 3), ("points", _vp), ("n_points", C.c_int64),
        ("cell_start", _vp), ("ids", _vp),
    ]


# name -> (restype, argtypes); every symbol include/gs2mesh_b200.h declares
SIGNATURES = {
    "gsb_last_error": (C.c_char_p, []),
    "gsb_version": (C.c_int, []),
    "gsb_kernel_launch_count": (C.c_uint64, []),
    "gsb_profile_num_stages": (C.c_int, []),
    "gsb_profile_stage_name": (C.c_char_p, [C.c_int]),
    "gsb_profile_enable": (C.c_int, [C.c_int]),
    "gsb_profile_collect": (C.c_int, [C.POINTER(C.c_double), C.POINTER(C.c_uint64), C.c_int]),
    "gsb_raster_workspace_bytes": (C.c_size_t, [C.c_int32, C.c_int32, C.c_int32, C.c_int64]),
    "gsb_raster_forward": (C.c_int, [C.POINTER(GsbRasterArgs), _vp]),
    "gsb_raster_forward_pair": (C.c_int, [C.POINTER(GsbRasterArgs), C.POINTER(GsbRasterArgs), _vp, _vp]),
    "gsb_raster_mark_visible": (C.c_int, [C.c_int32, _vp, _vp, _vp, _vp, _vp]),
    "gsb_image_to_u8": (C.c_int, [_vp, C.c_int32, C.c_int32, _vp, _vp]),
    "gsb_tsdf_create": (_vp, [C.POINTER(GsbVolumeDesc)]),
    "gsb_tsdf_destroy": (None, [_vp]),
    "gsb_tsdf_prepare_depth": (C.c_int, [_vp, _vp, _vp, C.c_int32, C.c_int32, C.c_float, C.c_float, C.c_double, C.c_double, _vp, _vp]),
    "gsb_mask_morphology": (C.c_int, [_vp, C.c_int32, C.c_int32, C.c_int32, C.c_int32, _vp, _vp]),
    "gsb_tsdf_integrate": (C.c_int, [_vp, _vp, _vp, C.c_int32, C.c_int32, C.c_double, C.c_double, C.c_double, C.c_double,
                                     C.POINTER(C.c_double), _vp]),
    "gsb_tsdf_touch": (C.c_int, [_vp, _vp, C.c_int32, C.c_int32, C.c_double, C.c_double, C.c_double, C.c_double, C.POINTER(C.c_double), _vp]),
    "gsb_tsdf_to_sums": (C.c_int, [_vp, _vp]),
    "gsb_tsdf_from_sums": (C.c_int, [_vp, _vp]),
    "gsb_tsdf_find_bricks": (C.c_int, [_vp, _vp, C.c_uint32, C.c_int, _vp, _vp, _vp]),
    "gsb_tsdf_export_dense": (C.c_int, [_vp, C.POINTER(C.c_int32), C.POINTER(C.c_int32), _vp, _vp, _vp]),
    "gsb_tsdf_last_stats": (C.c_int, [_vp, _vp, _vp]),
    "gsb_tsdf_reduce_scratch_bytes": (C.c_size_t, [_vp, C.c_int, C.c_uint32]),
    "gsb_tsdf_reduce": (C.c_int, [_vp, _vp, C.c_int, C.c_int, C.c_int, _vp, C.c_size_t, C.POINTER(C.c_size_t), _vp]),
    "gsb_comm_unique_id": (C.c_int, [_vp]),
    "gsb_comm_create": (_vp, [_vp, C.c_int, C.c_int]),
    "gsb_comm_destroy": (None, [_vp]),
    "gsb_mesh_count": (C.c_int, [_vp, C.POINTER(C.c_int32), _vp, C.c_uint32, _vp, _vp]),
    "gsb_mesh_emit": (C.c_int, [_vp, C.POINTER(C.c_int32), _vp, C.c_uint32, _vp, _vp, _vp]),
    "gsb_mesh_vertices": (C.c_int, [_vp, C.POINTER(C.c_int32), _vp, C.c_int64, _vp, _vp, _vp]),
    "gsb_mesh_vertex_normals": (C.c_int, [_vp, C.c_int64, _vp, C.c_int64, _vp, _vp, _vp, _vp]),
    "gsb_mesh_cluster_workspace_bytes": (C.c_size_t, [C.c_int64, C.c_int64]),
    "gsb_mesh_clusters": (C.c_int, [_vp, C.c_int64, C.c_int64, _vp, _vp, C.c_size_t, _vp, _vp, _vp, _vp, _vp]),
    "gsb_mesh_remove_small_clusters": (C.c_int, [_vp, C.c_int64, C.c_int64, _vp, _vp, C.c_double, _vp, C.c_size_t, _vp, _vp,
                                                 _vp, _vp]),
    "gsb_mesh_simplify_workspace_bytes": (C.c_size_t, [C.c_int64, C.c_int64]),
    "gsb_mesh_simplify": (C.c_int, [_vp, _vp, _vp, C.c_int64, _vp, C.c_int64, C.POINTER(C.c_double), C.POINTER(C.c_double),
                                    C.c_double, C.c_int, _vp, C.c_size_t, _vp, _vp, _vp, _vp, _vp, _vp]),
    "gsb_mesh_filter_workspace_bytes": (C.c_size_t, [C.c_int64, C.c_int, C.c_int]),
    "gsb_mesh_filter": (C.c_int, [C.c_int, _vp, _vp, _vp, C.c_int64, _vp, _vp, C.c_int32, C.c_double, C.c_double, C.c_int,
                                  _vp, C.c_size_t, _vp, _vp, _vp, _vp]),
    "gsb_mesh_edge_topology_workspace_bytes": (C.c_size_t, [C.c_int64, C.c_int64]),
    "gsb_mesh_edge_topology": (C.c_int, [_vp, C.c_int64, C.c_int64, C.c_int, _vp, C.c_size_t, _vp, _vp, _vp]),
    "gsb_mesh_vertex_topology_workspace_bytes": (C.c_size_t, [C.c_int64, C.c_int64]),
    "gsb_mesh_non_manifold_vertices": (C.c_int, [_vp, C.c_int64, C.c_int64, _vp, C.c_size_t, _vp, _vp, _vp]),
    "gsb_mesh_self_intersections_workspace_bytes": (C.c_size_t, [C.c_int64, C.c_int64, C.c_int64]),
    "gsb_mesh_self_intersections": (C.c_int, [_vp, C.c_int64, _vp, C.c_int64, C.POINTER(C.c_double), C.POINTER(C.c_double),
                                              _vp, C.c_size_t, _vp, C.c_int64, _vp, _vp]),
    "gsb_mesh_area_volume_workspace_bytes": (C.c_size_t, [C.c_int64, C.c_int64]),
    "gsb_mesh_area_volume": (C.c_int, [_vp, C.c_int64, _vp, C.c_int64, _vp, C.c_size_t, _vp, _vp]),
    "gsb_pcd_count":(C.c_int, [_vp, C.POINTER(C.c_int32), _vp, C.c_uint32, C.c_int, _vp, _vp]),
    "gsb_pcd_emit": (C.c_int, [_vp, C.POINTER(C.c_int32), _vp, C.c_uint32, C.c_int, _vp, _vp, _vp]),
    "gsb_pcd_points": (C.c_int, [_vp, C.POINTER(C.c_int32), _vp, C.c_int64, C.c_int, _vp, _vp, _vp, _vp]),
    "gsb_tsdf_raycast": (C.c_int, [_vp, C.c_int32, C.c_int32, C.c_double, C.c_double, C.c_double, C.c_double,
                                   C.POINTER(C.c_double), C.c_double, C.c_double, _vp, _vp, _vp, _vp]),
    "gsb_eval_sample_count": (C.c_int, [_vp, C.c_int64, _vp, C.c_int64, C.c_double, _vp, _vp]),
    "gsb_eval_sample_emit": (C.c_int, [_vp, C.c_int64, _vp, C.c_int64, C.c_double, _vp, _vp, _vp]),
    "gsb_eval_grid_workspace_bytes": (C.c_size_t, [C.c_int64, C.c_int64]),
    "gsb_eval_grid_build": (C.c_int, [C.POINTER(GsbPointGrid), _vp, C.c_size_t, _vp]),
    "gsb_eval_nearest": (C.c_int, [C.POINTER(GsbPointGrid), _vp, C.c_int64, C.c_double, _vp, _vp, _vp]),
    "gsb_eval_radius_downsample": (C.c_int, [C.POINTER(GsbPointGrid), C.c_double, _vp, _vp, _vp, C.POINTER(C.c_int32), _vp]),
    "gsb_eval_knn": (C.c_int, [C.POINTER(GsbPointGrid), _vp, C.c_int64, C.c_int32, _vp, _vp, _vp]),
    "gsb_eval_estimate_normals": (C.c_int, [C.POINTER(GsbPointGrid), _vp, C.c_int64, C.c_int32, _vp, _vp]),
    "gsb_pcd_statistical_workspace_bytes": (C.c_size_t, [C.c_int64]),
    "gsb_pcd_statistical_outliers": (C.c_int, [C.POINTER(GsbPointGrid), C.c_int32, C.c_double, _vp, C.c_size_t, _vp, _vp, _vp,
                                               _vp]),
    "gsb_pcd_radius_outliers": (C.c_int, [C.POINTER(GsbPointGrid), C.c_int64, C.c_double, _vp, _vp]),
    "gsb_pcd_dbscan_workspace_bytes": (C.c_size_t, [C.c_int64]),
    "gsb_pcd_dbscan": (C.c_int, [C.POINTER(GsbPointGrid), C.c_double, C.c_int64, _vp, C.c_size_t, _vp, _vp, _vp]),
    "gsb_eval_transform_points": (C.c_int, [_vp, C.c_int64, C.POINTER(C.c_double), _vp, _vp]),
    "gsb_eval_crop_polygon": (C.c_int, [_vp, C.c_int64, _vp, C.c_int32, C.c_int32, C.c_double, C.c_double, _vp, _vp, _vp, _vp]),
    "gsb_eval_voxel_workspace_bytes": (C.c_size_t, [C.c_int64]),
    "gsb_pcd_voxel_downsample": (C.c_int, [_vp, _vp, _vp, C.c_int64, C.POINTER(C.c_double), C.POINTER(C.c_double), C.c_double,
                                           _vp, C.c_size_t, _vp, _vp, _vp, _vp, _vp]),
    "gsb_eval_icp_correspond": (C.c_int, [C.POINTER(GsbPointGrid), _vp, C.c_int64, C.c_double, _vp, _vp, _vp]),
    "gsb_eval_icp_moments": (C.c_int, [_vp, _vp, _vp, C.c_int64, _vp, C.c_int, C.POINTER(C.c_double), _vp, _vp, _vp]),
    "gsb_eval_mask_dilate_disk":(C.c_int, [_vp, C.c_int32, C.c_int32, C.c_int32, C.c_int32, _vp, _vp, _vp]),
    "gsb_eval_cull_vertices_by_masks": (C.c_int, [_vp, C.c_int64, _vp, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                                  _vp, _vp, _vp]),
    "gsb_eval_triangle_areas": (C.c_int, [_vp, C.c_int64, _vp, C.c_int64, _vp, _vp]),
    "gsb_eval_sample_uniform": (C.c_int, [_vp, C.c_int64, _vp, C.c_int64, _vp, _vp, C.c_int64, _vp, _vp]),
    "gsb_eval_poisson_neighbours": (C.c_int, [C.POINTER(GsbPointGrid), C.c_double, C.c_double, _vp, _vp, _vp, _vp, _vp]),
    "gsb_eval_poisson_eliminate": (C.c_int, [_vp, _vp, _vp, C.c_int64, _vp, _vp, _vp, _vp, C.POINTER(C.c_int32), _vp]),
    "gsb_eval_visibility": (C.c_int, [_vp, C.c_int64, C.POINTER(C.c_double), C.c_double, C.POINTER(C.c_int32), _vp, _vp,
                                      _vp]),
    "gsb_stereo_pack_inputs": (C.c_int, [_vp, _vp, C.c_int32, C.c_int32, _vp, _vp]),
    "gsb_stereo_disparities": (C.c_int, [_vp, _vp, C.c_int32, C.c_int32, C.c_float, _vp, _vp, _vp]),
    "gsb_stereo_occlusion_depth": (C.c_int, [_vp, _vp, C.c_int32, C.c_int32, C.c_int64, C.c_double, C.c_float, _vp, _vp, _vp]),
}

_lib = None


class GsbError(RuntimeError):
    def __init__(self, code, message):
        super().__init__(message)
        self.code = code


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing: the CUDA extension has not been built (run `python -m gs2mesh_b200.build` or "
                "__graft_entry__.build()).  gs2mesh_b200 has no CPU fallback.")
        handle = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(handle, name)  # AttributeError if the library does not export a declared symbol
            fn.restype = res
            fn.argtypes = args
        _lib = handle
    return _lib


def check(code: int, invalid_is_value_error: bool = False) -> None:
    """Raises GsbError for a failed call; with invalid_is_value_error, ValueError for GSB_ERR_INVALID instead (arguments
    the caller passed on from its own caller)."""
    if code != GSB_OK:
        message = lib().gsb_last_error().decode("utf-8", "replace")
        if invalid_is_value_error and code == GSB_ERR_INVALID:
            raise ValueError(message)
        raise GsbError(code, message)


def ptr(t):
    """torch tensor (or None) -> c_void_p of its storage start."""
    return None if t is None else C.c_void_p(t.data_ptr())


def stream(dev) -> C.c_void_p:
    """The current torch stream of CUDA device dev, as a library call's stream argument."""
    import torch

    return C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def device(device=None, like=None):
    """`device` if given, else the device of `like` when it is a CUDA tensor, else the current CUDA device."""
    import torch

    if device is not None:
        return torch.device(device)
    if isinstance(like, torch.Tensor) and like.is_cuda:
        return like.device
    return torch.device("cuda", torch.cuda.current_device())


def profile_enable(on: bool) -> None:
    check(lib().gsb_profile_enable(1 if on else 0))


def profile_collect():
    """{stage name: (total ms, samples)} since the last collect; synchronises the device."""
    L = lib()
    n = L.gsb_profile_num_stages()
    ms = (C.c_double * n)()
    cnt = (C.c_uint64 * n)()
    check(L.gsb_profile_collect(ms, cnt, n))
    return {L.gsb_profile_stage_name(i).decode(): (float(ms[i]), int(cnt[i])) for i in range(n)}
