"""Open3D-shaped facade over the CUDA TSDF / mesh kernels: exactly the slice of the `open3d` API that
gs2mesh_utils/tsdf_utils.py touches, so its body (lines 51-142) reads the same with

    import gs2mesh_b200.o3d_compat as o3d

    volume = o3d.pipelines.integration.ScalableTSDFVolume(voxel_length=..., sdf_trunc=..., color_type=...RGB8)   # :53-56
    rgbd   = o3d.geometry.RGBDImage.create_from_color_and_depth(o3d.geometry.Image(rgb), o3d.geometry.Image(depth),
                 depth_scale=..., depth_trunc=..., convert_rgb_to_intensity=False)                               # :88-93
    intr   = o3d.camera.PinholeCameraIntrinsic(w, h, fx, fy, cx, cy)                                            # :106
    volume.integrate(rgbd, intr, np.linalg.inv(extrinsic))                                                       # :107
    mesh = volume.extract_triangle_mesh(); mesh.scale(s, (0, 0, 0)); mesh.compute_vertex_normals()               # :108-110
    o3d.io.write_triangle_mesh(path, mesh)                                                                       # :119
    clusters, n_tri, area = mesh.cluster_connected_triangles(); mesh.remove_triangles_by_mask(mask);
    mesh.remove_unreferenced_vertices()                                                                          # :132-140

Differences from Open3D, by construction: the volume lives in GPU memory (an unbounded, hashed set of 16^3 bricks on
the same voxel lattice, like Open3D's; `window_resolution=` only sets the window dense read-backs look at); images are uploaded on
integrate().  Everything else (argument names, the RuntimeError on mismatching image sizes, float32 depth
conversion rule `d / scale; d >= trunc -> 0`) follows Open3D 0.17.
"""
from __future__ import annotations

import contextlib
from types import SimpleNamespace

import numpy as np

from .mesh import TriangleMesh as _Mesh
from .mesh import extract_triangle_mesh as _extract


class Image:
    """open3d.geometry.Image: a thin holder of a host array (uint8 HxWx3 colour or float32 HxW depth)."""

    def __init__(self, array):
        self.array = np.ascontiguousarray(array)

    def __array__(self, dtype=None):
        return self.array if dtype is None else self.array.astype(dtype)

    @property
    def width(self):
        return int(self.array.shape[1])

    @property
    def height(self):
        return int(self.array.shape[0])


class RGBDImage:
    def __init__(self, color, depth, depth_scale=1.0, depth_trunc=float("inf")):
        self.color = color
        self.depth = depth  # RAW depth; scale / trunc are applied by the fused prepare kernel at integrate()
        self._depth_scale = float(depth_scale)
        self._depth_trunc = float(depth_trunc)

    @staticmethod
    def create_from_color_and_depth(color, depth, depth_scale=1000.0, depth_trunc=3.0, convert_rgb_to_intensity=True):
        if convert_rgb_to_intensity:
            raise NotImplementedError("gs2mesh passes convert_rgb_to_intensity=False (tsdf_utils.py:93); intensity images are not supported")
        c, d = np.asarray(color), np.asarray(depth)
        if c.shape[0] != d.shape[0] or c.shape[1] != d.shape[1]:
            raise RuntimeError("[CreateFromColorAndDepth] Unsupported image format.")
        return RGBDImage(color if isinstance(color, Image) else Image(c), depth if isinstance(depth, Image) else Image(d),
                         depth_scale, depth_trunc)


class PinholeCameraIntrinsic:
    def __init__(self, width, height, fx, fy, cx, cy):
        self.width, self.height = int(width), int(height)
        self.fx, self.fy, self.cx, self.cy = float(fx), float(fy), float(cx), float(cy)
        self.intrinsic_matrix = np.array([[self.fx, 0, self.cx], [0, self.fy, self.cy], [0, 0, 1.0]])

    def get_focal_length(self):
        return self.fx, self.fy

    def get_principal_point(self):
        return self.cx, self.cy


class TSDFVolumeColorType:
    NoColor = 0
    RGB8 = 1
    Gray32 = 2


class TriangleMesh(_Mesh):
    """open3d.geometry.TriangleMesh members used by tsdf_utils.py:108-142."""

    def remove_triangles_by_mask(self, mask):
        self.triangles = self.triangles[~np.asarray(mask, dtype=bool)]
        return self

    def remove_unreferenced_vertices(self):
        used = np.zeros(len(self.vertices), bool)
        used[self.triangles.reshape(-1)] = True
        remap = np.cumsum(used) - 1
        self.triangles = remap[self.triangles]
        self.vertices = self.vertices[used]
        if self.vertex_colors is not None:
            self.vertex_colors = self.vertex_colors[used]
        if self.vertex_normals is not None:
            self.vertex_normals = self.vertex_normals[used]
        return self

    def __deepcopy__(self, memo):
        return TriangleMesh(self.vertices.copy(), self.triangles.copy(), None if self.vertex_colors is None else self.vertex_colors.copy(),
                            None if self.vertex_normals is None else self.vertex_normals.copy(), device=self.device)


class ScalableTSDFVolume:
    def __init__(self, voxel_length, sdf_trunc, color_type=TSDFVolumeColorType.RGB8, volume_unit_resolution=16,
                 depth_sampling_stride=4, *, window_resolution=512, device="cuda", pool_bricks=None):
        if volume_unit_resolution != 16 or depth_sampling_stride != 4:
            raise NotImplementedError("only Open3D's defaults (volume_unit_resolution=16, depth_sampling_stride=4) are built; "
                                      "gs2mesh does not override them (tsdf_utils.py:53-56)")
        if color_type == TSDFVolumeColorType.Gray32:
            raise NotImplementedError("Gray32 volumes are not supported (gs2mesh uses RGB8)")
        from .tsdf import TSDFVolume, default_window

        origin, count = default_window(window_resolution)
        self.voxel_length, self.sdf_trunc, self.color_type = float(voxel_length), float(sdf_trunc), color_type
        self._vol = TSDFVolume(self.voxel_length, self.sdf_trunc, origin, count, with_color=color_type == TSDFVolumeColorType.RGB8,
                               device=device, pool_bricks=pool_bricks)

    def integrate(self, image, intrinsic, extrinsic):
        d = np.asarray(image.depth)
        c = np.asarray(image.color)
        if d.ndim != 2 or d.shape[1] != intrinsic.width or d.shape[0] != intrinsic.height or \
                (self._vol.color is not None and (c.ndim != 3 or c.shape[2] != 3 or c.dtype != np.uint8)):
            raise RuntimeError("[ScalableTSDFVolume::Integrate] Unsupported image format.")
        prepared = self._vol.prepare_depth(d.astype(np.float32), intrinsic.width, intrinsic.height, depth_scale=image._depth_scale,
                                           depth_trunc=image._depth_trunc)
        # unbounded like Open3D's hash map: bricks are opened (and the pool grown if need be) before any voxel is updated
        self._vol.integrate_exact(prepared, c if self._vol.color is not None else None, intrinsic.width, intrinsic.height,
                                  intrinsic.fx, intrinsic.fy, intrinsic.cx, intrinsic.cy, np.asarray(extrinsic, dtype=np.float64))

    def extract_triangle_mesh(self):
        m = _extract(self._vol)
        return TriangleMesh(m.vertices, m.triangles, m.vertex_colors, m.vertex_normals, device=m.device)

    def reset(self):
        self._vol.reset()


def _write_triangle_mesh(path, mesh, **_):
    mesh.write_ply(path)
    return True


@contextlib.contextmanager
def _verbosity(_level):
    yield None


# module tree mirroring `open3d`
geometry = SimpleNamespace(Image=Image, RGBDImage=RGBDImage, TriangleMesh=TriangleMesh)
camera = SimpleNamespace(PinholeCameraIntrinsic=PinholeCameraIntrinsic)
pipelines = SimpleNamespace(integration=SimpleNamespace(ScalableTSDFVolume=ScalableTSDFVolume, TSDFVolumeColorType=TSDFVolumeColorType))
io = SimpleNamespace(write_triangle_mesh=_write_triangle_mesh)
utility = SimpleNamespace(VerbosityContextManager=_verbosity, VerbosityLevel=SimpleNamespace(Debug=0, Info=1, Warning=2, Error=3))
__version__ = "0.17.0-gs2mesh_b200"
