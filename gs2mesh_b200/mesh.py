"""Mesh extraction + post-processing for the TSDF stage: the part of gs2mesh_utils/tsdf_utils.py the
reference delegates to Open3D's TriangleMesh (lines 108-110 extract / scale / vertex normals,
112-120 save, 122-142 cluster cleaning).

Marching cubes, vertex attributes and vertex normals run on the GPU (gsb_mesh_* in
include/gs2mesh_b200.h); vertex de-duplication is a sort/unique of 64-bit edge keys (what Open3D
does with a hash map).  Connected-component cleaning runs on the GPU for a mesh extracted from a
GPU volume (`TriangleMesh.device` is set) and with numpy / scipy for a mesh built from host arrays;
both give the same labels, counts and cleaned mesh.  PLY writing stays on the host like in the
reference.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import numpy as np
import torch

from . import _lib
from ._lib import ptr


def color_to_uint8(colors):
    """Open3D's utility::ColorToUint8, which its PLY writer applies to vertex colours:
    uint8_t(std::round(std::min(1., std::max(0., c)) * 255.)).  std::round rounds halves away from zero (np.rint would
    round them to even), and std::max(0., NaN) is 0."""
    c = np.asarray(colors, dtype=np.float64)
    c = np.where(c > 0.0, c, 0.0)
    s = np.where(c < 1.0, c, 1.0) * 255.0
    lo = np.floor(s)
    return (lo + (s - lo >= 0.5)).astype(np.uint8)


class TriangleMesh:
    """Minimal stand-in for open3d.geometry.TriangleMesh (the members tsdf_utils.py touches)."""

    def __init__(self, vertices, triangles, vertex_colors=None, vertex_normals=None, device=None):
        # the CUDA device a mesh extracted from a GPU volume came from; None for a mesh built from host arrays.  Cluster
        # cleaning runs there (the arrays themselves are host numpy either way).
        self.device = None if device is None else torch.device(device)
        self.vertices = np.asarray(vertices, dtype=np.float64).reshape(-1, 3)
        self.triangles = np.asarray(triangles, dtype=np.int64).reshape(-1, 3)
        self.vertex_colors = None if vertex_colors is None else np.asarray(vertex_colors, dtype=np.float64).reshape(-1, 3)
        self.vertex_normals = None if vertex_normals is None else np.asarray(vertex_normals, dtype=np.float64).reshape(-1, 3)

    # -- tsdf_utils.py:109
    def scale(self, scale, center=(0, 0, 0)):
        c = np.asarray(center, dtype=np.float64)
        self.vertices = (self.vertices - c) * float(scale) + c
        return self

    # -- tsdf_utils.py:110 (area-weighted, normalised; TriangleMesh::ComputeVertexNormals, bit for bit)
    def compute_vertex_normals(self, device=None):
        nv, nt = len(self.vertices), len(self.triangles)
        if nv == 0:
            self.vertex_normals = np.zeros((0, 3))
            return self
        if nt and (self.triangles.min() < 0 or self.triangles.max() >= nv):
            raise ValueError("compute_vertex_normals: triangle vertex index out of range")
        dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        with torch.cuda.device(dev):
            xyz = torch.as_tensor(self.vertices).to(dev).contiguous()
            tri = torch.as_tensor(self.triangles).to(dev).contiguous()
            # vertex -> triangle incidence as CSR; the stable sort keeps each vertex's triangles in triangle order, the
            # order Open3D adds them in
            flat = tri.reshape(-1)
            incidence = torch.sort(flat, stable=True).indices
            offsets = torch.zeros(nv + 1, dtype=torch.int64, device=dev)
            offsets[1:] = torch.cumsum(torch.bincount(flat, minlength=nv), 0)
            out = torch.empty(nv, 3, dtype=torch.float64, device=dev)
            stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            _lib.check(_lib.lib().gsb_mesh_vertex_normals(ptr(xyz), nv, ptr(tri), nt, ptr(incidence), ptr(offsets), ptr(out),
                                                          stream))
            self.vertex_normals = out.cpu().numpy()
        return self

    def _clusters_on_device(self, with_area):
        """gsb_mesh_clusters on self.device: (device triangles, workspace, labels, counts, n_clusters, cluster areas or
        None), all enqueued on the device's current stream."""
        nv, nt = len(self.vertices), len(self.triangles)
        if nt and (self.triangles.min() < 0 or self.triangles.max() >= nv):
            raise ValueError("cluster_connected_triangles: triangle vertex index out of range")
        dev = self.device
        L = _lib.lib()
        stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        tri = torch.as_tensor(self.triangles, dtype=torch.int64).to(dev).contiguous()
        work = torch.empty(L.gsb_mesh_cluster_workspace_bytes(nt, nv), dtype=torch.uint8, device=dev)
        labels = torch.empty(nt, dtype=torch.int64, device=dev)
        counts = torch.empty(nt, dtype=torch.int64, device=dev)
        n = torch.empty(1, dtype=torch.int64, device=dev)
        xyz = torch.as_tensor(self.vertices).to(dev).contiguous() if with_area else None
        area = torch.empty(nt, dtype=torch.float64, device=dev) if with_area else None
        _lib.check(L.gsb_mesh_clusters(ptr(tri), nt, nv, ptr(xyz), ptr(work), work.numel(), ptr(labels), ptr(counts), ptr(n),
                                       ptr(area), stream))
        return tri, work, labels, counts, n, area

    # -- tsdf_utils.py:132-133 (TriangleMesh::ClusterConnectedTriangles: triangles sharing an edge)
    def cluster_connected_triangles(self):
        if self.device is not None:
            with torch.cuda.device(self.device):
                _, _, labels, counts, n, area = self._clusters_on_device(with_area=True)
                k = int(n.item())
                return labels.cpu().numpy(), counts[:k].cpu().numpy(), area[:k].cpu().numpy()
        from scipy.sparse import coo_matrix
        from scipy.sparse.csgraph import connected_components

        nt = len(self.triangles)
        if nt == 0:
            return np.zeros(0, np.int64), np.zeros(0, np.int64), np.zeros(0)
        t = self.triangles
        e = np.concatenate([t[:, [0, 1]], t[:, [1, 2]], t[:, [2, 0]]], axis=0)
        e.sort(axis=1)
        owner = np.tile(np.arange(nt), 3)
        key = e[:, 0] * (int(self.vertices.shape[0]) + 1) + e[:, 1]
        order = np.argsort(key, kind="stable")
        ks, os_ = key[order], owner[order]
        same = ks[1:] == ks[:-1]
        a, b = os_[:-1][same], os_[1:][same]
        graph = coo_matrix((np.ones(len(a), np.int8), (a, b)), shape=(nt, nt))
        _, labels = connected_components(graph, directed=False)
        counts = np.bincount(labels)
        v = self.vertices
        area = 0.5 * np.linalg.norm(np.cross(v[t[:, 1]] - v[t[:, 0]], v[t[:, 2]] - v[t[:, 0]]), axis=1)
        return labels.astype(np.int64), counts.astype(np.int64), np.bincount(labels, weights=area)

    # -- tsdf_utils.py:137-140
    def remove_small_clusters(self, min_triangles):
        if self.device is not None:
            return self._remove_small_clusters_on_device(min_triangles)
        labels, counts, _ = self.cluster_connected_triangles()
        keep = ~(counts[labels] < min_triangles) if len(labels) else np.zeros(0, bool)
        tris = self.triangles[keep]
        used = np.zeros(len(self.vertices), bool)
        used[tris.reshape(-1)] = True  # remove_unreferenced_vertices
        remap = np.cumsum(used) - 1
        pick = lambda a: None if a is None else a[used]
        return TriangleMesh(self.vertices[used], remap[tris], pick(self.vertex_colors), pick(self.vertex_normals))

    def _remove_small_clusters_on_device(self, min_triangles):
        """remove_small_clusters on self.device: the triangles go up once, the kept triangles (renumbered) and the old ids
        of the kept vertices come back, and the vertex arrays are gathered where they live."""
        nv, nt = len(self.vertices), len(self.triangles)
        with torch.cuda.device(self.device):
            dev = self.device
            stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            tri, work, labels, counts, _, _ = self._clusters_on_device(with_area=False)
            out_tri = torch.empty(nt, 3, dtype=torch.int64, device=dev)
            ids = torch.empty(nv, dtype=torch.int64, device=dev)
            sizes = torch.empty(2, dtype=torch.int64, device=dev)
            _lib.check(_lib.lib().gsb_mesh_remove_small_clusters(ptr(tri), nt, nv, ptr(labels), ptr(counts), float(min_triangles),
                                                                 ptr(work), work.numel(), ptr(out_tri), ptr(ids), ptr(sizes),
                                                                 stream))
            kt, kv = (int(x) for x in sizes.cpu().tolist())
            tris, used = out_tri[:kt].cpu().numpy(), ids[:kv].cpu().numpy()
        pick = lambda a: None if a is None else a[used]
        return TriangleMesh(self.vertices[used], tris, pick(self.vertex_colors), pick(self.vertex_normals), device=self.device)

    # -- o3d.io.write_triangle_mesh(path, mesh): binary little-endian PLY, double coordinates
    def write_ply(self, path):
        nv, nt = len(self.vertices), len(self.triangles)
        props = [("x", "<f8"), ("y", "<f8"), ("z", "<f8")]
        header = ["ply", "format binary_little_endian 1.0", "comment Created by gs2mesh_b200", f"element vertex {nv}",
                  "property double x", "property double y", "property double z"]
        if self.vertex_normals is not None:
            props += [("nx", "<f8"), ("ny", "<f8"), ("nz", "<f8")]
            header += ["property double nx", "property double ny", "property double nz"]
        if self.vertex_colors is not None:
            props += [("red", "u1"), ("green", "u1"), ("blue", "u1")]
            header += ["property uchar red", "property uchar green", "property uchar blue"]
        header += [f"element face {nt}", "property list uchar uint vertex_indices", "end_header"]
        vert = np.zeros(nv, dtype=props)
        vert["x"], vert["y"], vert["z"] = self.vertices.T if nv else (np.zeros(0),) * 3
        if self.vertex_normals is not None and nv:
            vert["nx"], vert["ny"], vert["nz"] = self.vertex_normals.T
        if self.vertex_colors is not None and nv:
            vert["red"], vert["green"], vert["blue"] = color_to_uint8(self.vertex_colors).T
        face = np.zeros(nt, dtype=[("n", "u1"), ("v", "<u4", (3,))])
        face["n"] = 3
        face["v"] = self.triangles.astype(np.uint32)
        with open(path, "wb") as f:
            f.write(("\n".join(header) + "\n").encode("ascii"))
            f.write(vert.tobytes())
            f.write(face.tobytes())
        return path


def extract_triangle_mesh(volume, with_colors: Optional[bool] = None) -> TriangleMesh:
    """`volume.extract_triangle_mesh()` for a gs2mesh_b200.tsdf.TSDFVolume."""
    dev = volume.device
    L = _lib.lib()
    with_colors = (volume.color is not None) if with_colors is None else with_colors
    with torch.cuda.device(dev):
        stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        nb = volume.num_bricks()  # every brick ever opened = pool slots [0, nb)
        if nb == 0:
            return TriangleMesh(np.zeros((0, 3)), np.zeros((0, 3), np.int64), np.zeros((0, 3)) if with_colors else None,
                                device=dev)
        bricks = torch.arange(nb, dtype=torch.int32, device=dev)
        # edge keys are voxel indices inside the bounding box of the open bricks (+1: a cube reaches into its +1 neighbours)
        idx = volume._index[:nb, :3]
        lo = idx.min(dim=0).values.cpu().numpy().astype(np.int64)
        hi = idx.max(dim=0).values.cpu().numpy().astype(np.int64)
        window = (C.c_int32 * 6)(*[int(v) for v in lo], *[int(v) for v in (hi - lo + 2)])
        counts = torch.zeros(nb, dtype=torch.int32, device=dev)
        _lib.check(L.gsb_mesh_count(volume._h, window, ptr(bricks), nb, ptr(counts), stream))
        offsets = torch.cumsum(counts.to(torch.int64), 0) - counts.to(torch.int64)
        n_tri = int(counts.sum().item())
        if n_tri == 0:
            return TriangleMesh(np.zeros((0, 3)), np.zeros((0, 3), np.int64), np.zeros((0, 3)) if with_colors else None,
                                device=dev)
        keys = torch.empty(n_tri * 3, dtype=torch.int64, device=dev)
        _lib.check(L.gsb_mesh_emit(volume._h, window, ptr(bricks), nb, ptr(offsets.contiguous()), ptr(keys), stream))
        uniq, inverse = torch.unique(keys, return_inverse=True)  # vertex ids = rank of the edge key
        nv = int(uniq.numel())
        xyz = torch.empty(nv, 3, dtype=torch.float64, device=dev)
        rgb = torch.empty(nv, 3, dtype=torch.float64, device=dev) if with_colors else None
        _lib.check(L.gsb_mesh_vertices(volume._h, window, ptr(uniq.contiguous()), nv, ptr(xyz), ptr(rgb), stream))
        tris = inverse.reshape(-1, 3)
        mesh = TriangleMesh(xyz.cpu().numpy(), tris.cpu().numpy(), None if rgb is None else rgb.cpu().numpy(), device=dev)
        mesh.edge_keys = uniq.cpu().numpy()  # (voxel index inside `key_window` * 3 + axis) per vertex, for tests
        mesh.key_window = (tuple(int(v) for v in lo), tuple(int(v) for v in (hi - lo + 2)))  # (brick origin, brick count)
    return mesh
