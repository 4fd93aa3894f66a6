"""Mesh extraction + post-processing for the TSDF stage: the part of gs2mesh_utils/tsdf_utils.py the
reference delegates to Open3D's TriangleMesh (lines 108-110 extract / scale / vertex normals,
112-120 save, 122-142 cluster cleaning).

Marching cubes, vertex attributes and vertex normals run on the GPU (gsb_mesh_* in
include/gs2mesh_b200.h); vertex de-duplication is a sort/unique of 64-bit edge keys (what Open3D
does with a hash map).  Connected-component cleaning runs on the GPU for a mesh extracted from a
GPU volume (`TriangleMesh.device` is set) and with numpy / scipy for a mesh built from host arrays;
both give the same labels, counts and cleaned mesh.  Vertex-clustering simplification (Open3D's
simplify_vertex_clustering) and the smoothing and sharpening filters (filter_smooth_simple / _laplacian / _taubin,
filter_sharpen) run on the GPU, and so do the topology queries (manifoldness, orientability, self-intersection,
watertightness, Euler characteristic, surface area and volume).  The extracted PointCloud is cleaned and thinned on the GPU
too (gs2mesh_b200/pointcloud.py): remove_statistical_outlier, remove_radius_outlier, cluster_dbscan, select_by_index,
voxel_down_sample with colours and normals, uniform_down_sample, compute_nearest_neighbor_distance and
compute_point_cloud_distance.  PLY writing stays on the host like in the reference.
"""
from __future__ import annotations

import ctypes as C
import enum
from typing import Optional

import numpy as np
import torch

from . import _lib
from . import pointcloud as _pcd
from ._lib import ptr
from .io import color_to_uint8, write_point_cloud_ply  # noqa: F401  (color_to_uint8: callers also import it from here)


class SimplificationContraction(enum.IntEnum):
    """open3d.geometry.SimplificationContraction: where simplify_vertex_clustering places a cell's vertex."""

    Average = 0  # GSB_SIMPLIFY_AVERAGE: the mean of the cell's vertices
    Quadric = 1  # GSB_SIMPLIFY_QUADRIC: the minimum of the cell's plane quadrics


class FilterScope(enum.IntEnum):
    """open3d.geometry.FilterScope: which vertex attributes the smoothing and sharpening filters change."""

    All = 0  # GSB_FILTER_SCOPE_ALL: positions, and colours and normals where the mesh has them
    Color = 1
    Normal = 2
    Vertex = 3  # positions only


def _adjacency(tri, nv):
    """Open3D's ComputeAdjacencyList as CSR on tri's device: (offsets int64 [nv + 1], neighbours int64), each vertex's
    run holding the distinct ids it shares a triangle with at another corner position, ascending."""
    src = tri[:, [0, 0, 1, 1, 2, 2]].reshape(-1)
    dst = tri[:, [1, 2, 0, 2, 0, 1]].reshape(-1)
    keys = torch.unique(src * nv + dst)  # sorted: by vertex, then by neighbour
    owner = keys // nv
    offsets = torch.zeros(nv + 1, dtype=torch.int64, device=tri.device)
    offsets[1:] = torch.cumsum(torch.bincount(owner, minlength=nv), 0)
    return offsets, (keys - owner * nv).contiguous()


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

    def _check(self, who, attributes=False):
        """(n_vertices, n_triangles); ValueError prefixed `who: ` for a triangle index outside [0, n_vertices) and, with
        `attributes`, for vertex colours or normals without one row per vertex."""
        nv, nt = len(self.vertices), len(self.triangles)
        if nt and (self.triangles.min() < 0 or self.triangles.max() >= nv):
            raise ValueError(f"{who}: triangle vertex index out of range")
        for name in ("vertex_colors", "vertex_normals") if attributes else ():
            a = getattr(self, name)
            if a is not None and len(a) != nv:
                raise ValueError(f"{who}: {name} must have one row per vertex")
        return nv, nt

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
        self._check("compute_vertex_normals")
        dev = _lib.device(device)
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
            stream = _lib.stream(dev)
            _lib.check(_lib.lib().gsb_mesh_vertex_normals(ptr(xyz), nv, ptr(tri), nt, ptr(incidence), ptr(offsets), ptr(out),
                                                          stream))
            self.vertex_normals = out.cpu().numpy()
        return self

    def _clusters_on_device(self, with_area):
        """gsb_mesh_clusters on self.device: (device triangles, workspace, labels, counts, n_clusters, cluster areas or
        None), all enqueued on the device's current stream."""
        nv, nt = self._check("cluster_connected_triangles")
        dev = self.device
        L = _lib.lib()
        stream = _lib.stream(dev)
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
            stream = _lib.stream(dev)
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

    # -- TriangleMesh::SimplifyVertexClustering (DESIGN.md section 7, "Simplification")
    def simplify_vertex_clustering(self, voxel_size, contraction=None):
        """A new mesh of the same class with one vertex per occupied cell of a `voxel_size` grid anchored half a cell
        below the vertices' minimum.  Cells are numbered in the order of their smallest vertex id (Open3D's numbering).
        SimplificationContraction.Average (the default) places each at the mean of its vertices, Quadric at the
        minimum of its triangles' area-weighted plane quadrics where |det A| > 1e-4 (the mean elsewhere); colours and
        normals are means either way.  Triangles whose corners fall into fewer than three cells are dropped, the rest
        start at their smallest vertex id (winding kept) and each such triple is kept once, in input order.

        Runs on `self.device` (the current CUDA device for a mesh built from host arrays); the result records that
        device and holds host arrays.  `self.last_simplify_stats` gives the cells, the triangles and the cells that
        took the quadric solve.  RuntimeError("voxel_size <= 0.0") / ("voxel_size is too small.") as in Open3D;
        ValueError for non-finite vertices or voxel size, bad indices or a cell box past 63-bit keys."""
        contraction = SimplificationContraction.Average if contraction is None else SimplificationContraction(contraction)
        s = float(voxel_size)
        if not s > 0.0:
            raise RuntimeError("voxel_size <= 0.0")
        nv, nt = self._check("simplify_vertex_clustering", attributes=True)
        lo = self.vertices.min(axis=0) if nv else np.zeros(3)
        hi = self.vertices.max(axis=0) if nv else np.zeros(3)
        dev = _lib.device(self.device)
        L = _lib.lib()
        dbl3 = C.c_double * 3
        with torch.cuda.device(dev):
            up = lambda a: None if a is None else torch.as_tensor(a).to(dev).contiguous()
            xyz, rgb, nrm, tri = up(self.vertices), up(self.vertex_colors), up(self.vertex_normals), up(self.triangles)
            like = lambda a: None if a is None else torch.empty_like(a)
            out_v, out_c, out_n, out_t = like(xyz), like(rgb), like(nrm), like(tri)
            work = torch.empty(L.gsb_mesh_simplify_workspace_bytes(nv, nt), dtype=torch.uint8, device=dev)
            sizes = torch.empty(3, dtype=torch.int64, device=dev)
            rc = L.gsb_mesh_simplify(ptr(xyz), ptr(rgb), ptr(nrm), nv, ptr(tri), nt, dbl3(*lo.tolist()), dbl3(*hi.tolist()), s,
                                     int(contraction), ptr(work), work.numel(), ptr(out_v), ptr(out_c), ptr(out_n), ptr(out_t),
                                     ptr(sizes), _lib.stream(dev))
            if rc == _lib.GSB_ERR_INVALID and L.gsb_last_error().endswith(b"voxel_size is too small."):
                raise RuntimeError("voxel_size is too small.")
            _lib.check(rc, invalid_is_value_error=True)
            k, kt, kq = (int(x) for x in sizes.cpu().tolist())
            host = lambda a, n: None if a is None else a[:n].cpu().numpy()
            out = type(self)(host(out_v, k), host(out_t, kt), host(out_c, k), host(out_n, k), device=dev)
        self.last_simplify_stats = {"vertices": k, "triangles": kt, "quadric_cells": kq}
        return out

    # -- TriangleMesh::FilterSmoothSimple / FilterSmoothLaplacian / FilterSmoothTaubin / FilterSharpen (DESIGN.md
    # section 7, "Smoothing and sharpening").  Each returns a new mesh of the same class with the same triangles; it runs
    # on `self.device` (the current CUDA device for a mesh built from host arrays), and the result records that device
    # and holds host arrays.  Neighbours are the vertices sharing a triangle; each pass reads only the previous pass's
    # values.  `filter_scope` picks positions (Vertex), colours (Color), normals (Normal) or all three (All); colours and
    # normals only where the mesh has them, normals not renormalised, colours not clamped.
    def filter_smooth_simple(self, number_of_iterations=1, filter_scope=FilterScope.All):
        """x' = (x + sum of the neighbours' x) / (1 + number of neighbours), per pass."""
        return self._filter("filter_smooth_simple", _lib.GSB_FILTER_SIMPLE, number_of_iterations, 0.0, 0.0, filter_scope)

    def filter_smooth_laplacian(self, number_of_iterations=1, lambda_filter=0.5, filter_scope=FilterScope.All):
        """x' = x + lambda_filter * (the neighbours' x weighted by 1 / (distance + 1e-12), averaged, - x), per pass; a
        vertex without neighbours keeps its values."""
        return self._filter("filter_smooth_laplacian", _lib.GSB_FILTER_LAPLACIAN, number_of_iterations, lambda_filter, 0.0,
                            filter_scope)

    def filter_smooth_taubin(self, number_of_iterations=1, lambda_filter=0.5, mu=-0.53, filter_scope=FilterScope.All):
        """Per iteration one Laplacian pass with lambda_filter, then one with mu: smooths without shrinking."""
        return self._filter("filter_smooth_taubin", _lib.GSB_FILTER_TAUBIN, number_of_iterations, lambda_filter, mu,
                            filter_scope)

    def filter_sharpen(self, number_of_iterations=1, strength=1, filter_scope=FilterScope.All):
        """x' = x + strength * sum over the neighbours of (x - neighbour's x), per pass."""
        return self._filter("filter_sharpen", _lib.GSB_FILTER_SHARPEN, number_of_iterations, strength, 0.0, filter_scope)

    def _filter(self, name, kind, number_of_iterations, param0, param1, filter_scope):
        """gsb_mesh_filter on the mesh's CSR adjacency: the one call path of the four filters."""
        scope = FilterScope(filter_scope)
        iterations = int(number_of_iterations)
        if not 0 <= iterations <= 2**31 - 1:
            raise ValueError(f"{name}: number_of_iterations must be in [0, 2^31 - 1], got {iterations}")
        nv, nt = self._check(name, attributes=True)
        dev = _lib.device(self.device)
        L = _lib.lib()
        with torch.cuda.device(dev):
            up = lambda a: None if a is None else torch.as_tensor(a).to(dev).contiguous()
            xyz, rgb, nrm = up(self.vertices), up(self.vertex_colors), up(self.vertex_normals)
            offsets, neighbours = _adjacency(up(self.triangles), nv)
            like = lambda a: None if a is None else torch.empty_like(a)
            out_v, out_c, out_n = like(xyz), like(rgb), like(nrm)
            work = torch.empty(L.gsb_mesh_filter_workspace_bytes(nv, rgb is not None, nrm is not None), dtype=torch.uint8,
                               device=dev)
            _lib.check(L.gsb_mesh_filter(kind, ptr(xyz), ptr(rgb), ptr(nrm), nv, ptr(offsets), ptr(neighbours), iterations,
                                         float(param0), float(param1), int(scope), ptr(work), work.numel(), ptr(out_v),
                                         ptr(out_c), ptr(out_n), _lib.stream(dev)), invalid_is_value_error=True)
            host = lambda a: None if a is None else a.cpu().numpy()
            return type(self)(host(out_v), self.triangles.copy(), host(out_c), host(out_n), device=dev)

    # -- TriangleMesh::GetNonManifoldEdges / IsEdgeManifold / GetNonManifoldVertices / IsVertexManifold /
    # GetSelfIntersectingTriangles / IsSelfIntersecting / IsOrientable / IsWatertight / EulerPoincareCharacteristic /
    # GetSurfaceArea / GetVolume (DESIGN.md section 7, "Topology queries").  Each runs on `self.device` (the current CUDA
    # device for a mesh built from host arrays), returns host values and leaves the mesh unchanged.  ValueError for an
    # out-of-range triangle index, non-finite vertices or a size past 32-bit ids.
    def get_non_manifold_edges(self, allow_boundary_edges=True):
        """int64 (k, 2): the edges (min, max), ascending, with more than two incident triangles, or with
        allow_boundary_edges=False any count but two.  (a, a, b) puts two incidences on (a, b)."""
        with _Topology(self) as q:
            return q.edges(allow_boundary_edges, with_list=True)[0]

    def is_edge_manifold(self, allow_boundary_edges=True):
        with _Topology(self) as q:
            return q.edges(allow_boundary_edges)[1] == 0

    def get_non_manifold_vertices(self):
        """int64 (k,), ascending: the vertices whose link graph (one edge per incident triangle: its first corner pair
        without the vertex) has more than one component."""
        with _Topology(self) as q:
            return q.vertices(with_list=True)[0]

    def is_vertex_manifold(self):
        with _Topology(self) as q:
            return q.vertices()[1] == 0

    def get_self_intersecting_triangles(self):
        """int64 (k, 2), t0 < t1, ascending by (t0, t1): the pairs that share no vertex id, whose boxes overlap and
        that Open3D's TriangleTriangle3d reports as intersecting."""
        with _Topology(self) as q:
            return q.self_intersections(with_list=True)[0]

    def is_self_intersecting(self):
        with _Topology(self) as q:
            return q.self_intersections()[1] > 0

    def is_orientable(self):
        with _Topology(self) as q:
            return q.edges(True)[3]

    def is_watertight(self):
        """is_edge_manifold(False) and is_vertex_manifold() and not is_self_intersecting(), on one upload."""
        with _Topology(self) as q:
            return q.watertight()

    def euler_poincare_characteristic(self):
        """V + F - E: every vertex, every triangle, the distinct undirected edges including (a, a)."""
        with _Topology(self) as q:
            return len(self.vertices) + len(self.triangles) - q.edges(True)[2]

    def get_surface_area(self):
        """The sum of 0.5 ||(p0 - p1) x (p0 - p2)|| in a fixed two-stage order."""
        with _Topology(self) as q:
            return q.area_volume()[0]

    def get_volume(self):
        """|sum of p0 . (p1 x p2) / 6|; RuntimeError as Open3D's for a mesh that is not watertight or not orientable."""
        with _Topology(self) as q:
            if not q.watertight():
                raise RuntimeError("The mesh is not watertight, and the volume cannot be computed.")
            if not q.edges(False)[3]:
                raise RuntimeError("The mesh is not orientable, and the volume cannot be computed.")
            return abs(q.area_volume()[1])

    # -- o3d.io.write_triangle_mesh(path, mesh): binary little-endian PLY, double coordinates and normals, uchar colours
    def write_ply(self, path):
        return write_point_cloud_ply(path, self.vertices, self.vertex_colors, self.vertex_normals, self.triangles)


class _Topology:
    """One upload of a mesh for the topology entries: the checks, the device arrays, and each edge pass's results kept
    so that is_watertight and get_volume run it once."""

    def __init__(self, mesh):
        nv, nt = mesh._check("topology")
        if not np.isfinite(mesh.vertices).all():
            raise ValueError("topology: the vertices are not finite")
        self.mesh, self.nv, self.nt = mesh, nv, nt
        self.dev = _lib.device(mesh.device)
        self.L = _lib.lib()
        self._edges = {}
        self._xyz = None

    def __enter__(self):
        self._ctx = torch.cuda.device(self.dev)
        self._ctx.__enter__()
        self.stream = _lib.stream(self.dev)
        self.tri = torch.as_tensor(self.mesh.triangles, dtype=torch.int64).to(self.dev).contiguous()
        return self

    def __exit__(self, *exc):
        return self._ctx.__exit__(*exc)

    def _work(self, nbytes):
        return torch.empty(nbytes, dtype=torch.uint8, device=self.dev)

    def xyz(self):
        if self._xyz is None:
            self._xyz = torch.as_tensor(self.mesh.vertices).to(self.dev).contiguous()
        return self._xyz

    def edges(self, allow_boundary_edges, with_list=False):
        """(non-manifold edges or None, their count, distinct edges, orientable)."""
        allow = bool(allow_boundary_edges)
        if (allow, with_list) not in self._edges and (allow, True) not in self._edges:
            L = self.L
            work = self._work(L.gsb_mesh_edge_topology_workspace_bytes(self.nt, self.nv))
            out = torch.empty(3 * self.nt, 2, dtype=torch.int64, device=self.dev) if with_list else None
            sizes = torch.empty(3, dtype=torch.int64, device=self.dev)
            _lib.check(L.gsb_mesh_edge_topology(ptr(self.tri), self.nt, self.nv, int(allow), ptr(work), work.numel(), ptr(out),
                                                ptr(sizes), self.stream), invalid_is_value_error=True)
            k, e, orientable = (int(x) for x in sizes.cpu().tolist())
            self._edges[(allow, with_list)] = (None if out is None else out[:k].cpu().numpy(), k, e, bool(orientable))
        return self._edges.get((allow, with_list)) or self._edges[(allow, True)]

    def vertices(self, with_list=False):
        """(non-manifold vertices, their count)."""
        L = self.L
        work = self._work(L.gsb_mesh_vertex_topology_workspace_bytes(self.nt, self.nv))
        out = torch.empty(self.nv, dtype=torch.int64, device=self.dev) if with_list else None
        count = torch.empty(1, dtype=torch.int64, device=self.dev)
        _lib.check(L.gsb_mesh_non_manifold_vertices(ptr(self.tri), self.nt, self.nv, ptr(work), work.numel(), ptr(out), ptr(count),
                                                    self.stream), invalid_is_value_error=True)
        k = int(count.item())
        return (out[:k].cpu().numpy() if with_list else None), k

    def self_intersections(self, with_list=False):
        """(pairs or None, their count); self.stats = (pairs, candidate pairs, registrations, grid level)."""
        L = self.L
        # the grid spans the referenced vertices only: a vertex no triangle uses must not stretch the cells
        v = self.mesh.vertices[self.mesh.triangles.reshape(-1)] if self.nt else np.zeros((1, 3))
        dbl3 = C.c_double * 3
        lo = dbl3(*v.min(axis=0).tolist())
        hi = dbl3(*v.max(axis=0).tolist())
        stats = torch.empty(4, dtype=torch.int64, device=self.dev)

        def run(out, capacity):
            work = self._work(L.gsb_mesh_self_intersections_workspace_bytes(self.nt, self.nv, capacity))
            _lib.check(L.gsb_mesh_self_intersections(ptr(self.xyz()), self.nv, ptr(self.tri), self.nt, lo, hi, ptr(work),
                                                     work.numel(), ptr(out), capacity, ptr(stats), self.stream),
                       invalid_is_value_error=True)
            return [int(x) for x in stats.cpu().tolist()]

        self.stats = run(None, 0)
        k = self.stats[0]
        if not with_list:
            return None, k
        out = torch.empty(k, 2, dtype=torch.int64, device=self.dev)
        if k:
            if run(out, k)[0] != k:
                raise RuntimeError("get_self_intersecting_triangles: the emit pass found a different number of pairs")
        return out.cpu().numpy(), k

    def watertight(self):
        return self.edges(False)[1] == 0 and self.vertices()[1] == 0 and self.self_intersections()[1] == 0

    def area_volume(self):
        """(surface area, signed volume sum)."""
        L = self.L
        work = self._work(L.gsb_mesh_area_volume_workspace_bytes(self.nt, self.nv))
        out = torch.empty(2, dtype=torch.float64, device=self.dev)
        _lib.check(L.gsb_mesh_area_volume(ptr(self.xyz()), self.nv, ptr(self.tri), self.nt, ptr(work), work.numel(), ptr(out),
                                          self.stream), invalid_is_value_error=True)
        a, v = out.cpu().tolist()
        return a, v


def remove_vertices_by_mask(vertices, triangles, vertex_mask, vertex_colors=None, vertex_normals=None):
    """TriangleMesh.remove_vertices_by_mask(mask): drops the vertices where vertex_mask is True, keeping the rest (and
    their colours and normals) in order; keeps the triangles whose three vertices survive, in order, re-indexed.
    Vertices no triangle uses stay.  Returns (vertices, triangles, colours or None, normals or None) as device tensors."""
    v = torch.as_tensor(vertices)
    dev = _lib.device(like=v)
    v = v.to(dev).to(torch.float64).reshape(-1, 3)
    t = torch.as_tensor(triangles).to(dev).to(torch.int64).reshape(-1, 3)
    keep = ~torch.as_tensor(vertex_mask).to(dev).to(torch.bool).reshape(-1)
    if keep.shape[0] != v.shape[0]:
        raise ValueError("remove_vertices_by_mask: the mask must have one entry per vertex")
    vmap = torch.cumsum(keep.to(torch.int64), 0) - 1
    vmap = torch.where(keep, vmap, torch.full_like(vmap, -1))
    mt = vmap[t]
    mt = mt[(mt >= 0).all(dim=1)]
    pick = lambda a: None if a is None else torch.as_tensor(a).to(dev).to(torch.float64).reshape(-1, 3)[keep]
    return v[keep], mt, pick(vertex_colors), pick(vertex_normals)


def extract_triangle_mesh(volume, with_colors: Optional[bool] = None) -> TriangleMesh:
    """`volume.extract_triangle_mesh()` for a gs2mesh_b200.tsdf.TSDFVolume.  Vertices are in ascending edge key; triangles
    in Open3D's loop order with the volume units visited in lattice order: bricks in ascending lattice index (bx, by, bz),
    inside a brick cubes in pool-layout order x*256 + y*16 + z, inside a cube the case table's triangles."""
    dev = volume.device
    L = _lib.lib()
    with_colors = (volume.color is not None) if with_colors is None else with_colors
    with torch.cuda.device(dev):
        stream = _lib.stream(dev)
        nb = volume.num_bricks()  # every brick ever opened = pool slots [0, nb)
        if nb == 0:
            return TriangleMesh(np.zeros((0, 3)), np.zeros((0, 3), np.int64), np.zeros((0, 3)) if with_colors else None,
                                device=dev)
        # edge keys are voxel indices inside the bounding box of the open bricks (+1: a cube reaches into its +1 neighbours)
        idx = volume._index[:nb, :3].to(torch.int64)
        lo_t = idx.min(dim=0).values
        n_t = idx.max(dim=0).values - lo_t + 2
        lo, n = lo_t.cpu().numpy(), n_t.cpu().numpy()
        window = (C.c_int32 * 6)(*[int(v) for v in lo], *[int(v) for v in n])
        # bricks in ascending lattice index, not in pool order: triangles come out brick after brick in this order, so the
        # mesh does not depend on the order the pool handed out its slots in
        rel = idx - lo_t
        bricks = torch.sort((rel[:, 0] * n_t[1] + rel[:, 1]) * n_t[2] + rel[:, 2]).indices.to(torch.int32)
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
        mesh.key_window = (tuple(int(v) for v in lo), tuple(int(v) for v in n))  # (brick origin, brick count)
    return mesh


class PointCloud:
    """Minimal stand-in for open3d.geometry.PointCloud: fp64 points, colours and normals as host arrays (None when
    absent)."""

    def __init__(self, points, colors=None, normals=None, device=None):
        self.device = None if device is None else torch.device(device)
        self.points = np.asarray(points, dtype=np.float64).reshape(-1, 3)
        self.colors = None if colors is None else np.asarray(colors, dtype=np.float64).reshape(-1, 3)
        self.normals = None if normals is None else np.asarray(normals, dtype=np.float64).reshape(-1, 3)

    # Open3D: non-empty, one entry per point
    def has_colors(self):
        return len(self.points) > 0 and self.colors is not None and len(self.colors) == len(self.points)

    def has_normals(self):
        return len(self.points) > 0 and self.normals is not None and len(self.normals) == len(self.points)

    def scale(self, scale, center=(0, 0, 0)):
        c = np.asarray(center, dtype=np.float64)
        self.points = (self.points - c) * float(scale) + c
        return self

    # -- PointCloud::RemoveStatisticalOutliers / RemoveRadiusOutliers / ClusterDBSCAN / SelectByIndex / VoxelDownSample /
    # UniformDownSample / ComputeNearestNeighborDistance / ComputePointCloudDistance (DESIGN.md section 7, "Point-cloud
    # cleaning and downsampling" and "Density clustering"; gs2mesh_b200/pointcloud.py).  Each runs on `self.device` (the
    # current CUDA device for a cloud built from host arrays), returns a new cloud of the same class holding host arrays
    # with that device set, or host values, and leaves the cloud unchanged; colours and normals travel with their points.
    # ValueError for non-finite points, a colour or normal array without one row per point, or 2^31 points or more.
    def remove_statistical_outlier(self, nb_neighbors, std_ratio, print_progress=False):
        """(cloud, int64 indices ascending): keeps point i iff its mean distance m_i to its nb_neighbors nearest points
        (itself included) satisfies 0 < m_i < mean + std_ratio * std of the positive m_i over the cloud's n points."""
        return _pcd.remove_statistical_outlier(self, nb_neighbors, std_ratio)

    def remove_radius_outlier(self, nb_points, radius, print_progress=False):
        """(cloud, int64 indices ascending): keeps point i iff more than nb_points points (itself included) lie at squared
        distance strictly below radius * radius."""
        return _pcd.remove_radius_outlier(self, nb_points, radius)

    def cluster_dbscan(self, eps, min_points, print_progress=False):
        """int32 numpy (n,): DBSCAN cluster labels, numbered by each cluster's smallest core point index, -1 for noise
        (DESIGN.md section 7, "Density clustering")."""
        return _pcd.cluster_dbscan(self, eps, min_points)

    def select_by_index(self, indices, invert=False):
        """The points at `indices` (or, with invert, the others) in ascending index order, each once."""
        return _pcd.select_by_index(self, indices, invert)

    def voxel_down_sample(self, voxel_size):
        """The mean point, colour and normal of each occupied voxel, in ascending (x, y, z) voxel order."""
        return _pcd.voxel_down_sample(self, voxel_size)

    def uniform_down_sample(self, every_k_points):
        """Points 0, k, 2k, ... with their colours and normals."""
        return _pcd.uniform_down_sample(self, every_k_points)

    def compute_nearest_neighbor_distance(self):
        """fp64 numpy (n,): each point's distance to its nearest other point."""
        return _pcd.compute_nearest_neighbor_distance(self)

    def compute_point_cloud_distance(self, target):
        """fp64 numpy (n,): each point's distance to the nearest point of `target`."""
        return _pcd.compute_point_cloud_distance(self, target)

    # -- o3d.io.write_point_cloud(path, pcd): binary little-endian PLY, double coordinates and normals, uchar colours
    def write_ply(self, path):
        return write_point_cloud_ply(path, self.points, self.colors, self.normals)


def _extract_cloud(volume, mode, with_colors, with_normals):
    """The sorted keys of `volume`'s cloud and their attributes: count -> scan -> emit -> sort -> points."""
    dev = volume.device
    L = _lib.lib()
    empty = lambda on: np.zeros((0, 3)) if on else None
    with torch.cuda.device(dev):
        stream = _lib.stream(dev)
        nb = volume.num_bricks()  # every brick ever opened = pool slots [0, nb)
        if nb == 0:
            return PointCloud(np.zeros((0, 3)), empty(with_colors), empty(with_normals), device=dev)
        bricks = torch.arange(nb, dtype=torch.int32, device=dev)
        # the key window of extract_triangle_mesh: the bounding box of the open bricks and their +1 neighbours
        idx = volume._index[:nb, :3]
        lo = idx.min(dim=0).values.cpu().numpy().astype(np.int64)
        hi = idx.max(dim=0).values.cpu().numpy().astype(np.int64)
        window = (C.c_int32 * 6)(*[int(v) for v in lo], *[int(v) for v in (hi - lo + 2)])
        counts = torch.zeros(nb, dtype=torch.int32, device=dev)
        _lib.check(L.gsb_pcd_count(volume._h, window, ptr(bricks), nb, mode, ptr(counts), stream))
        offsets = torch.cumsum(counts.to(torch.int64), 0) - counts.to(torch.int64)
        n = int(counts.sum().item())
        key_window = (tuple(int(v) for v in lo), tuple(int(v) for v in (hi - lo + 2)))
        if n == 0:
            pcd = PointCloud(np.zeros((0, 3)), empty(with_colors), empty(with_normals), device=dev)
            pcd.keys, pcd.key_window = np.zeros(0, np.int64), key_window
            return pcd
        keys = torch.empty(n, dtype=torch.int64, device=dev)
        _lib.check(L.gsb_pcd_emit(volume._h, window, ptr(bricks), nb, mode, ptr(offsets.contiguous()), ptr(keys), stream))
        keys = torch.sort(keys).values  # every key has one owner brick: no duplicates to remove
        xyz = torch.empty(n, 3, dtype=torch.float64, device=dev)
        rgb = torch.empty(n, 3, dtype=torch.float64, device=dev) if with_colors else None
        nrm = torch.empty(n, 3, dtype=torch.float64, device=dev) if with_normals else None
        _lib.check(L.gsb_pcd_points(volume._h, window, ptr(keys), n, mode, ptr(xyz), ptr(rgb), ptr(nrm), stream))
        host = lambda t: None if t is None else t.cpu().numpy()
        pcd = PointCloud(host(xyz), host(rgb), host(nrm), device=dev)
        pcd.keys = keys.cpu().numpy()  # window voxel index (* 3 + axis for the surface cloud) per point, for tests
        pcd.key_window = key_window  # (brick origin, brick count)
    return pcd


def extract_point_cloud(volume, with_colors: Optional[bool] = None, with_normals: bool = True) -> PointCloud:
    """`volume.extract_point_cloud()` for a gs2mesh_b200.tsdf.TSDFVolume: Open3D's ScalableTSDFVolume::ExtractPointCloud,
    the zero crossings of the TSDF along the lattice axes with interpolated colours and TSDF-gradient normals, in
    ascending edge key (window voxel index * 3 + axis)."""
    with_colors = (volume.color is not None) if with_colors is None else bool(with_colors)
    if with_colors and volume.color is None:
        raise ValueError("extract_point_cloud: the volume has no colour")
    return _extract_cloud(volume, _lib.GSB_PCD_SURFACE, with_colors, bool(with_normals))


def extract_voxel_point_cloud(volume) -> PointCloud:
    """`volume.extract_voxel_point_cloud()`: Open3D's ScalableTSDFVolume::ExtractVoxelPointCloud, the centre of every
    voxel with weight != 0 and -0.98 <= tsdf < 0.98, grey (tsdf + 1) / 2, in ascending window voxel index."""
    return _extract_cloud(volume, _lib.GSB_PCD_VOXELS, True, False)
