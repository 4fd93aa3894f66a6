// Mesh extraction from the brick TSDF volume: `volume.extract_triangle_mesh()` of
// gs2mesh_utils/tsdf_utils.py:108, i.e. Open3D 0.17.0 ScalableTSDFVolume::ExtractTriangleMesh
// (SURVEY.md row T3), plus the vertex normals of tsdf_utils.py:110.
//
// Open3D walks every voxel of every allocated volume unit serially, looks the 8 cube corners up
// (through the hash map when they fall into a neighbouring unit), skips the cube if ANY corner has
// weight 0, classifies corners with `tsdf < 0`, and de-duplicates vertices by (global voxel, axis).
// Here: one CTA per touched brick stages the brick plus its +1 halo (17^3 (tsdf, weight) pairs)
// in shared memory; a count pass and an emit pass write three 64-bit edge keys per triangle
// (key = global voxel index * 3 + axis); the caller uniques the keys (vertex ids) and a vertex
// kernel evaluates positions / colours per unique edge in fp64 with Open3D's formulas.
// Triangle order: the caller lists the bricks in ascending lattice index; the emit pass places a brick's triangles by a
// block-wide scan of the per-cube counts, so cubes follow in pool-layout order x*256 + y*16 + z and each cube's triangles
// in the case table's order.  The mesh therefore does not depend on pool order or on warp scheduling.
//
// Cluster cleaning (tsdf_utils.py:122-142, TriangleMesh::ClusterConnectedTriangles + removal of small clusters and
// unreferenced vertices): triangles sharing an edge are grouped by a radix sort of 64-bit edge keys, joined by a
// lock-free union-find whose roots are the smallest triangle of each cluster, and numbered by an exclusive scan of the
// root flags -- the order Open3D's BFS loop and scipy's connected_components number them in.
#include <cub/cub.cuh>
#include <cuda/atomic>

#include "gs2mesh_b200.h"
#include "gsb_common.h"
#include "gsb_mc_tables.h"
#include "gsb_union_find.cuh"
#include "gsb_volume_view.cuh"


namespace gsb {
namespace {

constexpr int kHalo = GSB_BRICK + 1;  // 17

__device__ __forceinline__ int cube_case(const float2* s, int x, int y, int z) {
  int c = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float2 v = s[((x + kMcShift[i][0]) * kHalo + (y + kMcShift[i][1])) * kHalo + (z + kMcShift[i][2])];
    if (v.y == 0.0f) return 0;  // any corner never observed: no surface here
    if (v.x < 0.0f) c |= 1 << i;
  }
  return c == 255 ? 0 : c;
}

constexpr int kMcThreads = 256;
using McScan = cub::BlockScan<uint32_t, kMcThreads>;

// mode 0: tri_counts[b] = number of triangles of brick b.  mode 1: write the edge keys, cube i's triangles after those of
// cubes 0 .. i-1 of the brick.  Launched with kMcThreads threads: each of the 16 rounds covers cubes [256k, 256k + 256).
__global__ void __launch_bounds__(kMcThreads) mc_brick_kernel(const VolView v, const uint32_t* __restrict__ bricks, int mode,
                                                              uint32_t* __restrict__ tri_counts,
                                                              const long long* __restrict__ tri_offsets,
                                                              long long* __restrict__ edge_keys) {
  __shared__ float2 s[kHalo * kHalo * kHalo];
  __shared__ uint32_t s_count;
  __shared__ uint32_t s_nb[8];  // pool slots of the brick and its +1 neighbours (bit 2: x+1, bit 1: y+1, bit 0: z+1)
  __shared__ McScan::TempStorage s_scan;
  const uint32_t brick = bricks[blockIdx.x];
  const int4 bi = v.index[brick];
  // window-relative brick coordinates (the edge keys are relative to the key window)
  const int bx = bi.x - v.b0[0], by = bi.y - v.b0[1], bz = bi.z - v.b0[2];
  if (threadIdx.x == 0) s_count = 0;
  if (threadIdx.x < 8)
    s_nb[threadIdx.x] = threadIdx.x == 0 ? brick
                                         : slot_of_brick(v, bi.x + ((threadIdx.x >> 2) & 1), bi.y + ((threadIdx.x >> 1) & 1),
                                                         bi.z + (threadIdx.x & 1));
  __syncthreads();
  for (int i = threadIdx.x; i < kHalo * kHalo * kHalo; i += blockDim.x) {
    const int z = i % kHalo, y = (i / kHalo) % kHalo, x = i / (kHalo * kHalo);
    const uint32_t slot = s_nb[((x >> 4) << 2) | ((y >> 4) << 1) | (z >> 4)];
    s[i] = slot == kSlotNone ? make_float2(0.f, 0.f)
                             : v.tw[(size_t)slot * GSB_BRICK_VOXELS + ((x & 15) * 16 + (y & 15)) * 16 + (z & 15)];
  }
  __syncthreads();
  long long base = mode ? tri_offsets[blockIdx.x] : 0;  // emit: where this round's first triangle goes
  const long long NY = (long long)v.nb[1] * GSB_BRICK, NZ = (long long)v.nb[2] * GSB_BRICK;
  for (int i = threadIdx.x; i < GSB_BRICK_VOXELS; i += kMcThreads) {
    const int z = i & 15, y = (i >> 4) & 15, x = i >> 8;
    const int c = cube_case(s, x, y, z);
    int ntri = 0;
    while (ntri < 5 && kMcTriTable[c][3 * ntri] >= 0) ++ntri;
    if (mode == 0) {
      if (ntri) atomicAdd(&s_count, (uint32_t)ntri);  // an integer sum: the same whatever the order
    } else {
      uint32_t slot, round_total;
      McScan(s_scan).ExclusiveSum((uint32_t)ntri, slot, round_total);
      for (int t = 0; t < ntri; ++t) {
        // Open3D pushes (e0, e2, e1): ScalableTSDFVolume.cpp ExtractTriangleMesh
        const int order[3] = {0, 2, 1};
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          const int e = kMcTriTable[c][3 * t + order[k]];
          const long long gx = bx * 16 + x + kMcEdgeShift[e][0], gy = by * 16 + y + kMcEdgeShift[e][1],
                          gz = bz * 16 + z + kMcEdgeShift[e][2];
          edge_keys[3 * (base + slot + t) + k] = ((gx * NY + gy) * NZ + gz) * 3 + kMcEdgeShift[e][3];
        }
      }
      base += round_total;
      __syncthreads();  // s_scan is reused by the next round
    }
  }
  __syncthreads();
  if (mode == 0 && threadIdx.x == 0) tri_counts[blockIdx.x] = s_count;
}

// One unique edge -> vertex position and colour, fp64 with one rounding per operation in Open3D's order (no FMA
// contraction, no reciprocal), so both equal Open3D's doubles bit for bit:
//   pt(k) = half_voxel_length + voxel_length * index(k);  pt(axis) += f0 * voxel_length / (f0 + f1)
//   colour = (f1 * c0 + f0 * c1) / (f0 + f1),  c = voxel colour / 255.0
__global__ void __launch_bounds__(256) mc_vertices_kernel(const VolView v, const long long* __restrict__ keys, long long n,
                                                          double* __restrict__ xyz, double* __restrict__ rgb) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const long long NY = (long long)v.nb[1] * GSB_BRICK, NZ = (long long)v.nb[2] * GSB_BRICK;
  const long long key = keys[i];
  const int axis = (int)(key % 3);
  long long lin = key / 3;
  const int gz = (int)(lin % NZ);
  lin /= NZ;
  const int gy = (int)(lin % NY);
  const int gx = (int)(lin / NY);
  const int dx = axis == 0, dy = axis == 1, dz = axis == 2;
  const float2 a = load_voxel(v, gx, gy, gz), b = load_voxel(v, gx + dx, gy + dy, gz + dz);
  const double f0 = fabs((double)a.x), f1 = fabs((double)b.x);
  const double vl = v.voxel_length, half = __dmul_rn(vl, 0.5), sum = __dadd_rn(f0, f1);
  // global (lattice) voxel index = window origin + window-relative index
  double p[3] = {__dadd_rn(half, __dmul_rn(vl, (double)(v.b0[0] * GSB_BRICK + gx))),
                 __dadd_rn(half, __dmul_rn(vl, (double)(v.b0[1] * GSB_BRICK + gy))),
                 __dadd_rn(half, __dmul_rn(vl, (double)(v.b0[2] * GSB_BRICK + gz)))};
  p[axis] = __dadd_rn(p[axis], __ddiv_rn(__dmul_rn(f0, vl), sum));
  xyz[3 * i] = p[0];
  xyz[3 * i + 1] = p[1];
  xyz[3 * i + 2] = p[2];
  if (rgb != nullptr && v.color != nullptr) {
    const size_t ia = voxel_address(v, gx, gy, gz), ib = voxel_address(v, gx + dx, gy + dy, gz + dz);
    const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
    const float4 c0 = ia == (size_t)-1 ? zero : v.color[ia], c1 = ib == (size_t)-1 ? zero : v.color[ib];
    const float k0[3] = {c0.x, c0.y, c0.z}, k1[3] = {c1.x, c1.y, c1.z};
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const double w0 = __dmul_rn(f1, __ddiv_rn((double)k0[k], 255.0)), w1 = __dmul_rn(f0, __ddiv_rn((double)k1[k], 255.0));
      rgb[3 * i + k] = __ddiv_rn(__dadd_rn(w0, w1), sum);
    }
  }
}

// Vertex normals of TriangleMesh::ComputeVertexNormals(normalized=true), bit for bit and run to run.  Open3D sums the
// unnormalised triangle normals (v1-v0).cross(v2-v0) into each vertex of triangle 0, 1, 2, ... in turn, then calls
// MeshBase::NormalizeNormals().  One thread per vertex walks its incidences (positions 3*t+k of the flattened triangle
// array, in ascending order) and adds them in that same order, one rounding per operation -- no atomics, so the sum
// does not depend on scheduling.  NormalizeNormals() is Eigen's normalize(), which (Eigen >= 3.3, MatrixBase::normalize
// in Dot.h) divides by sqrt(squaredNorm()) only if squaredNorm() > 0, followed by Open3D's `isnan(n(0))` -> (0,0,1);
// a zero sum therefore stays (0,0,0).  squaredNorm() of a Vector3d is Eigen's vectorised redux: (x*x + y*y) + z*z.
__global__ void __launch_bounds__(256) mesh_vertex_normals_kernel(const double* __restrict__ xyz,
                                                                  const long long* __restrict__ tris,
                                                                  const long long* __restrict__ incidence,
                                                                  const long long* __restrict__ offsets, long long nv,
                                                                  double* __restrict__ normals) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nv) return;
  double sx = 0.0, sy = 0.0, sz = 0.0;
  for (long long j = offsets[i], end = offsets[i + 1]; j < end; ++j) {
    const long long t = incidence[j] / 3;
    const long long i0 = tris[3 * t], i1 = tris[3 * t + 1], i2 = tris[3 * t + 2];
    const double x0 = xyz[3 * i0], y0 = xyz[3 * i0 + 1], z0 = xyz[3 * i0 + 2];
    const double ax = __dsub_rn(xyz[3 * i1], x0), ay = __dsub_rn(xyz[3 * i1 + 1], y0), az = __dsub_rn(xyz[3 * i1 + 2], z0);
    const double bx = __dsub_rn(xyz[3 * i2], x0), by = __dsub_rn(xyz[3 * i2 + 1], y0), bz = __dsub_rn(xyz[3 * i2 + 2], z0);
    sx = __dadd_rn(sx, __dsub_rn(__dmul_rn(ay, bz), __dmul_rn(az, by)));
    sy = __dadd_rn(sy, __dsub_rn(__dmul_rn(az, bx), __dmul_rn(ax, bz)));
    sz = __dadd_rn(sz, __dsub_rn(__dmul_rn(ax, by), __dmul_rn(ay, bx)));
  }
  const double sq = __dadd_rn(__dadd_rn(__dmul_rn(sx, sx), __dmul_rn(sy, sy)), __dmul_rn(sz, sz));
  if (sq > 0.0) {
    const double len = __dsqrt_rn(sq);
    sx = __ddiv_rn(sx, len);
    sy = __ddiv_rn(sy, len);
    sz = __ddiv_rn(sz, len);
  }
  if (isnan(sx)) {
    sx = 0.0;
    sy = 0.0;
    sz = 1.0;
  }
  normals[3 * i] = sx;
  normals[3 * i + 1] = sy;
  normals[3 * i + 2] = sz;
}

// ---------------------------------------------------------------------------------------------------------------------
// Edge-connected triangle clusters: the union-find of gsb_union_find.cuh over triangle ids, so the surviving root of a
// cluster is its smallest triangle.
// ---------------------------------------------------------------------------------------------------------------------
// Three (key, triangle) pairs per triangle, edges (a,b), (b,c), (c,a) in that order; key = min*(n_vertices+1) + max,
// the host's key (mesh.py) and Open3D's GetEdgeToTrianglesMap.  Degenerate edges (a,a) get keys like any other.
__global__ void __launch_bounds__(256) cluster_edge_keys_kernel(const long long* __restrict__ tris, int nt,
                                                                unsigned long long stride, unsigned long long* __restrict__ keys,
                                                                uint32_t* __restrict__ owner, int* __restrict__ parent) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nt) return;
  const long long v[3] = {tris[3 * (size_t)t], tris[3 * (size_t)t + 1], tris[3 * (size_t)t + 2]};
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    keys[(size_t)k * nt + t] = edge_key(v[k], v[(k + 1) % 3], stride);
    owner[(size_t)k * nt + t] = (uint32_t)t;
  }
  parent[t] = t;
}

// Neighbours in the sorted key array with equal keys share an edge: joining each with its predecessor joins every run.
__global__ void __launch_bounds__(256) cluster_union_kernel(const unsigned long long* __restrict__ keys,
                                                            const uint32_t* __restrict__ owner, long long n, int* parent) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x + 1;
  if (i >= n || keys[i] != keys[i - 1]) return;
  uf_union(parent, (int)owner[i], (int)owner[i - 1]);
}

// After every hook: parent[t] = its root, root_flag[t] = 1 for the roots.  The walk here does not halve: a halving
// store into parent[x] could land after thread x wrote its root there and leave x pointing at a non-root.  Each
// parent[t] is written once, by thread t, and every value a walk can read is an ancestor, so every walk ends at the root.
__global__ void __launch_bounds__(256) cluster_compress_kernel(int* parent, int nt, int* __restrict__ root_flag) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nt) return;
  int r = t, p = uf_load(parent, t);
  while (p != r) {
    r = p;
    p = uf_load(parent, r);
  }
  ParentRef(parent[t]).store(r, cuda::memory_order_relaxed);
  root_flag[t] = r == t;
}

// label[t] = the rank of t's root among the roots (clusters numbered by their smallest triangle); counts by integer
// atomics (exact, so the same on every run); the last thread writes the number of clusters.
__global__ void __launch_bounds__(256) cluster_label_kernel(const int* __restrict__ parent, const int* __restrict__ root_flag,
                                                            const int* __restrict__ rank, int nt, long long* __restrict__ labels,
                                                            unsigned long long* counts, long long* __restrict__ n_clusters,
                                                            uint32_t* __restrict__ label32) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nt) return;
  const int l = rank[parent[t]];
  labels[t] = l;
  if (label32) label32[t] = (uint32_t)l;
  atomicAdd(&counts[l], 1ull);
  if (t == nt - 1) *n_clusters = (long long)rank[t] + root_flag[t];
}

// 0.5 * ||(v1-v0) x (v2-v0)|| with numpy's roundings: np.cross computes each component as one product minus another,
// np.linalg.norm(axis=1) as sqrt((x*x + y*y) + z*z); no FMA contraction.
__global__ void __launch_bounds__(256) triangle_area_kernel(const double* __restrict__ xyz, const long long* __restrict__ tris,
                                                            int nt, double* __restrict__ area) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nt) return;
  const long long i0 = tris[3 * (size_t)t], i1 = tris[3 * (size_t)t + 1], i2 = tris[3 * (size_t)t + 2];
  const double x0 = xyz[3 * i0], y0 = xyz[3 * i0 + 1], z0 = xyz[3 * i0 + 2];
  const double ax = __dsub_rn(xyz[3 * i1], x0), ay = __dsub_rn(xyz[3 * i1 + 1], y0), az = __dsub_rn(xyz[3 * i1 + 2], z0);
  const double bx = __dsub_rn(xyz[3 * i2], x0), by = __dsub_rn(xyz[3 * i2 + 1], y0), bz = __dsub_rn(xyz[3 * i2 + 2], z0);
  const double cx = __dsub_rn(__dmul_rn(ay, bz), __dmul_rn(az, by));
  const double cy = __dsub_rn(__dmul_rn(az, bx), __dmul_rn(ax, bz));
  const double cz = __dsub_rn(__dmul_rn(ax, by), __dmul_rn(ay, bx));
  area[t] = __dmul_rn(0.5, __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(cx, cx), __dmul_rn(cy, cy)), __dmul_rn(cz, cz))));
}

// One warp per cluster sums its triangles' areas (sorted by label, ascending triangle id inside a label) in a fixed
// order: lane-strided partial sums, then a fixed butterfly.  No floating-point atomics, so the bits repeat run to run.
__global__ void __launch_bounds__(256) cluster_area_sum_kernel(const double* __restrict__ sorted_area,
                                                               const long long* __restrict__ offsets,
                                                               const unsigned long long* __restrict__ counts, int nt,
                                                               double* __restrict__ cluster_area) {
  const long long c = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (c >= nt) return;
  const long long begin = offsets[c], n = (long long)counts[c];
  double s = 0.0;
  for (long long j = lane; j < n; j += 32) s = __dadd_rn(s, sorted_area[begin + j]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s = __dadd_rn(s, __shfl_xor_sync(0xffffffffu, s, o));
  if (lane == 0) cluster_area[c] = s;
}

// keep[t] = !(counts[labels[t]] < threshold), the comparison numpy makes between int64 counts and a float threshold.
__global__ void __launch_bounds__(256) cluster_keep_kernel(const long long* __restrict__ labels,
                                                           const long long* __restrict__ counts, int nt, double threshold,
                                                           int* __restrict__ keep) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nt) return;
  keep[t] = !((double)counts[labels[t]] < threshold);
}

__global__ void __launch_bounds__(256) mark_referenced_kernel(const long long* __restrict__ tris, const int* __restrict__ keep,
                                                              int nt, int* __restrict__ referenced) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nt || !keep[t]) return;
#pragma unroll
  for (int k = 0; k < 3; ++k) referenced[tris[3 * (size_t)t + k]] = 1;
}

__global__ void __launch_bounds__(256) remap_triangles_kernel(const long long* __restrict__ tris, const int* __restrict__ keep,
                                                              const int* __restrict__ tri_pos, const int* __restrict__ new_id,
                                                              int nt, long long* __restrict__ out_tris) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nt || !keep[t]) return;
  const size_t o = 3 * (size_t)tri_pos[t];
#pragma unroll
  for (int k = 0; k < 3; ++k) out_tris[o + k] = new_id[tris[3 * (size_t)t + k]];
}

__global__ void __launch_bounds__(256) kept_vertices_kernel(const int* __restrict__ referenced, const int* __restrict__ new_id,
                                                            int nv, long long* __restrict__ vertex_ids) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v < nv && referenced[v]) vertex_ids[new_id[v]] = v;
}

__global__ void clean_sizes_kernel(const int* __restrict__ keep, const int* __restrict__ tri_pos, int nt,
                                   const int* __restrict__ referenced, const int* __restrict__ new_id, int nv,
                                   long long* __restrict__ sizes) {
  sizes[0] = nt ? (long long)tri_pos[nt - 1] + keep[nt - 1] : 0;
  sizes[1] = nv ? (long long)new_id[nv - 1] + referenced[nv - 1] : 0;
}

// Workspace layout of the two cluster entries (each carves its own regions from the start of the block); with a NULL
// base only `total` is meaningful.
struct ClusterWork {
  unsigned long long* keys;  // [2][3 nt] edge keys (DoubleBuffer); later [2 nt] sorted-by-label areas + [nt] offsets
  uint32_t* owner;           // [2][3 nt] triangle of each key (DoubleBuffer); later [2 nt] labels as sort keys
  int* parent;               // [nt]
  int* flag;                 // [nt]
  int* rank;                 // [nt]
  void* tmp;
  size_t tmp_bytes, total;
};
struct CleanWork {
  int *keep, *tri_pos, *referenced, *new_id;  // [nt], [nt], [nv], [nv]
  void* tmp;
  size_t tmp_bytes, total;
};

size_t cub_tmp_bytes(int64_t nt, int64_t nv) {
  const long long n3 = 3 * nt;
  size_t a = 0, b = 0, c = 0, d = 0, e = 0;
  cub::DoubleBuffer<unsigned long long> k(nullptr, nullptr);
  cub::DoubleBuffer<uint32_t> o(nullptr, nullptr);
  cub::DeviceRadixSort::SortPairs(nullptr, a, k, o, n3);
  cub::DoubleBuffer<uint32_t> lk(nullptr, nullptr);
  cub::DoubleBuffer<double> av(nullptr, nullptr);
  cub::DeviceRadixSort::SortPairs(nullptr, b, lk, av, (long long)nt);
  cub::DeviceScan::ExclusiveSum(nullptr, c, (int*)nullptr, (int*)nullptr, (long long)nt);
  cub::DeviceScan::ExclusiveSum(nullptr, d, (int*)nullptr, (int*)nullptr, (long long)nv);
  cub::DeviceScan::ExclusiveSum(nullptr, e, (unsigned long long*)nullptr, (long long*)nullptr, (long long)nt);
  size_t m = a;
  for (size_t x : {b, c, d, e}) m = x > m ? x : m;
  return m;
}

ClusterWork carve_cluster(void* base, int64_t nt, int64_t nv) {
  Carver c(base);
  ClusterWork w;
  w.keys = c.take<unsigned long long>(6 * (size_t)nt);
  w.owner = c.take<uint32_t>(6 * (size_t)nt);
  w.parent = c.take<int>((size_t)nt);
  w.flag = c.take<int>((size_t)nt);
  w.rank = c.take<int>((size_t)nt);
  w.tmp_bytes = cub_tmp_bytes(nt, nv);
  w.tmp = c.take<char>(w.tmp_bytes);
  w.total = c.total();
  return w;
}

CleanWork carve_clean(void* base, int64_t nt, int64_t nv) {
  Carver c(base);
  CleanWork w;
  w.keep = c.take<int>((size_t)nt);
  w.tri_pos = c.take<int>((size_t)nt);
  w.referenced = c.take<int>((size_t)nv);
  w.new_id = c.take<int>((size_t)nv);
  w.tmp_bytes = cub_tmp_bytes(nt, nv);
  w.tmp = c.take<char>(w.tmp_bytes);
  w.total = c.total();
  return w;
}

}  // namespace
}  // namespace gsb

using namespace gsb;

extern "C" {

int gsb_mesh_count(const GsbVolume* vol, const int32_t* window, const uint32_t* bricks, uint32_t n_bricks, uint32_t* tri_counts,
                   void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (!vol || (n_bricks && (!bricks || !tri_counts))) return fail(GSB_ERR_INVALID, "mesh_count: bad arguments");
  if (const int rc = window_check("mesh_count", window)) return rc;
  if (n_bricks == 0) return GSB_OK;
  mc_brick_kernel<<<n_bricks, kMcThreads, 0, stream>>>(view_of(vol, window), bricks, 0, tri_counts, nullptr, nullptr);
  count_launch();
  return check_launch("mc_brick_kernel(count)", stream, false);
}

int gsb_mesh_emit(const GsbVolume* vol, const int32_t* window, const uint32_t* bricks, uint32_t n_bricks, const int64_t* tri_offsets,
                  int64_t* edge_keys, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (!vol || (n_bricks && (!bricks || !tri_offsets || !edge_keys))) return fail(GSB_ERR_INVALID, "mesh_emit: bad arguments");
  if (const int rc = window_check("mesh_emit", window)) return rc;
  if (n_bricks == 0) return GSB_OK;
  mc_brick_kernel<<<n_bricks, kMcThreads, 0, stream>>>(view_of(vol, window), bricks, 1, nullptr, reinterpret_cast<const long long*>(tri_offsets),
                                                reinterpret_cast<long long*>(edge_keys));
  count_launch();
  return check_launch("mc_brick_kernel(emit)", stream, false);
}

int gsb_mesh_vertices(const GsbVolume* vol, const int32_t* window, const int64_t* keys, int64_t n, double* xyz, double* rgb,
                      void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (!vol || n < 0 || (n && (!keys || !xyz))) return fail(GSB_ERR_INVALID, "mesh_vertices: bad arguments");
  if (const int rc = window_check("mesh_vertices", window)) return rc;
  if (n == 0) return GSB_OK;
  mc_vertices_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(view_of(vol, window), reinterpret_cast<const long long*>(keys),
                                                                     n, xyz, rgb);
  count_launch();
  return check_launch("mc_vertices_kernel", stream, false);
}

int gsb_mesh_vertex_normals(const double* xyz, int64_t n_vertices, const int64_t* triangles, int64_t n_triangles,
                            const int64_t* incidence, const int64_t* incidence_offsets, double* normals, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (n_vertices < 0 || n_triangles < 0 || (n_vertices && (!xyz || !normals || !incidence_offsets)) ||
      (n_triangles && (!triangles || !incidence)))
    return fail(GSB_ERR_INVALID, "mesh_vertex_normals: bad arguments");
  if (n_vertices == 0) return GSB_OK;
  mesh_vertex_normals_kernel<<<(unsigned)((n_vertices + 255) / 256), 256, 0, stream>>>(
      xyz, reinterpret_cast<const long long*>(triangles), reinterpret_cast<const long long*>(incidence),
      reinterpret_cast<const long long*>(incidence_offsets), n_vertices, normals);
  count_launch();
  return check_launch("mesh_vertex_normals_kernel", stream, false);
}

size_t gsb_mesh_cluster_workspace_bytes(int64_t n_triangles, int64_t n_vertices) {
  if (!mesh_sizes_ok(n_triangles, n_vertices, kMaxMeshIds)) return 0;
  const size_t a = carve_cluster(nullptr, n_triangles, n_vertices).total, b = carve_clean(nullptr, n_triangles, n_vertices).total;
  return a > b ? a : b;
}

int gsb_mesh_clusters(const int64_t* triangles, int64_t n_triangles, int64_t n_vertices, const double* vertices, void* workspace,
                      size_t workspace_bytes, int64_t* labels, int64_t* counts, int64_t* n_clusters, double* cluster_area,
                      void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (!mesh_sizes_ok(n_triangles, n_vertices, kMaxMeshIds))
    return mesh_size_error("mesh_clusters", n_triangles, n_vertices, kMaxMeshIds);
  if (!n_clusters || (n_triangles && (!triangles || !workspace || !labels || !counts || (cluster_area && !vertices))))
    return fail(GSB_ERR_INVALID, "mesh_clusters: bad arguments");
  if (n_triangles == 0) {
    GSB_CUDA_OK(cudaMemsetAsync(n_clusters, 0, sizeof(int64_t), stream));
    return GSB_OK;
  }
  const size_t need = gsb_mesh_cluster_workspace_bytes(n_triangles, n_vertices);
  if (workspace_bytes < need) return fail(GSB_ERR_WORKSPACE, "mesh_clusters: workspace %zu < %zu bytes", workspace_bytes, need);
  const int nt = (int)n_triangles;
  const long long n3 = 3 * (long long)nt;
  const ClusterWork w = carve_cluster(workspace, n_triangles, n_vertices);
  const auto* tris = reinterpret_cast<const long long*>(triangles);
  const unsigned long long stride = (unsigned long long)n_vertices + 1;
  const int key_bits = bits_of(stride * stride - 1);  // keys < (n_vertices+1)^2 <= 2^62: 32-bit ids

  cluster_edge_keys_kernel<<<blocks_for(nt), 256, 0, stream>>>(tris, nt, stride, w.keys, w.owner, w.parent);
  count_launch();
  cub::DoubleBuffer<unsigned long long> keys(w.keys, w.keys + n3);
  cub::DoubleBuffer<uint32_t> owner(w.owner, w.owner + n3);
  size_t tmp_bytes = w.tmp_bytes;
  GSB_CUDA_OK(cub::DeviceRadixSort::SortPairs(w.tmp, tmp_bytes, keys, owner, n3, 0, key_bits, stream));
  if (n3 > 1) {
    cluster_union_kernel<<<blocks_for(n3 - 1), 256, 0, stream>>>(keys.Current(), owner.Current(), n3, w.parent);
    count_launch();
  }
  cluster_compress_kernel<<<blocks_for(nt), 256, 0, stream>>>(w.parent, nt, w.flag);
  count_launch();
  tmp_bytes = w.tmp_bytes;
  GSB_CUDA_OK(cub::DeviceScan::ExclusiveSum(w.tmp, tmp_bytes, w.flag, w.rank, (long long)nt, stream));
  auto* ucounts = reinterpret_cast<unsigned long long*>(counts);
  GSB_CUDA_OK(cudaMemsetAsync(counts, 0, sizeof(int64_t) * (size_t)nt, stream));
  // the edge sort's buffers are free from here on: labels as sort keys in `owner`, areas and offsets in `keys`
  uint32_t* label32 = cluster_area ? w.owner : nullptr;
  cluster_label_kernel<<<blocks_for(nt), 256, 0, stream>>>(w.parent, w.flag, w.rank, nt, reinterpret_cast<long long*>(labels),
                                                          ucounts, reinterpret_cast<long long*>(n_clusters), label32);
  count_launch();
  if (int rc = check_launch("mesh_clusters", stream, false)) return rc;
  if (!cluster_area) return GSB_OK;

  auto* area = reinterpret_cast<double*>(w.keys);
  auto* offsets = reinterpret_cast<long long*>(w.keys + 2 * (size_t)nt);
  triangle_area_kernel<<<blocks_for(nt), 256, 0, stream>>>(vertices, tris, nt, area);
  count_launch();
  cub::DoubleBuffer<uint32_t> by_label(label32, label32 + nt);
  cub::DoubleBuffer<double> areas(area, area + nt);
  tmp_bytes = w.tmp_bytes;  // a stable sort: each cluster's areas stay in triangle order
  GSB_CUDA_OK(cub::DeviceRadixSort::SortPairs(w.tmp, tmp_bytes, by_label, areas, (long long)nt, 0, bits_of((unsigned long long)nt),
                                              stream));
  tmp_bytes = w.tmp_bytes;
  GSB_CUDA_OK(cub::DeviceScan::ExclusiveSum(w.tmp, tmp_bytes, ucounts, offsets, (long long)nt, stream));
  cluster_area_sum_kernel<<<blocks_for(32 * (long long)nt), 256, 0, stream>>>(areas.Current(), offsets, ucounts, nt, cluster_area);
  count_launch();
  return check_launch("mesh_clusters(area)", stream, false);
}

int gsb_mesh_remove_small_clusters(const int64_t* triangles, int64_t n_triangles, int64_t n_vertices, const int64_t* labels,
                                   const int64_t* counts, double threshold, void* workspace, size_t workspace_bytes,
                                   int64_t* out_triangles, int64_t* vertex_ids, int64_t* sizes, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (!mesh_sizes_ok(n_triangles, n_vertices, kMaxMeshIds))
    return mesh_size_error("mesh_remove_small_clusters", n_triangles, n_vertices, kMaxMeshIds);
  if (!sizes || (n_triangles && (!triangles || !labels || !counts || !out_triangles)) ||
      ((n_triangles || n_vertices) && !workspace) || (n_vertices && !vertex_ids))
    return fail(GSB_ERR_INVALID, "mesh_remove_small_clusters: bad arguments");
  const size_t need = gsb_mesh_cluster_workspace_bytes(n_triangles, n_vertices);
  if ((n_triangles || n_vertices) && workspace_bytes < need)
    return fail(GSB_ERR_WORKSPACE, "mesh_remove_small_clusters: workspace %zu < %zu bytes", workspace_bytes, need);
  const int nt = (int)n_triangles, nv = (int)n_vertices;
  const CleanWork w = carve_clean(workspace, n_triangles, n_vertices);
  const auto* tris = reinterpret_cast<const long long*>(triangles);
  size_t tmp_bytes;
  if (nt) {
    cluster_keep_kernel<<<blocks_for(nt), 256, 0, stream>>>(reinterpret_cast<const long long*>(labels),
                                                           reinterpret_cast<const long long*>(counts), nt, threshold, w.keep);
    count_launch();
    tmp_bytes = w.tmp_bytes;
    GSB_CUDA_OK(cub::DeviceScan::ExclusiveSum(w.tmp, tmp_bytes, w.keep, w.tri_pos, (long long)nt, stream));
  }
  if (nv) {
    GSB_CUDA_OK(cudaMemsetAsync(w.referenced, 0, sizeof(int) * (size_t)nv, stream));
    if (nt) {
      mark_referenced_kernel<<<blocks_for(nt), 256, 0, stream>>>(tris, w.keep, nt, w.referenced);
      count_launch();
    }
    tmp_bytes = w.tmp_bytes;
    GSB_CUDA_OK(cub::DeviceScan::ExclusiveSum(w.tmp, tmp_bytes, w.referenced, w.new_id, (long long)nv, stream));
    kept_vertices_kernel<<<blocks_for(nv), 256, 0, stream>>>(w.referenced, w.new_id, nv, reinterpret_cast<long long*>(vertex_ids));
    count_launch();
  }
  if (nt) {
    remap_triangles_kernel<<<blocks_for(nt), 256, 0, stream>>>(tris, w.keep, w.tri_pos, w.new_id, nt,
                                                              reinterpret_cast<long long*>(out_triangles));
    count_launch();
  }
  clean_sizes_kernel<<<1, 1, 0, stream>>>(w.keep, w.tri_pos, nt, w.referenced, w.new_id, nv, reinterpret_cast<long long*>(sizes));
  count_launch();
  return check_launch("mesh_remove_small_clusters", stream, false);
}

}  // extern "C"
