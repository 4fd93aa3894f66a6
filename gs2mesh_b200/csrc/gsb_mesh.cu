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
#include "gs2mesh_b200.h"
#include "gsb_common.h"
#include "gsb_mc_tables.h"


namespace gsb {
namespace {

constexpr int kHalo = GSB_BRICK + 1;  // 17

struct VolView {
  const float2* tw;
  const float4* color;
  const unsigned long long* keys;  // brick hash
  const uint32_t* vals;
  const int4* index;               // lattice index of every pool slot
  uint32_t mask, pool;
  int nb[3];                       // key window: brick count
  int b0[3];                       // key window: first brick
  double voxel_length;
};

// pool slot of the brick with lattice index (bx,by,bz), or kSlotNone (Open3D: volume_units_.find() == end())
__device__ __forceinline__ uint32_t slot_of_brick(const VolView& v, int bx, int by, int bz) {
  if (!brick_key_ok(bx, by, bz)) return kSlotNone;
  const uint32_t h = brick_find(v.keys, v.mask, brick_key(bx, by, bz));
  if (h == kSlotNone) return kSlotNone;
  const uint32_t s = v.vals[h];
  return s < v.pool ? s : kSlotNone;
}

// (gx,gy,gz) = voxel coordinates relative to the key window's first voxel; a brick that was never opened -> weight 0
__device__ __forceinline__ size_t voxel_address(const VolView& v, int gx, int gy, int gz) {
  const uint32_t slot = slot_of_brick(v, v.b0[0] + (gx >> 4), v.b0[1] + (gy >> 4), v.b0[2] + (gz >> 4));
  if (slot == kSlotNone) return (size_t)-1;
  return (size_t)slot * GSB_BRICK_VOXELS + ((gx & 15) * 16 + (gy & 15)) * 16 + (gz & 15);
}
__device__ __forceinline__ float2 load_voxel(const VolView& v, int gx, int gy, int gz) {
  const size_t a = voxel_address(v, gx, gy, gz);
  return a == (size_t)-1 ? make_float2(0.f, 0.f) : v.tw[a];
}

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

// mode 0: tri_counts[b] = number of triangles of brick b.  mode 1: write the edge keys.
__global__ void __launch_bounds__(256) mc_brick_kernel(const VolView v, const uint32_t* __restrict__ bricks, int mode,
                                                       uint32_t* __restrict__ tri_counts,
                                                       const long long* __restrict__ tri_offsets,
                                                       long long* __restrict__ edge_keys) {
  __shared__ float2 s[kHalo * kHalo * kHalo];
  __shared__ uint32_t s_count;
  __shared__ uint32_t s_nb[8];  // pool slots of the brick and its +1 neighbours (bit 2: x+1, bit 1: y+1, bit 0: z+1)
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
  const long long base = mode ? tri_offsets[blockIdx.x] : 0;
  const long long NY = (long long)v.nb[1] * GSB_BRICK, NZ = (long long)v.nb[2] * GSB_BRICK;
  for (int i = threadIdx.x; i < GSB_BRICK_VOXELS; i += blockDim.x) {
    const int z = i & 15, y = (i >> 4) & 15, x = i >> 8;
    const int c = cube_case(s, x, y, z);
    if (c == 0) continue;
    int ntri = 0;
    while (ntri < 5 && kMcTriTable[c][3 * ntri] >= 0) ++ntri;
    const uint32_t slot = atomicAdd(&s_count, (uint32_t)ntri);
    if (mode) {
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

VolView view_of(const GsbVolume* vol, const int32_t* window) {
  VolView v;
  v.tw = reinterpret_cast<const float2*>(vol->d.tsdf_weight);
  v.color = reinterpret_cast<const float4*>(vol->d.color);
  v.keys = reinterpret_cast<const unsigned long long*>(vol->d.hash_keys);
  v.vals = vol->d.hash_vals;
  v.index = reinterpret_cast<const int4*>(vol->d.brick_index);
  v.mask = vol->d.hash_slots - 1u;
  v.pool = vol->d.pool_bricks;
  for (int k = 0; k < 3; ++k) {
    v.b0[k] = window[k];
    v.nb[k] = window[3 + k];
  }
  v.voxel_length = vol->d.voxel_length;
  return v;
}

// GSB_OK, or the error for a key window that is malformed or too large.  A window may span the whole lattice plus the
// +1 brick past its end: 2^21 + 1 bricks per axis.
int window_check(const char* who, const int32_t* w) {
  if (!w) return fail(GSB_ERR_INVALID, "%s: bad arguments", who);
  for (int k = 0; k < 3; ++k)
    if (w[3 + k] <= 0 || w[3 + k] > (1 << 21) + 1 || w[k] < -kBrickBias || w[k] >= kBrickBias)
      return fail(GSB_ERR_INVALID, "%s: bad key window", who);
  // keys = ((gx*NY + gy)*NZ + gz)*3 + axis must fit 63 bits
  const double vox = 16.0 * 16.0 * 16.0 * (double)w[3] * (double)w[4] * (double)w[5] * 3.0;
  if (vox >= 9.0e18)
    return fail(GSB_ERR_INVALID,
                "%s: the bounding box of the open bricks (%d x %d x %d bricks) is too large for 63-bit edge keys "
                "(16^3 * nbx * nby * nbz * 3 must be < 9e18)",
                who, w[3], w[4], w[5]);
  return GSB_OK;
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
  mc_brick_kernel<<<n_bricks, 256, 0, stream>>>(view_of(vol, window), bricks, 0, tri_counts, nullptr, nullptr);
  count_launch();
  return check_launch("mc_brick_kernel(count)", stream, false);
}

int gsb_mesh_emit(const GsbVolume* vol, const int32_t* window, const uint32_t* bricks, uint32_t n_bricks, const int64_t* tri_offsets,
                  int64_t* edge_keys, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (!vol || (n_bricks && (!bricks || !tri_offsets || !edge_keys))) return fail(GSB_ERR_INVALID, "mesh_emit: bad arguments");
  if (const int rc = window_check("mesh_emit", window)) return rc;
  if (n_bricks == 0) return GSB_OK;
  mc_brick_kernel<<<n_bricks, 256, 0, stream>>>(view_of(vol, window), bricks, 1, nullptr, reinterpret_cast<const long long*>(tri_offsets),
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

}  // extern "C"
