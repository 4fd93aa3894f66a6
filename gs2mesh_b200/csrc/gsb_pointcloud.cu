// Point clouds from the brick TSDF volume: Open3D 0.17.0 ScalableTSDFVolume::ExtractPointCloud (the zero crossings of
// the TSDF along the three lattice axes, with colours and TSDF-gradient normals) and ::ExtractVoxelPointCloud (the
// centre of every observed voxel near the surface, grey by its tsdf).  DESIGN.md section 7, "Point clouds", restates both.
//
// Open3D walks every voxel of every volume unit serially.  Here one CTA per open brick applies the predicate to each of
// its voxels (count pass, then emit pass of one 64-bit key per point: window voxel index * 3 + axis for the surface
// cloud, window voxel index for the voxel cloud); the caller sorts the keys, and one thread per key computes the point,
// its colour and (surface cloud) its normal in Open3D's operation order, one rounding per operation.
#include "gs2mesh_b200.h"
#include "gsb_common.h"
#include "gsb_volume_view.cuh"

namespace gsb {
namespace {

constexpr int kHalo = GSB_BRICK + 1;  // 17

// Open3D's test for a voxel that may carry a point: `w != 0 && f < 0.98f && f >= -0.98f`
__device__ __forceinline__ bool near_surface(float2 v) { return v.y != 0.0f && v.x < 0.98f && v.x >= -0.98f; }

// Count (offsets == nullptr: counts[b] = points of brick b) or emit (keys from offsets[b] on) the points of each listed
// brick.  The surface cloud stages the brick plus the +1 voxel layer on each of its three +faces (the neighbour an edge
// reaches; edges and corner of the 17^3 cube are never read); the voxel cloud reads the brick where it lies.
template <bool kSurface>
__global__ void __launch_bounds__(256) pcd_brick_kernel(const VolView v, const uint32_t* __restrict__ bricks,
                                                        uint32_t* __restrict__ counts, const long long* __restrict__ offsets,
                                                        long long* __restrict__ keys) {
  __shared__ float2 s[kSurface ? kHalo * kHalo * kHalo : 1];
  __shared__ uint32_t s_count;
  __shared__ uint32_t s_nb[3];  // pool slots of the +x, +y, +z neighbours
  const uint32_t brick = bricks[blockIdx.x];
  const int4 bi = v.index[brick];
  const int bx = bi.x - v.b0[0], by = bi.y - v.b0[1], bz = bi.z - v.b0[2];
  if (threadIdx.x == 0) s_count = 0;
  if (kSurface) {
    if (threadIdx.x < 3)
      s_nb[threadIdx.x] = slot_of_brick(v, bi.x + (threadIdx.x == 0), bi.y + (threadIdx.x == 1), bi.z + (threadIdx.x == 2));
    __syncthreads();
    for (int i = threadIdx.x; i < kHalo * kHalo * kHalo; i += blockDim.x) {
      const int z = i % kHalo, y = (i / kHalo) % kHalo, x = i / (kHalo * kHalo);
      const int out = (x >> 4) + (y >> 4) + (z >> 4);
      if (out > 1) continue;  // never read
      const uint32_t slot = out == 0 ? brick : s_nb[(x >> 4) ? 0 : (y >> 4) ? 1 : 2];
      s[i] = slot == kSlotNone ? make_float2(0.f, 0.f)
                               : v.tw[(size_t)slot * GSB_BRICK_VOXELS + ((x & 15) * 16 + (y & 15)) * 16 + (z & 15)];
    }
  }
  __syncthreads();
  const long long base = offsets ? offsets[blockIdx.x] : 0;
  const long long NY = (long long)v.nb[1] * GSB_BRICK, NZ = (long long)v.nb[2] * GSB_BRICK;
  for (int i = threadIdx.x; i < GSB_BRICK_VOXELS; i += blockDim.x) {
    const int z = i & 15, y = (i >> 4) & 15, x = i >> 8;
    const long long lin = ((long long)(bx * 16 + x) * NY + (by * 16 + y)) * NZ + (bz * 16 + z);
    if (!kSurface) {
      if (!near_surface(v.tw[(size_t)brick * GSB_BRICK_VOXELS + i])) continue;
      const uint32_t at = atomicAdd(&s_count, 1u);
      if (offsets) keys[base + at] = lin;
      continue;
    }
    const float2 a = s[(x * kHalo + y) * kHalo + z];
    if (!near_surface(a)) continue;
    const float2 nbr[3] = {s[((x + 1) * kHalo + y) * kHalo + z], s[(x * kHalo + y + 1) * kHalo + z],
                           s[(x * kHalo + y) * kHalo + z + 1]};
    int mask = 0;
#pragma unroll
    for (int k = 0; k < 3; ++k)
      if (near_surface(nbr[k]) && __fmul_rn(a.x, nbr[k].x) < 0.0f) mask |= 1 << k;  // float product, as Open3D's
    if (mask == 0) continue;
    const uint32_t at = atomicAdd(&s_count, (uint32_t)__popc(mask));
    if (offsets) {
      int j = 0;
#pragma unroll
      for (int k = 0; k < 3; ++k)
        if (mask & (1 << k)) keys[base + at + j++] = lin * 3 + k;
    }
  }
  __syncthreads();
  if (!offsets && threadIdx.x == 0) counts[blockIdx.x] = s_count;
}

// One sorted key -> point, colour and normal.  Surface cloud (ExtractPointCloud), for the edge from voxel (x,y,z) of
// unit index0 to its +1 neighbour on `axis`:
//   p0 = (vl/2 + vl*x, vl/2 + vl*y, vl/2 + vl*z) + index0 * U    (per unit, not vl/2 + vl*(16*b + x))
//   p1 = p0, p1(axis) += vl;  r0 = |f0|, r1 = |f1| (float)
//   point  = (p0 * (double)r1 + p1 * (double)r0) / (double)(r0 + r1 in float)
//   colour = (double)((c0 * r1 + c1 * r0) / (r0 + r1) / 255.0f), all float
//   normal = normalized(n), n(j) = GetTSDFAt(point + 0.99 vl e_j) - GetTSDFAt(point - 0.99 vl e_j)
// Eigen's normalized() divides by sqrt((x*x + y*y) + z*z) only when that is > 0.  Voxel cloud (ExtractVoxelPointCloud):
// point = p0, grey = ((double)f + 1.0) * 0.5.
template <bool kSurface>
__global__ void __launch_bounds__(256) pcd_points_kernel(const VolView v, const long long* __restrict__ keys, long long n,
                                                         double* __restrict__ xyz, double* __restrict__ rgb,
                                                         double* __restrict__ normals) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const long long NY = (long long)v.nb[1] * GSB_BRICK, NZ = (long long)v.nb[2] * GSB_BRICK;
  const long long key = keys[i];
  const int axis = kSurface ? (int)(key % 3) : 0;
  long long lin = kSurface ? key / 3 : key;
  const int g[3] = {(int)(lin / (NY * NZ)), (int)((lin / NZ) % NY), (int)(lin % NZ)};
  const double vl = v.voxel_length, half = __dmul_rn(vl, 0.5), U = __dmul_rn(vl, (double)GSB_BRICK);
  double p0[3];
#pragma unroll
  for (int k = 0; k < 3; ++k)
    p0[k] = __dadd_rn(__dadd_rn(half, __dmul_rn(vl, (double)(g[k] & 15))), __dmul_rn((double)(v.b0[k] + (g[k] >> 4)), U));
  const size_t ia = voxel_address(v, g[0], g[1], g[2]);
  const float f0 = v.tw[ia].x;
  if (!kSurface) {
#pragma unroll
    for (int k = 0; k < 3; ++k) xyz[3 * i + k] = p0[k];
    if (rgb) {
      const double c = __dmul_rn(__dadd_rn((double)f0, 1.0), 0.5);
#pragma unroll
      for (int k = 0; k < 3; ++k) rgb[3 * i + k] = c;
    }
    return;
  }
  const size_t ib = voxel_address(v, g[0] + (axis == 0), g[1] + (axis == 1), g[2] + (axis == 2));
  const float f1 = v.tw[ib].x;
  const float r0 = fabsf(f0), r1 = fabsf(f1), rs = __fadd_rn(r0, r1);
  const double d0 = (double)r0, d1 = (double)r1, ds = (double)rs;
  double p[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const double p1 = k == axis ? __dadd_rn(p0[k], vl) : p0[k];
    p[k] = __ddiv_rn(__dadd_rn(__dmul_rn(p0[k], d1), __dmul_rn(p1, d0)), ds);
    xyz[3 * i + k] = p[k];
  }
  if (rgb) {
    const float4 c0 = v.color[ia], c1 = v.color[ib];
    const float k0[3] = {c0.x, c0.y, c0.z}, k1[3] = {c1.x, c1.y, c1.z};
#pragma unroll
    for (int k = 0; k < 3; ++k)
      rgb[3 * i + k] = (double)__fdiv_rn(__fdiv_rn(__fadd_rn(__fmul_rn(k0[k], r1), __fmul_rn(k1[k], r0)), rs), 255.0f);
  }
  if (normals) {
    double nv[3];
    tsdf_normal(v, vl, U, half, p, nv);
#pragma unroll
    for (int j = 0; j < 3; ++j) normals[3 * i + j] = nv[j];
  }
}

bool mode_ok(int mode) { return mode == GSB_PCD_SURFACE || mode == GSB_PCD_VOXELS; }

}  // namespace
}  // namespace gsb

using namespace gsb;

extern "C" {

int gsb_pcd_count(const GsbVolume* vol, const int32_t* window, const uint32_t* bricks, uint32_t n_bricks, int mode,
                  uint32_t* counts, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (!vol || !mode_ok(mode) || (n_bricks && (!bricks || !counts))) return fail(GSB_ERR_INVALID, "pcd_count: bad arguments");
  if (const int rc = window_check("pcd_count", window)) return rc;
  if (n_bricks == 0) return GSB_OK;
  const VolView v = view_of(vol, window);
  if (mode == GSB_PCD_SURFACE)
    pcd_brick_kernel<true><<<n_bricks, 256, 0, stream>>>(v, bricks, counts, nullptr, nullptr);
  else
    pcd_brick_kernel<false><<<n_bricks, 256, 0, stream>>>(v, bricks, counts, nullptr, nullptr);
  count_launch();
  return check_launch("pcd_brick_kernel(count)", stream, false);
}

int gsb_pcd_emit(const GsbVolume* vol, const int32_t* window, const uint32_t* bricks, uint32_t n_bricks, int mode,
                 const int64_t* offsets, int64_t* keys, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (!vol || !mode_ok(mode) || (n_bricks && (!bricks || !offsets || !keys))) return fail(GSB_ERR_INVALID, "pcd_emit: bad arguments");
  if (const int rc = window_check("pcd_emit", window)) return rc;
  if (n_bricks == 0) return GSB_OK;
  const VolView v = view_of(vol, window);
  const auto* off = reinterpret_cast<const long long*>(offsets);
  auto* k = reinterpret_cast<long long*>(keys);
  if (mode == GSB_PCD_SURFACE)
    pcd_brick_kernel<true><<<n_bricks, 256, 0, stream>>>(v, bricks, nullptr, off, k);
  else
    pcd_brick_kernel<false><<<n_bricks, 256, 0, stream>>>(v, bricks, nullptr, off, k);
  count_launch();
  return check_launch("pcd_brick_kernel(emit)", stream, false);
}

int gsb_pcd_points(const GsbVolume* vol, const int32_t* window, const int64_t* keys, int64_t n, int mode, double* xyz,
                   double* rgb, double* normals, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (!vol || !mode_ok(mode) || n < 0 || (n && (!keys || !xyz))) return fail(GSB_ERR_INVALID, "pcd_points: bad arguments");
  if (mode == GSB_PCD_VOXELS && normals) return fail(GSB_ERR_INVALID, "pcd_points: the voxel cloud has no normals");
  if (mode == GSB_PCD_SURFACE && rgb && !vol->d.color)
    return fail(GSB_ERR_INVALID, "pcd_points: colours asked of a volume without colour");
  if (const int rc = window_check("pcd_points", window)) return rc;
  if (n == 0) return GSB_OK;
  const VolView v = view_of(vol, window);
  const auto* k = reinterpret_cast<const long long*>(keys);
  if (mode == GSB_PCD_SURFACE)
    pcd_points_kernel<true><<<blocks_for(n), 256, 0, stream>>>(v, k, n, xyz, rgb, normals);
  else
    pcd_points_kernel<false><<<blocks_for(n), 256, 0, stream>>>(v, k, n, xyz, rgb, nullptr);
  count_launch();
  return check_launch("pcd_points_kernel", stream, false);
}

}  // extern "C"
