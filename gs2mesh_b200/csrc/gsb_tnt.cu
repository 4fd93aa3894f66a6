// Tanks and Temples evaluation (evaluation/TNT/eval_code/python_toolbox/evaluation/{registration,evaluation}.py) without
// Open3D: the point-cloud transform, the selection-polygon crop, voxel downsampling and the moments of point-to-point ICP
// with scaling.  The correspondence search shares gsb_eval.cu's grid (gsb_eval_icp_correspond).
//
// Every floating-point operation is fp64 with an explicit rounding intrinsic, in the operation order DESIGN.md section 7d
// restates from Open3D 0.17 and Eigen, so nvcc cannot contract a multiply and an add into an FMA.
#include <cub/cub.cuh>

#include "gs2mesh_b200.h"
#include "gsb_common.h"

namespace gsb {
namespace {

struct Mat4 {
  double m[16];
};

// PointCloud::Transform: v = T (x, y, z, 1) with each row ((T_i0*x + T_i1*y) + T_i2*z) + T_i3, then xyz / v_3.
__global__ void __launch_bounds__(256) transform_kernel(const double* __restrict__ in, long long n, Mat4 T,
                                                        double* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double x = in[3 * i], y = in[3 * i + 1], z = in[3 * i + 2];
  double v[4];
#pragma unroll
  for (int r = 0; r < 4; ++r)
    v[r] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T.m[4 * r], x), __dmul_rn(T.m[4 * r + 1], y)), __dmul_rn(T.m[4 * r + 2], z)),
                     T.m[4 * r + 3]);
#pragma unroll
  for (int k = 0; k < 3; ++k) out[3 * i + k] = __ddiv_rn(v[k], v[3]);
}

// SelectionPolygonVolume::CropInPolygon: a point is kept iff axis_min <= p_w <= axis_max and an odd number of the edge
// crossings P_i.u + (p_v - P_i.v) / (P_j.v - P_i.v) * (P_j.u - P_i.u) lie strictly below p_u (the index std::lower_bound
// returns on the sorted crossings).  The polygon's (u, v) coordinates are staged in shared memory.
__global__ void __launch_bounds__(256) crop_kernel(const double* __restrict__ pts, long long n, const double* __restrict__ poly,
                                                   int m, int u, int v, int w, double axis_min, double axis_max,
                                                   uint8_t* __restrict__ keep, unsigned int* __restrict__ non_finite) {
  extern __shared__ double suv[];  // [m][2]
  for (int k = threadIdx.x; k < m; k += blockDim.x) {
    suv[2 * k] = poly[3 * k + u];
    suv[2 * k + 1] = poly[3 * k + v];
  }
  __syncthreads();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double x = pts[3 * i], y = pts[3 * i + 1], z = pts[3 * i + 2];
  if (!isfinite(x) || !isfinite(y) || !isfinite(z)) {
    keep[i] = 0;
    atomicAdd(non_finite, 1u);
    return;
  }
  auto coord = [&](int a) { return a == 0 ? x : (a == 1 ? y : z); };
  const double pw = coord(w);
  if (pw < axis_min || pw > axis_max) {
    keep[i] = 0;
    return;
  }
  const double pu = coord(u), pv = coord(v);
  int below = 0;
  for (int a = 0; a < m; ++a) {
    const int b = a + 1 == m ? 0 : a + 1;
    const double au = suv[2 * a], av = suv[2 * a + 1], bu = suv[2 * b], bv = suv[2 * b + 1];
    if ((av < pv && bv >= pv) || (bv < pv && av >= pv)) {
      const double x = __dadd_rn(au, __dmul_rn(__ddiv_rn(__dsub_rn(pv, av), __dsub_rn(bv, av)), __dsub_rn(bu, au)));
      below += x < pu;
    }
  }
  keep[i] = below & 1;
}

// VoxelDownSample: voxel index floor((p - lo) / voxel) per axis; key = (ix << (by + bz)) | (iy << bz) | iz, so ascending
// keys are ascending (x, y, z) voxels.  The (key, point index) pairs are stably sorted, then one thread per voxel sums its
// points in input order (from 0.0, like Open3D's AccumulatedPoint) and divides by the count.
struct VoxelGrid {
  double lo[3];
  double voxel;
  int shift_x, shift_y;
};

__global__ void __launch_bounds__(256) voxel_key_kernel(const double* __restrict__ pts, long long n, VoxelGrid g,
                                                        unsigned long long* __restrict__ keys, long long* __restrict__ ids) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  unsigned long long c[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) c[a] = (unsigned long long)(int)floor(__ddiv_rn(__dsub_rn(pts[3 * i + a], g.lo[a]), g.voxel));
  keys[i] = (c[0] << g.shift_x) | (c[1] << g.shift_y) | c[2];
  ids[i] = i;
}

__global__ void __launch_bounds__(256) voxel_head_kernel(const unsigned long long* __restrict__ keys, long long n,
                                                         uint8_t* __restrict__ head) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) head[i] = i == 0 || keys[i] != keys[i - 1];
}

// The mean of each voxel's values v (points, colours or normals) in input order from 0.0, divided by the voxel's point
// count.  With skip_nan a row with a NaN component adds nothing but still counts (Open3D's AccumulatedPoint normal).
__global__ void __launch_bounds__(256) voxel_mean_kernel(const double* __restrict__ v, long long n,
                                                         const long long* __restrict__ ids, const long long* __restrict__ starts,
                                                         const long long* __restrict__ n_voxels, bool skip_nan,
                                                         double* __restrict__ out) {
  const long long vx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long nv = *n_voxels;
  if (vx >= nv) return;
  const long long s = starts[vx], e = vx + 1 < nv ? starts[vx + 1] : n;
  double sum[3] = {0.0, 0.0, 0.0};
  for (long long k = s; k < e; ++k) {
    const double* r = v + 3 * ids[k];
    if (skip_nan && (isnan(r[0]) || isnan(r[1]) || isnan(r[2]))) continue;
#pragma unroll
    for (int a = 0; a < 3; ++a) sum[a] = __dadd_rn(sum[a], r[a]);
  }
  const double cnt = (double)(e - s);
#pragma unroll
  for (int a = 0; a < 3; ++a) out[3 * vx + a] = __ddiv_rn(sum[a], cnt);
}

// ICP moments over the correspondences (index[i] >= 0), with a fixed reduction tree and no floating-point atomics:
// lane t (of kMomBlocks * kMomThreads) adds the values of points t, t + T, t + 2T, ... in turn from 0.0; each block
// halves its lanes (s[l] += s[l + h], h = 128 .. 1), and one block halves the block partials the same way.
//   pass 0: d2, source xyz, target xyz                                  (7 sums)
//   pass 1: (t - mu_t)_j (s - mu_s)_k for j, k in 0..2 (j-major), then (s - mu_s)_k^2   (12 sums)
// out[kMomSums] receives the number of correspondences.
constexpr int kMomBlocks = 256, kMomThreads = 256, kMomSums = 12;
static_assert((kMomSums + 1) * kMomBlocks == GSB_EVAL_ICP_MOMENT_WORKSPACE, "workspace: the partials and partial counts");

struct Means {
  double s[3], t[3];
};

__device__ void block_halve(double (*s)[kMomThreads], long long* sc, int lane) {
  for (int h = kMomThreads / 2; h > 0; h >>= 1) {
    if (lane < h) {
#pragma unroll
      for (int q = 0; q < kMomSums; ++q) s[q][lane] = __dadd_rn(s[q][lane], s[q][lane + h]);
      sc[lane] += sc[lane + h];
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(kMomThreads) moments_kernel(const double* __restrict__ src, const double* __restrict__ tgt,
                                                              const long long* __restrict__ index, const double* __restrict__ d2,
                                                              long long n, int pass, Means mu, double* __restrict__ partial,
                                                              long long* __restrict__ partial_count) {
  __shared__ double s[kMomSums][kMomThreads];
  __shared__ long long sc[kMomThreads];
  const int lane = threadIdx.x;
  double acc[kMomSums];
#pragma unroll
  for (int q = 0; q < kMomSums; ++q) acc[q] = 0.0;
  long long cnt = 0;
  const long long stride = (long long)kMomBlocks * kMomThreads;
  for (long long i = (long long)blockIdx.x * kMomThreads + lane; i < n; i += stride) {
    const long long j = index[i];
    if (j < 0) continue;
    ++cnt;
    const double sp[3] = {src[3 * i], src[3 * i + 1], src[3 * i + 2]};
    const double tp[3] = {tgt[3 * j], tgt[3 * j + 1], tgt[3 * j + 2]};
    if (pass == 0) {
      acc[0] = __dadd_rn(acc[0], d2[i]);
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        acc[1 + k] = __dadd_rn(acc[1 + k], sp[k]);
        acc[4 + k] = __dadd_rn(acc[4 + k], tp[k]);
      }
    } else {
      double sd[3], td[3];
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        sd[k] = __dsub_rn(sp[k], mu.s[k]);
        td[k] = __dsub_rn(tp[k], mu.t[k]);
      }
#pragma unroll
      for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int k = 0; k < 3; ++k) acc[3 * r + k] = __dadd_rn(acc[3 * r + k], __dmul_rn(td[r], sd[k]));
#pragma unroll
      for (int k = 0; k < 3; ++k) acc[9 + k] = __dadd_rn(acc[9 + k], __dmul_rn(sd[k], sd[k]));
    }
  }
#pragma unroll
  for (int q = 0; q < kMomSums; ++q) s[q][lane] = acc[q];
  sc[lane] = cnt;
  __syncthreads();
  block_halve(s, sc, lane);
  if (lane < kMomSums) partial[lane * kMomBlocks + blockIdx.x] = s[lane][0];
  if (lane == 0) partial_count[blockIdx.x] = sc[0];
}

__global__ void __launch_bounds__(kMomThreads) moments_final_kernel(const double* __restrict__ partial,
                                                                    const long long* __restrict__ partial_count,
                                                                    double* __restrict__ out) {
  static_assert(kMomBlocks == kMomThreads, "the final pass gives one lane per block partial");
  __shared__ double s[kMomSums][kMomThreads];
  __shared__ long long sc[kMomThreads];
  const int lane = threadIdx.x;
#pragma unroll
  for (int q = 0; q < kMomSums; ++q) s[q][lane] = partial[q * kMomBlocks + lane];
  sc[lane] = partial_count[lane];
  __syncthreads();
  block_halve(s, sc, lane);
  if (lane < kMomSums) out[lane] = s[lane][0];
  if (lane == 0) out[kMomSums] = (double)sc[0];
}

int bits_for(long long extent) {  // bits that hold 0 .. extent - 1
  int b = 0;
  while (b < 63 && (1ll << b) < extent) ++b;
  return b;
}

bool host_finite(const double* v, int n) {
  for (int k = 0; k < n; ++k)
    if (!std::isfinite(v[k])) return false;
  return true;
}

size_t voxel_workspace_bytes(int64_t n_points) {
  if (n_points < 0 || n_points >= 2147483647) return 0;
  const int n = (int)n_points;
  size_t sort_bytes = 0, select_bytes = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                  (long long*)nullptr, (long long*)nullptr, n);
  cub::DeviceSelect::Flagged(nullptr, select_bytes, cub::CountingInputIterator<long long>(0), (uint8_t*)nullptr,
                             (long long*)nullptr, (long long*)nullptr, n);
  Carver c(nullptr);
  c.take<unsigned long long>(2 * (size_t)n);
  c.take<long long>(3 * (size_t)n);
  c.take<uint8_t>((size_t)n);
  c.take<char>(sort_bytes > select_bytes ? sort_bytes : select_bytes);
  return c.total();
}

}  // namespace
}  // namespace gsb

using namespace gsb;

extern "C" {

int gsb_eval_transform_points(const double* points, int64_t n_points, const double* transform, double* out, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (n_points < 0 || !transform || (n_points && (!points || !out)))
    return fail(GSB_ERR_INVALID, "eval_transform_points: bad arguments");
  if (n_points == 0) return GSB_OK;
  Mat4 T;
  for (int k = 0; k < 16; ++k) T.m[k] = transform[k];
  transform_kernel<<<blocks_for(n_points), 256, 0, stream>>>(points, n_points, T, out);
  count_launch();
  return check_launch("transform_kernel", stream, false);
}

int gsb_eval_crop_polygon(const double* points, int64_t n_points, const double* polygon, int32_t n_vertices,
                          int32_t orthogonal_axis, double axis_min, double axis_max, uint8_t* keep, uint32_t* counter,
                          uint32_t* host_non_finite, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (n_points < 0 || orthogonal_axis < 0 || orthogonal_axis > 2 || !polygon ||
      (n_points && (!points || !keep || !counter || !host_non_finite)))
    return fail(GSB_ERR_INVALID, "eval_crop_polygon: bad arguments");
  if (n_vertices < 3 || n_vertices > GSB_EVAL_MAX_POLYGON)
    return fail(GSB_ERR_INVALID, "eval_crop_polygon: the polygon has %d vertices (3 .. %d are supported)", n_vertices,
                GSB_EVAL_MAX_POLYGON);
  if (n_points == 0) return GSB_OK;
  static const int kAxes[3][3] = {{1, 2, 0}, {0, 2, 1}, {0, 1, 2}};  // (u, v, w) for orthogonal axis x, y, z
  const int* a = kAxes[orthogonal_axis];
  GSB_CUDA_OK(cudaMemsetAsync(counter, 0, sizeof(uint32_t), stream));
  crop_kernel<<<blocks_for(n_points), 256, sizeof(double) * 2 * n_vertices, stream>>>(
      points, n_points, polygon, n_vertices, a[0], a[1], a[2], axis_min, axis_max, keep, counter);
  count_launch();
  if (int rc = check_launch("crop_kernel", stream, false)) return rc;
  GSB_CUDA_OK(cudaMemcpyAsync(host_non_finite, counter, sizeof(uint32_t), cudaMemcpyDeviceToHost, stream));
  GSB_CUDA_OK(cudaStreamSynchronize(stream));
  if (*host_non_finite)
    return fail(GSB_ERR_INVALID, "eval_crop_polygon: %u points are not finite", (unsigned)*host_non_finite);
  return GSB_OK;
}

size_t gsb_eval_voxel_workspace_bytes(int64_t n_points) { return voxel_workspace_bytes(n_points); }

// Keys, stable sort, voxel heads, their starts, then the mean of the points and of the colours and normals that are given.
int gsb_pcd_voxel_downsample(const double* points, const double* colors, const double* normals, int64_t n_points,
                             const double* min_bound, const double* max_bound, double voxel_size, void* workspace,
                             size_t workspace_bytes, double* out, double* out_colors, double* out_normals, int64_t* n_out,
                             void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (!colors != !out_colors || !normals != !out_normals)
    return fail(GSB_ERR_INVALID, "pcd_voxel_downsample: colours and normals need both their input and their output");
  if (n_points < 0 || n_points >= 2147483647 || !(voxel_size > 0.0) || !(voxel_size < INFINITY) || !min_bound || !max_bound ||
      !n_out || (n_points && (!points || !out || !workspace)))
    return fail(GSB_ERR_INVALID, "pcd_voxel_downsample: bad arguments");
  if (n_points == 0) {
    GSB_CUDA_OK(cudaMemsetAsync(n_out, 0, sizeof(int64_t), stream));
    return GSB_OK;
  }
  if (!host_finite(min_bound, 3) || !host_finite(max_bound, 3))
    return fail(GSB_ERR_INVALID, "pcd_voxel_downsample: the points are not finite");
  VoxelGrid g;
  g.voxel = voxel_size;
  double span = 0.0;
  for (int a = 0; a < 3; ++a) {
    g.lo[a] = min_bound[a] - voxel_size * 0.5;
    span = std::max(span, (max_bound[a] + voxel_size * 0.5) - g.lo[a]);
  }
  if (voxel_size * 2147483647.0 < span)  // Open3D: voxel_size * INT_MAX < (voxel_max_bound - voxel_min_bound).maxCoeff()
    return fail(GSB_ERR_INVALID, "pcd_voxel_downsample: voxel_size is too small (voxel_size * INT_MAX < %g)", span);
  long long extent[3];  // voxels per axis; the largest index is that of max_bound
  for (int a = 0; a < 3; ++a) extent[a] = (long long)std::floor((max_bound[a] - g.lo[a]) / voxel_size) + 1;
  const int bx = bits_for(extent[0]), by = bits_for(extent[1]), bz = bits_for(extent[2]);
  if (bx + by + bz > 63)
    return fail(GSB_ERR_INVALID,
                "pcd_voxel_downsample: %lld x %lld x %lld voxels need %d key bits; voxel keys are limited to 63 bits",
                extent[0], extent[1], extent[2], bx + by + bz);
  g.shift_x = by + bz;
  g.shift_y = bz;
  if (workspace_bytes < voxel_workspace_bytes(n_points))
    return fail(GSB_ERR_WORKSPACE, "pcd_voxel_downsample: workspace %zu < %zu bytes", workspace_bytes,
                voxel_workspace_bytes(n_points));
  const int n = (int)n_points;
  Carver c(workspace);
  unsigned long long* keys = c.take<unsigned long long>(2 * (size_t)n);
  long long* ids = c.take<long long>(3 * (size_t)n);
  uint8_t* head = c.take<uint8_t>((size_t)n);
  size_t tmp_bytes = workspace_bytes - c.total();
  void* tmp = c.take<char>(tmp_bytes);
  voxel_key_kernel<<<blocks_for(n), 256, 0, stream>>>(points, n, g, keys, ids);
  count_launch();
  GSB_CUDA_OK(cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, keys, keys + n, ids, ids + n, n, 0, bx + by + bz, stream));
  voxel_head_kernel<<<blocks_for(n), 256, 0, stream>>>(keys + n, n, head);
  count_launch();
  long long* starts = ids + 2 * (size_t)n;
  auto* n_voxels = reinterpret_cast<long long*>(n_out);
  GSB_CUDA_OK(cub::DeviceSelect::Flagged(tmp, tmp_bytes, cub::CountingInputIterator<long long>(0), head, starts, n_voxels, n,
                                         stream));
  voxel_mean_kernel<<<blocks_for(n), 256, 0, stream>>>(points, n, ids + n, starts, n_voxels, false, out);
  count_launch();
  if (colors) {
    voxel_mean_kernel<<<blocks_for(n), 256, 0, stream>>>(colors, n, ids + n, starts, n_voxels, false, out_colors);
    count_launch();
  }
  if (normals) {
    voxel_mean_kernel<<<blocks_for(n), 256, 0, stream>>>(normals, n, ids + n, starts, n_voxels, true, out_normals);
    count_launch();
  }
  return check_launch("voxel downsample", stream, false);
}

int gsb_eval_icp_moments(const double* source, const int64_t* index, const double* dist2, int64_t n_source,
                         const double* target, int pass, const double* means, double* workspace, double* out, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (n_source < 0 || (pass != 0 && pass != 1) || (pass == 1 && !means) || !workspace || !out ||
      (n_source && (!source || !index || !target || (pass == 0 && !dist2))))
    return fail(GSB_ERR_INVALID, "eval_icp_moments: bad arguments");
  Means mu{};
  if (pass == 1)
    for (int k = 0; k < 3; ++k) {
      mu.s[k] = means[k];
      mu.t[k] = means[3 + k];
    }
  double* partial = workspace;
  auto* partial_count = reinterpret_cast<long long*>(workspace + kMomSums * kMomBlocks);
  moments_kernel<<<kMomBlocks, kMomThreads, 0, stream>>>(source, target, reinterpret_cast<const long long*>(index), dist2,
                                                         n_source, pass, mu, partial, partial_count);
  moments_final_kernel<<<1, kMomThreads, 0, stream>>>(partial, partial_count, out);
  count_launch(2);
  return check_launch("icp moments", stream, false);
}

}  // extern "C"
