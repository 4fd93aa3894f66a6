// Mesh culling by object masks: DTU's cull_scan (evaluation/DTU/eval_code/evaluate_single_scene.py:21-116) without
// scikit-image.  A vertex is dropped when some view projects it strictly inside the image onto an unset pixel of that
// view's mask dilated by a disk.
//
// The projection is fp32 with an explicit rounding intrinsic per operation, so nvcc contracts nothing and the results
// equal the reference's torch expressions on the GPU (DESIGN.md section 7a records the operation order).  The dilation
// is integer-only.
#include "gs2mesh_b200.h"
#include "gsb_common.h"

namespace gsb {
namespace {

constexpr int kMaxRadius = 254;  // distances are stored as uint8, capped at radius + 1

// ---------------------------------------------------------------------------------------------------------------------
// Disk dilation, two passes.  rowdist[v][y][x] = distance from x to the nearest set pixel of row y, capped at r + 1.
// Output pixel (y, x) is set iff some dy in [-r, r] has rowdist[y+dy][x] <= floor(sqrt(r*r - dy*dy)), which is exactly
// "some set pixel (y', x') has (x'-x)^2 + (y'-y)^2 <= r^2" (skimage disk(r)); rows outside the image hold no set pixel.
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) row_distance_kernel(const uint8_t* __restrict__ masks, long long n_pixels, int width,
                                                           int radius, uint8_t* __restrict__ rowdist) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_pixels) return;
  const int x = (int)(i % width);
  const uint8_t* row = masks + (i - x);
  int d = 0;
  for (; d <= radius; ++d)
    if ((x - d >= 0 && row[x - d]) || (x + d < width && row[x + d])) break;
  rowdist[i] = (uint8_t)d;
}

// One warp per 32-pixel output word: lane = pixel, the word is the warp's ballot.  dy runs outward from 0, where the
// allowed row distance is largest, so pixels inside the object stop at once.
__global__ void __launch_bounds__(256) column_disk_kernel(const uint8_t* __restrict__ rowdist, int n_views, int height,
                                                          int width, int radius, uint32_t* __restrict__ packed) {
  __shared__ int half_width[kMaxRadius + 1];  // floor(sqrt(r*r - dy*dy)), integer square root
  for (int dy = threadIdx.x; dy <= radius; dy += blockDim.x) {
    const int n = radius * radius - dy * dy;
    int h = (int)sqrtf((float)n);
    while (h * h > n) --h;
    while ((h + 1) * (h + 1) <= n) ++h;
    half_width[dy] = h;
  }
  __syncthreads();
  const int words = (width + 31) >> 5;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= (long long)n_views * height * words) return;  // whole warps leave together
  const int word = (int)(warp % words);
  const long long row = warp / words;  // v * height + y
  const int y = (int)(row % height);
  const int x = word * 32 + lane;
  bool set = false;
  if (x < width) {
    const uint8_t* col = rowdist + (row - y) * width + x;  // column x of view v
    for (int dy = 0; dy <= radius && !set; ++dy) {
      const int h = half_width[dy];
      set = (y - dy >= 0 && col[(long long)(y - dy) * width] <= h) || (y + dy < height && col[(long long)(y + dy) * width] <= h);
    }
  }
  const uint32_t bits = __ballot_sync(0xffffffffu, set);
  if (lane == 0) packed[warp] = bits;
}

// ---------------------------------------------------------------------------------------------------------------------
// Projection and decision, one thread per vertex (evaluate_single_scene.py:57-99 in torch's fp32 operation order):
//   p = fp32(v); cam_r = fma(M[r][3], 1, fma(M[r][2], z, fma(M[r][1], y, fma(M[r][0], x, 0))))   (cuBLAS's k order)
//   pix = cam_{0,1} / (cam_2 + 1e-6f); pix.x *= fp32(1/(W-1)), pix.y *= fp32(1/(H-1))   (torch divides a CUDA tensor by
//   a scalar as a multiplication by its fp32 reciprocal); g = (pix - 0.5f) * 2; valid = -1 < g < 1 on both axes;
//   grid_sample(nearest, zeros, align_corners=True): i = nearbyint(((g + 1) / 2) * (size - 1)), outside the mask = 0.
// The vertex is culled iff some view has valid && mask == 0; the loop over views stops there.
// ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float project_row(const float* m, float x, float y, float z) {
  return __fmaf_rn(m[3], 1.0f, __fmaf_rn(m[2], z, __fmaf_rn(m[1], y, __fmaf_rn(m[0], x, 0.0f))));
}

__device__ __forceinline__ int nearest_index(float g, float size_m1) {
  return __float2int_rn(__fmul_rn(__fdiv_rn(__fadd_rn(g, 1.0f), 2.0f), size_m1));  // round half to even
}

__global__ void __launch_bounds__(256) cull_kernel(const double* __restrict__ vertices, long long n,
                                                   const float* __restrict__ matrices, int n_views, float inv_w, float inv_h,
                                                   int mask_w, int mask_h, const uint32_t* __restrict__ packed,
                                                   uint8_t* __restrict__ keep) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float x = __double2float_rn(vertices[3 * i]), y = __double2float_rn(vertices[3 * i + 1]),
              z = __double2float_rn(vertices[3 * i + 2]);
  const int words = (mask_w + 31) >> 5;
  const float mw1 = (float)(mask_w - 1), mh1 = (float)(mask_h - 1);
  uint8_t k = 1;
  for (int v = 0; v < n_views; ++v) {
    const float* M = matrices + 16 * v;
    const float c0 = project_row(M, x, y, z), c1 = project_row(M + 4, x, y, z), c2 = project_row(M + 8, x, y, z);
    const float den = __fadd_rn(c2, 1e-6f);
    const float gx = __fmul_rn(__fsub_rn(__fmul_rn(__fdiv_rn(c0, den), inv_w), 0.5f), 2.0f);
    const float gy = __fmul_rn(__fsub_rn(__fmul_rn(__fdiv_rn(c1, den), inv_h), 0.5f), 2.0f);
    if (!(gx > -1.0f && gx < 1.0f && gy > -1.0f && gy < 1.0f)) continue;  // NaN lands here too
    const int ix = nearest_index(gx, mw1), iy = nearest_index(gy, mh1);
    const bool set = ix >= 0 && ix < mask_w && iy >= 0 && iy < mask_h &&
                     ((packed[((long long)v * mask_h + iy) * words + (ix >> 5)] >> (ix & 31)) & 1u);
    if (!set) {
      k = 0;
      break;
    }
  }
  keep[i] = k;
}

}  // namespace
}  // namespace gsb

using namespace gsb;

extern "C" {

int gsb_eval_mask_dilate_disk(const uint8_t* masks, int32_t n_views, int32_t height, int32_t width, int32_t radius,
                              uint32_t* packed, uint8_t* workspace, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (n_views < 0 || height < 0 || width < 0 || radius < 0 || radius > kMaxRadius)
    return fail(GSB_ERR_INVALID, "eval_mask_dilate_disk: bad arguments (0 <= radius <= %d)", kMaxRadius);
  const long long pixels = (long long)n_views * height * width;
  if (pixels == 0) return GSB_OK;
  if (!masks || !packed || !workspace) return fail(GSB_ERR_INVALID, "eval_mask_dilate_disk: NULL buffer");
  row_distance_kernel<<<(unsigned)((pixels + 255) / 256), 256, 0, stream>>>(masks, pixels, width, radius, workspace);
  count_launch();
  const long long threads = (long long)n_views * height * ((width + 31) / 32) * 32;
  column_disk_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, stream>>>(workspace, n_views, height, width, radius, packed);
  count_launch();
  return check_launch("mask dilation", stream, false);
}

int gsb_eval_cull_vertices_by_masks(const double* vertices, int64_t n_vertices, const float* matrices, int32_t n_views,
                                    int32_t image_width, int32_t image_height, int32_t mask_width, int32_t mask_height,
                                    const uint32_t* packed_masks, uint8_t* keep, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (n_vertices < 0 || n_views < 0 || image_width < 2 || image_height < 2 || mask_width < 1 || mask_height < 1 ||
      (n_vertices && (!vertices || !keep || (n_views && (!matrices || !packed_masks)))))
    return fail(GSB_ERR_INVALID, "eval_cull_vertices_by_masks: bad arguments");
  if (n_vertices == 0) return GSB_OK;
  // torch's scalar division: the reciprocal is taken in fp32 on the host
  const float inv_w = 1.0f / (float)(image_width - 1), inv_h = 1.0f / (float)(image_height - 1);
  cull_kernel<<<(unsigned)((n_vertices + 255) / 256), 256, 0, stream>>>(vertices, n_vertices, matrices, n_views, inv_w, inv_h,
                                                                        mask_width, mask_height, packed_masks, keep);
  count_launch();
  return check_launch("cull_kernel", stream, false);
}

}  // extern "C"
