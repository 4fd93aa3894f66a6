// Stereo stage between the renderer and the TSDF (gs2mesh_utils/stereo_utils.py:82-179) without the PNG / npy round
// trip: the disparity model's padded inputs, the crop and flip of its outputs, the left-right occlusion mask and the
// depth conversion.  The model itself stays the caller's torch module.
//
// Padding is DLNR's InputPadder(dims, divis_by=32) in 'sintel' mode: ph = ((H/32 + 1)*32 - H) % 32, pad
// [l, r, t, b] = [pw/2, pw - pw/2, ph/2, ph - ph/2].  The occlusion test and the depth are evaluated in the dtypes numpy
// gives the reference's expressions, with one explicit rounding per operation (DESIGN.md section 7c).
#include <climits>
#include <cmath>

#include "gs2mesh_b200.h"
#include "gsb_common.h"

namespace gsb {
namespace {

struct Pad {
  int l, t, wp, hp;
};

Pad stereo_pad(int width, int height) {
  const int pw = ((width / 32 + 1) * 32 - width) % 32, ph = ((height / 32 + 1) * 32 - height) % 32;
  return {pw / 2, ph / 2, width + pw, height + ph};
}

bool frame_ok(int width, int height) {
  return width >= 1 && height >= 1 && width <= GSB_TSDF_MAX_WIDTH && height <= GSB_TSDF_MAX_HEIGHT;
}

// One thread per padded pixel of each of the 4 images: [0] = pad(left), [1] = pad(right), [2] = flip_x(pad(right)),
// [3] = flip_x(pad(left)); replicate padding, float(u8), channel planes [4][3][Hp][Wp].
__global__ void __launch_bounds__(256) pack_kernel(const uint8_t* __restrict__ left, const uint8_t* __restrict__ right, int width,
                                                   int height, Pad p, float* __restrict__ out) {
  const long long plane = (long long)p.hp * p.wp;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 4 * plane) return;
  const int k = (int)(i / plane);
  const long long j = i - k * plane;
  const int yp = (int)(j / p.wp), xp = (int)(j - (long long)yp * p.wp);
  const uint8_t* src = (k == 0 || k == 3) ? left : right;
  const int xs = k >= 2 ? p.wp - 1 - xp : xp;
  const int sy = min(max(yp - p.t, 0), height - 1), sx = min(max(xs - p.l, 0), width - 1);
  const uint8_t* px = src + ((long long)sy * width + sx) * 3;
  float* o = out + (long long)k * 3 * plane + j;
  o[0] = (float)px[0];
  o[plane] = (float)px[1];
  o[2 * plane] = (float)px[2];
}

// One thread per padded pixel: disp_rl = sign * flip_x(flow_rl) over the whole padded plane (the reference builds the
// RL padder from the already padded images, so nothing is cropped), disp_lr = sign * flow_lr cropped to the frame.
__global__ void __launch_bounds__(256) disparity_kernel(const float* __restrict__ flow_lr, const float* __restrict__ flow_rl,
                                                        int width, int height, Pad p, float sign, float* __restrict__ disp_lr,
                                                        float* __restrict__ disp_rl) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)p.hp * p.wp) return;
  const int yp = (int)(i / p.wp), xp = (int)(i - (long long)yp * p.wp);
  const long long row = (long long)yp * p.wp;
  disp_rl[i] = __fmul_rn(sign, flow_rl[row + (p.wp - 1 - xp)]);
  const int y = yp - p.t, x = xp - p.l;
  if (y >= 0 && y < height && x >= 0 && x < width) disp_lr[(long long)y * width + x] = __fmul_rn(sign, flow_lr[i]);
}

// get_occlusion_mask (stereo_utils.py:161-179) and depth (:133), one thread per pixel, in numpy's dtypes:
//   xp  = int32(fp64(x) - fp64(d_lr))      x86 cvttsd2si: NaN or out of range -> INT_MIN
//   xc  = clip(xp, 0, W-1);  xr = fp64(xc) + fp64(d_rl[y][xc])       (row y of d_rl's own plane)
//   xrc = clip(xr, 0, W-1)                 np.clip keeps NaN
//   visible = !(|fp64(x) - xrc| > thr) && 0 <= xp < W
//   depth = fp32(fx*B) / d_lr              NumPy 1.x value-based casting keeps float32
__global__ void __launch_bounds__(256) occlusion_depth_kernel(const float* __restrict__ disp_lr, const float* __restrict__ disp_rl,
                                                              int width, int height, long long rl_stride, double threshold,
                                                              float depth_numerator, uint8_t* __restrict__ visible,
                                                              float* __restrict__ depth) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)width * height) return;
  const int y = (int)(i / width), x = (int)(i - (long long)y * width);
  const float d = disp_lr[i];
  if (depth) depth[i] = __fdiv_rn(depth_numerator, d);
  if (!visible) return;
  const double xf = __dsub_rn((double)x, (double)d);
  // truncation fits int32 iff -2^31 - 1 < xf < 2^31; every other value (NaN included) converts to INT_MIN
  const int xp = (xf > -2147483649.0 && xf < 2147483648.0) ? __double2int_rz(xf) : INT_MIN;
  const int xc = min(max(xp, 0), width - 1);
  const double xr = __dadd_rn((double)xc, (double)disp_rl[(long long)y * rl_stride + xc]);
  const double hi = (double)(width - 1);
  const double xrc = isnan(xr) ? xr : (xr < 0.0 ? 0.0 : (xr > hi ? hi : xr));  // no fmin/fmax: they drop NaN
  const double diff = fabs(__dsub_rn((double)x, xrc));
  visible[i] = (uint8_t)(!(diff > threshold) && xp >= 0 && xp < width);
}

}  // namespace
}  // namespace gsb

using namespace gsb;

extern "C" {

int gsb_stereo_pack_inputs(const uint8_t* left, const uint8_t* right, int32_t width, int32_t height, float* out, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (!frame_ok(width, height))
    return fail(GSB_ERR_INVALID, "stereo_pack_inputs: frame %d x %d outside 1..%d x 1..%d", width, height, GSB_TSDF_MAX_WIDTH,
                GSB_TSDF_MAX_HEIGHT);
  if (!left || !right || !out) return fail(GSB_ERR_INVALID, "stereo_pack_inputs: NULL buffer");
  const Pad p = stereo_pad(width, height);
  pack_kernel<<<blocks_for(4LL * p.hp * p.wp), 256, 0, stream>>>(left, right, width, height, p, out);
  count_launch();
  return check_launch("stereo pack_kernel", stream, false);
}

int gsb_stereo_disparities(const float* flow_lr, const float* flow_rl, int32_t width, int32_t height, float sign, float* disp_lr,
                           float* disp_rl, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (!frame_ok(width, height))
    return fail(GSB_ERR_INVALID, "stereo_disparities: frame %d x %d outside 1..%d x 1..%d", width, height, GSB_TSDF_MAX_WIDTH,
                GSB_TSDF_MAX_HEIGHT);
  if (!isfinite(sign)) return fail(GSB_ERR_INVALID, "stereo_disparities: sign must be finite");
  if (!flow_lr || !flow_rl || !disp_lr || !disp_rl) return fail(GSB_ERR_INVALID, "stereo_disparities: NULL buffer");
  const Pad p = stereo_pad(width, height);
  disparity_kernel<<<blocks_for((long long)p.hp * p.wp), 256, 0, stream>>>(flow_lr, flow_rl, width, height, p, sign, disp_lr,
                                                                           disp_rl);
  count_launch();
  return check_launch("stereo disparity_kernel", stream, false);
}

int gsb_stereo_occlusion_depth(const float* disp_lr, const float* disp_rl, int32_t width, int32_t height, int64_t rl_stride,
                               double threshold, float depth_numerator, uint8_t* visible, float* depth, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (!frame_ok(width, height))
    return fail(GSB_ERR_INVALID, "stereo_occlusion_depth: frame %d x %d outside 1..%d x 1..%d", width, height,
                GSB_TSDF_MAX_WIDTH, GSB_TSDF_MAX_HEIGHT);
  if (!disp_lr || (!visible && !depth) || (visible && (!disp_rl || rl_stride < width)))
    return fail(GSB_ERR_INVALID, "stereo_occlusion_depth: bad arguments (NULL buffer or rl_stride < width)");
  occlusion_depth_kernel<<<blocks_for((long long)width * height), 256, 0, stream>>>(disp_lr, disp_rl, width, height, rl_stride,
                                                                                    threshold, depth_numerator, visible, depth);
  count_launch();
  return check_launch("stereo occlusion_depth_kernel", stream, false);
}

}  // extern "C"
