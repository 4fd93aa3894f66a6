// Ray casting of the brick TSDF volume: the depth, normal and colour images of the fused zero-level surface on the pixel
// grid of one pinhole camera.  Open3D's legacy ScalableTSDFVolume has no ray cast, so the semantics are ours; DESIGN.md
// section 7, "Ray casting", states them, and tests/raycast_oracle.py restates them in numpy.
//
// One thread per pixel, in 16 x 8 tiles so that neighbouring rays walk the same bricks.  Each ray marches from its
// near end: an empty unit is crossed in one step, a cube with an unobserved corner in one voxel, and a valid sample
// advances by its truncated distance (at least one voxel).  The first valid pair with f_prev > 0 >= f is the hit.  The
// slot of the unit a sample lies in is kept across steps, so a step inside one brick does not probe the hash again.
// Every fp64 operation is an explicit __d*_rn, so nothing is contracted and the restatement can match every bit.
#include <climits>
#include <cmath>

#include "gs2mesh_b200.h"
#include "gsb_common.h"
#include "gsb_volume_view.cuh"

namespace gsb {
namespace {

constexpr int kTileX = 16, kTileY = 8;

struct RayParams {
  double fx, fy, cx, cy;
  double E[12];  // world -> camera [R|t], row-major
  double zmin, zmax;
  double tau;    // sdf_trunc
  int W, H;
};

// The ray's parameter interval [z_in, z_out] inside the box of the lattice range, where unit indices lie in
// [-2^20, 2^20): p - vl/2 in [-2^20 U, 2^20 U).  false if the ray misses the box.  Axes with a zero direction component
// only test the origin against the slab (no division by zero).
__device__ __forceinline__ bool lattice_interval(const double o[3], const double d[3], double U, double half, double& z_in,
                                                 double& z_out) {
  const double lo = __dadd_rn(__dmul_rn(-(double)kBrickBias, U), half), hi = __dadd_rn(__dmul_rn((double)kBrickBias, U), half);
  z_in = -INFINITY;
  z_out = INFINITY;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    if (d[k] == 0.0) {
      if (!(o[k] >= lo && o[k] < hi)) return false;
      continue;
    }
    const double t1 = __ddiv_rn(__dsub_rn(lo, o[k]), d[k]), t2 = __ddiv_rn(__dsub_rn(hi, o[k]), d[k]);
    z_in = fmax(z_in, fmin(t1, t2));
    z_out = fmin(z_out, fmax(t1, t2));
  }
  return true;
}

__global__ void __launch_bounds__(kTileX * kTileY) raycast_kernel(const VolView v, const RayParams rp, float* __restrict__ depth,
                                                                   float* __restrict__ normals, float* __restrict__ colors) {
  const int u = blockIdx.x * kTileX + threadIdx.x, vv = blockIdx.y * kTileY + threadIdx.y;
  if (u >= rp.W || vv >= rp.H) return;
  const size_t pix = (size_t)vv * rp.W + u;
  const double vl = v.voxel_length, half = __dmul_rn(vl, 0.5), U = __dmul_rn(vl, (double)GSB_BRICK);
  // a = ((u - cx)/fx, (v - cy)/fy, 1); o = -R^T t; d = R^T a
  const double ax = __ddiv_rn(__dsub_rn((double)u, rp.cx), rp.fx), ay = __ddiv_rn(__dsub_rn((double)vv, rp.cy), rp.fy);
  const double* E = rp.E;
  double o[3], d[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    o[k] = -__dadd_rn(__dadd_rn(__dmul_rn(E[k], E[3]), __dmul_rn(E[4 + k], E[7])), __dmul_rn(E[8 + k], E[11]));
    d[k] = __dadd_rn(__dadd_rn(__dmul_rn(E[k], ax), __dmul_rn(E[4 + k], ay)), E[8 + k]);
  }
  const double dn = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(d[0], d[0]), __dmul_rn(d[1], d[1])), __dmul_rn(d[2], d[2])));
  const double step_vl = __ddiv_rn(vl, dn);

  bool found = false;
  double hit = 0.0;
  double z_in, z_out;
  if (dn > 0.0 && lattice_interval(o, d, U, half, z_in, z_out)) {
    const double z_end = fmin(rp.zmax, z_out);
    double z = fmax(rp.zmin, z_in);
    bool prev_valid = false;
    double f_prev = 0.0, z_prev = 0.0;
    int cached[3] = {INT_MIN, INT_MIN, INT_MIN};  // the unit whose slot `cached_slot` holds
    uint32_t cached_slot = kSlotNone;
    while (z <= z_end) {
      double p[3], q[3], fl[3];
#pragma unroll
      for (int k = 0; k < 3; ++k) p[k] = __dadd_rn(o[k], __dmul_rn(z, d[k]));
      double z_next;
      uint32_t s0 = kSlotNone;
      const bool in = unit_of(U, half, p, q, fl);
      int i0[3] = {0, 0, 0};
      if (in) {
#pragma unroll
        for (int k = 0; k < 3; ++k) i0[k] = (int)fl[k];
        if (i0[0] != cached[0] || i0[1] != cached[1] || i0[2] != cached[2]) {
          cached_slot = slot_of_brick(v, i0[0], i0[1], i0[2]);
#pragma unroll
          for (int k = 0; k < 3; ++k) cached[k] = i0[k];
        }
        s0 = cached_slot;
      }
      if (s0 == kSlotNone) {
        // EMPTY: to the ray's exit from the unit's box, p - vl/2 in [fl U, (fl + 1) U) per axis
        double exit = INFINITY;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          if (d[k] == 0.0) continue;
          const double face = __dadd_rn(__dmul_rn(d[k] > 0.0 ? __dadd_rn(fl[k], 1.0) : fl[k], U), half);
          exit = fmin(exit, __ddiv_rn(__dsub_rn(face, o[k]), d[k]));
        }
        prev_valid = false;
        z_next = exit > z ? exit : __dadd_rn(z, step_vl);
      } else {
        int c[3];
        double r[3], f8[8];
        cube_in_unit(vl, U, q, fl, c, r);
        bool valid = true;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          uint32_t voxel;
          const uint32_t slot = cube_corner(v, i0, s0, c, i, voxel);
          const float2 tw = slot == kSlotNone ? make_float2(0.f, 0.f) : v.tw[(size_t)slot * GSB_BRICK_VOXELS + voxel];
          valid = valid && tw.y != 0.0f;
          f8[i] = (double)tw.x;
        }
        if (!valid) {  // INVALID: a corner never observed
          prev_valid = false;
          z_next = __dadd_rn(z, step_vl);
        } else {
          const double f = cube_trilinear(f8, r);
          if (prev_valid && f_prev > 0.0 && f <= 0.0) {
            found = true;
            hit = __dadd_rn(z_prev, __dmul_rn(__dsub_rn(z, z_prev), __ddiv_rn(f_prev, __dsub_rn(f_prev, f))));
            break;
          }
          prev_valid = true;
          f_prev = f;
          z_prev = z;
          z_next = f > 0.0 ? __dadd_rn(z, __ddiv_rn(fmax(__dmul_rn(f, rp.tau), vl), dn)) : __dadd_rn(z, step_vl);
        }
      }
      if (!(z_next > z)) break;  // a step rounding cannot take: the ray ends here
      z = z_next;
    }
  }
  if (!found) {
    depth[pix] = 0.0f;
    if (normals) normals[3 * pix] = normals[3 * pix + 1] = normals[3 * pix + 2] = 0.0f;
    if (colors) colors[3 * pix] = colors[3 * pix + 1] = colors[3 * pix + 2] = 0.0f;
    return;
  }
  depth[pix] = (float)hit;
  double p[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) p[k] = __dadd_rn(o[k], __dmul_rn(hit, d[k]));
  if (normals) {
    double nv[3];
    tsdf_normal(v, vl, U, half, p, nv);
#pragma unroll
    for (int k = 0; k < 3; ++k) normals[3 * pix + k] = (float)nv[k];
  }
  if (colors) {
#pragma unroll 1
    for (int k = 0; k < 3; ++k) colors[3 * pix + k] = (float)__ddiv_rn(tsdf_at<true>(v, vl, U, half, p, k), 255.0);
  }
}

bool finite_value(double x) { return std::isfinite(x); }

}  // namespace
}  // namespace gsb

using namespace gsb;

extern "C" {

int gsb_tsdf_raycast(const GsbVolume* vol, int32_t width, int32_t height, double fx, double fy, double cx, double cy,
                     const double* extrinsic_w2c, double depth_min, double depth_max, float* depth, float* normals,
                     float* colors, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (!vol || !extrinsic_w2c || !depth) return fail(GSB_ERR_INVALID, "tsdf_raycast: bad arguments");
  if (width <= 0 || height <= 0 || width > GSB_TSDF_MAX_WIDTH || height > GSB_TSDF_MAX_HEIGHT)
    return fail(GSB_ERR_INVALID, "tsdf_raycast: image %dx%d outside 1..%d x 1..%d (width x height)", width, height,
                GSB_TSDF_MAX_WIDTH, GSB_TSDF_MAX_HEIGHT);
  bool ok = finite_value(fx) && finite_value(fy) && finite_value(cx) && finite_value(cy) && finite_value(depth_min) && finite_value(depth_max);
  for (int k = 0; k < 16; ++k) ok = ok && finite_value(extrinsic_w2c[k]);
  if (!ok) return fail(GSB_ERR_INVALID, "tsdf_raycast: non-finite intrinsics, extrinsic or depth range");
  if (!(fx > 0.0 && fy > 0.0)) return fail(GSB_ERR_INVALID, "tsdf_raycast: fx and fy must be > 0");
  if (!(depth_min >= 0.0 && depth_min < depth_max))
    return fail(GSB_ERR_INVALID, "tsdf_raycast: the depth range needs 0 <= depth_min < depth_max");
  if (colors && !vol->d.color) return fail(GSB_ERR_INVALID, "tsdf_raycast: colours asked of a volume without colour");
  RayParams rp;
  rp.fx = fx;
  rp.fy = fy;
  rp.cx = cx;
  rp.cy = cy;
  for (int k = 0; k < 12; ++k) rp.E[k] = extrinsic_w2c[k];
  rp.zmin = depth_min;
  rp.zmax = depth_max;
  rp.tau = vol->d.sdf_trunc;
  rp.W = width;
  rp.H = height;
  const int32_t window[6] = {0, 0, 0, 1, 1, 1};  // the ray caster addresses bricks by lattice index only
  const VolView v = view_of(vol, window);
  const dim3 grid((unsigned)((width + kTileX - 1) / kTileX), (unsigned)((height + kTileY - 1) / kTileY));
  raycast_kernel<<<grid, dim3(kTileX, kTileY), 0, stream>>>(v, rp, depth, normals, colors);
  count_launch();
  return check_launch("raycast_kernel", stream, false);
}

}  // extern "C"
