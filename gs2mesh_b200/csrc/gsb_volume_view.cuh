// Read-only view of the brick TSDF volume for the read-out kernels (mesh: gsb_mesh.cu, point clouds: gsb_pointcloud.cu,
// ray casting: gsb_raycast.cu): the pool, its hash, the key window the extraction's 64-bit keys index, and the
// GetTSDFAt interpolation the point clouds and the ray caster share.
#pragma once

#include "gs2mesh_b200.h"
#include "gsb_common.h"

namespace gsb {

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

// ---------------------------------------------------------------------------------------------------------------------
// ScalableTSDFVolume::GetTSDFAt's cube, in double with one rounding per operation (point clouds: gsb_pointcloud.cu, ray
// casting: gsb_raycast.cu).  For a point p: q = p - vl/2, the unit index0 = floor(q / U) (U = 16 vl), the grid position
// g = (q - index0 * U) / vl, the base voxel c = clamp(floor(g), 0, 15) and the trilinear weights r = g - c.  The eight
// corners c + kMcShift[i] past 15 lie in the +1 units.

// The unit of p - vl/2 as doubles fl[3] (floors compared before any conversion, so no position overflows an int), and
// whether it lies inside the lattice range [-2^20, 2^20).
__device__ __forceinline__ bool unit_of(double U, double half, const double p[3], double q[3], double fl[3]) {
  bool in = true;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    q[k] = __dsub_rn(p[k], half);
    fl[k] = floor(__ddiv_rn(q[k], U));
    in = in && fl[k] >= -(double)kBrickBias && fl[k] < (double)kBrickBias;
  }
  return in;
}

// base voxel c and trilinear weights r of q inside the unit fl
__device__ __forceinline__ void cube_in_unit(double vl, double U, const double q[3], const double fl[3], int c[3], double r[3]) {
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const double g = __ddiv_rn(__dsub_rn(q[k], __dmul_rn(fl[k], U)), vl);
    c[k] = min(max((int)floor(g), 0), GSB_BRICK - 1);
    r[k] = __dsub_rn(g, (double)c[k]);
  }
}

// pool slot and voxel offset of corner i of the cube (c in unit i0, slot s0); kSlotNone when its unit is not open
__device__ __forceinline__ uint32_t cube_corner(const VolView& v, const int i0[3], uint32_t s0, const int c[3], int i,
                                                uint32_t& voxel) {
  // corners in kMcShift order: (0,0,0) (1,0,0) (1,1,0) (0,1,0) (0,0,1) (1,0,1) (1,1,1) (0,1,1)
  constexpr int sx[8] = {0, 1, 1, 0, 0, 1, 1, 0}, sy[8] = {0, 0, 1, 1, 0, 0, 1, 1}, sz[8] = {0, 0, 0, 0, 1, 1, 1, 1};
  const int x = c[0] + sx[i], y = c[1] + sy[i], z = c[2] + sz[i];
  voxel = ((x & 15) * 16 + (y & 15)) * 16 + (z & 15);
  return (x | y | z) < GSB_BRICK ? s0 : slot_of_brick(v, i0[0] + (x >> 4), i0[1] + (y >> 4), i0[2] + (z >> 4));
}

// Open3D's trilinear sum over the eight corner values, in its order
__device__ __forceinline__ double cube_trilinear(const double f[8], const double r[3]) {
  const double a0 = __dsub_rn(1.0, r[0]), a1 = __dsub_rn(1.0, r[1]), a2 = __dsub_rn(1.0, r[2]);
  const double lo = __dadd_rn(__dmul_rn(a1, __dadd_rn(__dmul_rn(a2, f[0]), __dmul_rn(r[2], f[4]))),
                              __dmul_rn(r[1], __dadd_rn(__dmul_rn(a2, f[3]), __dmul_rn(r[2], f[7]))));
  const double hi = __dadd_rn(__dmul_rn(a1, __dadd_rn(__dmul_rn(a2, f[1]), __dmul_rn(r[2], f[5]))),
                              __dmul_rn(r[1], __dadd_rn(__dmul_rn(a2, f[2]), __dmul_rn(r[2], f[6]))));
  return __dadd_rn(__dmul_rn(a0, lo), __dmul_rn(r[0], hi));
}

// ScalableTSDFVolume::GetTSDFAt(p): a missing unit gives 0.0 for the whole sample, a missing +1 unit 0 for its corners;
// weights are not consulted.  kColor: the same interpolation of colour channel `ch` instead of the tsdf.
template <bool kColor = false>
__device__ double tsdf_at(const VolView& v, double vl, double U, double half, const double p[3], int ch = 0) {
  double q[3], fl[3], r[3];
  int c[3];
  if (!unit_of(U, half, p, q, fl)) return 0.0;
  const int i0[3] = {(int)fl[0], (int)fl[1], (int)fl[2]};
  const uint32_t s0 = slot_of_brick(v, i0[0], i0[1], i0[2]);
  if (s0 == kSlotNone) return 0.0;
  cube_in_unit(vl, U, q, fl, c, r);
  double f[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    uint32_t voxel;
    const uint32_t slot = cube_corner(v, i0, s0, c, i, voxel);
    const size_t a = (size_t)slot * GSB_BRICK_VOXELS + voxel;
    f[i] = slot == kSlotNone ? 0.0 : kColor ? (double)(&v.color[a].x)[ch] : (double)v.tw[a].x;
  }
  return cube_trilinear(f, r);
}

// ScalableTSDFVolume::GetNormalAt(p).normalized(): n(j) = GetTSDFAt(p + h e_j) - GetTSDFAt(p - h e_j), h = 0.99 vl;
// Eigen's normalized() divides by sqrt((x*x + y*y) + z*z) only when that is > 0.
__device__ __forceinline__ void tsdf_normal(const VolView& v, double vl, double U, double half, const double p[3],
                                            double nv[3]) {
  const double h = __dmul_rn(0.99, vl);
#pragma unroll 1
  for (int j = 0; j < 3; ++j) {
    double pm[3] = {p[0], p[1], p[2]}, pp[3] = {p[0], p[1], p[2]};
    pm[j] = __dsub_rn(pm[j], h);
    pp[j] = __dadd_rn(pp[j], h);
    nv[j] = __dsub_rn(tsdf_at(v, vl, U, half, pp), tsdf_at(v, vl, U, half, pm));
  }
  const double sq = __dadd_rn(__dadd_rn(__dmul_rn(nv[0], nv[0]), __dmul_rn(nv[1], nv[1])), __dmul_rn(nv[2], nv[2]));
  if (sq > 0.0) {
    const double len = __dsqrt_rn(sq);
#pragma unroll
    for (int j = 0; j < 3; ++j) nv[j] = __ddiv_rn(nv[j], len);
  }
}

inline VolView view_of(const GsbVolume* vol, const int32_t* window) {
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
inline int window_check(const char* who, const int32_t* w) {
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

}  // namespace gsb
