// Read-only view of the brick TSDF volume for the extraction kernels (mesh: gsb_mesh.cu, point clouds:
// gsb_pointcloud.cu): the pool, its hash, and the key window the extraction's 64-bit keys index.
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
