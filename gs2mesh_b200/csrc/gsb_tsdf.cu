// TSDF integration for sm_90a: Open3D's ScalableTSDFVolume (what gs2mesh_utils/tsdf_utils.py:53-56,107 drives) as an
// UNBOUNDED brick store -- a pool of 16^3-voxel bricks addressed through a device hash table keyed by the integer lattice
// index of the brick, allocated on first touch exactly like Open3D's unordered_map<Vector3i, VolumeUnit>.
//
// The reference integrates through Open3D 0.17.0 (CPU): per frame it back-projects every
// 4th pixel, opens all 16^3 "volume units" within +-sdf_trunc of those points and runs
// UniformTSDFVolume::IntegrateWithDepthToCameraDistanceMultiplier on each unit once
// (SURVEY.md rows T1/T2).  Here the same two steps are two kernels:
//
//   mark_bricks   one thread per sampled pixel; fp64 back-projection (Open3D builds the point
//                 cloud in double), brick box of the point +- trunc, find-or-insert of every brick of the box in the
//                 hash (a new key takes the next pool slot), de-duplication with a per-entry frame stamp (atomicExch)
//                 and an append-only work list of hash entries.  Nothing waits: an entry's pool slot is only read by the
//                 next kernel.
//   integrate     persistent CTAs pull entries from the list.  A brick is 32 KB of contiguous
//                 (tsdf, weight) pairs: thread t owns voxel pairs (2 consecutive z) and moves
//                 them with 16-byte loads/stores, 8 independent loads in flight per thread.
//                 Projection, truncated distance and the running weighted mean are fused; the
//                 depth-to-camera-distance multiplier is recomputed instead of read.
//
// fp32 arithmetic uses explicit round-to-nearest intrinsics (no FMA contraction) in Open3D's
// operation order, so results are bit-identical to oracle/tsdf_oracle.cpp.
#include "gsb_common.h"


namespace gsb {
namespace {

struct MarkParams {
  int W, H, nsx, nsy;
  double fx, fy, cx, cy;
  double pose[12];  // rows 0..2 of extrinsic^-1 (camera -> world)
  double trunc, unit_length;
};

__global__ void __launch_bounds__(256) mark_bricks_kernel(const MarkParams m, const HashView hv, const float* __restrict__ depth,
                                                          uint32_t* __restrict__ list, uint32_t* __restrict__ counters,
                                                          uint32_t frame) {
  // entries this CTA queues: collected in shared memory and appended to the frame's work list with ONE global atomic per
  // CTA (every append used to bump the same global counter: ~2200 same-address atomics per frame, serialised in L2)
  constexpr int kLocal = 1024;
  __shared__ uint32_t s_list[kLocal];
  __shared__ uint32_t s_n, s_base;
  if (threadIdx.x == 0) s_n = 0;
  __syncthreads();
  auto append = [&](uint32_t h) {
    const uint32_t k = atomicAdd(&s_n, 1u);
    if (k < (uint32_t)kLocal)
      s_list[k] = h;
    else
      list[atomicAdd(&counters[kCntQueued], 1u)] = h;  // more than the CTA's buffer holds: straight to the list
  };
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  const int lane = threadIdx.x & 31;
  bool valid = s < m.nsx * m.nsy;
  int lo[3] = {0, 0, 0}, hi[3] = {-1, -1, -1};
  if (valid) {
    const int i = (s / m.nsx) * 4, j = (s % m.nsx) * 4;  // depth_sampling_stride = 4
    const float p = depth[(size_t)i * m.W + j];
    valid = p > 0.f;
    if (valid) {
      // PointCloudFactory.cpp CreatePointCloudFromFloatDepthImage, all in double
      const double z = (double)p;
      const double x = __ddiv_rn(__dmul_rn((double)j - m.cx, z), m.fx);
      const double y = __ddiv_rn(__dmul_rn((double)i - m.cy, z), m.fy);
#pragma unroll
      for (int r = 0; r < 3; ++r) {
        const double w = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(m.pose[4 * r], x), __dmul_rn(m.pose[4 * r + 1], y)),
                                             __dmul_rn(m.pose[4 * r + 2], z)),
                                   m.pose[4 * r + 3]);
        lo[r] = (int)floor(__ddiv_rn(__dadd_rn(w, -m.trunc), m.unit_length));
        hi[r] = (int)floor(__ddiv_rn(__dadd_rn(w, m.trunc), m.unit_length));
      }
    }
  }
  // The 32 samples of a warp are neighbours on an image row: their boxes mostly name the same few bricks.  The warp walks
  // the boxes in lockstep; lanes that hold the same brick elect one of them (match.any), and only that lane touches the hash
  // table -- about a tenth of the probes, stamp reads and atomics of one-probe-per-sample.
  const int nx = hi[0] - lo[0] + 1, ny = hi[1] - lo[1] + 1, nz = hi[2] - lo[2] + 1;
  const int total = valid ? nx * ny * nz : 0;
  int most = total;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) most = max(most, __shfl_xor_sync(0xffffffffu, most, o));
  // Three box cells per trip: their votes and the leaders' first probes are independent, so the memory round trips of a trip
  // overlap (the kernel is one warp's chain of dependent L2 accesses: 39 us with one cell per trip on C1).
  constexpr int kPer = 3;
  for (int i0 = 0; i0 < most; i0 += kPer) {
    unsigned long long key[kPer], seen[kPer];
    uint32_t h[kPer], st[kPer];
    int bx[kPer], by[kPer], bz[kPer];
    bool lead[kPer];
#pragma unroll
    for (int u = 0; u < kPer; ++u) {
      const int i = i0 + u;
      key[u] = kHashEmpty;
      seen[u] = kHashEmpty;
      h[u] = 0;
      st[u] = 0;
      bx[u] = by[u] = bz[u] = 0;
      bool mine = i < total;
      if (mine) {
        bz[u] = lo[2] + i % nz;
        by[u] = lo[1] + (i / nz) % ny;
        bx[u] = lo[0] + i / (nz * ny);
        if (brick_key_ok(bx[u], by[u], bz[u])) {
          key[u] = brick_key(bx[u], by[u], bz[u]);
        } else {
          count_out_of_range(counters);  // not a pool drop: a larger pool cannot hold it
          mine = false;
        }
      }
      const unsigned peers = __match_any_sync(0xffffffffu, key[u]);
      lead[u] = mine && (int)(__ffs(peers) - 1) == lane;  // lanes naming the same brick elect the lowest one
      if (lead[u]) {  // first probe at the home slot + its stamp, issued before anything waits
        h[u] = brick_hash(key[u], hv.mask);
        seen[u] = hv.keys[h[u]];
        st[u] = hv.stamp[h[u]];
      }
    }
#pragma unroll
    for (int u = 0; u < kPer; ++u) {
      if (!lead[u]) continue;
      uint32_t hh = h[u];
      if (seen[u] != key[u]) {  // not at its home slot (collision or not yet opened): walk / insert
        hh = brick_find_or_insert(hv, counters, bx[u], by[u], bz[u]);
        if (hh == kSlotNone) {
          count_dropped(counters);  // reported by gsb_tsdf_last_stats; the stage class grows the pool
          continue;
        }
        st[u] = hv.stamp[hh];
      }
      if (st[u] == frame) continue;
      if (atomicExch(&hv.stamp[hh], frame) != frame) append(hh);
    }
  }
  __syncthreads();
  const uint32_t n_local = min(s_n, (uint32_t)kLocal);
  if (threadIdx.x == 0 && n_local) s_base = atomicAdd(&counters[kCntQueued], n_local);
  __syncthreads();
  for (uint32_t k = threadIdx.x; k < n_local; k += blockDim.x) list[s_base + k] = s_list[k];
}

struct FrameParams {
  float E[12];  // rows 0..2 of the world->camera extrinsic, cast to float
  float fx, fy, cx, cy, inv_fx, inv_fy;
  float vl, half, trunc, trunc_inv;
  float sx, sy, sz;  // E(:,2) * voxel_length
  float safe_w, safe_h;
  int W, H;
  double unit_length;
};

__device__ __forceinline__ float4 ld_stream(const float4* p) {
  float4 v;
  asm volatile("ld.global.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
  return v;
}
__device__ __forceinline__ void st_stream(float4* p, const float4& v) {
  asm volatile("st.global.L1::no_allocate.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

// UniformTSDFVolume::IntegrateWithDepthToCameraDistanceMultiplier, one voxel, split in two so that
// the depth-image gathers of all of a thread's voxels can be in flight together:
//   project_voxel: camera-space point -> packed pixel (v << 16 | u), or -1 if the voxel is skipped.  The packing holds
//                  u < 65536 and v < 32768 (GSB_TSDF_MAX_WIDTH / _HEIGHT, checked by the entry points), and then
//                  v * W + u < 2^31 as well.
//   fuse_voxel:    depth sample -> truncated distance -> running weighted mean
__device__ __forceinline__ int project_voxel(const FrameParams& f, float pcx, float pcy, float pcz) {
  if (pcz <= 0.f) return -1;
  const float u_f = __fadd_rn(__fadd_rn(__fdiv_rn(__fmul_rn(pcx, f.fx), pcz), f.cx), 0.5f);
  const float v_f = __fadd_rn(__fadd_rn(__fdiv_rn(__fmul_rn(pcy, f.fy), pcz), f.cy), 0.5f);
  if (!(u_f >= 0.0001f && u_f < f.safe_w && v_f >= 0.0001f && v_f < f.safe_h)) return -1;
  return ((int)v_f << 16) | (int)u_f;
}
// depth sample -> truncated distance `t` of one voxel; false if the voxel is not updated by this frame.  The decision does
// not depend on the stored (tsdf, weight), so it is taken BEFORE the volume is read and only updated voxels are loaded.
__device__ __forceinline__ bool sample_voxel(const FrameParams& f, int uv, float d, float pcz, float& t) {
  if (uv < 0 || d <= 0.0f) return false;
  const int u = uv & 0xffff, v = uv >> 16;
  // CreateDepthToCameraDistanceMultiplierFloatImage, recomputed per lookup
  const float xx = __fmul_rn(__fsub_rn((float)u, f.cx), f.inv_fx);
  const float yy = __fmul_rn(__fsub_rn((float)v, f.cy), f.inv_fy);
  const float mult = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(xx, xx), __fmul_rn(yy, yy)), 1.0f));
  const float sdf = __fmul_rn(__fsub_rn(d, pcz), mult);
  if (!(sdf > -f.trunc)) return false;
  t = fminf(1.0f, __fmul_rn(sdf, f.trunc_inv));
  return true;
}
// running weighted mean of one voxel (tsdf, weight) and its colour
__device__ __forceinline__ void fuse_voxel(float t, float& tsdf, float& w) {
  tsdf = __fdiv_rn(__fadd_rn(__fmul_rn(tsdf, w), t), __fadd_rn(w, 1.0f));
  w = __fadd_rn(w, 1.0f);
}
__device__ __forceinline__ void fuse_color(float4& c, float w_before, uint32_t rgb) {
  const float r = (float)(rgb & 0xffu), g = (float)((rgb >> 8) & 0xffu), b = (float)((rgb >> 16) & 0xffu);
  const float den = __fadd_rn(w_before, 1.0f);
  c.x = __fdiv_rn(__fadd_rn(__fmul_rn(c.x, w_before), r), den);
  c.y = __fdiv_rn(__fadd_rn(__fmul_rn(c.y, w_before), g), den);
  c.z = __fdiv_rn(__fadd_rn(__fmul_rn(c.z, w_before), b), den);
}
__device__ __forceinline__ uint32_t load_rgb(const uint8_t* __restrict__ rgb, int pix) {
  const uint8_t* p = rgb + 3 * (size_t)pix;
  return (uint32_t)__ldg(p) | (uint32_t)__ldg(p + 1) << 8 | (uint32_t)__ldg(p + 2) << 16;
}

constexpr int kIntThreads = 256;
constexpr int kPasses = GSB_BRICK_VOXELS / 2 / kIntThreads;  // 8 voxel-pair passes per brick
constexpr int kSweep = 2;                                    // passes handled together (4 voxels per thread)

// One brick per CTA iteration, in sweeps of kSweep voxel-pair passes:
//   (A) project the sweep's voxels, all depth gathers in flight (image reads hit L2)
//   (B) per voxel: updated by this frame? -> t.  Threads with nothing to update skip the rest of the sweep.
//   (C) loads of the UPDATED pairs only: (tsdf, weight), colour, rgb -- all in flight together
//   (D) fuse + store
// ~60% of the voxels of a touched brick lie outside the truncation band and are never read or written.
// Compiled for 4 CTAs per SM: 64 registers and a few spilled bytes at sm_90a, where 3 CTAs would give 80 and no spills.
__global__ void __launch_bounds__(kIntThreads, 4) integrate_kernel(const FrameParams f, const float* __restrict__ depth,
                                                                   const uint8_t* __restrict__ rgb, float4* __restrict__ tw,
                                                                   float4* __restrict__ color,
                                                                   const uint32_t* __restrict__ list,
                                                                   uint32_t* __restrict__ counters,
                                                                   const unsigned long long* __restrict__ hash_keys,
                                                                   const uint32_t* __restrict__ hash_vals, uint32_t pool) {
  // a frame cannot queue more entries than the list holds (one per pool slot + the few a full pool refused)
  const uint32_t n = counters[kCntQueued];
  const int t = threadIdx.x;
  // thread -> voxel pair: pair q = pass*256 + t, first voxel 2q = (x, y, z) with
  //   x = 2*pass + (t >> 7), y = (t >> 3) & 15, z = 2 * (t & 7)
  const int y = (t >> 3) & 15, z0 = 2 * (t & 7), xo = t >> 7;
  const bool with_color = color != nullptr && rgb != nullptr;
  for (uint32_t it = blockIdx.x; it < n; it += gridDim.x) {
    const uint32_t entry = list[it];
    const uint32_t brick = hash_vals[entry];  // pool slot
    if (brick >= pool) {                      // dead key: the pool was full when this brick was opened
      if (t == 0) count_dropped(counters);   // each entry is listed once per frame, so counted once per frame
      continue;
    }
    int bx, by, bz;
    brick_unkey(hash_keys[entry], bx, by, bz);
    const double ox = (double)bx * f.unit_length;  // origin = index * unit_length (OpenVolumeUnit)
    const double oy = (double)by * f.unit_length;
    const double oz = (double)bz * f.unit_length;
    float4* base = tw + (size_t)brick * (GSB_BRICK_VOXELS / 2) + t;
    float4* cbase = color + ((size_t)brick * GSB_BRICK_VOXELS + 2 * (size_t)t);
    const float py = (float)((double)__fadd_rn(f.half, __fmul_rn(f.vl, (float)y)) + oy);
    const float pz = (float)((double)f.half + oz);
    // the y/z part of extrinsic * (px,py,pz,1) is the same for all passes; the reference adds the four products left to right,
    // so only the products (not their sum) can be hoisted
    const float e1y = __fmul_rn(f.E[1], py), e2z = __fmul_rn(f.E[2], pz);
    const float e5y = __fmul_rn(f.E[5], py), e6z = __fmul_rn(f.E[6], pz);
    const float e9y = __fmul_rn(f.E[9], py), e10z = __fmul_rn(f.E[10], pz);
#pragma unroll 1
    for (int s = 0; s < kPasses; s += kSweep) {
      int uv[kSweep][2];
      float cz[kSweep][2];
#pragma unroll
      for (int p = 0; p < kSweep; ++p) {
        const int x = 2 * (s + p) + xo;
        const float px = (float)((double)__fadd_rn(f.half, __fmul_rn(f.vl, (float)x)) + ox);
        // pt_camera = extrinsic * (px,py,pz,1), then z0 incremental steps along the brick's z axis
        float cxm = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(f.E[0], px), e1y), e2z), f.E[3]);
        float cym = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(f.E[4], px), e5y), e6z), f.E[7]);
        float czm = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(f.E[8], px), e9y), e10z), f.E[11]);
        for (int k = 0; k < z0; ++k) {
          cxm = __fadd_rn(cxm, f.sx);
          cym = __fadd_rn(cym, f.sy);
          czm = __fadd_rn(czm, f.sz);
        }
        uv[p][0] = project_voxel(f, cxm, cym, czm);
        cz[p][0] = czm;
        cxm = __fadd_rn(cxm, f.sx);
        cym = __fadd_rn(cym, f.sy);
        czm = __fadd_rn(czm, f.sz);
        uv[p][1] = project_voxel(f, cxm, cym, czm);
        cz[p][1] = czm;
      }
      float dd[kSweep][2];
#pragma unroll
      for (int p = 0; p < kSweep; ++p)
#pragma unroll
        for (int e = 0; e < 2; ++e)
          dd[p][e] = uv[p][e] >= 0 ? __ldg(depth + (uv[p][e] >> 16) * f.W + (uv[p][e] & 0xffff)) : 0.f;
      uint32_t upd = 0;  // bit 2p+e
      float tt[kSweep][2];
#pragma unroll
      for (int p = 0; p < kSweep; ++p)
#pragma unroll
        for (int e = 0; e < 2; ++e) upd |= (sample_voxel(f, uv[p][e], dd[p][e], cz[p][e], tt[p][e]) ? 1u : 0u) << (2 * p + e);
      if (upd == 0) continue;

      float4 v[kSweep];
      float4 c[kSweep][2];
      uint32_t px8[kSweep][2];
#pragma unroll
      for (int p = 0; p < kSweep; ++p)
        if (upd >> (2 * p) & 3u) v[p] = ld_stream(base + (s + p) * kIntThreads);
      if (with_color) {
#pragma unroll
        for (int p = 0; p < kSweep; ++p)
#pragma unroll
          for (int e = 0; e < 2; ++e)
            if (upd >> (2 * p + e) & 1u) {
              c[p][e] = ld_stream(cbase + 2 * (size_t)((s + p) * kIntThreads) + e);
              px8[p][e] = load_rgb(rgb, (uv[p][e] >> 16) * f.W + (uv[p][e] & 0xffff));
            }
      }
#pragma unroll
      for (int p = 0; p < kSweep; ++p) {
        if (!(upd >> (2 * p) & 3u)) continue;
        const float w0 = v[p].y, w1 = v[p].w;
        if (upd >> (2 * p) & 1u) fuse_voxel(tt[p][0], v[p].x, v[p].y);
        if (upd >> (2 * p + 1) & 1u) fuse_voxel(tt[p][1], v[p].z, v[p].w);
        st_stream(base + (s + p) * kIntThreads, v[p]);
        if (with_color) {
          if (upd >> (2 * p) & 1u) {
            fuse_color(c[p][0], w0, px8[p][0]);
            st_stream(cbase + 2 * (size_t)((s + p) * kIntThreads), c[p][0]);
          }
          if (upd >> (2 * p + 1) & 1u) {
            fuse_color(c[p][1], w1, px8[p][1]);
            st_stream(cbase + 2 * (size_t)((s + p) * kIntThreads) + 1, c[p][1]);
          }
        }
      }
    }
  }
}

__global__ void __launch_bounds__(256) prepare_depth_kernel(const float* __restrict__ in, const float* __restrict__ final_T,
                                                            const uint8_t* __restrict__ mask, size_t n, float alpha_min,
                                                            float min_depth, float depth_scale, double depth_trunc,
                                                            float* __restrict__ out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float d = in[i];
  if (final_T) {
    const float alpha = 1.0f - final_T[i];
    d = alpha > alpha_min ? __fdiv_rn(d, alpha) : 0.f;
  }
  if (mask) d = d * (float)mask[i];
  if (d < min_depth) d = 0.f;          // tsdf_utils.py:83
  d = __fdiv_rn(d, depth_scale);       // ConvertDepthToFloatImage
  if ((double)d >= depth_trunc) d = 0.f;
  out[i] = d;
}

// k x k rectangular min (erode) / max (dilate) filter over a uint8 mask with OpenCV's window: anchor k/2, i.e. offsets
// -(k/2) .. k-1-k/2 on both axes, pixels outside the image ignored (cv2.erode / cv2.dilate / MORPH_CLOSE with the default
// border value; tsdf_utils.py:73-77).  One 64x16 output tile per CTA: halo tile -> smem, row pass, column pass.
constexpr int kMorphTX = 64, kMorphTY = 16, kMorphMaxK = 64;
__global__ void __launch_bounds__(256) morph_kernel(const uint8_t* __restrict__ in, uint8_t* __restrict__ out, int W, int H, int k,
                                                    int dilate) {
  extern __shared__ uint8_t morph_sm[];
  const int tw = kMorphTX + k - 1, th = kMorphTY + k - 1;
  uint8_t* tile = morph_sm;            // [th][tw]
  uint8_t* rows = morph_sm + th * tw;  // [th][kMorphTX]
  const int ax = k / 2;
  const int x0 = blockIdx.x * kMorphTX - ax, y0 = blockIdx.y * kMorphTY - ax;
  const uint8_t neutral = dilate ? 0 : 255;
  for (int i = threadIdx.x; i < th * tw; i += blockDim.x) {
    const int x = x0 + i % tw, y = y0 + i / tw;
    tile[i] = (x >= 0 && x < W && y >= 0 && y < H) ? in[(size_t)y * W + x] : neutral;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < th * kMorphTX; i += blockDim.x) {
    const uint8_t* src = tile + (i / kMorphTX) * tw + i % kMorphTX;
    uint8_t v = neutral;
    for (int j = 0; j < k; ++j) v = dilate ? max(v, src[j]) : min(v, src[j]);
    rows[i] = v;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < kMorphTY * kMorphTX; i += blockDim.x) {
    const int lx = i % kMorphTX, ly = i / kMorphTX;
    const int x = blockIdx.x * kMorphTX + lx, y = blockIdx.y * kMorphTY + ly;
    if (x >= W || y >= H) continue;
    uint8_t v = neutral;
    for (int j = 0; j < k; ++j) {
      const uint8_t s = rows[(ly + j) * kMorphTX + lx];
      v = dilate ? max(v, s) : min(v, s);
    }
    out[(size_t)y * W + x] = v;
  }
}

// sums_pair in place over the voxel pairs [0, n_pairs) of the pool slots in use
__global__ void __launch_bounds__(256) sums_kernel(float4* __restrict__ tw, float4* __restrict__ color, size_t n_pairs, int to_sums,
                                                   const uint32_t* __restrict__ counters) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_pairs || i / (GSB_BRICK_VOXELS / 2) >= counters[kCntPool]) return;
  float4 v = tw[i];
  if (v.y == 0.f && v.w == 0.f) return;
  float4 c[2];
  if (color)
#pragma unroll
    for (int k = 0; k < 2; ++k)
      if ((k ? v.w : v.y) != 0.f) c[k] = color[2 * i + k];
  sums_pair(v, c, color != nullptr, to_sums);
  tw[i] = v;
  if (color)
#pragma unroll
    for (int k = 0; k < 2; ++k)
      if ((k ? v.w : v.y) != 0.f) color[2 * i + k] = c[k];
}

// Window of the lattice -> dense x*NY*NZ + y*NZ + z grids (Open3D UniformTSDFVolume indexing); unallocated bricks read as 0.
__global__ void __launch_bounds__(256) export_dense_kernel(const float2* __restrict__ tw, const unsigned long long* __restrict__ keys,
                                                           const uint32_t* __restrict__ vals, uint32_t mask, uint32_t pool, int b0x,
                                                           int b0y, int b0z, int nbx, int nby, int nbz, float* __restrict__ tsdf,
                                                           float* __restrict__ weight) {
  const size_t n = (size_t)nbx * nby * nbz * GSB_BRICK_VOXELS;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;  // (window brick, voxel) index
  if (i >= n) return;
  const size_t wb = i / GSB_BRICK_VOXELS;
  const int vi = (int)(i % GSB_BRICK_VOXELS);
  const int bz = (int)(wb % nbz), by = (int)((wb / nbz) % nby), bx = (int)(wb / ((size_t)nbz * nby));
  const int x = bx * 16 + (vi >> 8), y = by * 16 + ((vi >> 4) & 15), z = bz * 16 + (vi & 15);
  const size_t o = ((size_t)x * (nby * 16) + y) * (nbz * 16) + z;
  float2 v = make_float2(0.f, 0.f);
  if (brick_key_ok(b0x + bx, b0y + by, b0z + bz)) {
    const uint32_t h = brick_find(keys, mask, brick_key(b0x + bx, b0y + by, b0z + bz));
    const uint32_t slot = h == kSlotNone ? kSlotNone : vals[h];
    if (slot < pool) v = tw[(size_t)slot * GSB_BRICK_VOXELS + vi];
  }
  if (tsdf) tsdf[o] = v.x;
  if (weight) weight[o] = v.y;
}

// lattice indices -> pool slots (kSlotNone if absent); insert != 0 opens missing bricks (zero-filled, like OpenVolumeUnit)
__global__ void __launch_bounds__(256) find_bricks_kernel(const HashView hv, uint32_t* __restrict__ counters,
                                                          const int32_t* __restrict__ indices, uint32_t n,
                                                          const uint32_t* __restrict__ n_dev, int insert,
                                                          uint32_t* __restrict__ slots, uint32_t* __restrict__ entries) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || (n_dev != nullptr && i >= *n_dev)) return;
  const int bx = indices[4 * (size_t)i], by = indices[4 * (size_t)i + 1], bz = indices[4 * (size_t)i + 2];
  uint32_t h = kSlotNone;
  if (insert && !brick_key_ok(bx, by, bz)) {
    count_out_of_range(counters);
  } else if (insert) {
    h = brick_find_or_insert(hv, counters, bx, by, bz);
    if (h == kSlotNone) count_dropped(counters);  // a dead key (h != kSlotNone) is counted by resolve_slots_kernel
  } else if (brick_key_ok(bx, by, bz)) {
    h = brick_find(hv.keys, hv.mask, brick_key(bx, by, bz));
  }
  if (entries) entries[i] = h;
  if (slots) slots[i] = kSlotNone;  // resolved by resolve_slots_kernel once every insertion of this launch has landed
}
// insert != 0: an entry without a pool slot (a dead key, found or just left by brick_find_or_insert) is a dropped brick
__global__ void __launch_bounds__(256) resolve_slots_kernel(const uint32_t* __restrict__ vals, const uint32_t* __restrict__ entries,
                                                            uint32_t n, const uint32_t* __restrict__ n_dev, uint32_t pool,
                                                            int insert, uint32_t* __restrict__ counters,
                                                            uint32_t* __restrict__ slots) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || (n_dev != nullptr && i >= *n_dev)) return;
  const uint32_t h = entries[i];
  const uint32_t s = h == kSlotNone ? kSlotNone : vals[h];
  if (insert && h != kSlotNone && s >= pool) count_dropped(counters);
  slots[i] = s < pool ? s : kSlotNone;
}

// gsb_tsdf_touch: the dead keys among the frame's listed entries (integrate_kernel counts them itself when it runs)
__global__ void __launch_bounds__(256) count_dead_kernel(const uint32_t* __restrict__ list, const uint32_t* __restrict__ vals,
                                                         uint32_t pool, uint32_t* __restrict__ counters) {
  const uint32_t n = counters[kCntQueued];
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    if (vals[list[i]] >= pool) count_dropped(counters);
}

__global__ void copy_stats_kernel(uint32_t* counters, uint32_t frame, uint32_t* out) {
  out[0] = counters[kCntQueued];
  out[1] = counters[kCntDropped];
  out[2] = frame;
  out[3] = counters[kCntPool];
  out[4] = counters[kCntDroppedTotal];
  out[5] = counters[kCntOutOfRange];
  out[6] = counters[kCntOutOfRangeTotal];
  out[7] = 0;
}

// general 4x4 inverse in double (Gauss-Jordan with partial pivoting)
bool invert4(const double* m, double* out) {
  double a[4][8];
  for (int r = 0; r < 4; ++r)
    for (int c = 0; c < 4; ++c) {
      a[r][c] = m[4 * r + c];
      a[r][4 + c] = r == c ? 1.0 : 0.0;
    }
  for (int c = 0; c < 4; ++c) {
    int piv = c;
    for (int r = c + 1; r < 4; ++r)
      if (fabs(a[r][c]) > fabs(a[piv][c])) piv = r;
    if (a[piv][c] == 0.0) return false;
    if (piv != c)
      for (int k = 0; k < 8; ++k) {
        double tmp = a[c][k];
        a[c][k] = a[piv][k];
        a[piv][k] = tmp;
      }
    const double d = a[c][c];
    for (int k = 0; k < 8; ++k) a[c][k] /= d;
    for (int r = 0; r < 4; ++r)
      if (r != c) {
        const double fct = a[r][c];
        for (int k = 0; k < 8; ++k) a[r][k] -= fct * a[c][k];
      }
  }
  for (int r = 0; r < 4; ++r)
    for (int c = 0; c < 4; ++c) out[4 * r + c] = a[r][4 + c];
  return true;
}

// SM count of the current device, which sizes the persistent grids launched on it
int num_sms() {
  int dev = 0, n = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return 132;
  return n;
}

}  // namespace

int tsdf_sums(GsbVolume* vol, bool to_sums, uint32_t bricks, cudaStream_t stream) {
  if (!vol) return fail(GSB_ERR_INVALID, "tsdf: volume is NULL");
  const size_t n_pairs = (size_t)(bricks < vol->d.pool_bricks ? bricks : vol->d.pool_bricks) * (GSB_BRICK_VOXELS / 2);
  if (n_pairs == 0) return GSB_OK;
  sums_kernel<<<(unsigned)((n_pairs + 255) / 256), 256, 0, stream>>>(reinterpret_cast<float4*>(vol->d.tsdf_weight),
                                                                     reinterpret_cast<float4*>(vol->d.color), n_pairs, to_sums,
                                                                     vol->d.counters);
  count_launch();
  return check_launch("sums_kernel", stream, false);
}

}  // namespace gsb

using namespace gsb;

extern "C" {

GsbVolume* gsb_tsdf_create(const GsbVolumeDesc* desc) {
  if (!desc || !desc->tsdf_weight || !desc->brick_index || !desc->hash_keys || !desc->hash_vals || !desc->hash_stamp ||
      !desc->brick_list || !desc->counters) {
    fail(GSB_ERR_INVALID, "tsdf_create: tsdf_weight, brick_index, hash_keys, hash_vals, hash_stamp, brick_list and counters are required");
    return nullptr;
  }
  if (desc->pool_bricks == 0 || desc->pool_bricks > 0x7fffffffu) {
    fail(GSB_ERR_INVALID, "tsdf_create: pool_bricks must be in 1 .. 2^31-1");
    return nullptr;
  }
  if (desc->hash_slots < 2 * (uint64_t)desc->pool_bricks || (desc->hash_slots & (desc->hash_slots - 1u)) != 0) {
    fail(GSB_ERR_INVALID, "tsdf_create: hash_slots must be a power of two >= 2 * pool_bricks");
    return nullptr;
  }
  if (!(desc->voxel_length > 0) || !(desc->sdf_trunc > 0)) {
    fail(GSB_ERR_INVALID, "tsdf_create: voxel_length and sdf_trunc must be positive");
    return nullptr;
  }
  GsbVolume* v = new GsbVolume();
  v->d = *desc;
  return v;
}

void gsb_tsdf_destroy(GsbVolume* vol) { delete vol; }

int gsb_tsdf_prepare_depth(const float* depth_in, const float* final_T, const uint8_t* mask, int32_t width, int32_t height,
                           float alpha_min, float min_depth, double depth_scale, double depth_trunc, float* depth_out,
                           void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (!depth_in || !depth_out || width <= 0 || height <= 0) return fail(GSB_ERR_INVALID, "prepare_depth: bad arguments");
  const size_t n = (size_t)width * height;
  {
    StageTimer tm(kStDepthPrep, stream);
    prepare_depth_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(depth_in, final_T, mask, n, alpha_min, min_depth,
                                                                          (float)depth_scale, depth_trunc, depth_out);
  }
  count_launch();
  return check_launch("prepare_depth_kernel", stream, false);
}

int gsb_mask_morphology(const uint8_t* mask_in, int32_t width, int32_t height, int32_t kernel_size, int32_t dilate, uint8_t* mask_out,
                        void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (!mask_in || !mask_out || mask_in == mask_out || width <= 0 || height <= 0)
    return fail(GSB_ERR_INVALID, "mask_morphology: bad arguments (in-place filtering is not supported)");
  if (kernel_size < 1 || kernel_size > kMorphMaxK) return fail(GSB_ERR_INVALID, "mask_morphology: kernel_size must be in 1..64");
  const int tw = kMorphTX + kernel_size - 1, th = kMorphTY + kernel_size - 1;
  const size_t smem = (size_t)th * tw + (size_t)th * kMorphTX;
  dim3 grid((width + kMorphTX - 1) / kMorphTX, (height + kMorphTY - 1) / kMorphTY);
  morph_kernel<<<grid, 256, smem, stream>>>(mask_in, mask_out, width, height, kernel_size, dilate != 0);
  count_launch();
  return check_launch("morph_kernel", stream, false);
}

// block discovery of one frame (T1): opens every brick within +-sdf_trunc of the sampled depth points and queues it
static int run_mark(GsbVolume* vol, const float* depth, int32_t width, int32_t height, double fx, double fy, double cx, double cy,
                    const double* extrinsic, cudaStream_t stream, double* unit_length_out) {
  const GsbVolumeDesc& d = vol->d;
  double pose[16];
  if (!invert4(extrinsic, pose)) return fail(GSB_ERR_INVALID, "tsdf_integrate: extrinsic is singular");
  vol->frame += 1;
  if (vol->frame == 0) {  // stamp wrap-around: start over
    GSB_CUDA_OK(cudaMemsetAsync(d.hash_stamp, 0, (size_t)d.hash_slots * sizeof(uint32_t), stream));
    vol->frame = 1;
  }
  GSB_CUDA_OK(cudaMemsetAsync(d.counters, 0, 4 * sizeof(uint32_t), stream));  // the per-frame words; [4..] persist

  MarkParams m{};
  m.W = width;
  m.H = height;
  m.nsx = (width + 3) / 4;
  m.nsy = (height + 3) / 4;
  m.fx = fx;
  m.fy = fy;
  m.cx = cx;
  m.cy = cy;
  for (int k = 0; k < 12; ++k) m.pose[k] = pose[k];
  m.trunc = d.sdf_trunc;
  m.unit_length = d.voxel_length * GSB_BRICK;
  *unit_length_out = m.unit_length;
  const int ns = m.nsx * m.nsy;
  {
    StageTimer tm(kStMarkBricks, stream);
    mark_bricks_kernel<<<(ns + 255) / 256, 256, 0, stream>>>(m, hash_view(d), depth, d.brick_list, d.counters, vol->frame);
  }
  count_launch();
  return check_launch("mark_bricks_kernel", stream, false);
}

// the packed pixel index of integrate_kernel (project_voxel) holds u < 65536, v < 32768
static int check_frame_size(const char* fn, int32_t width, int32_t height) {
  if (width > GSB_TSDF_MAX_WIDTH || height > GSB_TSDF_MAX_HEIGHT)
    return fail(GSB_ERR_INVALID, "%s: frame %dx%d exceeds the supported %dx%d (width x height)", fn, width, height,
                GSB_TSDF_MAX_WIDTH, GSB_TSDF_MAX_HEIGHT);
  return GSB_OK;
}

int gsb_tsdf_touch(GsbVolume* vol, const float* depth, int32_t width, int32_t height, double fx, double fy, double cx, double cy,
                   const double* extrinsic, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (!vol || !depth || !extrinsic || width <= 0 || height <= 0) return fail(GSB_ERR_INVALID, "tsdf_touch: bad arguments");
  int rc;
  if ((rc = check_frame_size("tsdf_touch", width, height))) return rc;
  double unit_length = 0;
  if ((rc = run_mark(vol, depth, width, height, fx, fy, cx, cy, extrinsic, stream, &unit_length))) return rc;
  count_dead_kernel<<<num_sms(), 256, 0, stream>>>(vol->d.brick_list, vol->d.hash_vals, vol->d.pool_bricks, vol->d.counters);
  count_launch();
  return check_launch("count_dead_kernel", stream, false);
}

int gsb_tsdf_integrate(GsbVolume* vol, const float* depth, const uint8_t* rgb, int32_t width, int32_t height, double fx,
                       double fy, double cx, double cy, const double* extrinsic, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (!vol || !depth || !extrinsic || width <= 0 || height <= 0) return fail(GSB_ERR_INVALID, "tsdf_integrate: bad arguments");
  if (int rc = check_frame_size("tsdf_integrate", width, height)) return rc;
  const GsbVolumeDesc& d = vol->d;
  double unit_length = 0;
  int rc;
  if ((rc = run_mark(vol, depth, width, height, fx, fy, cx, cy, extrinsic, stream, &unit_length))) return rc;

  FrameParams f{};
  for (int k = 0; k < 12; ++k) f.E[k] = (float)extrinsic[k];
  f.fx = (float)fx;
  f.fy = (float)fy;
  f.cx = (float)cx;
  f.cy = (float)cy;
  f.inv_fx = 1.0f / f.fx;
  f.inv_fy = 1.0f / f.fy;
  f.vl = (float)d.voxel_length;
  f.half = f.vl * 0.5f;
  f.trunc = (float)d.sdf_trunc;
  f.trunc_inv = 1.0f / f.trunc;
  f.sx = f.E[2] * f.vl;
  f.sy = f.E[6] * f.vl;
  f.sz = f.E[10] * f.vl;
  f.safe_w = width - 0.0001f;
  f.safe_h = height - 0.0001f;
  f.W = width;
  f.H = height;
  f.unit_length = unit_length;
  const size_t resident = (size_t)num_sms() * 8;
  const int grid = (int)(resident < (size_t)d.pool_bricks ? resident : (size_t)d.pool_bricks);
  const unsigned long long* hkeys = reinterpret_cast<const unsigned long long*>(d.hash_keys);
  {
    StageTimer tm(kStIntegrate, stream);
    integrate_kernel<<<grid, kIntThreads, 0, stream>>>(f, depth, rgb, reinterpret_cast<float4*>(d.tsdf_weight),
                                                       reinterpret_cast<float4*>(d.color), d.brick_list, d.counters, hkeys,
                                                       d.hash_vals, d.pool_bricks);
  }
  count_launch();
  return check_launch("integrate_kernel", stream, false);
}

int gsb_tsdf_to_sums(GsbVolume* vol, void* stream) { return tsdf_sums(vol, true, UINT32_MAX, static_cast<cudaStream_t>(stream)); }
int gsb_tsdf_from_sums(GsbVolume* vol, void* stream) { return tsdf_sums(vol, false, UINT32_MAX, static_cast<cudaStream_t>(stream)); }

int gsb_tsdf_export_dense(const GsbVolume* vol, const int32_t* brick_origin, const int32_t* brick_count, float* tsdf, float* weight,
                          void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (!vol || !brick_origin || !brick_count || (!tsdf && !weight)) return fail(GSB_ERR_INVALID, "tsdf_export_dense: bad arguments");
  for (int k = 0; k < 3; ++k)
    if (brick_count[k] <= 0) return fail(GSB_ERR_INVALID, "tsdf_export_dense: brick_count must be positive");
  const size_t n = (size_t)brick_count[0] * brick_count[1] * brick_count[2] * GSB_BRICK_VOXELS;
  if (n > 0xffffffffull * 256) return fail(GSB_ERR_INVALID, "tsdf_export_dense: window too large");
  const GsbVolumeDesc& d = vol->d;
  export_dense_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(
      reinterpret_cast<const float2*>(d.tsdf_weight), reinterpret_cast<const unsigned long long*>(d.hash_keys), d.hash_vals,
      d.hash_slots - 1u, d.pool_bricks, brick_origin[0], brick_origin[1], brick_origin[2], brick_count[0], brick_count[1],
      brick_count[2], tsdf, weight);
  count_launch();
  return check_launch("export_dense_kernel", stream, false);
}

int gsb_tsdf_find_bricks(GsbVolume* vol, const int32_t* indices, uint32_t n, int insert, uint32_t* slots, uint32_t* scratch,
                         void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (!vol || (n && (!indices || !slots || !scratch))) return fail(GSB_ERR_INVALID, "tsdf_find_bricks: bad arguments");
  if (n == 0) return GSB_OK;
  const GsbVolumeDesc& d = vol->d;
  find_bricks_kernel<<<(n + 255) / 256, 256, 0, stream>>>(hash_view(d), d.counters, indices, n, nullptr, insert, slots, scratch);
  resolve_slots_kernel<<<(n + 255) / 256, 256, 0, stream>>>(d.hash_vals, scratch, n, nullptr, d.pool_bricks, insert, d.counters,
                                                            slots);
  count_launch(2);
  return check_launch("find_bricks_kernel", stream, false);
}

int gsb_tsdf_last_stats(const GsbVolume* vol, uint32_t* out, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (!vol || !out) return fail(GSB_ERR_INVALID, "tsdf_last_stats: bad arguments");
  copy_stats_kernel<<<1, 1, 0, stream>>>(vol->d.counters, vol->frame, out);
  count_launch();
  return check_launch("copy_stats_kernel", stream, false);
}

}  // extern "C"
