// Shared host/device helpers for the gs2mesh_b200 CUDA library (sm_90a only).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <mutex>
#include <vector>

#include "gs2mesh_b200.h"

// Opaque handle of include/gs2mesh_b200.h: a copy of the caller's descriptor (owns no device memory).
struct GsbVolume {
  GsbVolumeDesc d;
  uint32_t frame = 0;
};

namespace gsb {

constexpr int kTile = 16;          // DGR/cuda_rasterizer/config.h:16-17 (BLOCK_X, BLOCK_Y)
constexpr int kTilePixels = 256;

extern thread_local char g_error[512];
extern std::atomic<uint64_t> g_launches;

inline int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_error, sizeof(g_error), fmt, ap);
  va_end(ap);
  return code;
}

inline void count_launch(uint64_t n = 1) { g_launches.fetch_add(n, std::memory_order_relaxed); }

#define GSB_CUDA_OK(expr)                                                                          \
  do {                                                                                             \
    cudaError_t e__ = (expr);                                                                      \
    if (e__ != cudaSuccess)                                                                        \
      return ::gsb::fail(GSB_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__),    \
                         __FILE__, __LINE__);                                                      \
  } while (0)

// Cheap launch check (cudaPeekAtLastError); with `sync` also waits for the stream, like the
// reference's debug mode (auxiliary.h:166-173).
inline int check_launch(const char* what, cudaStream_t s, bool sync) {
  cudaError_t e = cudaPeekAtLastError();
  if (e == cudaSuccess && sync) e = cudaStreamSynchronize(s);
  if (e != cudaSuccess) {
    cudaGetLastError();
    return fail(GSB_ERR_CUDA, "%s: %s", what, cudaGetErrorString(e));
  }
  return GSB_OK;
}

// ---------------------------------------------------------------------------------------------
// Optional per-stage device timing (bench.py's roofline numbers): CUDA events recorded on the
// launching stream around each stage when enabled; read back with gsb_profile_collect().
// ---------------------------------------------------------------------------------------------
enum Stage {
  kStPreprocess = 0,
  kStScan,
  kStEmit,
  kStSort,
  kStRanges,
  kStRender,
  kStToU8,
  kStDepthPrep,
  kStMarkBricks,
  kStIntegrate,
  kStMergeIndex,   // gsb_tsdf_reduce: brick index exchange (all-gather, union, broadcast) incl. the host read of the union size
  kStMergePack,    //                  pack + to-sums (in-place to-sums on the canonical rank)
  kStMergeReduce,  //                  the NCCL reduce / all-reduce of the payload
  kStMergeUnpack,  //                  from-sums (+ unpack) where the result lives
  kStCount
};

struct Profiler {
  std::atomic<bool> enabled{false};
  struct Rec {
    int stage;
    cudaEvent_t a, b;
  };
  std::mutex mu;
  std::vector<Rec> recs;
  std::vector<cudaEvent_t> pool;
  cudaEvent_t get() {
    if (!pool.empty()) {
      cudaEvent_t e = pool.back();
      pool.pop_back();
      return e;
    }
    cudaEvent_t e = nullptr;
    cudaEventCreate(&e);
    return e;
  }
};
extern Profiler g_prof;

struct StageTimer {
  cudaStream_t s;
  int stage;
  cudaEvent_t a = nullptr, b = nullptr;
  StageTimer(int stage_, cudaStream_t s_) : s(s_), stage(stage_) {
    if (!g_prof.enabled.load(std::memory_order_relaxed)) return;
    std::lock_guard<std::mutex> lk(g_prof.mu);
    a = g_prof.get();
    b = g_prof.get();
    cudaEventRecord(a, s);
  }
  ~StageTimer() {
    if (!a) return;
    cudaEventRecord(b, s);
    std::lock_guard<std::mutex> lk(g_prof.mu);
    g_prof.recs.push_back({stage, a, b});
  }
};

inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// blocks of `threads` threads that cover n items
inline unsigned blocks_for(long long n, int threads = 256) { return (unsigned)((n + threads - 1) / threads); }

// Mesh entries index vertices and triangles with 32-bit ids.  A mesh they accept has non-negative sizes, no triangles
// without vertices, at most kMaxMeshIds vertices and at most max_triangles triangles (kMaxMeshIds, or fewer where an entry
// keeps several ids per triangle).  mesh_size_error gives the refusal of a mesh mesh_sizes_ok rejects, prefixed `who: `.
constexpr int64_t kMaxMeshIds = 2147483647;

inline bool mesh_sizes_ok(int64_t nt, int64_t nv, int64_t max_triangles) {
  return nt >= 0 && nv >= 0 && nt <= max_triangles && nv <= kMaxMeshIds && (nt == 0 || nv > 0);
}

inline int mesh_size_error(const char* who, int64_t nt, int64_t nv, int64_t max_triangles) {
  if (nt < 0 || nv < 0)
    return fail(GSB_ERR_INVALID, "%s: negative size (n_triangles %lld, n_vertices %lld)", who, (long long)nt, (long long)nv);
  if (nt > 0 && nv == 0 && nt <= max_triangles)
    return fail(GSB_ERR_INVALID, "%s: %lld triangles but no vertices", who, (long long)nt);
  return fail(GSB_ERR_INVALID, "%s: %lld triangles / %lld vertices; ids are 32-bit (at most %lld triangles and %lld vertices)",
              who, (long long)nt, (long long)nv, (long long)max_triangles, (long long)kMaxMeshIds);
}

// ---------------------------------------------------------------------------------------------
// Brick hash of the TSDF volume (Open3D's unordered_map<Vector3i, VolumeUnit>): open addressing, linear probing,
// 64-bit keys = three 21-bit biased lattice indices.  An entry's position in the table identifies the brick inside a
// frame (work list, frame stamp); hash_vals[position] is its slot in the brick pool.
// ---------------------------------------------------------------------------------------------
constexpr unsigned long long kHashEmpty = ~0ull;
constexpr uint32_t kSlotNone = 0xffffffffu;   // key present, no pool slot (pool exhausted) / not found
constexpr int kBrickBias = 1 << 20;           // lattice indices in [-2^20, 2^20)

__host__ __device__ inline bool brick_key_ok(int bx, int by, int bz) {
  return bx >= -kBrickBias && bx < kBrickBias && by >= -kBrickBias && by < kBrickBias && bz >= -kBrickBias && bz < kBrickBias;
}
__host__ __device__ inline unsigned long long brick_key(int bx, int by, int bz) {
  return ((unsigned long long)(uint32_t)(bx + kBrickBias) << 42) | ((unsigned long long)(uint32_t)(by + kBrickBias) << 21) |
         (unsigned long long)(uint32_t)(bz + kBrickBias);
}
__host__ __device__ inline void brick_unkey(unsigned long long key, int& bx, int& by, int& bz) {
  bx = (int)((key >> 42) & 0x1fffffu) - kBrickBias;
  by = (int)((key >> 21) & 0x1fffffu) - kBrickBias;
  bz = (int)(key & 0x1fffffu) - kBrickBias;
}
__host__ __device__ inline uint32_t brick_hash(unsigned long long key, uint32_t mask) {
  key ^= key >> 33;  // splitmix64 finaliser
  key *= 0xff51afd7ed558ccdull;
  key ^= key >> 33;
  key *= 0xc4ceb9fe1a85ec53ull;
  key ^= key >> 33;
  return (uint32_t)key & mask;
}
// counters (uint32[8]): [0] entries queued this frame  [1] bricks dropped this frame (pool full)
//                       [2] brick-box cells outside the lattice this frame
//                       [4] pool slots in use (persistent)  [5] bricks dropped since creation (persistent)
//                       [6] brick-box cells outside the lattice since creation (persistent)
// Every drop and every out-of-range cell is added to its per-frame word and its persistent word with atomics where it is
// found, so no kernel folds one into the other.
constexpr int kCntQueued = 0, kCntDropped = 1, kCntOutOfRange = 2, kCntPool = 4, kCntDroppedTotal = 5, kCntOutOfRangeTotal = 6;

struct HashView {
  unsigned long long* keys;
  uint32_t* vals;
  uint32_t* stamp;
  int32_t* index;  // [pool][4]
  uint32_t mask, pool;
};

inline HashView hash_view(const GsbVolumeDesc& d) {
  HashView hv;
  hv.keys = reinterpret_cast<unsigned long long*>(d.hash_keys);
  hv.vals = d.hash_vals;
  hv.stamp = d.hash_stamp;
  hv.index = d.brick_index;
  hv.mask = d.hash_slots - 1u;
  hv.pool = d.pool_bricks;
  return hv;
}

// sums_pair in place over the pool slots in use among the first `bricks` (gsb_tsdf.cu): gsb_tsdf_to_sums / from_sums over
// the whole pool, the merge's canonical rank over the union at the front of its pool
int tsdf_sums(GsbVolume* vol, bool to_sums, uint32_t bricks, cudaStream_t stream);

#ifdef __CUDACC__
// position of `key` in the table, or kSlotNone
__device__ inline uint32_t brick_find(const unsigned long long* __restrict__ keys, uint32_t mask, unsigned long long key) {
  uint32_t h = brick_hash(key, mask);
  for (uint32_t probe = 0; probe <= mask; ++probe, h = (h + 1) & mask) {
    const unsigned long long k = keys[h];
    if (k == key) return h;
    if (k == kHashEmpty) return kSlotNone;
  }
  return kSlotNone;
}

__device__ __forceinline__ void count_dropped(uint32_t* counters) {
  atomicAdd(&counters[kCntDropped], 1u);
  atomicAdd(&counters[kCntDroppedTotal], 1u);
}
__device__ __forceinline__ void count_out_of_range(uint32_t* counters) {
  atomicAdd(&counters[kCntOutOfRange], 1u);
  atomicAdd(&counters[kCntOutOfRangeTotal], 1u);
}

// position of brick (bx,by,bz) in the table, inserting it (and giving it the next pool slot) if absent; kSlotNone if the
// brick cannot be stored.  The pool slot of a fresh key is written by the inserting thread with a plain store: readers of
// hash_vals are always a later kernel.  Threads that pass the pool check together can all insert; those whose slot lands
// past the pool leave a dead key (hash_vals = kSlotNone) and still return its position.  A dead key is therefore counted
// as dropped by whoever reads its slot: integrate_kernel, count_dead_kernel (touch), resolve_slots_kernel and
// insert_gathered_kernel (merge).
__device__ __forceinline__ uint32_t brick_find_or_insert(const HashView& hv, uint32_t* __restrict__ counters, int bx, int by,
                                                         int bz) {
  if (!brick_key_ok(bx, by, bz)) return kSlotNone;
  const unsigned long long key = brick_key(bx, by, bz);
  uint32_t h = brick_hash(key, hv.mask);
  for (uint32_t probe = 0; probe <= hv.mask; ++probe, h = (h + 1) & hv.mask) {
    unsigned long long k = hv.keys[h];
    if (k == kHashEmpty) {
      // pool exhausted: do not grow the table any further (racy by a few entries at most, bounded by the probe limit)
      if (*(volatile uint32_t*)&counters[kCntPool] >= hv.pool) return kSlotNone;
      k = atomicCAS(&hv.keys[h], kHashEmpty, key);
      if (k == kHashEmpty) {  // inserted: OpenVolumeUnit
        const uint32_t slot = atomicAdd(&counters[kCntPool], 1u);
        if (slot < hv.pool) {
          hv.vals[h] = slot;
          reinterpret_cast<int4*>(hv.index)[slot] = make_int4(bx, by, bz, 0);
        } else {
          hv.vals[h] = kSlotNone;
          atomicSub(&counters[kCntPool], 1u);
        }
        return h;
      }
    }
    if (k == key) return h;
  }
  return kSlotNone;
}

// (mean, weight) <-> (sum, weight) of one voxel pair in registers, the one statement of the conversion: v = (tsdf0, w0,
// tsdf1, w1), c[k] the colour of voxel k (with_color).  to_sums: tsdf*w, rgb*w; else tsdf/w (0 where w is 0), rgb/w.
// Callers skip a pair whose two weights are 0 (it is not stored back in place), and the colour of a voxel of weight 0 is
// not converted (callers need not load it).  Skipping gives the bits converting would give, because a voxel of weight 0
// holds tsdf 0 and colour 0: pools start zero-filled, integrate_kernel writes only the voxels it fuses and fuse_voxel
// leaves them with weight >= 1, and the merge's from-sums step writes tsdf 0 and a colour of 0 where the summed weight is
// 0 (a sum of weights >= 0 is 0 only if every rank's weight was, and so were their tsdf and colour).
__device__ __forceinline__ void sums_pair(float4& v, float4 (&c)[2], bool with_color, bool to_sums) {
  const float w0 = v.y, w1 = v.w;
  if (to_sums) {
    v.x *= w0;
    v.z *= w1;
  } else {
    v.x = w0 > 0.f ? v.x / w0 : 0.f;
    v.z = w1 > 0.f ? v.z / w1 : 0.f;
  }
  if (!with_color) return;
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    const float w = k ? w1 : w0;
    if (w == 0.f) continue;
    if (to_sums) {
      c[k].x *= w;
      c[k].y *= w;
      c[k].z *= w;
    } else {
      c[k].x /= w;
      c[k].y /= w;
      c[k].z /= w;
    }
  }
}
#endif

// Carves consecutive 256-byte aligned regions out of one caller-owned block.
struct Carver {
  char* base;
  size_t off = 0;
  explicit Carver(void* p) : base(static_cast<char*>(p)) {}
  template <typename T>
  T* take(size_t count) {
    off = align_up(off, 256);
    T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
    off += count * sizeof(T);
    return p;
  }
  size_t total() const { return align_up(off, 256); }
};

}  // namespace gsb
