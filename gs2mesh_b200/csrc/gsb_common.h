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
