// Stable LSD radix sort building block for (uint32 key, uint32 value) pairs, 8-bit digits.
//
// Replaces cub::DeviceRadixSort in the rasterizer's binning stage (the reference sorts R
// 64-bit tile|depth keys in ~6 passes, rasterizer_impl.cu:303-308).  Here the ordering work is
// split so that the R-sized stream is only touched for the tile bits:
//   1. the P Gaussians are sorted by view depth (4 passes over P, P << R);
//   2. instances are emitted in that order (tile id, Gaussian id);
//   3. a stable sort on the tile id alone (2 passes for <= 65536 tiles) groups them per tile while
//      preserving the (depth, index) order inside every tile.
// A sort = one histogram kernel (all digits of all passes in a single read of the keys) + ONE
// kernel per pass: block-local stable ranking with warp match-any votes, block offsets by chained
// (decoupled look-back) prefix over per-block status words, items staged in digit order in shared
// memory and written out in runs.
#pragma once

#include "gsb_common.h"

namespace gsb {
namespace {

constexpr int kRdxThreads = 256;
constexpr int kRdxWarps = kRdxThreads / 32;
constexpr int kRdxItems = 16;                          // items per thread of the R-sized (instance) sorts
constexpr int kRdxBlock = kRdxThreads * kRdxItems;     // 4096 items per CTA
constexpr int kRdxBins = 256;
constexpr int kRdxMaxPasses = 4;
constexpr int kRdxWindow = 8;                          // predecessors inspected per look-back round
constexpr int kRdxSmallItems = 8;                      // items per thread of small sorts
constexpr size_t kRdxSmallSort = 1u << 22;             // sorts of up to 4M items count as "small" (the P-sized depth sort)

// status word of (block, digit): [31:30] 0 = not ready, 1 = block aggregate, 2 = inclusive prefix
constexpr uint32_t kStAgg = 1u << 30, kStIncl = 2u << 30, kStVal = (1u << 30) - 1u;

// Number of items the sort works on: host value, or a device counter clamped by `capacity`
// (0 when the frame overflowed its workspace: counters[2] != 0).
__device__ __forceinline__ uint32_t radix_count(uint32_t n_host, const unsigned long long* counters, int64_t capacity) {
  if (counters == nullptr) return n_host;
  if (counters[2] != 0) return 0u;
  const unsigned long long n = counters[1];
  return (int64_t)n > capacity ? 0u : (uint32_t)n;
}

// Digit histograms of every pass in one read of the keys: ghist[pass][digit].
template <int kItems>
__global__ void __launch_bounds__(kRdxThreads) radix_histogram_kernel(const uint32_t* __restrict__ keys, uint32_t n_host,
                                                                     const unsigned long long* __restrict__ counters,
                                                                     int64_t capacity, int passes, int digit_bits,
                                                                     uint32_t* __restrict__ ghist) {
  __shared__ uint32_t hist[kRdxMaxPasses][kRdxBins];
  const uint32_t dmask = (1u << digit_bits) - 1u;
  const uint32_t n = radix_count(n_host, counters, capacity);
  const uint32_t base = blockIdx.x * (kRdxThreads * kItems);
  if (base >= n) return;
  for (int p = 0; p < passes; ++p) hist[p][threadIdx.x] = 0;
  __syncthreads();
  uint32_t kreg[kItems];
#pragma unroll
  for (int k = 0; k < kItems; ++k) {  // every load in flight before the first vote waits for one
    const uint32_t i = base + k * kRdxThreads + threadIdx.x;
    kreg[k] = i < n ? keys[i] : 0u;
  }
#pragma unroll
  for (int k = 0; k < kItems; ++k) {
    const uint32_t i = base + k * kRdxThreads + threadIdx.x;
    const uint32_t wbase = i - (threadIdx.x & 31);  // first item of this warp's 32
    if (wbase + 32 <= n) {
      // full warp.  Depth keys of one view share their upper bytes, tile ids of neighbouring instances their
      // upper byte: when all 32 lanes agree on a digit one lane adds 32 instead of 32 serialised atomics.
      const uint32_t key = kreg[k];
      for (int p = 0; p < passes; ++p) {
        const uint32_t dgt = (key >> (digit_bits * p)) & dmask;
        int same;
        __match_all_sync(0xffffffffu, dgt, &same);
        if (same) {
          if ((threadIdx.x & 31) == 0) atomicAdd(&hist[p][dgt], 32u);
        } else {
          atomicAdd(&hist[p][dgt], 1u);
        }
      }
    } else if (i < n) {
      const uint32_t key = kreg[k];
      for (int p = 0; p < passes; ++p) atomicAdd(&hist[p][(key >> (digit_bits * p)) & dmask], 1u);
    }
  }
  __syncthreads();
  for (int p = 0; p < passes; ++p) {
    const uint32_t c = hist[p][threadIdx.x];
    if (c) atomicAdd(&ghist[p * kRdxBins + threadIdx.x], c);
  }
}

__device__ __forceinline__ uint32_t ld_status(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_status(uint32_t* p, uint32_t v) {
  asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// One stable pass.  `ghist` = this pass's 256 global digit counts, `status` = [nblocks][256] words and
// `ticket` = block-order counter, both zeroed before the sort.  When `ranges` != NULL this is the last
// pass of the tile sort: keys are then fully sorted tile ids and the first / last instance of every
// tile seen by the block updates ranges[tile] = (start, end) with atomicMin / atomicMax.
// kItems = items per thread: 16 for the R-sized instance sorts; the P-sized depth sort, whose whole grid is co-resident
// and therefore runs at the latency of ONE block, uses 8 (more, shorter critical paths).
template <int kItems>
__global__ void __launch_bounds__(kRdxThreads, kItems >= 16 ? 3 : 4) radix_pass_kernel(const uint32_t* __restrict__ keys_in,
                                                                const uint32_t* __restrict__ vals_in,
                                                                uint32_t* __restrict__ keys_out,
                                                                uint32_t* __restrict__ vals_out, uint32_t n_host,
                                                                const unsigned long long* __restrict__ counters,
                                                                int64_t capacity, int shift, uint32_t dmask,
                                                                const uint32_t* __restrict__ ghist,
                                                                uint32_t* __restrict__ status, uint32_t* __restrict__ ticket,
                                                                uint2* __restrict__ ranges, int write_keys,
                                                                const uint32_t* __restrict__ gather_src,
                                                                uint32_t* __restrict__ gather_dst,
                                                                const uint32_t* __restrict__ gather_src2,
                                                                uint32_t* __restrict__ gather_dst2) {
  constexpr int kBlock = kRdxThreads * kItems;
  __shared__ uint32_t s_key[kBlock];
  __shared__ uint32_t s_val[kBlock];
  __shared__ uint32_t warp_hist[kRdxWarps][kRdxBins];  // per-warp digit counts -> per-warp bases
  __shared__ uint32_t digit_start[kRdxBins];           // first local slot of each digit in this block
  __shared__ uint32_t global_off[kRdxBins];            // global output position of that slot
  __shared__ uint32_t scan_tmp[kRdxWarps];
  __shared__ uint32_t s_bid;

  const uint32_t n = radix_count(n_host, counters, capacity);
  // blocks are numbered in arrival order, so every predecessor of a block is already running
  if (threadIdx.x == 0) s_bid = atomicAdd(ticket, 1u);
#pragma unroll
  for (int w = 0; w < kRdxWarps; ++w) warp_hist[w][threadIdx.x] = 0;
  __syncthreads();
  const uint32_t bid = s_bid;
  const uint32_t base = bid * kBlock;
  if (base >= n) return;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t lt_mask = (1u << lane) - 1u;
  const uint32_t count = min((uint32_t)kBlock, n - base);

  // ---- phase 1: each warp walks its contiguous (32 * kItems)-item segment in order and ranks its items
  uint32_t key[kItems], val[kItems];
  uint32_t lrank[kItems];  // rank among same-digit items of this warp's segment
  const uint32_t seg = base + warp * (kBlock / kRdxWarps);
  // (a) every load of the thread is issued before anything waits for one
#pragma unroll
  for (int k = 0; k < kItems; ++k) {
    const uint32_t i = seg + k * 32 + lane;
    const bool ok = i < n;
    key[k] = ok ? keys_in[i] : 0xffffffffu;
    val[k] = ok ? (vals_in != nullptr ? vals_in[i] : i) : 0u;  // no payload array: the payload is the item's index
  }
  // (b) same-digit groups of each 32-item row (independent votes, pipelined)
  uint32_t peers[kItems];
#pragma unroll
  for (int k = 0; k < kItems; ++k) {
    const bool ok = seg + k * 32 + lane < n;
    const uint32_t d = ok ? ((key[k] >> shift) & dmask) : (uint32_t)kRdxBins;  // 256 = "no item"
    peers[k] = __match_any_sync(0xffffffffu, d);
  }
  // (c) one shared-memory atomic per group, by its lowest lane, rows in order: the value it returns is the number of
  //     same-digit items in the warp's earlier rows.  __syncwarp() orders the atomics of consecutive rows (their
  //     leaders may be different lanes); nothing waits for a returned value inside this loop.
#pragma unroll
  for (int k = 0; k < kItems; ++k) {
    const bool ok = seg + k * 32 + lane < n;
    uint32_t before = 0;
    if (ok && (peers[k] & lt_mask) == 0)
      before = atomicAdd(&warp_hist[warp][(key[k] >> shift) & dmask], (uint32_t)__popc(peers[k]));
    lrank[k] = before;
    __syncwarp();
  }
  // (d) the group's count-before comes from its leader
#pragma unroll
  for (int k = 0; k < kItems; ++k) {
    const uint32_t before = __shfl_sync(0xffffffffu, lrank[k], __ffs(peers[k]) - 1);
    lrank[k] = before + __popc(peers[k] & lt_mask);
  }
  __syncthreads();

  // ---- phase 2: thread d owns digit d
  {
    const int d = threadIdx.x;
    uint32_t run = 0;
#pragma unroll
    for (int w = 0; w < kRdxWarps; ++w) {
      const uint32_t c = warp_hist[w][d];
      warp_hist[w][d] = run;  // base of warp w inside digit d
      run += c;
    }
    // publish this block's count of digit d, then chain back over the predecessors
    uint32_t* my = status + (size_t)bid * kRdxBins + d;
    st_status(my, (bid == 0 ? kStIncl : kStAgg) | run);
    uint32_t prev = 0;
    if (bid > 0) {
      // Windowed look-back: the status words of kRdxWindow predecessors are requested at once (independent
      // loads), then consumed newest-first.  When every block of a pass starts at the same time (the whole
      // P-sized grid is co-resident) a one-word-at-a-time walk costs ~nblocks/2 dependent L2 round trips;
      // this cuts the chain by the window length.  Every word is self-contained (flag + count), so a
      // speculative read of an older word is valid whatever state the newer ones were in.
      bool closed = false;
      for (int64_t b = (int64_t)bid - 1; !closed; b -= kRdxWindow) {
        uint32_t sv[kRdxWindow];
#pragma unroll
        for (int j = 0; j < kRdxWindow; ++j)
          sv[j] = b - j >= 0 ? ld_status(status + (size_t)(b - j) * kRdxBins + d) : kStIncl;  // before block 0: prefix 0
#pragma unroll
        for (int j = 0; j < kRdxWindow; ++j) {
          if (!closed) {
            uint32_t v = sv[j];
            for (uint32_t spin = 0; (v >> 30) == 0; ++spin) {
              if (spin > (1u << 24)) __trap();  // a predecessor never published: fail loudly instead of hanging
              v = ld_status(status + (size_t)(b - j) * kRdxBins + d);
            }
            prev += v & kStVal;
            closed = (v >> 30) == 2;
          }
        }
      }
      st_status(my, kStIncl | (prev + run));
    }
    // local digit starts: exclusive scan of `run` over the 256 digits
    uint32_t incl = run;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += v;
    }
    if (lane == 31) scan_tmp[warp] = incl;
    __syncthreads();
    uint32_t wbase = 0;
#pragma unroll
    for (int w = 0; w < kRdxWarps; ++w)
      if (w < warp) wbase += scan_tmp[w];
    digit_start[d] = wbase + incl - run;
    __syncthreads();
    // global digit base: exclusive scan of the global histogram over the 256 digits
    const uint32_t tot = ghist[d];
    uint32_t tincl = tot;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t v = __shfl_up_sync(0xffffffffu, tincl, o);
      if (lane >= o) tincl += v;
    }
    if (lane == 31) scan_tmp[warp] = tincl;
    __syncthreads();
    uint32_t tbase = 0;
#pragma unroll
    for (int w = 0; w < kRdxWarps; ++w)
      if (w < warp) tbase += scan_tmp[w];
    global_off[d] = tbase + tincl - tot + prev;
  }
  __syncthreads();

  // ---- phase 3: stage the block's items in digit order
#pragma unroll
  for (int k = 0; k < kItems; ++k) {
    const uint32_t i = seg + k * 32 + lane;
    if (i < n) {
      const uint32_t d = (key[k] >> shift) & dmask;
      const uint32_t slot = digit_start[d] + warp_hist[warp][d] + lrank[k];
      s_key[slot] = key[k];
      s_val[slot] = val[k];
    }
  }
  __syncthreads();

  // ---- phase 4: write runs (consecutive slots of one digit go to consecutive addresses)
  for (uint32_t sidx = threadIdx.x; sidx < count; sidx += kRdxThreads) {
    const uint32_t kk = s_key[sidx];
    const uint32_t d = (kk >> shift) & dmask;
    const uint32_t dst = global_off[d] + (sidx - digit_start[d]);
    if (write_keys) keys_out[dst] = kk;  // nobody reads the keys of a sort's last pass
    const uint32_t vv = s_val[sidx];
    vals_out[dst] = vv;
    if (gather_dst != nullptr) gather_dst[dst] = gather_src[vv];  // a per-value attribute, delivered in sorted order
    if (gather_dst2 != nullptr) gather_dst2[dst] = gather_src2[vv];
    if (ranges != nullptr) {
      // slots are in ascending tile order inside the block (stable LSD => low digit sorted within high digit)
      if (sidx == 0 || s_key[sidx - 1] != kk) atomicMin(&ranges[kk].x, dst);
      if (sidx + 1 == count || s_key[sidx + 1] != kk) atomicMax(&ranges[kk].y, dst + 1);
    }
  }
}

// Items per thread of a sort over at most `max_items` items.
inline int radix_items_for(size_t max_items) { return max_items <= kRdxSmallSort ? kRdxSmallItems : kRdxItems; }
inline size_t radix_blocks_for(size_t max_items) {
  const size_t block = (size_t)kRdxThreads * radix_items_for(max_items);
  return (max_items + block - 1) / block;
}

// Bits per digit of a sort over `bits` key bits: the passes share the bits evenly (13 tile-id bits -> 7 + 6 instead
// of 8 + 5: fewer, longer same-digit runs per block in the first pass).
inline int radix_digit_bits(int bits) {
  const int passes = (bits + 7) / 8;
  return (bits + passes - 1) / passes;
}

// Scratch words one sort needs for `max_items` items.  Sized for blocks of 4 items per thread, half the smallest block
// either sort uses: a margin that keeps every gsb_raster_workspace_bytes value as it was.
inline size_t radix_scratch_words(size_t max_items) {
  const size_t nblocks = (max_items + kRdxThreads * 4 - 1) / (kRdxThreads * 4);
  return (size_t)kRdxMaxPasses * (kRdxBins + nblocks * kRdxBins + 1) + 64;
}

// Scratch layout: ghist [kRdxMaxPasses][256] | tickets [64] | status [passes][nblocks][256]
inline uint32_t* radix_ghist(uint32_t* scratch) { return scratch; }

// Zeroes the histogram / ticket / status words one sort over `max_items` items with `bits` key bits needs.
inline void radix_prepare(uint32_t* scratch, size_t max_items, int bits, cudaStream_t stream) {
  const size_t nblocks = radix_blocks_for(max_items);
  const int passes = (bits + 7) / 8;
  const size_t words = (size_t)kRdxMaxPasses * kRdxBins + 64 + (size_t)passes * nblocks * kRdxBins;
  cudaMemsetAsync(scratch, 0, words * sizeof(uint32_t), stream);
}

// Enqueues ceil(bits/8) stable passes sorting (keys, vals) by key bits [0, bits).  identity_payload: the payload of item i
// is i (the first pass synthesises it instead of reading vals_a).  gather_dst != NULL: the last pass also writes
// gather_dst[j] = gather_src[value of sorted item j] (likewise gather_dst2 / gather_src2).  `a`/`b` are
// ping-pong buffers; returns which buffer holds the result (0 = a, 1 = b).  n is either the host
// value (counters == NULL) or read on the device from counters[1] (clamped by capacity).
// histogram_ready: the caller already ran radix_prepare() and filled the digit histograms.
template <int kItems>
inline int radix_sort_pairs_t(uint32_t* keys_a, uint32_t* vals_a, uint32_t* keys_b, uint32_t* vals_b, uint32_t n_host,
                              const unsigned long long* counters, int64_t capacity, size_t max_items, int bits,
                              uint32_t* scratch, uint2* ranges_on_last_pass, cudaStream_t stream, uint64_t* launches,
                              bool histogram_ready, const uint32_t* gather_src, uint32_t* gather_dst,
                              const uint32_t* gather_src2, uint32_t* gather_dst2, bool identity_payload) {
  const uint32_t nblocks = (uint32_t)radix_blocks_for(max_items);
  if (nblocks == 0) return 0;
  const int passes = (bits + 7) / 8;
  const int db = radix_digit_bits(bits);
  uint32_t* ghist = scratch;                                    // [kRdxMaxPasses][256]
  uint32_t* tickets = ghist + kRdxMaxPasses * kRdxBins;          // [64]
  uint32_t* status = tickets + 64;                               // [passes][nblocks][256]
  if (!histogram_ready) {
    radix_prepare(scratch, max_items, bits, stream);
    radix_histogram_kernel<kItems><<<nblocks, kRdxThreads, 0, stream>>>(keys_a, n_host, counters, capacity, passes, db, ghist);
    *launches += 1;
  }
  int cur = 0;
  for (int p = 0; p < passes; ++p) {
    const uint32_t* kin = cur ? keys_b : keys_a;
    const uint32_t* vin = (p == 0 && identity_payload) ? nullptr : (cur ? vals_b : vals_a);
    uint32_t* kout = cur ? keys_a : keys_b;
    uint32_t* vout = cur ? vals_a : vals_b;
    radix_pass_kernel<kItems><<<nblocks, kRdxThreads, 0, stream>>>(
        kin, vin, kout, vout, n_host, counters, capacity, db * p, (1u << db) - 1u, ghist + p * kRdxBins,
        status + (size_t)p * nblocks * kRdxBins,
        tickets + p, p == passes - 1 ? ranges_on_last_pass : nullptr, p != passes - 1,
        gather_src, p == passes - 1 ? gather_dst : nullptr, gather_src2, p == passes - 1 ? gather_dst2 : nullptr);
    *launches += 1;
    cur ^= 1;
  }
  return cur;
}

inline int radix_sort_pairs(uint32_t* keys_a, uint32_t* vals_a, uint32_t* keys_b, uint32_t* vals_b, uint32_t n_host,
                            const unsigned long long* counters, int64_t capacity, size_t max_items, int bits,
                            uint32_t* scratch, uint2* ranges_on_last_pass, cudaStream_t stream, uint64_t* launches,
                            bool histogram_ready, const uint32_t* gather_src = nullptr, uint32_t* gather_dst = nullptr,
                            const uint32_t* gather_src2 = nullptr, uint32_t* gather_dst2 = nullptr,
                            bool identity_payload = false) {
  const auto sort = radix_items_for(max_items) == kRdxSmallItems ? radix_sort_pairs_t<kRdxSmallItems> : radix_sort_pairs_t<kRdxItems>;
  return sort(keys_a, vals_a, keys_b, vals_b, n_host, counters, capacity, max_items, bits, scratch, ranges_on_last_pass, stream,
              launches, histogram_ready, gather_src, gather_dst, gather_src2, gather_dst2, identity_payload);
}

}  // namespace
}  // namespace gsb
