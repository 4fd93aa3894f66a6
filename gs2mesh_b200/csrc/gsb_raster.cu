// Forward Gaussian-splat rasterizer for sm_90a (H100).
//
// Behavioural contract = the reference's forward pass
//   DGR/cuda_rasterizer/rasterizer_impl.cu:198-336 (Rasterizer::forward)
//   DGR/cuda_rasterizer/forward.cu:155-256 (preprocess), :261-374 (render)
// (DGR = third_party/gaussian-splatting/submodules/diff-gaussian-rasterization), called twice per stereo pair by
// gs2mesh_utils/renderer_utils.py:378-389 -- but the pipeline is organised differently:
//
//   preprocess   one WARP per 32 consecutive Gaussians, ONE launch for both eyes of a stereo pair.  The warp's parameter
//                block is contiguous in every reference tensor ([P,3] xyz / scales, [P,4] quaternions,
//                [P] opacities, [P,M,3] SH = 6 KB per warp) and is staged into shared memory once
//                with 1-D bulk TMA copies (cp.async.bulk + mbarrier); the 3-D covariance is computed once; projection,
//                binning and SH shading run per eye.  The 6 KB SH block is only fetched when at least one Gaussian of the
//                warp survives culling in some eye, and is read back with 16-byte loads.  Per eye three coalesced record
//                planes: recA = (px, py, z_view, opacity)  recB = (conic a, b, c, red)  recC = (green, blue)
//   binning      exact (Gaussian,tile) test: a pair is kept only if the tile's pixel lattice can
//                reach alpha >= 1/255 -- the image is bit-identical to rectangle binning
//                (rasterizer_impl.cu:88-107) with far fewer instances to sort and blend.
//   sort         the reference's order inside a tile is (depth bits, Gaussian index) ascending
//                (stable radix sort of tile << 32 | depth keys emitted in index order).  Here: stable
//                LSD radix sort of the P (depth bits, index) pairs -- ONE sort per pair when both eyes see every Gaussian at
//                the same view depth --, a one-pass scan of the tile counts in that order, instances emitted in that order,
//                then a stable sort of the R instances on the tile id alone (gsb_radix.cuh).
//   render       per 16x16 tile, four warps that never wait for each other: each streams the tile's
//                list, keeps the records its 8x8 pixel block can see (exact footprint test) in a
//                private compacted shared-memory list -- stored as per-column / per-row terms of the exponent -- and blends
//                them with predicated accumulation, two pixels per lane;
//                also accumulates the expected-depth channel (sum z*alpha*T) the TSDF stage consumes.
//
// All kernels run on the caller's stream(s).
#include <algorithm>

#include <cub/cub.cuh>

#include "gsb_common.h"
#include "gsb_radix.cuh"

namespace gsb {

thread_local char g_error[512] = {0};
std::atomic<uint64_t> g_launches{0};
Profiler g_prof;
static const char* kStageNames[kStCount] = {"preprocess", "depth_sort", "emit", "tile_sort", "tile_ranges",
                                            "render",     "to_u8", "prepare_depth", "mark_bricks", "integrate",
                                            "merge_index", "merge_pack", "merge_reduce", "merge_unpack"};

namespace {

constexpr int kWarpsPerBlock = 4;
constexpr int kPreThreads = kWarpsPerBlock * 32;
constexpr int kMaxShFloats = 48;  // 16 coefficients x RGB

// ---------------------------------------------------------------------------------------------
// PTX wrappers: mbarrier + 1-D bulk TMA (global -> shared)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a bulk copy that never lands (bad pointer / size) traps instead of hanging the GPU.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  for (uint32_t spin = 0; !mbar_try_wait(bar, parity); ++spin)
    if (spin > (1u << 22)) __trap();
}
__device__ __forceinline__ void tma_load_1d(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst_smem)),
               "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// ---------------------------------------------------------------------------------------------
// Per-Gaussian maths.  Expressions are kept in the reference's algebraic form so nvcc contracts
// them the same way it contracts the reference's device code.
// ---------------------------------------------------------------------------------------------
struct Mat3 {  // column-major, m[col][row] (glm convention)
  float m[3][3];
};
__device__ __forceinline__ Mat3 mat_mul(const Mat3& a, const Mat3& b) {
  Mat3 r;
#pragma unroll
  for (int j = 0; j < 3; ++j)
#pragma unroll
    for (int i = 0; i < 3; ++i) r.m[j][i] = a.m[0][i] * b.m[j][0] + a.m[1][i] * b.m[j][1] + a.m[2][i] * b.m[j][2];
  return r;
}
__device__ __forceinline__ Mat3 mat_t(const Mat3& a) {
  Mat3 r;
#pragma unroll
  for (int j = 0; j < 3; ++j)
#pragma unroll
    for (int i = 0; i < 3; ++i) r.m[j][i] = a.m[i][j];
  return r;
}

struct TileRect {
  uint32_t x0, y0, x1, y1;
};
// auxiliary.h:46-56
__device__ __forceinline__ TileRect tile_rect(float px, float py, int radius, uint32_t gx, uint32_t gy) {
  TileRect r;
  r.x0 = min(gx, (uint32_t)max(0, (int)((px - radius) / kTile)));
  r.y0 = min(gy, (uint32_t)max(0, (int)((py - radius) / kTile)));
  r.x1 = min(gx, (uint32_t)max(0, (int)((px + radius + kTile - 1) / kTile)));
  r.y1 = min(gy, (uint32_t)max(0, (int)((py + radius + kTile - 1) / kTile)));
  return r;
}

// Exact footprint test.  A pixel of the box [x0,x1] x [y0,y1] (pixel centres) can only be blended if
//   power = -0.5*(a dx^2 + c dy^2) - b dx dy <= 0  and  opacity*exp(power) >= 1/255
// (forward.cu:336-346), i.e. q(d) = a dx^2 + 2b dx dy + c dy^2 <= 2 ln(255*opacity).  q is convex,
// so its minimum over the tile's pixel box is 0 if the centre lies inside and otherwise sits on
// one of the four box edges.  A safety margin covers fp32 rounding of both evaluations; pairs
// inside the margin are kept, so no contributing pair is ever dropped.
// __noinline__: the counting and the emitting kernel must execute the same instructions.
struct Footprint {  // per-Gaussian constants of the test
  float a, b, c;      // conic
  float nb_a, nb_c;   // -b/a, -b/c: minimiser slopes along horizontal / vertical box edges
  float two_tau;      // 2 ln(255 * opacity)
  bool degenerate;    // non positive-definite conic: never culled
};
__device__ __forceinline__ Footprint make_footprint(float a, float b, float c, float two_tau) {
  Footprint f;
  f.a = a;
  f.b = b;
  f.c = c;
  f.degenerate = !(a > 0.f && c > 0.f && a * c - b * b > 0.f);
  // approximate division is enough: an error of a few ulp in the clamped minimiser changes q in second order only
  f.nb_a = f.degenerate ? 0.f : __fdividef(-b, a);
  f.nb_c = f.degenerate ? 0.f : __fdividef(-b, c);
  f.two_tau = two_tau;
  return f;
}
__device__ __forceinline__ bool rect_can_contribute(float gxp, float gyp, const Footprint& f, float x0, float y0, float x1,
                                                    float y1) {
  if (f.degenerate) return true;
  const float dx_lo = gxp - x1, dx_hi = gxp - x0;
  const float dy_lo = gyp - y1, dy_hi = gyp - y0;
  if (dx_lo <= 0.f && dx_hi >= 0.f && dy_lo <= 0.f && dy_hi >= 0.f) return true;
  const float DX = fmaxf(fabsf(dx_lo), fabsf(dx_hi)), DY = fmaxf(fabsf(dy_lo), fabsf(dy_hi));
  const float margin = 1e-3f + 8e-6f * (f.a * DX * DX + f.c * DY * DY + 2.f * fabsf(f.b) * DX * DY);
  // The centre lies outside the box, so the minimum of the (convex) quadratic over the box sits on an edge that faces the
  // centre: the vertical edge nearer to it and the horizontal edge nearer to it.  (d = centre - pixel: the nearer edge is
  // the one with the smaller |d|.)  An edge that does not face the centre only yields a value >= the minimum.
  const float dx = fabsf(dx_lo) < fabsf(dx_hi) ? dx_lo : dx_hi;
  const float dy = fminf(dy_hi, fmaxf(dy_lo, f.nb_c * dx));
  const float qv = f.a * dx * dx + 2.f * f.b * dx * dy + f.c * dy * dy;
  const float ey = fabsf(dy_lo) < fabsf(dy_hi) ? dy_lo : dy_hi;
  const float ex = fminf(dx_hi, fmaxf(dx_lo, f.nb_a * ey));
  const float qh = f.a * ex * ex + 2.f * f.b * ex * ey + f.c * ey * ey;
  return fminf(qv, qh) <= f.two_tau + margin;
}
// A non-degenerate footprint and its centre as two float4 (x, y, a, b), (c, nb_a, nb_c, two_tau), as lanes share it.
__device__ __forceinline__ void publish_footprint(float4* slot, float px, float py, const Footprint& f) {
  slot[0] = make_float4(px, py, f.a, f.b);
  slot[1] = make_float4(f.c, f.nb_a, f.nb_c, f.two_tau);
}
__device__ __forceinline__ Footprint read_footprint(const float4& q0, const float4& q1) {
  return Footprint{q0.z, q0.w, q1.x, q1.y, q1.z, q1.w, false};
}
// __noinline__: the counting and the emitting kernel must execute the same instructions.
__device__ __noinline__ bool tile_can_contribute(float gxp, float gyp, float a, float b, float c, float nb_a, float nb_c,
                                                 float two_tau, uint32_t tx, uint32_t ty) {
  const Footprint f = read_footprint(make_float4(gxp, gyp, a, b), make_float4(c, nb_a, nb_c, two_tau));
  const float x0 = (float)(tx * kTile), y0 = (float)(ty * kTile);
  return rect_can_contribute(gxp, gyp, f, x0, y0, x0 + (kTile - 1), y0 + (kTile - 1));
}

// Candidate tiles under the exact test: the reference rectangle intersected with the tiles that overlap the axis-aligned
// bounding box of the ellipse q(d) <= tau (half extents sqrt(tau c / det), sqrt(tau a / det)).  tau carries the same
// rounding allowance as rect_can_contribute's margin (its S term is <= 4 tau k over the box, k = ac/det); very elongated
// conics (k > 1000) keep the reference rectangle.  Explicitly rounded operations only: the binning, the emitting and the
// validation kernel must all arrive at the same rectangle.
__device__ __forceinline__ TileRect shrink_rect(TileRect r, float px, float py, const Footprint& f) {
  if (f.degenerate) return r;
  const float ac = __fmul_rn(f.a, f.c);
  const float det = __fsub_rn(ac, __fmul_rn(f.b, f.b));
  const float k = __fdiv_rn(ac, det);
  if (!(k <= 1000.f)) return r;
  const float tau = __fmul_rn(__fadd_rn(f.two_tau, 2e-3f), __fadd_rn(1.f, __fmul_rn(5e-5f, k)));
  if (!(tau > 0.f)) {  // opacity < 1/255: nothing can be blended
    r.x1 = r.x0;
    r.y1 = r.y0;
    return r;
  }
  const float hx = __fadd_rn(__fmul_rn(__fsqrt_rn(__fdiv_rn(__fmul_rn(tau, f.c), det)), 1.0001f), 0.01f);
  const float hy = __fadd_rn(__fmul_rn(__fsqrt_rn(__fdiv_rn(__fmul_rn(tau, f.a), det)), 1.0001f), 0.01f);
  const float inv = 1.0f / kTile;  // power of two: exact
  const float lox = floorf(__fmul_rn(__fsub_rn(px, hx), inv)), hix = floorf(__fmul_rn(__fadd_rn(px, hx), inv));
  const float loy = floorf(__fmul_rn(__fsub_rn(py, hy), inv)), hiy = floorf(__fmul_rn(__fadd_rn(py, hy), inv));
  // compare in float (the bounds may be negative or huge), then convert
  const float x0 = fmaxf((float)r.x0, lox), x1 = fminf((float)r.x1, hix + 1.f);
  const float y0 = fmaxf((float)r.y0, loy), y1 = fminf((float)r.y1, hiy + 1.f);
  if (!(x0 < x1 && y0 < y1)) {
    r.x1 = r.x0;
    r.y1 = r.y0;
    return r;
  }
  r.x0 = (uint32_t)x0;
  r.x1 = (uint32_t)x1;
  r.y0 = (uint32_t)y0;
  r.y1 = (uint32_t)y1;
  return r;
}

// A Gaussian's candidate tiles: the reference rectangle, under exact culling shrunk to the ellipse's (shrink_rect), and
// whether each of its tiles must be tested.  The binning, the emitting and the validation kernel all decide here.
struct Candidate {
  TileRect rc;
  Footprint fp;  // make_footprint(1, 0, 1, 0) without exact culling
  bool test;     // exact culling of a positive-definite conic: tiles are tested, not all kept
  uint32_t w, area;
};
__device__ __forceinline__ Candidate no_candidate() {  // a Gaussian binned nowhere
  return Candidate{TileRect{0, 0, 0, 0}, make_footprint(1.f, 0.f, 1.f, 0.f), false, 0u, 0u};
}
// conic = (a, b, c, ·) as in recB; taken by reference so that the emit kernels only load it under exact culling
__device__ __forceinline__ Candidate make_candidate(float px, float py, int radius, const float4& conic, float opacity,
                                                    uint32_t gx, uint32_t gy, bool exact) {
  Candidate cd = no_candidate();
  cd.rc = tile_rect(px, py, radius, gx, gy);
  if (exact) {
    cd.fp = make_footprint(conic.x, conic.y, conic.z, 2.f * logf(255.f * opacity));
    cd.test = !cd.fp.degenerate;
    cd.rc = shrink_rect(cd.rc, px, py, cd.fp);
  }
  cd.w = cd.rc.x1 - cd.rc.x0;
  cd.area = cd.w * (cd.rc.y1 - cd.rc.y0);
  return cd;
}

// A candidate rectangle of at most kMaskTiles tiles packed into the word the emit pass replays its mask with:
// x0 | y0 << kRectCoordBits | (w - 1) << 2 kRectCoordBits.  kRectLarge: no mask stored, re-test when emitting.
constexpr uint32_t kMaskTiles = 64;
constexpr uint32_t kRectCoordBits = 13, kRectWidthBits = 6;
constexpr uint32_t kRectCoordMax = (1u << kRectCoordBits) - 1u;
constexpr uint32_t kRectLarge = 0xffffffffu;
static_assert(2 * kRectCoordBits + kRectWidthBits == 32, "the packed rectangle is one word");
static_assert(kMaskTiles == 1u << kRectWidthBits, "w - 1 of a rectangle of up to kMaskTiles tiles fills the width field");
__device__ __forceinline__ uint32_t pack_rect(uint32_t x0, uint32_t y0, uint32_t w) {
  return x0 | (y0 << kRectCoordBits) | ((w - 1u) << (2 * kRectCoordBits));
}
__device__ __forceinline__ uint3 unpack_rect(uint32_t word) {  // (x0, y0, w)
  return make_uint3(word & kRectCoordMax, (word >> kRectCoordBits) & kRectCoordMax, (word >> (2 * kRectCoordBits)) + 1u);
}

// Slot k of a rectangle w tiles wide, row-major -> (column, row).  For k < 64, w <= 64, (k + 0.5) / w is never within
// rounding distance of an integer, so the approximate division floors to the exact row.
__device__ __forceinline__ uint2 rect_slot(uint32_t k, uint32_t w) {
  const uint32_t row = (uint32_t)__float2int_rd(__fdividef((float)k + 0.5f, (float)w));
  return make_uint2(k - row * w, row);
}

// Warp-flattened slots: each lane's `cand` slots laid end to end in lane order.  warp_inclusive_sum gives a lane the end
// of its slots; slot_owner the lane holding flattened slot fidx, the first whose inclusive sum exceeds fidx (for a valid
// slot one of the 32 lanes: 5 halvings settle it).
__device__ __forceinline__ uint32_t warp_inclusive_sum(uint32_t cand) {
  const int lane = threadIdx.x & 31;
  uint32_t incl = cand;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += v;
  }
  return incl;
}
__device__ __forceinline__ int slot_owner(uint32_t incl, uint32_t fidx) {
  int lo = 0, hi = 31;
#pragma unroll
  for (int step = 0; step < 5; ++step) {
    const int mid = (lo + hi) >> 1;
    const uint32_t v = __shfl_sync(0xffffffffu, incl, mid);
    if (v <= fidx)
      lo = mid + 1;
    else
      hi = mid;
  }
  return lo;
}

// Rectangles too large for a mask: the whole warp tests the tiles of each lane with `large` set, in lane order, 32 per
// step.  For each such lane it calls source(lane), which returns the callback run after every step:
// step(tiles kept in earlier steps, keep, ballot, tx, ty).
template <class Source>
__device__ __forceinline__ void walk_large_rects(bool large, float px, float py, const Candidate& cd, Source source) {
  const int lane = threadIdx.x & 31;
  unsigned todo = __ballot_sync(0xffffffffu, large);
  while (todo) {
    const int src = __ffs(todo) - 1;
    todo &= todo - 1;
    const float spx = __shfl_sync(0xffffffffu, px, src), spy = __shfl_sync(0xffffffffu, py, src);
    const float sa = __shfl_sync(0xffffffffu, cd.fp.a, src), sb = __shfl_sync(0xffffffffu, cd.fp.b, src);
    const float sc = __shfl_sync(0xffffffffu, cd.fp.c, src), st = __shfl_sync(0xffffffffu, cd.fp.two_tau, src);
    const float sna = __shfl_sync(0xffffffffu, cd.fp.nb_a, src), snc = __shfl_sync(0xffffffffu, cd.fp.nb_c, src);
    const bool stest = __shfl_sync(0xffffffffu, (int)cd.test, src) != 0;
    const uint32_t sx0 = __shfl_sync(0xffffffffu, cd.rc.x0, src), sy0 = __shfl_sync(0xffffffffu, cd.rc.y0, src);
    const uint32_t sw = __shfl_sync(0xffffffffu, cd.w, src), sarea = __shfl_sync(0xffffffffu, cd.area, src);
    auto step = source(src);
    uint32_t done = 0;
    for (uint32_t base = 0; base < sarea; base += 32) {
      const uint32_t k = base + lane;
      const uint32_t tx = sx0 + k % sw, ty = sy0 + k / sw;
      const bool keep = k < sarea && (!stest || tile_can_contribute(spx, spy, sa, sb, sc, sna, snc, st, tx, ty));
      const unsigned votes = __ballot_sync(0xffffffffu, keep);
      step(done, keep, votes, tx, ty);
      done += __popc(votes);
    }
  }
}

// Warp-flattened binning.  The candidate tiles of the warp's 32 Gaussians (rectangles of up to
// kMaskTiles tiles) are laid end to end and tested 32 at a time with every lane busy, instead of
// each lane looping over its own rectangle.  Returns this lane's kept-tile count; for rectangles
// of <= kMaskTiles tiles `mask` gets one bit per rectangle tile (row-major) so the emit pass can
// replay the decision without re-testing.  Larger rectangles are counted cooperatively (and
// re-tested by the emit pass with the same __noinline__ routine, so both passes agree).
// `stage` = 32 x 2 float4 of per-warp shared memory the lanes publish their footprint in.
__device__ __forceinline__ uint32_t bin_gaussians_warp(bool active, float px, float py, float ca, float cb, float cc,
                                                       float opacity, int radius, uint32_t gx, uint32_t gy, bool exact,
                                                       float4* stage, uint64_t& mask, uint32_t& rect_word) {
  const int lane = threadIdx.x & 31;
  Candidate cd = no_candidate();
  if (active) cd = make_candidate(px, py, radius, make_float4(ca, cb, cc, 0.f), opacity, gx, gy, exact);
  mask = 0ull;
  const bool small = active && cd.area <= kMaskTiles;
  rect_word = (small && cd.area != 0) ? pack_rect(cd.rc.x0, cd.rc.y0, cd.w) : kRectLarge;
  if (small && !cd.test) mask = cd.area == 64 ? ~0ull : ((1ull << cd.area) - 1ull);  // rectangle binning: everything kept
  const uint32_t cand = (small && cd.test) ? cd.area : 0u;
  const uint32_t incl = warp_inclusive_sum(cand);
  const uint32_t excl = incl - cand;
  const uint32_t total = __shfl_sync(0xffffffffu, incl, 31);
  publish_footprint(stage + 2 * lane, px, py, cd.fp);
  const uint32_t pack0 = cd.rc.x0 | (cd.rc.y0 << 16);  // tile coordinates < 65536
  const uint32_t pack1 = cd.w | (excl << 8);             // w <= 64, excl <= 31 * 64
  __syncwarp();
  for (uint32_t w0 = 0; w0 < total; w0 += 32) {
    const uint32_t fidx = w0 + lane;
    const int owner = slot_owner(incl, fidx);
    const uint32_t o0 = __shfl_sync(0xffffffffu, pack0, owner), o1 = __shfl_sync(0xffffffffu, pack1, owner);
    bool keep = false;
    if (fidx < total) {
      const float4 q0 = stage[2 * owner], q1 = stage[2 * owner + 1];
      const uint2 slot = rect_slot(fidx - (o1 >> 8), o1 & 0xffu);
      const uint32_t tx = (o0 & 0xffffu) + slot.x, ty = (o0 >> 16) + slot.y;
      const float x0 = (float)(tx * kTile), y0 = (float)(ty * kTile);
      keep = rect_can_contribute(q0.x, q0.y, read_footprint(q0, q1), x0, y0, x0 + (kTile - 1), y0 + (kTile - 1));
    }
    const unsigned votes = __ballot_sync(0xffffffffu, keep);
    // collect the votes that belong to my own rectangle
    const uint32_t my_lo = max(excl, w0), my_hi = min(excl + cand, w0 + 32);
    if (my_lo < my_hi) {
      const uint32_t nbits = my_hi - my_lo;
      const uint32_t bits = (votes >> (my_lo - w0)) & (nbits == 32 ? 0xffffffffu : ((1u << nbits) - 1u));
      mask |= (uint64_t)bits << (my_lo - excl);
    }
  }
  uint32_t kept = small ? (uint32_t)__popcll(mask) : 0u;
  // rectangles too large for a mask are only counted here
  walk_large_rects(active && !small, px, py, cd, [&](int src) {
    return [&, src](uint32_t done, bool, unsigned votes, uint32_t, uint32_t) {
      if (lane == src) kept = done + __popc(votes);
    };
  });
  return kept;
}

// forward.cu:20-71 (computeColorFromSH): `sh(i)` = i-th float of the Gaussian's [M,3] coefficient block.
template <class Acc>
__device__ __forceinline__ void eval_sh(int D, Acc sh, float3 dir, float res[3]) {
  const float SH_C0 = 0.28209479177387814f, SH_C1 = 0.4886025119029199f;
  const float SH_C2[5] = {1.0925484305920792f, -1.0925484305920792f, 0.31539156525252005f, -1.0925484305920792f,
                          0.5462742152960396f};
  const float SH_C3[7] = {-0.5900435899266435f, 2.890611442640554f, -0.4570457994644658f, 0.3731763325901154f,
                          -0.4570457994644658f, 1.445305721320277f, -0.5900435899266435f};
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) {
    float v = SH_C0 * sh(ch);
    if (D > 0) {
      const float x = dir.x, y = dir.y, z = dir.z;
      v = v - SH_C1 * y * sh(3 + ch) + SH_C1 * z * sh(6 + ch) - SH_C1 * x * sh(9 + ch);
      if (D > 1) {
        const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
        v = v + SH_C2[0] * xy * sh(12 + ch) + SH_C2[1] * yz * sh(15 + ch) + SH_C2[2] * (2.0f * zz - xx - yy) * sh(18 + ch) +
            SH_C2[3] * xz * sh(21 + ch) + SH_C2[4] * (xx - yy) * sh(24 + ch);
        if (D > 2) {
          v = v + SH_C3[0] * y * (3.0f * xx - yy) * sh(27 + ch) + SH_C3[1] * xy * z * sh(30 + ch) +
              SH_C3[2] * y * (4.0f * zz - xx - yy) * sh(33 + ch) + SH_C3[3] * z * (2.0f * zz - 3.0f * xx - 3.0f * yy) * sh(36 + ch) +
              SH_C3[4] * x * (4.0f * zz - xx - yy) * sh(39 + ch) + SH_C3[5] * z * (xx - yy) * sh(42 + ch) +
              SH_C3[6] * x * (xx - 3.0f * yy) * sh(45 + ch);
        }
      }
    }
    v += 0.5f;
    res[ch] = max(v, 0.0f);
  }
}

struct PreEye {  // what differs between the two eyes of a stereo pair (renderer_utils.py:378-389)
  const float* view;
  const float* proj;
  const float* campos;
  float tan_fovx, tan_fovy, focal_x, focal_y;
  float4* recA;
  float4* recB;
  float2* recC;
  uint32_t* tiles;
  int* radii;
  unsigned long long* counters;   // [0] += sum of reference tile rectangles, [3] |= 1 if the eyes' view depths differ
  uint64_t* masks;                // kept-tile bitmask of candidate rectangles with <= 64 tiles
  uint32_t* rects;                // packed candidate rectangle the mask refers to (kRectLarge: none)
  uint32_t* depth_keys;           // view-depth sort key per Gaussian, or NULL (validation path / shared with the other eye)
};
struct PreParams {
  int P, D, M, W, H;
  const float* means3D;
  const float* shs;
  const float* colors;
  const float* opacities;
  const float* scales;
  const float* rotations;
  const float* cov3D;
  float scale_modifier;
  uint32_t gx, gy;
  uint32_t flags;
  int use_tma;
  int binned;        // 0: validation path (no depth keys, no tile masks)
  int shared_depth;  // stereo pair whose eyes see every Gaussian at the same view depth: one key array (eye 0's), verified
  PreEye eye[2];
};

struct WarpStage {  // one warp's staged parameter block; every member offset is a multiple of 128 B
  float sh[32 * (kMaxShFloats + 4)];  // 6656 B, 512 B more than the SH block: the 8 KB stage the kernels were timed with
  float rot[32 * 4];            // 512 B
  float xyz[32 * 3];            // 384 B
  float scale[32 * 3];          // 384 B
  float opac[32];               // 128 B
  uint64_t bar;
  uint64_t pad[15];
};

// kEyes = 1: one view.  kEyes = 2: the two eyes of a stereo pair in ONE pass over the Gaussian parameters -- the 236-byte
// parameter block of every Gaussian (positions, scales, rotations, opacities, 192 B of SH) is staged once, the 3-D
// covariance is computed once, and projection / binning / SH shading run per eye from the staged block.  The eyes of a
// rig share the camera rotation and differ by a translation along the camera x axis (transformation_utils.py:219-223),
// so a Gaussian's view depth is THE SAME float in both eyes whenever the z rows of the two view matrices are bitwise
// equal; then one depth key per Gaussian (and one depth sort) serves both eyes.  The kernel verifies that and raises
// counters[3] otherwise (the caller then renders the eyes separately).
template <int kEyes, int kMinBlocks>
__global__ void __launch_bounds__(kPreThreads, kMinBlocks) preprocess_kernel(const PreParams p) {
  __shared__ __align__(128) WarpStage stage[kWarpsPerBlock];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  WarpStage& st = stage[warp];
  const int base = (blockIdx.x * kWarpsPerBlock + warp) * 32;
  if (base >= p.P) return;
  const int idx = base + lane;
  const int count = min(32, p.P - base);
  const bool has_sr = p.cov3D == nullptr;
  const bool full_tma = p.use_tma && count == 32;

  // ---- stage 1: positions, scales, rotations, opacities -------------------------------------
  if (full_tma) {
    if (lane == 0) {
      mbar_init(&st.bar, 1);
      uint32_t bytes = 384 + 128 + (has_sr ? 384 + 512 : 0);
      mbar_expect_tx(&st.bar, bytes);
      tma_load_1d(st.xyz, p.means3D + (size_t)base * 3, 384, &st.bar);
      tma_load_1d(st.opac, p.opacities + base, 128, &st.bar);
      if (has_sr) {
        tma_load_1d(st.scale, p.scales + (size_t)base * 3, 384, &st.bar);
        tma_load_1d(st.rot, p.rotations + (size_t)base * 4, 512, &st.bar);
      }
    }
    __syncwarp();
    mbar_wait(&st.bar, 0);
  } else {
    for (int k = lane; k < count * 3; k += 32) {
      st.xyz[k] = p.means3D[(size_t)base * 3 + k];
      if (has_sr) st.scale[k] = p.scales[(size_t)base * 3 + k];
    }
    if (lane < count) st.opac[lane] = p.opacities[base + lane];
    if (has_sr)
      for (int k = lane; k < count * 4; k += 32) st.rot[k] = p.rotations[(size_t)base * 4 + k];
    __syncwarp();
  }

  const bool valid = lane < count;
  bool visible[kEyes], front[kEyes];
  float px[kEyes], py[kEyes], zv[kEyes], ca[kEyes], cb[kEyes], cc[kEyes];
  int radius[kEyes];
  uint32_t ntiles[kEyes], nref[kEyes];
  float3 pos = make_float3(0.f, 0.f, 0.f);
  float3 tv[kEyes];
  float opacity = 0.f;
  bool any_front = false;
#pragma unroll
  for (int e = 0; e < kEyes; ++e) {
    visible[e] = front[e] = false;
    px[e] = py[e] = zv[e] = ca[e] = cb[e] = cc[e] = 0.f;
    radius[e] = 0;
    ntiles[e] = nref[e] = 0;
    tv[e] = make_float3(0.f, 0.f, 0.f);
  }
  if (valid) {
    pos = make_float3(st.xyz[lane * 3], st.xyz[lane * 3 + 1], st.xyz[lane * 3 + 2]);
    opacity = st.opac[lane];
#pragma unroll
    for (int e = 0; e < kEyes; ++e) {
      const float* vm = p.eye[e].view;
      // auxiliary.h:139-164 (in_frustum): view-space point, near cull at 0.2
      tv[e] = make_float3(vm[0] * pos.x + vm[4] * pos.y + vm[8] * pos.z + vm[12],
                          vm[1] * pos.x + vm[5] * pos.y + vm[9] * pos.z + vm[13],
                          vm[2] * pos.x + vm[6] * pos.y + vm[10] * pos.z + vm[14]);
      front[e] = tv[e].z > 0.2f;
      any_front = any_front || front[e];
    }
  }
  // forward.cu:118-152: Sigma = (S R)^T (S R); quaternion is w-first and NOT renormalised.  View independent: once per pair.
  float c3[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (any_front) {
    if (has_sr) {
      const float4 q = reinterpret_cast<const float4*>(st.rot)[lane];
      const float r = q.x, x = q.y, y = q.z, z = q.w;
      Mat3 S;
#pragma unroll
      for (int j = 0; j < 3; ++j)
#pragma unroll
        for (int i = 0; i < 3; ++i) S.m[j][i] = 0.f;
      S.m[0][0] = p.scale_modifier * st.scale[lane * 3];
      S.m[1][1] = p.scale_modifier * st.scale[lane * 3 + 1];
      S.m[2][2] = p.scale_modifier * st.scale[lane * 3 + 2];
      // Explicitly rounded, in the contraction nvcc gives the reference for sm_90a (which product of a sum is fused
      // decides the last bit of the conic): y*y + z*z is not fused, x*z is rounded before r*y is fused onto it.
      Mat3 R;
      R.m[0][0] = 1.f - 2.f * __fadd_rn(__fmul_rn(y, y), __fmul_rn(z, z));
      R.m[0][1] = 2.f * __fmaf_rn(x, y, -__fmul_rn(r, z));
      R.m[0][2] = 2.f * __fmaf_rn(r, y, __fmul_rn(x, z));
      R.m[1][0] = 2.f * __fmaf_rn(x, y, __fmul_rn(r, z));
      R.m[1][1] = 1.f - 2.f * __fmaf_rn(x, x, __fmul_rn(z, z));
      R.m[1][2] = 2.f * __fmaf_rn(y, z, -__fmul_rn(r, x));
      R.m[2][0] = 2.f * __fmaf_rn(-r, y, __fmul_rn(x, z));
      R.m[2][1] = 2.f * __fmaf_rn(y, z, __fmul_rn(r, x));
      R.m[2][2] = 1.f - 2.f * __fmaf_rn(x, x, __fmul_rn(y, y));
      const Mat3 Mx = mat_mul(S, R);
      const Mat3 Sg = mat_mul(mat_t(Mx), Mx);
      c3[0] = Sg.m[0][0];
      c3[1] = Sg.m[0][1];
      c3[2] = Sg.m[0][2];
      c3[3] = Sg.m[1][1];
      c3[4] = Sg.m[1][2];
      c3[5] = Sg.m[2][2];
    } else {
#pragma unroll
      for (int k = 0; k < 6; ++k) c3[k] = p.cov3D[(size_t)idx * 6 + k];
    }
  }
#pragma unroll
  for (int e = 0; e < kEyes; ++e) {
    if (!front[e]) continue;
    const float* vm = p.eye[e].view;
    const float* pm = p.eye[e].proj;
    float3 t = tv[e];
    zv[e] = t.z;
    const float hx = pm[0] * pos.x + pm[4] * pos.y + pm[8] * pos.z + pm[12];
    const float hy = pm[1] * pos.x + pm[5] * pos.y + pm[9] * pos.z + pm[13];
    const float hw = pm[3] * pos.x + pm[7] * pos.y + pm[11] * pos.z + pm[15];
    const float p_w = 1.0f / (hw + 0.0000001f);
    const float projx = hx * p_w, projy = hy * p_w;

    // forward.cu:74-113: EWA projection with the 1.3*tan(fov) guard band and +0.3 low-pass
    const float limx = 1.3f * p.eye[e].tan_fovx, limy = 1.3f * p.eye[e].tan_fovy;
    const float txtz = t.x / t.z, tytz = t.y / t.z;
    t.x = min(limx, max(-limx, txtz)) * t.z;
    t.y = min(limy, max(-limy, tytz)) * t.z;
    Mat3 J;
    J.m[0][0] = p.eye[e].focal_x / t.z;
    J.m[0][1] = 0.f;
    J.m[0][2] = -(p.eye[e].focal_x * t.x) / (t.z * t.z);
    J.m[1][0] = 0.f;
    J.m[1][1] = p.eye[e].focal_y / t.z;
    J.m[1][2] = -(p.eye[e].focal_y * t.y) / (t.z * t.z);
    J.m[2][0] = 0.f;
    J.m[2][1] = 0.f;
    J.m[2][2] = 0.f;
    Mat3 Wm;
    Wm.m[0][0] = vm[0];
    Wm.m[0][1] = vm[4];
    Wm.m[0][2] = vm[8];
    Wm.m[1][0] = vm[1];
    Wm.m[1][1] = vm[5];
    Wm.m[1][2] = vm[9];
    Wm.m[2][0] = vm[2];
    Wm.m[2][1] = vm[6];
    Wm.m[2][2] = vm[10];
    const Mat3 T = mat_mul(Wm, J);
    Mat3 V;
    V.m[0][0] = c3[0];
    V.m[0][1] = c3[1];
    V.m[0][2] = c3[2];
    V.m[1][0] = c3[1];
    V.m[1][1] = c3[3];
    V.m[1][2] = c3[4];
    V.m[2][0] = c3[2];
    V.m[2][1] = c3[4];
    V.m[2][2] = c3[5];
    const Mat3 cov = mat_mul(mat_mul(mat_t(T), mat_t(V)), T);
    const float cxx = cov.m[0][0] + 0.3f, cxy = cov.m[0][1], cyy = cov.m[1][1] + 0.3f;

    const float det = (cxx * cyy - cxy * cxy);
    if (det != 0.0f) {
      const float det_inv = 1.f / det;
      ca[e] = cyy * det_inv;
      cb[e] = -cxy * det_inv;
      cc[e] = cxx * det_inv;
      const float mid = 0.5f * (cxx + cyy);
      const float lambda1 = mid + sqrt(max(0.1f, mid * mid - det));
      const float lambda2 = mid - sqrt(max(0.1f, mid * mid - det));
      const float my_radius = ceil(3.f * sqrt(max(lambda1, lambda2)));
      // auxiliary.h:41-44: ndc2Pix is evaluated in double
      px[e] = (float)(((projx + 1.0) * p.W - 1.0) * 0.5);
      py[e] = (float)(((projy + 1.0) * p.H - 1.0) * 0.5);
      const TileRect rc = tile_rect(px[e], py[e], (int)my_radius, p.gx, p.gy);
      nref[e] = (rc.x1 - rc.x0) * (rc.y1 - rc.y0);
      if (nref[e] != 0) {
        visible[e] = true;
        radius[e] = (int)my_radius;
      }
    }
  }
  // The 6 KB SH block is only fetched when some lane survived culling in some eye; the bulk copy is issued NOW so that it
  // lands while the warp is busy binning.
  bool vis_any = false;
#pragma unroll
  for (int e = 0; e < kEyes; ++e) vis_any = vis_any || visible[e];
  const bool any_visible = __any_sync(0xffffffffu, vis_any);
  const int shf = p.M * 3;  // SH floats per Gaussian
  const bool need_sh = p.colors == nullptr && any_visible;
  const bool tma_sh = need_sh && full_tma && (shf * 4) % 16 == 0 && shf <= kMaxShFloats;
  // full-degree blocks (M = 16, 192 B per lane) are read as 16-byte vectors; smaller ones as scalars
  const bool vec_sh = shf == kMaxShFloats;
  if (tma_sh && lane == 0) {
    mbar_expect_tx(&st.bar, (uint32_t)(32 * shf * 4));
    tma_load_1d(st.sh, p.shs + (size_t)base * shf, (uint32_t)(32 * shf * 4), &st.bar);
  }
  // binning, pass 1: how many tiles this Gaussian is binned into.  The staged rotations / positions / scales are dead by
  // now: their 1280 bytes carry the lanes' footprints during binning (32 x 2 float4 = 1024 bytes)
  uint64_t tile_mask[kEyes];
  uint32_t rect_word[kEyes];
#pragma unroll
  for (int e = 0; e < kEyes; ++e) {
    __syncwarp();
    tile_mask[e] = 0ull;
    rect_word[e] = kRectLarge;
    ntiles[e] = bin_gaussians_warp(visible[e], px[e], py[e], ca[e], cb[e], cc[e], opacity, radius[e], p.gx, p.gy,
                                   (p.flags & GSB_RASTER_EXACT_TILE_CULL) != 0, reinterpret_cast<float4*>(st.rot), tile_mask[e],
                                   rect_word[e]);
  }

  // ---- stage 2: colour ------------------------------------------------------------------------
  float cr[kEyes], cg[kEyes], cbl[kEyes];
#pragma unroll
  for (int e = 0; e < kEyes; ++e) cr[e] = cg[e] = cbl[e] = 0.f;
  if (p.colors == nullptr) {
    if (any_visible) {
      if (tma_sh) {
        mbar_wait(&st.bar, 1);
      } else {
        for (int k = lane; k < count * shf; k += 32) st.sh[k] = p.shs[(size_t)base * shf + k];
        __syncwarp();
      }
      if (vis_any) {
        const float* sh = st.sh + lane * shf;
        float shreg[kMaxShFloats];
        if (vec_sh) {  // 12 x 16-byte reads, then the arithmetic from registers (both eyes share the reads)
          const float4* s4 = reinterpret_cast<const float4*>(sh);
#pragma unroll
          for (int k = 0; k < kMaxShFloats / 4; ++k) {
            const float4 v4 = s4[k];
            shreg[4 * k] = v4.x;
            shreg[4 * k + 1] = v4.y;
            shreg[4 * k + 2] = v4.z;
            shreg[4 * k + 3] = v4.w;
          }
        }
#pragma unroll
        for (int e = 0; e < kEyes; ++e) {
          if (!visible[e]) continue;
          const float* cp = p.eye[e].campos;
          const float3 cam = make_float3(cp[0], cp[1], cp[2]);
          float3 dir = make_float3(pos.x - cam.x, pos.y - cam.y, pos.z - cam.z);
          const float len = sqrt(dir.x * dir.x + dir.y * dir.y + dir.z * dir.z);
          dir.x = dir.x / len;
          dir.y = dir.y / len;
          dir.z = dir.z / len;
          float res[3];
          if (vec_sh)
            eval_sh(p.D, [&](int i) { return shreg[i]; }, dir, res);
          else
            eval_sh(p.D, [&](int i) { return sh[i]; }, dir, res);
          cr[e] = res[0];
          cg[e] = res[1];
          cbl[e] = res[2];
        }
      }
    }
  } else {
#pragma unroll
    for (int e = 0; e < kEyes; ++e)
      if (visible[e]) {
        cr[e] = p.colors[(size_t)idx * 3];
        cg[e] = p.colors[(size_t)idx * 3 + 1];
        cbl[e] = p.colors[(size_t)idx * 3 + 2];
      }
  }

  // ---- outputs --------------------------------------------------------------------------------
#pragma unroll
  for (int e = 0; e < kEyes; ++e) {
    const PreEye& o = p.eye[e];
    if (valid) {
      if (visible[e]) {
        o.recA[idx] = make_float4(px[e], py[e], zv[e], opacity);
        o.recB[idx] = make_float4(ca[e], cb[e], cc[e], cr[e]);
        o.recC[idx] = make_float2(cg[e], cbl[e]);
      }
      o.tiles[idx] = ntiles[e];
      o.radii[idx] = radius[e];
      if (p.binned && ntiles[e]) {
        o.masks[idx] = tile_mask[e];
        o.rects[idx] = rect_word[e];
      }
    }
    unsigned long long wsum = nref[e];
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) wsum += __shfl_xor_sync(0xffffffffu, wsum, off);
    if (lane == 0 && wsum) atomicAdd(&o.counters[0], wsum);
  }
  if (p.binned) {
    // Depth key = the bits of z_view (z > 0.2: bit order == float order).  A Gaussian that is binned nowhere emits no
    // instance, so where it lands in the depth order is irrelevant (key 0).
    if (kEyes == 2 && p.shared_depth) {
      if (valid) p.eye[0].depth_keys[idx] = any_front ? __float_as_uint(tv[0].z) : 0u;
      const bool differ = valid && any_front && __float_as_uint(tv[0].z) != __float_as_uint(tv[kEyes - 1].z);
      if (__any_sync(0xffffffffu, differ) && lane == 0) {
        atomicOr(&p.eye[0].counters[3], 1ull);
        atomicOr(&p.eye[kEyes - 1].counters[3], 1ull);
      }
    } else if (valid) {
#pragma unroll
      for (int e = 0; e < kEyes; ++e) p.eye[e].depth_keys[idx] = front[e] ? __float_as_uint(tv[e].z) : 0u;
    }
  }
}

// rasterizer_impl.cu:70-111: one (key, value) per kept (Gaussian, tile) pair, written at the
// Gaussian's prefix-sum offset in ascending tile order (the stable sort then preserves ascending
// Gaussian index among equal keys).
__global__ void __launch_bounds__(256) emit_instances_kernel(int P, const float4* __restrict__ recA,
                                                             const float4* __restrict__ recB,
                                                             const uint32_t* __restrict__ tiles,
                                                             const uint32_t* __restrict__ offsets,
                                                             const int* __restrict__ radii, uint32_t gx, uint32_t gy,
                                                             uint32_t flags, int64_t capacity,
                                                             uint64_t* __restrict__ keys, uint32_t* __restrict__ vals) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= P) return;
  const uint32_t n = tiles[idx];
  if (n == 0) return;
  const uint32_t end = offsets[idx];
  uint32_t off = end - n;
  if ((int64_t)end > capacity) return;  // host reports GSB_ERR_WORKSPACE
  const float4 A = recA[idx];
  const Candidate cd =
      make_candidate(A.x, A.y, radii[idx], recB[idx], A.w, gx, gy, (flags & GSB_RASTER_EXACT_TILE_CULL) != 0);
  const Footprint& fp = cd.fp;
  const uint32_t depth_bits = __float_as_uint(A.z);
  for (uint32_t ty = cd.rc.y0; ty < cd.rc.y1; ++ty)
    for (uint32_t tx = cd.rc.x0; tx < cd.rc.x1; ++tx) {
      if (cd.test && !tile_can_contribute(A.x, A.y, fp.a, fp.b, fp.c, fp.nb_a, fp.nb_c, fp.two_tau, tx, ty)) continue;
      if (off >= end) return;
      keys[off] = ((uint64_t)(ty * gx + tx) << 32) | depth_bits;
      vals[off] = (uint32_t)idx;
      ++off;
    }
}

// ---------------------------------------------------------------------------------------------
// Default binning pipeline: depth-sort the P Gaussians, emit their (tile, id) instances in that
// order, then split the instance stream by tile with a STABLE sort on the tile id alone.  Inside
// every tile the order is (depth bits, Gaussian index) ascending -- exactly what the reference's
// global stable radix sort on tile|depth keys emitted in Gaussian order produces
// (rasterizer_impl.cu:88-107,303) -- but the R-sized stream is sorted on <= 16 bits instead of 45,
// and nothing waits for the host.
// counters (unsigned long long[8]): [0] reference instance count  [1] binned instances R
//                                   [2] overflow flag (R > capacity)
// ---------------------------------------------------------------------------------------------
constexpr int kEmitThreads = 256;
constexpr int kScanThreads = 1024;
constexpr int kScanItems = 8;
constexpr int kScanBlock = kScanThreads * kScanItems;

// Exclusive scan of the tiles-per-Gaussian counts in depth order (delivered contiguously by the depth sort's last pass) ->
// instance offsets.  One pass: per-block scan + chained look-back over per-block status words (blocks take tickets in
// arrival order, so every predecessor of a block is already running; a full warp inspects 32 predecessors per round).
// With 8192 items per block the whole grid (123 blocks for 1M Gaussians) is co-resident and the chain is a few rounds deep.
// (The scan used to be fused into the emit pass; there every one of ~4000 heavy blocks paid the look-back latency before
// it could start writing: 104 us instead of 57 + this kernel's ~8.)  The last block publishes R (counters[1]) and the
// overflow flag (counters[2]).  status words: [31:30] 0 = not ready, 1 = block aggregate, 2 = inclusive prefix | 30-bit
// value (capacity < 2^30; values saturate, so an oversized frame still raises the flag).
__global__ void __launch_bounds__(kScanThreads) scan_tiles_kernel(int P, const uint32_t* __restrict__ tiles_sorted,
                                                                 uint32_t* __restrict__ offsets, int64_t capacity,
                                                                 unsigned long long* __restrict__ counters,
                                                                 uint32_t* __restrict__ scan_status, uint32_t* __restrict__ scan_ticket) {
  __shared__ uint32_t warp_tot[kScanThreads / 32];
  __shared__ uint32_t s_bid, s_prefix;
  if (threadIdx.x == 0) s_bid = atomicAdd(scan_ticket, 1u);
  __syncthreads();
  const uint32_t bid = s_bid;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int base = (int)(bid * kScanBlock + threadIdx.x * kScanItems);
  uint32_t v[kScanItems];
  uint32_t tsum = 0;
  if (base + kScanItems <= P) {  // two 16-byte loads
    const uint4 a = reinterpret_cast<const uint4*>(tiles_sorted + base)[0], b = reinterpret_cast<const uint4*>(tiles_sorted + base)[1];
    v[0] = a.x, v[1] = a.y, v[2] = a.z, v[3] = a.w, v[4] = b.x, v[5] = b.y, v[6] = b.z, v[7] = b.w;
  } else {
#pragma unroll
    for (int k = 0; k < kScanItems; ++k) v[k] = base + k < P ? tiles_sorted[base + k] : 0u;
  }
#pragma unroll
  for (int k = 0; k < kScanItems; ++k) tsum += v[k];
  uint32_t incl = tsum;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t u = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += u;
  }
  if (lane == 31) warp_tot[warp] = incl;
  __syncthreads();
  uint32_t wbase = 0, block_total = 0;
#pragma unroll
  for (int w = 0; w < kScanThreads / 32; ++w) {
    const uint32_t t = warp_tot[w];
    if (w < warp) wbase += t;
    block_total += t;
  }
  if (warp == 0) {
    uint32_t* my = scan_status + bid;
    if (lane == 0) st_status(my, (bid == 0 ? kStIncl : kStAgg) | min(block_total, kStVal));
    uint32_t prev = 0;
    if (bid > 0) {
      for (int64_t b = (int64_t)bid - 1;; b -= 32) {
        const int64_t src = b - lane;
        uint32_t sv = src >= 0 ? ld_status(scan_status + src) : kStIncl;  // before block 0: prefix 0
        for (uint32_t spin = 0; (sv >> 30) == 0; ++spin) {
          if (spin > (1u << 24)) __trap();  // a predecessor never published: fail loudly instead of hanging
          sv = ld_status(scan_status + src);
        }
        const unsigned closed = __ballot_sync(0xffffffffu, (sv >> 30) == 2);
        const int first = closed ? __ffs(closed) - 1 : 31;  // nearest predecessor holding an inclusive prefix
        unsigned long long part = lane <= first ? (unsigned long long)(sv & kStVal) : 0ull;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
        prev = (uint32_t)min(part + prev, (unsigned long long)kStVal);
        if (closed) break;
      }
      if (lane == 0) st_status(my, kStIncl | (uint32_t)min((unsigned long long)prev + block_total, (unsigned long long)kStVal));
    }
    if (lane == 0) {
      s_prefix = prev;
      if (bid == gridDim.x - 1) {  // blocks are numbered in arrival order: the last ticket covers the last Gaussians
        const unsigned long long total = (unsigned long long)prev + block_total;
        counters[1] = total;
        if ((int64_t)total > capacity) counters[2] = 1;
      }
    }
  }
  __syncthreads();
  uint32_t run = s_prefix + wbase + incl - tsum;
  if (base + kScanItems <= P) {
    uint4 a, b;
    a.x = run, run += v[0];
    a.y = run, run += v[1];
    a.z = run, run += v[2];
    a.w = run, run += v[3];
    b.x = run, run += v[4];
    b.y = run, run += v[5];
    b.z = run, run += v[6];
    b.w = run;
    reinterpret_cast<uint4*>(offsets + base)[0] = a;
    reinterpret_cast<uint4*>(offsets + base)[1] = b;
  } else {
#pragma unroll
    for (int k = 0; k < kScanItems; ++k) {
      if (base + k < P) offsets[base + k] = run;
      run += v[k];
    }
  }
}

// thread k = k-th Gaussian in depth order; the warp writes the (tile id, Gaussian id) instances of its 32 Gaussians at the
// offsets the scan produced.  Rectangles with a stored bitmask are replayed from it, flattened across the
// warp (every lane busy, stores run along the output); larger ones are re-tested cooperatively.  Stores beyond `capacity`
// are dropped (the frame is then flagged by the scan and re-rendered with a larger scratch).
__global__ void __launch_bounds__(kEmitThreads) emit_sorted_kernel(int P, const uint32_t* __restrict__ ids_sorted,
                                                                    const uint32_t* __restrict__ tiles_sorted,
                                                                    const uint32_t* __restrict__ offsets,
                                                                    const float4* __restrict__ recA, const float4* __restrict__ recB,
                                                                    const int* __restrict__ radii, const uint64_t* __restrict__ masks,
                                                                    const uint32_t* __restrict__ rects, uint32_t gx, uint32_t gy,
                                                                    uint32_t flags, int64_t capacity,
                                                                    uint32_t* __restrict__ tile_keys, uint32_t* __restrict__ tile_vals,
                                                                    uint32_t* __restrict__ ghist, int hist_passes, int digit_bits) {
  // digit histograms of the tile ids this block emits (what the tile sort's passes need), so the
  // sort does not have to read the instance stream once more just to count
  __shared__ uint32_t shist[kRdxMaxPasses][kRdxBins];
  for (int p = 0; p < hist_passes; ++p) shist[p][threadIdx.x] = 0;
  __syncthreads();
  auto tally = [&](uint32_t tile) {
    for (int p = 0; p < hist_passes; ++p) atomicAdd(&shist[p][(tile >> (digit_bits * p)) & ((1u << digit_bits) - 1u)], 1u);
  };
  const int k = (int)(blockIdx.x * kEmitThreads + threadIdx.x);
  const int lane = threadIdx.x & 31;
  uint32_t cnt = 0, off = 0, gid = 0;
  if (k < P) {  // three independent loads
    cnt = tiles_sorted[k];
    off = offsets[k];
    gid = ids_sorted[k];
  }
  const int64_t cap = capacity;

  uint32_t rect = kRectLarge;
  const bool active = cnt != 0;
  uint64_t mask = 0ull;
  if (active) {  // both gathers in flight together (the mask is only meaningful for a packed rectangle)
    rect = rects[gid];
    mask = masks[gid];
  }
  const bool small = active && rect != kRectLarge;
  if (!small) mask = 0ull;
  // ---- flattened replay of the stored masks (bits up to the highest kept tile of each rectangle)
  const uint32_t cand = small ? 64u - (uint32_t)__clzll((long long)mask) : 0u;
  const uint32_t incl = warp_inclusive_sum(cand);
  const uint32_t excl = incl - cand;
  const uint32_t total = __shfl_sync(0xffffffffu, incl, 31);
  const uint32_t mlo = (uint32_t)mask, mhi = (uint32_t)(mask >> 32);
  for (uint32_t w0 = 0; w0 < total; w0 += 32) {
    const uint32_t fidx = w0 + lane;
    const int owner = slot_owner(incl, fidx);
    const uint32_t olo = __shfl_sync(0xffffffffu, mlo, owner), ohi = __shfl_sync(0xffffffffu, mhi, owner);
    const uint32_t orect = __shfl_sync(0xffffffffu, rect, owner), oex = __shfl_sync(0xffffffffu, excl, owner);
    const uint32_t ooff = __shfl_sync(0xffffffffu, off, owner), ogid = __shfl_sync(0xffffffffu, gid, owner);
    if (fidx < total) {
      const uint32_t kk = fidx - oex;
      const uint64_t om = ((uint64_t)ohi << 32) | olo;
      if ((om >> kk) & 1ull) {
        const uint32_t ordinal = (uint32_t)__popcll(om & ((1ull << kk) - 1ull));
        const uint3 r = unpack_rect(orect);
        const uint2 slot = rect_slot(kk, r.z);
        const uint32_t tile = (r.y + slot.y) * gx + r.x + slot.x;
        const uint32_t dst = ooff + ordinal;
        if ((int64_t)dst < cap) {
          tile_keys[dst] = tile;
          tile_vals[dst] = ogid;
          tally(tile);
        }
      }
    }
  }
  // ---- rectangles without a mask: re-test, whole warp per Gaussian, ordered by ballot
  float4 A = make_float4(0.f, 0.f, 0.f, 0.f);
  Candidate cd = no_candidate();
  if (active && !small) {
    A = recA[gid];
    cd = make_candidate(A.x, A.y, radii[gid], recB[gid], A.w, gx, gy, (flags & GSB_RASTER_EXACT_TILE_CULL) != 0);
  }
  const uint32_t lt_mask = (1u << lane) - 1u;
  walk_large_rects(active && !small, A.x, A.y, cd, [&](int src) {
    const uint32_t soff = __shfl_sync(0xffffffffu, off, src), sgid = __shfl_sync(0xffffffffu, gid, src);
    return [&, soff, sgid](uint32_t done, bool keep, unsigned votes, uint32_t tx, uint32_t ty) {
      if (!keep) return;
      const uint32_t dst = soff + done + __popc(votes & lt_mask);
      if ((int64_t)dst < cap) {
        tile_keys[dst] = ty * gx + tx;
        tile_vals[dst] = sgid;
        tally(ty * gx + tx);
      }
    };
  });
  __syncthreads();
  for (int p = 0; p < hist_passes; ++p) {
    const uint32_t c = shist[p][threadIdx.x];
    if (c) atomicAdd(&ghist[p * kRdxBins + threadIdx.x], c);
  }
}

__global__ void __launch_bounds__(256) init_ranges_kernel(uint2* __restrict__ ranges, uint32_t ntiles) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < ntiles) ranges[t] = make_uint2(0xffffffffu, 0u);  // atomicMin / atomicMax targets; y <= x means empty
}

// rasterizer_impl.cu:116-138
__global__ void __launch_bounds__(256) tile_ranges_kernel(int64_t L, const uint64_t* __restrict__ keys,
                                                          uint2* __restrict__ ranges) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= L) return;
  const uint32_t cur = (uint32_t)(keys[idx] >> 32);
  if (idx == 0) {
    ranges[cur].x = 0;
  } else {
    const uint32_t prev = (uint32_t)(keys[idx - 1] >> 32);
    if (cur != prev) {
      ranges[prev].y = (uint32_t)idx;
      ranges[cur].x = (uint32_t)idx;
    }
  }
  if (idx == L - 1) ranges[cur].y = (uint32_t)L;
}

__device__ __forceinline__ float4 lds128(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr) : "memory");
  return v;
}
__device__ __forceinline__ float2 lds64(uint32_t addr) {
  float2 v;
  asm volatile("ld.shared.v2.f32 {%0,%1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(addr) : "memory");
  return v;
}
__device__ __forceinline__ void sts128(uint32_t addr, const float4& v) {
  asm volatile("st.shared.v4.f32 [%0], {%1,%2,%3,%4};" ::"r"(addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
__device__ __forceinline__ void sts64(uint32_t addr, const float2& v) {
  asm volatile("st.shared.v2.f32 [%0], {%1,%2};" ::"r"(addr), "f"(v.x), "f"(v.y) : "memory");
}

// forward.cu:261-374, re-organised: the blend without GSB_RASTER_FAST_EXP, with the reference's own exponent expression
// and full-precision expf (transmittance bit-identical to the reference's; the default table kernel below restructures
// the exponent).  Per 16x16 tile four warps that never wait for each other: every warp streams the tile's sorted
// instance list on its own, 32 Gaussians at a time -- each lane
// gathers ONE record (the warps of the CTA hit the same lines, so all but the first gather is an L1 hit) and tests it
// against the warp's 8x8 pixel block with the exact footprint test straight from registers.  The lanes whose Gaussian
// passed store their record at consecutive 48-byte slots (ballot rank) of the warp's private double-buffered list, so the
// blend loop walks plain consecutive addresses and is branch-free: the three thresholds of forward.cu:336-353 become
// predicates that gate a weight w = alpha*T (0 when the pixel skips the Gaussian) and the transmittance update.  An
// all-zero sentinel record (opacity 0 -> alpha 0 -> skipped) pads an odd hit count so the loop always takes two records
// per trip.  The next chunk's gathers are in flight while the current one is blended; a warp leaves as soon as its own 64
// pixels are saturated.  Skipped Gaussians are exactly the ones every pixel of the block would `continue` past in the
// reference loop; colours accumulate as fma(c, alpha*T, C) (the reference: fma(c*alpha, T, C), <= 1 ulp per term).
constexpr int kSlotBytes = 48;               // A (16) | B (16) | green, blue (8) | pad (8)
constexpr int kSlotsPerBuf = 33;             // 32 hits + sentinel
// kPix = 2 pixels per lane: 4 warps per tile, each an 8x8 block whose lanes own (x, y) and (x, y + 4): the list walk,
// the footprint test and the record loads are shared by 64 pixels.
constexpr int kPix = 2;
__global__ void __launch_bounds__(kTilePixels / kPix, 8)
    render_compact_kernel(const uint2* __restrict__ ranges, const uint32_t* __restrict__ point_list, int W, int H,
                          const float4* __restrict__ recA, const float4* __restrict__ recB, const float2* __restrict__ recC,
                          const float* __restrict__ bg, float* __restrict__ out_color, float* __restrict__ out_depth,
                          float* __restrict__ out_T, int64_t capacity) {
  constexpr int kWarps = 8 / kPix;
  __shared__ __align__(16) unsigned char slots[kWarps][2][kSlotsPerBuf * kSlotBytes];
  const uint32_t tiles_x = (W + kTile - 1) / kTile;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t a0 = smem_u32(&slots[warp][0][0]);
  const uint32_t blk_x = blockIdx.x * kTile + (warp & 1) * 8, blk_y = blockIdx.y * kTile + (warp >> 1) * (4 * kPix);
  const uint32_t pix_x = blk_x + (lane & 7), pix_y = blk_y + (lane >> 3);
  const float pfx = (float)pix_x;
  const float bx0 = (float)blk_x, by0 = (float)blk_y, bx1 = (float)(blk_x + 7), by1 = (float)(blk_y + 4 * kPix - 1);
  uint2 range = ranges[blockIdx.y * tiles_x + blockIdx.x];
  if (range.y <= range.x || (int64_t)range.y > capacity) range = make_uint2(0u, 0u);
  const int total = range.y - range.x;
  const uint32_t lt_mask = (1u << lane) - 1u;
  bool inside[kPix], done[kPix];
  float pfy[kPix], T[kPix], C0[kPix], C1[kPix], C2[kPix], Dz[kPix];
#pragma unroll
  for (int k = 0; k < kPix; ++k) {
    inside[k] = pix_x < (uint32_t)W && pix_y + 4 * k < (uint32_t)H;
    done[k] = !inside[k];
    pfy[k] = (float)(pix_y + 4 * k);
    T[k] = 1.0f;
    C0[k] = C1[k] = C2[k] = Dz[k] = 0.f;
  }

  float4 cA = make_float4(0.f, 0.f, 0.f, 0.f), cB = cA, nA = cA, nB = cA;
  float2 cC = make_float2(0.f, 0.f), nC = cC;
  if (lane < total) {
    const uint32_t g = point_list[range.x + lane];
    cA = recA[g];
    cB = recB[g];
    cC = recC[g];
  }
  // one Gaussian of the warp's list against this lane's pixel(s)
  auto blend = [&](uint32_t addr) {
    const float4 A = lds128(addr), B = lds128(addr + 16);
    const float2 gb = lds64(addr + 32);
    const float dx = A.x - pfx;
#pragma unroll
    for (int k = 0; k < kPix; ++k) {
      const float dy = A.y - pfy[k];
      const float power = -0.5f * (B.x * dx * dx + B.z * dy * dy) - B.y * dx * dy;
      const float alpha = min(0.99f, A.w * exp(power));
      const float test_T = T[k] * (1 - alpha);
      const bool cand = !done[k] && !(power > 0.0f) && !(alpha < 1.0f / 255.0f);
      const bool sat = cand && test_T < 0.0001f;
      const bool ok = cand && !sat;
      done[k] = done[k] || sat;
      const float w = ok ? alpha * T[k] : 0.f;
      C0[k] = fmaf(B.w, w, C0[k]);
      C1[k] = fmaf(gb.x, w, C1[k]);
      C2[k] = fmaf(gb.y, w, C2[k]);
      Dz[k] = fmaf(A.z, w, Dz[k]);
      T[k] = ok ? test_T : T[k];
    }
  };
  for (int c0 = 0; c0 < total; c0 += 32) {
    bool all_done = done[0];
#pragma unroll
    for (int k = 1; k < kPix; ++k) all_done = all_done && done[k];
    if (__all_sync(0xffffffffu, all_done)) break;
    const int nxt = c0 + 32 + lane;
    if (nxt < total) {  // next chunk's gathers fly while this one is tested and blended
      const uint32_t g = point_list[range.x + nxt];
      nA = recA[g];
      nB = recB[g];
      nC = recC[g];
    }
    bool hit = false;
    if (c0 + lane < total) {
      const Footprint fp = make_footprint(cB.x, cB.y, cB.z, 2.f * __logf(255.f * cA.w) + 1e-3f);
      hit = rect_can_contribute(cA.x, cA.y, fp, bx0, by0, bx1, by1);
    }
    const unsigned votes = __ballot_sync(0xffffffffu, hit);
    const int n = __popc(votes);
    const uint32_t buf = a0 + ((c0 >> 5) & 1) * (kSlotsPerBuf * kSlotBytes);
    if (hit) {
      const uint32_t dst = buf + __popc(votes & lt_mask) * kSlotBytes;
      sts128(dst, cA);
      sts128(dst + 16, cB);
      sts64(dst + 32, cC);
    }
    if (lane == 0) {  // sentinel after the last hit
      const uint32_t dst = buf + n * kSlotBytes;
      const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
      sts128(dst, z);
      sts128(dst + 16, z);
      sts64(dst + 32, make_float2(0.f, 0.f));
    }
    __syncwarp();  // the list is visible to every lane of the warp
    uint32_t addr = buf;
    for (int j = 0; j < n; j += 2, addr += 2 * kSlotBytes) {
      blend(addr);
      blend(addr + kSlotBytes);
    }
    cA = nA;
    cB = nB;
    cC = nC;
  }
  const size_t plane = (size_t)H * W;
#pragma unroll
  for (int k = 0; k < kPix; ++k)
    if (inside[k]) {
      const size_t pid = (size_t)(pix_y + 4 * k) * W + pix_x;
      out_color[pid] = C0[k] + T[k] * bg[0];
      out_color[plane + pid] = C1[k] + T[k] * bg[1];
      out_color[2 * plane + pid] = C2[k] + T[k] * bg[2];
      if (out_depth) out_depth[pid] = Dz[k];
      if (out_T) out_T[pid] = T[k];
    }
}

// ---------------------------------------------------------------------------------------------
// Table kernel (the GSB_RASTER_FAST_EXP blend, default): render_compact_kernel's per-warp compacted hit list, but the blend
// loop -- 29 issue slots per (record, pixel) in that kernel's shape with ex2.approx -- is cut to ~16 by moving everything
// that does not depend on the pixel out of it.
// FSETP / FSEL / FMNMX issue on the ALU pipe, which has half the FMA pipe's rate, and MUFU.EX2 is slower still.  Here:
//  * the exponent is evaluated in the log2 domain as  e = u'(x) + v(x)*dy(y) + w(y)  with
//        u'(x) = -0.5 log2e a dx^2 + log2(opacity),  v(x) = -log2e b dx,  w(y) = -0.5 log2e c dy^2 ;
//    the lane that compacts a record writes u', v for the warp block's 8 columns and dy, w for its 8 rows into the
//    record's slot (once per record and warp), so a pixel costs one FFMA + one FADD, and alpha = ex2(e)
//    needs no opacity multiply;
//  * both pixels of a lane (rows y and y+4) share the record's loads; (T0, T1) stay in one aligned register pair;
//  * the three thresholds of forward.cu:336-353 are three FSETPs with two predicate outputs each; the colour / depth
//    accumulation and the transmittance update are PREDICATED scalar FFMA/FMULs (FMA pipe) instead of FSELs (ALU pipe);
//  * "done" lives in the sign of T: a saturated pixel keeps its transmittance with the sign bit set, every later
//    test_T = T*(1-alpha) is negative, i.e. < 1e-4, so nothing is accumulated any more; |T| is written out.
// The exponent's rounding differs from the reference's expression by a few ulp of its largest term (as any
// re-association does); gated on the full-size parity tests against the reference binary (tests/test_gpu_pipeline.py).
constexpr int kTabSlotBytes = 160;  // X table 8 x (u',v) | Y table 4 x (dy0,dy1,w0,w1) | (r,g,b,z) | (thr,0,0,0)
constexpr int kTabSlots = 36;       // 32 hits + sentinel + the pair the pipelined loop reads ahead
constexpr int kTabX = 0, kTabY = 64, kTabC = 128, kTabThr = 144;

__device__ __forceinline__ float lds32(uint32_t addr) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr) : "memory");
  return v;
}

// One record against the lane's two pixels.  (u, v) = this lane's column entry, (dy0, dy1, w0, w1) = its row entry,
// thr = log2(opacity) (e > thr <=> power > 0), TT = packed (T0, T1) with the sign bit as the "done" flag.
// Written in PTX so that the thresholds are exactly three compares per pixel with chained predicates, the accumulation
// and the transmittance update are predicated FMA-pipe instructions, and T stays in one aligned register pair.
// NaNs fall through the tests like in the reference (leu / geu are true for unordered operands).
// The record is blended in two stages, for the software-pipelined loop of render_table_kernel: stage A is everything that does
// not depend on the transmittance (alpha of the lane's two pixels, forced to 0 where the reference `continue`s, so the
// record becomes inert: T * (1 - 0) = T, colour += c * 0), stage B the short serial part.  A warp left alone on its SM (the
// silhouette tiles that walk their whole list end the kernel as a handful of serial chains) then pays ~the T chain per
// record instead of load + exponent + exp + chain (tests/test_blend_formulation.py states the equivalence on the CPU).
__device__ __forceinline__ unsigned long long blend_stage_alpha(float u, float v, float dy0, float dy1, float w0, float w1, float thr) {
  unsigned long long al;
  asm("{\n"
      ".reg .f32 e0, e1, x0, x1, a0, a1;\n"
      ".reg .pred p1a, p2a, p1b, p2b;\n"
      "fma.rn.f32 e0, %6, %1, %5;\n"              // u'(x) + v(x) * dy(y)
      "fma.rn.f32 e1, %6, %2, %5;\n"
      "add.rn.f32 e0, e0, %3;\n"                  //   + w(y): log2-domain exponent incl. log2(opacity)
      "add.rn.f32 e1, e1, %4;\n"
      "ex2.approx.ftz.f32 x0, e0;\n"
      "ex2.approx.ftz.f32 x1, e1;\n"
      "min.f32 a0, x0, 0f3F7D70A4;\n"             // forward.cu:341  alpha = min(0.99f, ...)
      "min.f32 a1, x1, 0f3F7D70A4;\n"
      "setp.leu.f32 p1a, e0, %7;\n"                    // forward.cu:336  if (power > 0.0f) continue;
      "setp.leu.f32 p1b, e1, %7;\n"
      "setp.geu.and.f32 p2a, a0, 0f3B808081, p1a;\n"    // forward.cu:344  if (alpha < 1.0f / 255.0f) continue;
      "setp.geu.and.f32 p2b, a1, 0f3B808081, p1b;\n"
      "selp.f32 a0, a0, 0f00000000, p2a;\n"
      "selp.f32 a1, a1, 0f00000000, p2b;\n"
      "mov.b64 %0, {a0, a1};\n"
      "}\n"
      : "=l"(al)
      : "f"(dy0), "f"(dy1), "f"(w0), "f"(w1), "f"(u), "f"(v), "f"(thr));
  return al;
}

__device__ __forceinline__ void blend_stage_apply(unsigned long long al, float r, float g, float b, float z, unsigned long long& TT,
                                                  float& C00, float& C10, float& C20, float& Dz0, float& C01, float& C11, float& C21,
                                                  float& Dz1) {
  asm("{\n"
      ".reg .f32 al0, al1, oma0, oma1, tn0, tn1, ww0, ww1, t0, t1;\n"
      ".reg .pred oka, okb;\n"
      "mov.b64 {al0, al1}, %9;\n"
      "mov.b64 {t0, t1}, %0;\n"
      "fma.rn.f32 oma0, al0, 0fBF800000, 0f3F800000;\n"  // 1 - alpha (exactly rounded, like the reference's subtraction)
      "fma.rn.f32 oma1, al1, 0fBF800000, 0f3F800000;\n"
      "mul.rn.f32 tn0, t0, oma0;\n"               // test_T = T * (1 - alpha)
      "mul.rn.f32 tn1, t1, oma1;\n"
      "mul.rn.f32 ww0, al0, t0;\n"                // alpha * T
      "mul.rn.f32 ww1, al1, t1;\n"
      "setp.geu.f32 oka, tn0, 0f38D1B717;\n"      // forward.cu:347  if (test_T < 0.0001f) { done = true; continue; }
      "setp.geu.f32 okb, tn1, 0f38D1B717;\n"      //   (T >= 1e-4 while the pixel lives, negative once done: an inert record passes)
      "@oka fma.rn.f32 %1, %10, ww0, %1;\n"
      "@oka fma.rn.f32 %2, %11, ww0, %2;\n"
      "@oka fma.rn.f32 %3, %12, ww0, %3;\n"
      "@oka fma.rn.f32 %4, %13, ww0, %4;\n"
      "@okb fma.rn.f32 %5, %10, ww1, %5;\n"
      "@okb fma.rn.f32 %6, %11, ww1, %6;\n"
      "@okb fma.rn.f32 %7, %12, ww1, %7;\n"
      "@okb fma.rn.f32 %8, %13, ww1, %8;\n"
      "@oka mov.f32 t0, tn0;\n"                   // T = test_T
      "@okb mov.f32 t1, tn1;\n"
      "@!oka or.b32 t0, t0, 0x80000000;\n"        // done: keep |T|, set the sign
      "@!okb or.b32 t1, t1, 0x80000000;\n"
      "mov.b64 %0, {t0, t1};\n"
      "}\n"
      : "+l"(TT), "+f"(C00), "+f"(C10), "+f"(C20), "+f"(Dz0), "+f"(C01), "+f"(C11), "+f"(C21), "+f"(Dz1)
      : "l"(al), "f"(r), "f"(g), "f"(b), "f"(z));
}

__device__ __forceinline__ unsigned long long pack_f32x2(float lo, float hi) {
  return (unsigned long long)__float_as_uint(lo) | ((unsigned long long)__float_as_uint(hi) << 32);
}

// One CTA per tile in the hardware's block order: it mixes long and short lists on every SM, so the gather latency of the
// short ones hides behind the arithmetic of the long ones; a queue sorted by list length would end the kernel in a long
// phase of latency-bound tiles, and a persistent grid would keep the kernels of the other in-flight views off the SMs.
__global__ void __launch_bounds__(kTilePixels / 2, 7)
    render_table_kernel(const uint2* __restrict__ ranges, const uint32_t* __restrict__ point_list, int W, int H,
                        const float4* __restrict__ recA, const float4* __restrict__ recB, const float2* __restrict__ recC,
                        const float* __restrict__ bg, float* __restrict__ out_color, float* __restrict__ out_depth,
                        float* __restrict__ out_T, int64_t capacity) {
  constexpr int kWarps = 4;
  __shared__ __align__(16) unsigned char slots[kWarps][kTabSlots * kTabSlotBytes];
  const uint32_t tiles_x = (W + kTile - 1) / kTile;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t a0 = smem_u32(&slots[warp][0]);
  const uint32_t xoff = kTabX + (lane & 7) * 8, yoff = kTabY + (lane >> 3) * 16;
  const uint32_t lt_mask = (1u << lane) - 1u;
  // per-lane bases of the column / row entries; `off` (byte offset of the record's slot) is warp-uniform
  const uint32_t xbase = a0 + xoff, ybase = a0 + yoff;
  const float bg0 = bg[0], bg1 = bg[1], bg2 = bg[2];
  {
    const uint32_t tile = blockIdx.y * tiles_x + blockIdx.x;
    const uint32_t blk_x = blockIdx.x * kTile + (warp & 1) * 8, blk_y = blockIdx.y * kTile + (warp >> 1) * 8;
    const uint32_t pix_x = blk_x + (lane & 7), pix_y = blk_y + (lane >> 3);
    const float bx0 = (float)blk_x, by0 = (float)blk_y, bx1 = (float)(blk_x + 7), by1 = (float)(blk_y + 7);
    uint2 range = ranges[tile];
    if (range.y <= range.x || (int64_t)range.y > capacity) range = make_uint2(0u, 0u);
    const int total = range.y - range.x;
    const bool inside0 = pix_x < (uint32_t)W && pix_y < (uint32_t)H, inside1 = pix_x < (uint32_t)W && pix_y + 4 < (uint32_t)H;
    // the sign of T is the pixel's "done" flag
    unsigned long long TT = pack_f32x2(inside0 ? 1.0f : -1.0f, inside1 ? 1.0f : -1.0f);
    float C00 = 0.f, C10 = 0.f, C20 = 0.f, Dz0 = 0.f, C01 = 0.f, C11 = 0.f, C21 = 0.f, Dz1 = 0.f;

    float4 cA = make_float4(0.f, 0.f, 0.f, 0.f), cB = cA, nA = cA, nB = cA;
    float2 cC = make_float2(0.f, 0.f), nC = cC;
    // record indices run two chunks ahead of the blend, records one: the record gather of the next chunk never waits for
    // its index (in-order issue would stall the whole chunk on that dependent load)
    uint32_t g_next = 0;
    if (lane < total) {
      const uint32_t g = point_list[range.x + lane];
      if (32 + lane < total) g_next = point_list[range.x + 32 + lane];
      cA = recA[g];
      cB = recB[g];
      cC = recC[g];
    }
    auto alpha_of = [&](uint32_t off) {  // stage A of the record in slot `off`
      const float2 X = lds64(xbase + off);       // u', v of this lane's column
      const float4 Y = lds128(ybase + off);      // dy, w of this lane's two rows
      const float thr = lds32(a0 + kTabThr + off);
      return blend_stage_alpha(X.x, X.y, Y.x, Y.y, Y.z, Y.w, thr);
    };
    auto apply = [&](uint32_t off, unsigned long long al) {  // stage B
      const float4 Q = lds128(a0 + kTabC + off);  // r, g, b, z
      blend_stage_apply(al, Q.x, Q.y, Q.z, Q.w, TT, C00, C10, C20, Dz0, C01, C11, C21, Dz1);
    };
    for (int c0 = 0; c0 < total; c0 += 32) {
      if (__all_sync(0xffffffffu, (TT & 0x8000000080000000ull) == 0x8000000080000000ull)) break;  // both pixels done
      const int nxt = c0 + 32 + lane;
      if (nxt < total) {  // next chunk's gathers fly while this one is tested and blended
        nA = recA[g_next];
        nB = recB[g_next];
        nC = recC[g_next];
        if (nxt + 32 < total) g_next = point_list[range.x + nxt + 32];
      }
      bool hit = false;
      if (c0 + lane < total) {
        const Footprint fp = make_footprint(cB.x, cB.y, cB.z, 2.f * __logf(255.f * cA.w) + 1e-3f);
        hit = rect_can_contribute(cA.x, cA.y, fp, bx0, by0, bx1, by1);
      }
      const unsigned votes = __ballot_sync(0xffffffffu, hit);
      const int n = __popc(votes);
      if (hit) {  // this lane's record goes to slot `rank`: per-column and per-row terms of the exponent, colour, depth
        const uint32_t dst = a0 + __popc(votes & lt_mask) * kTabSlotBytes;
        const float ap = -0.72134752044448170f * cB.x, bp = -1.4426950408889634f * cB.y, cp = -0.72134752044448170f * cB.z;
        const float l2o = __log2f(cA.w);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float dx = cA.x - (bx0 + (float)i);
          sts64(dst + kTabX + 8 * i, make_float2(fmaf(ap * dx, dx, l2o), bp * dx));
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float dy0 = cA.y - (by0 + (float)j), dy1 = cA.y - (by0 + (float)(j + 4));
          sts128(dst + kTabY + 16 * j, make_float4(dy0, dy1, cp * dy0 * dy0, cp * dy1 * dy1));
        }
        sts128(dst + kTabC, make_float4(cB.w, cC.x, cC.y, cA.z));
        sts128(dst + kTabThr, make_float4(l2o, 0.f, 0.f, 0.f));
      }
      if (n != 0) {  // (a chunk none of whose records reaches the block costs no more than the test)
        if ((n & 1) && lane < kTabSlotBytes / 16) {  // odd count: sentinel after the last hit, u' = -1e30 -> alpha 0 -> skipped
          const float big = lane < 4 ? -1.0e30f : 0.f;  // quads 0..3 = the X table: (u', v, u', v)
          sts128(a0 + n * kTabSlotBytes + 16 * lane, make_float4(big, 0.f, big, 0.f));
        }
        __syncwarp();  // the list is visible to every lane of the warp
        const uint32_t end = (uint32_t)n * kTabSlotBytes;
        unsigned long long al0 = alpha_of(0), al1 = alpha_of(kTabSlotBytes);
        for (uint32_t off = 0; off < end; off += 2 * kTabSlotBytes) {
          // the next pair's alphas are in flight while this pair's T chain resolves (past the end: two slots of stale
          // bytes, computed and dropped)
          const unsigned long long nx0 = alpha_of(off + 2 * kTabSlotBytes), nx1 = alpha_of(off + 3 * kTabSlotBytes);
          apply(off, al0);
          apply(off + kTabSlotBytes, al1);
          al0 = nx0;
          al1 = nx1;
        }
        __syncwarp();  // every lane is done reading before the next chunk overwrites the slots
      }
      cA = nA;
      cB = nB;
      cC = nC;
    }
    const size_t plane = (size_t)H * W;
    const float Tf0 = fabsf(__uint_as_float((uint32_t)TT)), Tf1 = fabsf(__uint_as_float((uint32_t)(TT >> 32)));
    if (inside0) {
      const size_t pid = (size_t)pix_y * W + pix_x;
      out_color[pid] = C00 + Tf0 * bg0;
      out_color[plane + pid] = C10 + Tf0 * bg1;
      out_color[2 * plane + pid] = C20 + Tf0 * bg2;
      if (out_depth) out_depth[pid] = Dz0;
      if (out_T) out_T[pid] = Tf0;
    }
    if (inside1) {
      const size_t pid = (size_t)(pix_y + 4) * W + pix_x;
      out_color[pid] = C01 + Tf1 * bg0;
      out_color[plane + pid] = C11 + Tf1 * bg1;
      out_color[2 * plane + pid] = C21 + Tf1 * bg2;
      if (out_depth) out_depth[pid] = Dz1;
      if (out_T) out_T[pid] = Tf1;
    }
  }
}

__global__ void write_counts_kernel(const uint32_t* __restrict__ offsets, int P, const unsigned long long* counters,
                                    int64_t* out) {
  // offsets != NULL: validation path (instance total = last element of the per-Gaussian scan)
  out[0] = offsets ? (P > 0 ? (int64_t)offsets[P - 1] : 0) : (int64_t)counters[1];
  out[1] = (int64_t)counters[0];
  out[2] = (int64_t)counters[2];
  out[3] = (int64_t)counters[3];
}

__global__ void __launch_bounds__(256) mark_visible_kernel(int P, const float* __restrict__ means,
                                                           const float* __restrict__ vm, uint8_t* present) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= P) return;
  const float x = means[3 * (size_t)idx], y = means[3 * (size_t)idx + 1], z = means[3 * (size_t)idx + 2];
  present[idx] = (vm[2] * x + vm[6] * y + vm[10] * z + vm[14]) > 0.2f ? 1 : 0;
}

// cv::saturate_cast<uchar>(v): round half to even, clamp to [0,255]
__global__ void __launch_bounds__(256) to_u8_kernel(const float* __restrict__ chw, int W, int H, uint8_t* __restrict__ hwc) {
  const size_t n = (size_t)W * H;
  const size_t pid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (pid >= n) return;
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) {
    const float v = chw[ch * n + pid] * 255.f;
    int q = __float2int_rn(v);
    q = q < 0 ? 0 : (q > 255 ? 255 : q);
    if (!(v == v)) q = 0;
    hwc[pid * 3 + ch] = (uint8_t)q;
  }
}

// rasterizer_impl.cu:35-50
uint32_t higher_msb(uint32_t n) {
  uint32_t msb = sizeof(n) * 4, step = msb;
  while (step > 1) {
    step /= 2;
    if (n >> msb)
      msb += step;
    else
      msb -= step;
  }
  if (n >> msb) msb++;
  return msb;
}

struct Workspace {
  float4* recA;
  float4* recB;
  float2* recC;
  uint32_t* tiles;
  uint32_t* offsets;
  int* radii;
  unsigned long long* counters;  // [0] reference instance count
  uint2* ranges;
  uint32_t* depth_a;
  uint32_t* depth_b;
  uint32_t* ids_a;
  uint32_t* ids_b;
  uint32_t* sorted_offsets;
  uint64_t* masks;
  uint32_t* rects;
  uint32_t* scan_status;  // scan_tiles_kernel: [0] ticket, [64..] per-block status words
  uint32_t* radix_scratch;
  uint64_t* keys_in;
  uint64_t* keys_out;
  uint32_t* vals_in;
  uint32_t* vals_out;
  void* scan_temp;
  size_t scan_temp_bytes;
  void* sort_temp;
  size_t sort_temp_bytes;
  size_t total;
};

Workspace carve(void* base, int32_t P, int32_t W, int32_t H, int64_t R) {
  Workspace w{};
  Carver c(base);
  const size_t Pn = (size_t)(P > 1 ? P : 1), Rn = (size_t)(R > 1 ? R : 1);
  const size_t ntiles = (size_t)((W + kTile - 1) / kTile) * ((H + kTile - 1) / kTile);
  w.recA = c.take<float4>(Pn);
  w.recB = c.take<float4>(Pn);
  w.recC = c.take<float2>(Pn);
  w.tiles = c.take<uint32_t>(Pn);
  w.offsets = c.take<uint32_t>(Pn);
  w.radii = c.take<int>(Pn);
  w.counters = c.take<unsigned long long>(8);
  w.ranges = c.take<uint2>(ntiles);
  w.depth_a = c.take<uint32_t>(Pn);
  w.depth_b = c.take<uint32_t>(Pn);
  w.ids_a = c.take<uint32_t>(Pn);
  w.ids_b = c.take<uint32_t>(Pn);
  w.sorted_offsets = c.take<uint32_t>(Pn);
  w.masks = c.take<uint64_t>(Pn);
  w.rects = c.take<uint32_t>(Pn);
  w.scan_status = c.take<uint32_t>((Pn + kScanBlock - 1) / kScanBlock + 64);
  w.radix_scratch = c.take<uint32_t>(radix_scratch_words(std::max(Pn, Rn)));
  w.keys_in = c.take<uint64_t>(Rn);
  w.keys_out = c.take<uint64_t>(Rn);
  w.vals_in = c.take<uint32_t>(Rn);
  w.vals_out = c.take<uint32_t>(Rn);
  cub::DeviceScan::InclusiveSum(nullptr, w.scan_temp_bytes, (uint32_t*)nullptr, (uint32_t*)nullptr, (int)Pn);
  w.scan_temp = c.take<char>(w.scan_temp_bytes);
  cub::DeviceRadixSort::SortPairs(nullptr, w.sort_temp_bytes, (uint64_t*)nullptr, (uint64_t*)nullptr, (uint32_t*)nullptr,
                                  (uint32_t*)nullptr, (int64_t)Rn);
  w.sort_temp = c.take<char>(w.sort_temp_bytes);
  w.total = c.total();
  return w;
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// Zeroes every eye's counters and runs the preprocess pass over the pp.P Gaussians.
template <int kEyes, int kMinBlocks>
int preprocess(const PreParams& pp, cudaStream_t stream, bool dbg) {
  for (int e = 0; e < kEyes; ++e)
    GSB_CUDA_OK(cudaMemsetAsync(pp.eye[e].counters, 0, 8 * sizeof(unsigned long long), stream));
  {
    StageTimer tm(kStPreprocess, stream);
    preprocess_kernel<kEyes, kMinBlocks><<<(pp.P + kPreThreads - 1) / kPreThreads, kPreThreads, 0, stream>>>(pp);
  }
  count_launch();
  return check_launch(kEyes == 2 ? "preprocess_kernel<2>" : "preprocess_kernel", stream, dbg);
}

}  // namespace
}  // namespace gsb

using namespace gsb;

extern "C" {

const char* gsb_last_error(void) { return g_error; }
int gsb_version(void) { return GSB_VERSION; }
uint64_t gsb_kernel_launch_count(void) { return g_launches.load(); }

int gsb_profile_num_stages(void) { return kStCount; }
const char* gsb_profile_stage_name(int stage) { return stage >= 0 && stage < kStCount ? kStageNames[stage] : ""; }
int gsb_profile_enable(int on) {
  g_prof.enabled.store(on != 0);
  return GSB_OK;
}
int gsb_profile_collect(double* total_ms, uint64_t* samples, int n_stages) {
  if (!total_ms || !samples || n_stages < kStCount) return fail(GSB_ERR_INVALID, "profile_collect: need %d stages", (int)kStCount);
  GSB_CUDA_OK(cudaDeviceSynchronize());
  std::lock_guard<std::mutex> lk(g_prof.mu);
  for (int i = 0; i < n_stages; ++i) {
    total_ms[i] = 0.0;
    samples[i] = 0;
  }
  for (const Profiler::Rec& r : g_prof.recs) {
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, r.a, r.b) == cudaSuccess) {
      total_ms[r.stage] += ms;
      samples[r.stage] += 1;
    }
    g_prof.pool.push_back(r.a);
    g_prof.pool.push_back(r.b);
  }
  g_prof.recs.clear();
  return GSB_OK;
}

size_t gsb_raster_workspace_bytes(int32_t P, int32_t width, int32_t height, int64_t max_instances) {
  return carve(nullptr, P, width, height, max_instances).total;
}

struct Frame {  // one eye's call, validated and carved
  const GsbRasterArgs* a;
  Workspace ws;
  uint32_t gx, gy;
  size_t ntiles;
  int64_t cap;
  bool dbg, use_cub;
  int* radii;
};

static int render_frame_impl(const Frame& f, const uint32_t* point_list, cudaStream_t stream);

// One event per device for ordering the right eye's stream behind the shared part of a pair (a stream wait captures the
// event's state when it is enqueued, so the event can be re-recorded by the next pair).
static cudaEvent_t pair_event() {
  static std::mutex mu;
  static cudaEvent_t events[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  std::lock_guard<std::mutex> lk(mu);
  cudaEvent_t& e = events[dev & 63];
  if (!e) cudaEventCreateWithFlags(&e, cudaEventDisableTiming);
  return e;
}

constexpr uint32_t kRasterFlags = GSB_RASTER_EXACT_TILE_CULL | GSB_RASTER_NO_TMA | GSB_RASTER_DEBUG_SYNC | GSB_RASTER_CUB_SORT |
                                  GSB_RASTER_FAST_EXP | GSB_RASTER_PAIR_SHARED_DEPTH | GSB_RASTER_ASYNC;

static int validate_frame(const GsbRasterArgs* a, Frame& f) {
  if (!a) return fail(GSB_ERR_INVALID, "args is NULL");
  if (a->P < 0 || a->width <= 0 || a->height <= 0) return fail(GSB_ERR_INVALID, "bad P / image size");
  constexpr int kMaxSide = (int)kRectCoordMax * kTile;  // packed candidate rectangles hold kRectCoordBits-bit tile coordinates
  if (a->width > kMaxSide || a->height > kMaxSide) return fail(GSB_ERR_INVALID, "image side exceeds %d pixels", kMaxSide);
  if (!a->out_color || !a->background || !a->viewmatrix || !a->projmatrix || !a->cam_pos)
    return fail(GSB_ERR_INVALID, "out_color, background, viewmatrix, projmatrix and cam_pos are required");
  // DGR/diff_gaussian_rasterization/__init__.py:191-195
  if ((a->shs == nullptr) == (a->colors_precomp == nullptr))
    return fail(GSB_ERR_INVALID, "Please provide excatly one of either SHs or precomputed colors!");
  if (((a->scales == nullptr || a->rotations == nullptr) && a->cov3D_precomp == nullptr) ||
      ((a->scales != nullptr || a->rotations != nullptr) && a->cov3D_precomp != nullptr))
    return fail(GSB_ERR_INVALID,
                "Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!");
  if (a->shs && (a->sh_coeffs <= 0 || a->sh_coeffs > 16 || a->sh_degree < 0 || a->sh_degree > 3 ||
                 (a->sh_degree + 1) * (a->sh_degree + 1) > a->sh_coeffs))
    return fail(GSB_ERR_INVALID, "SH degree %d needs %d coefficients, tensor has %d (max 16)", a->sh_degree,
                (a->sh_degree + 1) * (a->sh_degree + 1), a->sh_coeffs);
  if (a->flags & ~kRasterFlags)
    return fail(GSB_ERR_INVALID, "flags 0x%x: undefined bits 0x%x (not a GSB_RASTER_* flag)", (unsigned)a->flags,
                (unsigned)(a->flags & ~kRasterFlags));
  if (!a->workspace)return fail(GSB_ERR_WORKSPACE, "workspace is NULL");
  if (a->max_instances >= (int64_t)kStVal)  // the emit pass's scan words hold 30-bit instance counts
    return fail(GSB_ERR_INVALID, "max_instances must be below 2^30 - 1");
  f.a = a;
  f.cap = a->max_instances;
  f.ws = carve(a->workspace, a->P, a->width, a->height, f.cap);
  if (f.ws.total > a->workspace_bytes)
    return fail(GSB_ERR_WORKSPACE, "workspace has %zu bytes, %zu needed", a->workspace_bytes, f.ws.total);
  f.dbg = (a->flags & GSB_RASTER_DEBUG_SYNC) != 0;
  f.use_cub = (a->flags & GSB_RASTER_CUB_SORT) != 0;
  f.gx = (a->width + kTile - 1) / kTile;
  f.gy = (a->height + kTile - 1) / kTile;
  f.ntiles = (size_t)f.gx * f.gy;
  f.radii = a->radii ? a->radii : f.ws.radii;
  return GSB_OK;
}

static int empty_frame(const GsbRasterArgs* a, cudaStream_t stream) {  // rasterize_points.cu:77: outputs stay zero-filled
  const size_t npix = (size_t)a->width * a->height;
  GSB_CUDA_OK(cudaMemsetAsync(a->out_color, 0, 3 * npix * sizeof(float), stream));
  if (a->out_depth) GSB_CUDA_OK(cudaMemsetAsync(a->out_depth, 0, npix * sizeof(float), stream));
  if (a->out_final_T) GSB_CUDA_OK(cudaMemsetAsync(a->out_final_T, 0, npix * sizeof(float), stream));
  if (a->num_rendered) GSB_CUDA_OK(cudaMemsetAsync(a->num_rendered, 0, 4 * sizeof(int64_t), stream));
  return GSB_OK;
}

static void fill_common(const Frame& f, PreParams& pp) {
  const GsbRasterArgs* a = f.a;
  const bool has_sr = a->scales != nullptr && a->rotations != nullptr;
  pp.P = a->P;
  pp.D = a->sh_degree;
  pp.M = a->sh_coeffs;
  pp.W = a->width;
  pp.H = a->height;
  pp.means3D = a->means3D;
  pp.shs = a->shs;
  pp.colors = a->colors_precomp;
  pp.opacities = a->opacities;
  pp.scales = a->scales;
  pp.rotations = a->rotations;
  pp.cov3D = a->cov3D_precomp;
  pp.scale_modifier = a->scale_modifier;
  pp.gx = f.gx;
  pp.gy = f.gy;
  pp.flags = a->flags;
  pp.use_tma = !(a->flags & GSB_RASTER_NO_TMA) && aligned16(a->means3D) && aligned16(a->opacities) &&
               (!has_sr || (aligned16(a->scales) && aligned16(a->rotations))) && (!a->shs || aligned16(a->shs));
}

static void fill_eye(const Frame& f, PreEye& e) {
  const GsbRasterArgs* a = f.a;
  e.view = a->viewmatrix;
  e.proj = a->projmatrix;
  e.campos = a->cam_pos;
  e.tan_fovx = a->tan_fovx;
  e.tan_fovy = a->tan_fovy;
  e.focal_y = a->height / (2.0f * a->tan_fovy);  // rasterizer_impl.cu:222-223
  e.focal_x = a->width / (2.0f * a->tan_fovx);
  e.recA = f.ws.recA;
  e.recB = f.ws.recB;
  e.recC = f.ws.recC;
  e.tiles = f.ws.tiles;
  e.radii = f.radii;
  e.counters = f.ws.counters;
  e.masks = f.ws.masks;
  e.rects = f.ws.rects;
  e.depth_keys = f.ws.depth_a;
}

// Stable sort of the P (depth bits, Gaussian index) pairs in `f`'s buffers; the last pass also delivers tiles-per-Gaussian in
// depth order for `f` (into f.ws.offsets) and, for a stereo pair, for `g` (into g->ws.offsets).
static int depth_sort(const Frame& f, const Frame* g, cudaStream_t stream, const uint32_t** ids_sorted) {
  uint64_t nl = 0;
  const int P = f.a->P;
  {
    StageTimer tm(kStScan, stream);
    const int which = radix_sort_pairs(f.ws.depth_a, f.ws.ids_a, f.ws.depth_b, f.ws.ids_b, (uint32_t)P, nullptr, 0, (size_t)P, 32,
                                       f.ws.radix_scratch, nullptr, stream, &nl, /*histogram_ready=*/false, f.ws.tiles, f.ws.offsets,
                                       g ? g->ws.tiles : nullptr, g ? g->ws.offsets : nullptr, /*identity_payload=*/true);
    *ids_sorted = which ? f.ws.ids_b : f.ws.ids_a;
  }
  count_launch(nl);
  return check_launch("depth sort", stream, f.dbg);
}

// emit (+ scan) -> stable tile split -> blend, for one eye whose Gaussians are already in depth order
static int bin_and_render(const Frame& f, const uint32_t* ids_sorted, cudaStream_t stream) {
  const GsbRasterArgs* a = f.a;
  const Workspace& ws = f.ws;
  const int P = a->P;
  const int64_t cap = f.cap;
  const uint32_t gx = f.gx, gy = f.gy;
  const size_t ntiles = f.ntiles;
  uint32_t* rs = ws.radix_scratch;
  uint64_t nl = 0;
  int rc;
  // tile-id sort buffers alias the 64-bit key arrays of the validation path
  uint32_t* tk_a = reinterpret_cast<uint32_t*>(ws.keys_in);
  uint32_t* tv_a = tk_a + cap;
  uint32_t* tk_b = reinterpret_cast<uint32_t*>(ws.keys_out);
  uint32_t* tv_b = tk_b + cap;
  const int tile_bits = (int)higher_msb((uint32_t)ntiles);
  const uint32_t* point_list;
  {
    StageTimer tm(kStEmit, stream);
    radix_prepare(rs, (size_t)cap, tile_bits, stream);
    const int sblocks = (P + kScanBlock - 1) / kScanBlock;
    GSB_CUDA_OK(cudaMemsetAsync(ws.scan_status, 0, ((size_t)sblocks + 64) * sizeof(uint32_t), stream));
    scan_tiles_kernel<<<sblocks, kScanThreads, 0, stream>>>(P, ws.offsets, ws.sorted_offsets, cap, ws.counters, ws.scan_status + 64,
                                                            ws.scan_status);
    emit_sorted_kernel<<<(P + kEmitThreads - 1) / kEmitThreads, kEmitThreads, 0, stream>>>(
        P, ids_sorted, ws.offsets, ws.sorted_offsets, ws.recA, ws.recB, f.radii, ws.masks, ws.rects, gx, gy, a->flags, cap, tk_a, tv_a,
        radix_ghist(rs), (tile_bits + 7) / 8, radix_digit_bits(tile_bits));
    init_ranges_kernel<<<(unsigned)((ntiles + 255) / 256), 256, 0, stream>>>(ws.ranges, (uint32_t)ntiles);
    nl += 3;
  }
  if ((rc = check_launch("emit_sorted_kernel", stream, f.dbg))) return rc;
  {
    StageTimer tm(kStSort, stream);
    const int which = radix_sort_pairs(tk_a, tv_a, tk_b, tv_b, 0u, ws.counters, cap, (size_t)cap, tile_bits, rs, ws.ranges, stream, &nl,
                                       /*histogram_ready=*/true);
    point_list = which ? tv_b : tv_a;
  }
  count_launch(nl);
  if ((rc = check_launch("tile sort", stream, f.dbg))) return rc;
  if (a->num_rendered) {
    write_counts_kernel<<<1, 1, 0, stream>>>(nullptr, P, ws.counters, a->num_rendered);
    count_launch();
  }
  return render_frame_impl(f, point_list, stream);
}

static int render_frame_impl(const Frame& f, const uint32_t* point_list, cudaStream_t stream) {
  const GsbRasterArgs* a = f.a;
  const Workspace& ws = f.ws;
  const int W = a->width, H = a->height;
  const int64_t cap = f.cap;
  const uint32_t gx = f.gx, gy = f.gy;
  {
    StageTimer tm(kStRender, stream);
#define GSB_LAUNCH_RENDER(KERNEL)                                                                                         \
  KERNEL<<<dim3(gx, gy), kTilePixels / 2, 0, stream>>>(ws.ranges, point_list, W, H, ws.recA, ws.recB, ws.recC, a->background, \
                                                       a->out_color, a->out_depth, a->out_final_T, cap)
    if (!(a->flags & GSB_RASTER_FAST_EXP)) {
      GSB_LAUNCH_RENDER(render_compact_kernel);
    } else {
      GSB_LAUNCH_RENDER(render_table_kernel);
    }
#undef GSB_LAUNCH_RENDER
  }
  count_launch();
  return check_launch("render_kernel", stream, f.dbg);
}

// synchronous contract: report an undersized workspace now (one wait at the END of the frame;
// GSB_RASTER_ASYNC callers read num_rendered[2] themselves after their own synchronisation)
static int finish_sync(const Frame& f, cudaStream_t stream) {
  if (f.use_cub || (f.a->flags & GSB_RASTER_ASYNC)) return GSB_OK;
  unsigned long long host_counters[4] = {0, 0, 0, 0};
  GSB_CUDA_OK(cudaMemcpyAsync(host_counters, f.ws.counters, sizeof(host_counters), cudaMemcpyDeviceToHost, stream));
  GSB_CUDA_OK(cudaStreamSynchronize(stream));
  if (host_counters[2])
    return fail(GSB_ERR_WORKSPACE, "frame needs %lld instances, workspace sized for %lld", (long long)host_counters[1],
                (long long)f.cap);
  return GSB_OK;
}

// the reference's own pipeline shape (P-sized scan, emit in Gaussian order, global radix sort of (tile | depth) keys,
// boundary detection), incl. its host round trip -- validation only
static int cub_path(const Frame& f, cudaStream_t stream) {
  const GsbRasterArgs* a = f.a;
  const Workspace& ws = f.ws;
  const int P = a->P;
  const int64_t cap = f.cap;
  int rc;
  {
    StageTimer tm(kStScan, stream);
    size_t temp_bytes = ws.scan_temp_bytes;
    GSB_CUDA_OK(cub::DeviceScan::InclusiveSum(ws.scan_temp, temp_bytes, ws.tiles, ws.offsets, P, stream));
  }
  if (a->num_rendered) {
    write_counts_kernel<<<1, 1, 0, stream>>>(ws.offsets, P, ws.counters, a->num_rendered);
    count_launch();
  }
  uint32_t R32 = 0;
  GSB_CUDA_OK(cudaMemcpyAsync(&R32, ws.offsets + (P - 1), sizeof(uint32_t), cudaMemcpyDeviceToHost, stream));
  GSB_CUDA_OK(cudaStreamSynchronize(stream));
  const int64_t R = (int64_t)R32;
  if (R > cap)
    return fail(GSB_ERR_WORKSPACE, "frame needs %lld instances, workspace sized for %lld", (long long)R, (long long)cap);
  if (R > 0) {
    {
      StageTimer tm(kStEmit, stream);
      emit_instances_kernel<<<(P + 255) / 256, 256, 0, stream>>>(P, ws.recA, ws.recB, ws.tiles, ws.offsets, f.radii, f.gx, f.gy, a->flags,
                                                                 cap, ws.keys_in, ws.vals_in);
    }
    count_launch();
    if ((rc = check_launch("emit_instances_kernel", stream, f.dbg))) return rc;
    const int bit = (int)higher_msb(f.gx * f.gy);
    {
      StageTimer tm(kStSort, stream);
      size_t temp_bytes = ws.sort_temp_bytes;
      GSB_CUDA_OK(cub::DeviceRadixSort::SortPairs(ws.sort_temp, temp_bytes, ws.keys_in, ws.keys_out, ws.vals_in, ws.vals_out, R, 0,
                                                  32 + bit, stream));
    }
    if ((rc = check_launch("radix sort", stream, f.dbg))) return rc;
  }
  GSB_CUDA_OK(cudaMemsetAsync(ws.ranges, 0, f.ntiles * sizeof(uint2), stream));
  if (R > 0) {
    {
      StageTimer tm(kStRanges, stream);
      tile_ranges_kernel<<<(unsigned)((R + 255) / 256), 256, 0, stream>>>(R, ws.keys_out, ws.ranges);
    }
    count_launch();
    if ((rc = check_launch("tile_ranges_kernel", stream, f.dbg))) return rc;
  }
  return render_frame_impl(f, ws.vals_out, stream);
}

int gsb_raster_forward(const GsbRasterArgs* a, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  Frame f{};
  int rc;
  if ((rc = validate_frame(a, f))) return rc;
  if (a->P == 0) return empty_frame(a, stream);
  PreParams pp{};
  fill_common(f, pp);
  fill_eye(f, pp.eye[0]);
  pp.eye[1] = pp.eye[0];
  pp.binned = f.use_cub ? 0 : 1;
  if ((rc = preprocess<1, 6>(pp, stream, f.dbg))) return rc;
  if (f.use_cub) return cub_path(f, stream);
  // ---- default pipeline: depth-sort P, emit in that order, stable split by tile; nothing waits
  const uint32_t* ids_sorted = nullptr;
  if ((rc = depth_sort(f, nullptr, stream, &ids_sorted))) return rc;
  if ((rc = bin_and_render(f, ids_sorted, stream))) return rc;
  return finish_sync(f, stream);
}

int gsb_raster_forward_pair(const GsbRasterArgs* left, const GsbRasterArgs* right, void* stream_left_v, void* stream_right_v) {
  cudaStream_t sl = static_cast<cudaStream_t>(stream_left_v);
  cudaStream_t sr = stream_right_v ? static_cast<cudaStream_t>(stream_right_v) : sl;
  Frame fl{}, fr{};
  int rc;
  if ((rc = validate_frame(left, fl))) return rc;
  if ((rc = validate_frame(right, fr))) return rc;
  if (left->P != right->P || left->means3D != right->means3D || left->shs != right->shs ||
      left->colors_precomp != right->colors_precomp || left->opacities != right->opacities || left->scales != right->scales ||
      left->rotations != right->rotations || left->cov3D_precomp != right->cov3D_precomp ||
      left->scale_modifier != right->scale_modifier || left->sh_degree != right->sh_degree || left->sh_coeffs != right->sh_coeffs ||
      left->width != right->width || left->height != right->height)
    return fail(GSB_ERR_INVALID, "forward_pair: both eyes must share the Gaussian tensors, SH settings and the image size");
  if (fl.use_cub || fr.use_cub) return fail(GSB_ERR_INVALID, "forward_pair: GSB_RASTER_CUB_SORT is a single-view validation path");
  if (left->workspace == right->workspace) return fail(GSB_ERR_INVALID, "forward_pair: each eye needs its own workspace");
  if (left->P == 0) {
    if ((rc = empty_frame(left, sl))) return rc;
    return empty_frame(right, sr);
  }
  PreParams pp{};
  fill_common(fl, pp);
  pp.flags = left->flags;
  fill_eye(fl, pp.eye[0]);
  fill_eye(fr, pp.eye[1]);
  pp.binned = 1;
  const bool shared = (left->flags & GSB_RASTER_PAIR_SHARED_DEPTH) != 0;
  pp.shared_depth = shared ? 1 : 0;
  // 5 CTAs per SM: measured on C1 at 0.194 ms (96 registers, 48 B of spills) vs 0.209 ms at 4 (114 registers, no spills)
  if ((rc = preprocess<2, 5>(pp, sl, fl.dbg))) return rc;
  const uint32_t* ids_l = nullptr;
  const uint32_t* ids_r = nullptr;
  if (shared) {  // one depth order for both eyes
    if ((rc = depth_sort(fl, &fr, sl, &ids_l))) return rc;
    ids_r = ids_l;
  }
  if (sr != sl) {  // the right eye continues on its own stream once the shared part (preprocess [+ depth sort]) is enqueued
    cudaEvent_t ev = pair_event();
    GSB_CUDA_OK(cudaEventRecord(ev, sl));
    GSB_CUDA_OK(cudaStreamWaitEvent(sr, ev, 0));
  }
  if (!shared) {
    if ((rc = depth_sort(fl, nullptr, sl, &ids_l))) return rc;
    if ((rc = depth_sort(fr, nullptr, sr, &ids_r))) return rc;
  }
  if ((rc = bin_and_render(fl, ids_l, sl))) return rc;
  if ((rc = bin_and_render(fr, ids_r, sr))) return rc;
  if ((rc = finish_sync(fl, sl))) return rc;
  return finish_sync(fr, sr);
}

int gsb_raster_mark_visible(int32_t P, const float* means3D, const float* viewmatrix, const float* projmatrix,
                            uint8_t* present, void* stream_v) {
  (void)projmatrix;  // the reference computes p_proj but only tests z_view (auxiliary.h:154)
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (P < 0 || (P > 0 && (!means3D || !viewmatrix || !present))) return fail(GSB_ERR_INVALID, "mark_visible: bad arguments");
  if (P == 0) return GSB_OK;
  mark_visible_kernel<<<(P + 255) / 256, 256, 0, stream>>>(P, means3D, viewmatrix, present);
  count_launch();
  return check_launch("mark_visible_kernel", stream, false);
}

int gsb_image_to_u8(const float* chw, int32_t width, int32_t height, uint8_t* hwc, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (!chw || !hwc || width <= 0 || height <= 0) return fail(GSB_ERR_INVALID, "image_to_u8: bad arguments");
  const size_t n = (size_t)width * height;
  {
    StageTimer tm(kStToU8, stream);
    to_u8_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(chw, width, height, hwc);
  }
  count_launch();
  return check_launch("to_u8_kernel", stream, false);
}

}  // extern "C"
