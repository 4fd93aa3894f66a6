// Multi-GPU merge of view-sharded TSDF volumes (SURVEY.md 8(b) seam 2 / 8(e)): every rank fuses its own views into a private
// brick pool; at the end ONE sum-reduce of (sum tsdf*w, w [, sum rgb*w]) over the union of the ranks' bricks gives the
// volume Open3D would have built from all views (the reference has no multi-GPU path: tsdf_utils.py:58 is one sequential loop).
//
// Everything is enqueued on the caller's stream: two NCCL exchanges of brick lattice indices (all-gather of every rank's
// list, broadcast of the canonical order), the hash insertions / look-ups that map the canonical order to local pool slots,
// one fused pack+to-sums kernel, ONE ncclReduce / ncclAllReduce of the packed payload, one fused unpack+from-sums kernel.
// The canonical rank (the root, or rank 0 for an all-reduce) exchanges its pool prefix in place -- no pack / unpack there.
// The only host synchronisation is the read of the union's size, which NCCL needs as the element count.
//
// NCCL is not linked: its entry points are resolved at run time from the libnccl.so.2 the process already carries
// (torch's), so that the library and torch.distributed share one NCCL.
#include <dlfcn.h>
#include <nccl.h>

#include <cstring>

#include "gsb_common.h"

namespace gsb {
namespace {

struct NcclApi {
  bool ok = false;
  char why[256] = {0};
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Broadcast)(const void*, void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Reduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*GroupStart)() = nullptr;
  ncclResult_t (*GroupEnd)() = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
};

NcclApi& nccl() {
  static NcclApi api = [] {
    NcclApi a;
    void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);  // the copy torch.distributed uses, if the process has one
    if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    if (!h) {
      snprintf(a.why, sizeof(a.why), "libnccl.so.2 not found: %s", dlerror());
      return a;
    }
    bool all = true;
#define GSB_NCCL_SYM(field, name)                                   \
  a.field = reinterpret_cast<decltype(a.field)>(dlsym(h, name));    \
  if (!a.field) {                                                   \
    all = false;                                                    \
    snprintf(a.why, sizeof(a.why), "libnccl lacks %s", name);       \
  }
    GSB_NCCL_SYM(GetUniqueId, "ncclGetUniqueId")
    GSB_NCCL_SYM(CommInitRank, "ncclCommInitRank")
    GSB_NCCL_SYM(CommDestroy, "ncclCommDestroy")
    GSB_NCCL_SYM(AllGather, "ncclAllGather")
    GSB_NCCL_SYM(Broadcast, "ncclBroadcast")
    GSB_NCCL_SYM(Reduce, "ncclReduce")
    GSB_NCCL_SYM(AllReduce, "ncclAllReduce")
    GSB_NCCL_SYM(GroupStart, "ncclGroupStart")
    GSB_NCCL_SYM(GroupEnd, "ncclGroupEnd")
    GSB_NCCL_SYM(GetErrorString, "ncclGetErrorString")
#undef GSB_NCCL_SYM
    a.ok = all;
    return a;
  }();
  return api;
}

#define GSB_NCCL_OK(expr)                                                                                             \
  do {                                                                                                                \
    ncclResult_t r__ = (expr);                                                                                        \
    if (r__ != ncclSuccess)                                                                                           \
      return ::gsb::fail(GSB_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, nccl().GetErrorString(r__), __FILE__, __LINE__); \
  } while (0)

// every rank's brick list (gathered: [nranks][pool] int4, counts[nranks]) -> this rank's hash; missing bricks are opened.
// A brick that cannot be stored counts as dropped: always in the thread that left it without a slot, and in a thread that
// finds it once its slot is stored (a copy of the brick from another rank may find the key first).
__global__ void __launch_bounds__(256) insert_gathered_kernel(const HashView hv, uint32_t* __restrict__ counters,
                                                              const int4* __restrict__ gathered, const uint32_t* __restrict__ counts,
                                                              int nranks, int self) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)nranks * hv.pool) return;
  const int r = (int)(i / hv.pool);
  const uint32_t j = (uint32_t)(i % hv.pool);
  if (r == self || j >= min(counts[r], hv.pool)) return;
  const int4 b = gathered[i];
  if (!brick_key_ok(b.x, b.y, b.z)) return;
  const uint32_t h = brick_find_or_insert(hv, counters, b.x, b.y, b.z);
  if (h == kSlotNone || hv.vals[h] >= hv.pool) count_dropped(counters);
}

// canonical order (the canonical rank's brick_index[0 .. n)) -> this rank's pool slots (kSlotNone: this rank never saw it)
__global__ void __launch_bounds__(256) map_canonical_kernel(const unsigned long long* __restrict__ keys, const uint32_t* __restrict__ vals,
                                                            uint32_t mask, uint32_t pool, const int4* __restrict__ canon,
                                                            const uint32_t* __restrict__ n_dev, uint32_t* __restrict__ slot_of) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= min(*n_dev, pool)) return;
  const int4 b = canon[i];
  uint32_t slot = kSlotNone;
  if (brick_key_ok(b.x, b.y, b.z)) {
    const uint32_t h = brick_find(keys, mask, brick_key(b.x, b.y, b.z));
    if (h != kSlotNone) slot = vals[h];
  }
  slot_of[i] = slot < pool ? slot : kSlotNone;
}

// the payload in canonical order <-> the pool, through slot_of (the pool slot of every payload brick): to_sums gathers
// pool -> payload, where a brick this rank never saw travels as zeros; else scatters payload -> pool, where a brick
// without a slot (only if this rank's pool was exhausted while opening the union, counted as dropped) is not written.
// A pair of weight 0 moves as it is and the colour of a voxel of weight 0 as zeros (sums_pair).
template <bool to_sums>
__global__ void __launch_bounds__(256) move_sums_kernel(float4* __restrict__ tw, float4* __restrict__ color,
                                                        const uint32_t* __restrict__ slot_of, uint32_t n, float4* __restrict__ ptw,
                                                        float4* __restrict__ pcolor) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;  // voxel pair of the payload
  if (i >= (size_t)n * (GSB_BRICK_VOXELS / 2)) return;
  const uint32_t slot = slot_of[i / (GSB_BRICK_VOXELS / 2)];
  if (slot == kSlotNone && !to_sums) return;
  const size_t p = (size_t)slot * (GSB_BRICK_VOXELS / 2) + i % (GSB_BRICK_VOXELS / 2);  // voxel pair of the pool
  float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
  if (slot != kSlotNone) v = to_sums ? tw[p] : ptw[i];
  float4 c[2] = {make_float4(0.f, 0.f, 0.f, 0.f), make_float4(0.f, 0.f, 0.f, 0.f)};
  if (color)
#pragma unroll
    for (int k = 0; k < 2; ++k)
      if ((k ? v.w : v.y) != 0.f) c[k] = to_sums ? color[2 * p + k] : pcolor[2 * i + k];
  sums_pair(v, c, color != nullptr, to_sums);
  (to_sums ? ptw[i] : tw[p]) = v;
  if (color)
#pragma unroll
    for (int k = 0; k < 2; ++k) (to_sums ? pcolor[2 * i + k] : color[2 * p + k]) = c[k];
}

struct ReduceScratch {
  uint32_t* counts;      // [nranks] pool slots in use on every rank
  uint32_t* n_union;     // [1] (+pad) bricks of the canonical rank after opening the union
  int4* gathered;        // [nranks][pool]
  int4* canon;           // [pool] canonical order on non-canonical ranks
  uint32_t* slot_of;     // [pool]
  float4* ptw;           // [n][2048]
  float4* pcolor;        // [n][4096] or NULL
  size_t fixed_bytes, total;
};

ReduceScratch carve_reduce(void* base, uint32_t pool, int nranks, uint32_t n_union, bool with_color) {
  ReduceScratch r{};
  Carver c(base);
  r.counts = c.take<uint32_t>((size_t)nranks + 16);
  r.n_union = c.take<uint32_t>(16);
  r.gathered = c.take<int4>((size_t)nranks * pool);
  r.canon = c.take<int4>(pool);
  r.slot_of = c.take<uint32_t>(pool);
  r.fixed_bytes = c.total();
  r.ptw = c.take<float4>((size_t)n_union * (GSB_BRICK_VOXELS / 2));
  r.pcolor = with_color ? c.take<float4>((size_t)n_union * GSB_BRICK_VOXELS) : nullptr;
  r.total = c.total();
  return r;
}

}  // namespace
}  // namespace gsb

using namespace gsb;

extern "C" {

int gsb_comm_unique_id(void* id128) {
  if (!id128) return fail(GSB_ERR_INVALID, "comm_unique_id: NULL");
  if (!nccl().ok) return fail(GSB_ERR_CUDA, "NCCL unavailable: %s", nccl().why);
  static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId is 128 bytes");
  ncclUniqueId id;
  GSB_NCCL_OK(nccl().GetUniqueId(&id));
  memcpy(id128, &id, sizeof(id));
  return GSB_OK;
}

void* gsb_comm_create(const void* id128, int nranks, int rank) {
  if (!id128 || nranks <= 0 || rank < 0 || rank >= nranks) {
    fail(GSB_ERR_INVALID, "comm_create: bad arguments");
    return nullptr;
  }
  if (!nccl().ok) {
    fail(GSB_ERR_CUDA, "NCCL unavailable: %s", nccl().why);
    return nullptr;
  }
  ncclUniqueId id;
  memcpy(&id, id128, sizeof(id));
  ncclComm_t comm = nullptr;
  ncclResult_t r = nccl().CommInitRank(&comm, nranks, id, rank);
  if (r != ncclSuccess) {
    fail(GSB_ERR_CUDA, "ncclCommInitRank failed: %s", nccl().GetErrorString(r));
    return nullptr;
  }
  return comm;
}

void gsb_comm_destroy(void* nccl_comm) {
  if (nccl_comm && nccl().ok) nccl().CommDestroy(static_cast<ncclComm_t>(nccl_comm));
}

size_t gsb_tsdf_reduce_scratch_bytes(const GsbVolume* vol, int nranks, uint32_t union_bricks) {
  if (!vol || nranks <= 0) return 0;
  return carve_reduce(nullptr, vol->d.pool_bricks, nranks, union_bricks, vol->d.color != nullptr).total;
}

int gsb_tsdf_reduce(GsbVolume* vol, void* nccl_comm, int nranks, int rank, int root, void* scratch, size_t scratch_bytes,
                    size_t* required_bytes, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (!vol || !nccl_comm || nranks <= 0 || rank < 0 || rank >= nranks || root >= nranks || !scratch)
    return fail(GSB_ERR_INVALID, "tsdf_reduce: bad arguments");
  if (!nccl().ok) return fail(GSB_ERR_CUDA, "NCCL unavailable: %s", nccl().why);
  if (nranks == 1) return GSB_OK;
  ncclComm_t comm = static_cast<ncclComm_t>(nccl_comm);
  const GsbVolumeDesc& d = vol->d;
  const uint32_t pool = d.pool_bricks, mask = d.hash_slots - 1u;
  const bool with_color = d.color != nullptr;
  const int canon_rank = root >= 0 ? root : 0;
  const bool all = root < 0;
  const bool canonical = rank == canon_rank;
  ReduceScratch rs = carve_reduce(scratch, pool, nranks, 0, with_color);
  if (rs.fixed_bytes > scratch_bytes) {
    if (required_bytes) *required_bytes = carve_reduce(nullptr, pool, nranks, pool / 8 + 1, with_color).total;
    return fail(GSB_ERR_WORKSPACE, "tsdf_reduce: scratch has %zu bytes, at least %zu needed", scratch_bytes, rs.fixed_bytes);
  }
  unsigned long long* keys = reinterpret_cast<unsigned long long*>(d.hash_keys);
  int4* index = reinterpret_cast<int4*>(d.brick_index);
  float4* tw = reinterpret_cast<float4*>(d.tsdf_weight);
  float4* color = reinterpret_cast<float4*>(d.color);

  uint32_t n_union = 0;  // the one host read of the merge: NCCL needs the payload size as a count
  {
    StageTimer tm(kStMergeIndex, stream);
    // 1. every rank's brick list
    GSB_NCCL_OK(nccl().GroupStart());
    GSB_NCCL_OK(nccl().AllGather(d.counters + kCntPool, rs.counts, 1, ncclUint32, comm, stream));
    GSB_NCCL_OK(nccl().AllGather(index, rs.gathered, (size_t)pool * 4, ncclInt32, comm, stream));
    GSB_NCCL_OK(nccl().GroupEnd());
    // 2. the ranks that receive the result open the bricks they lack
    if (canonical || all) {
      insert_gathered_kernel<<<blocks_for((long long)nranks * pool), 256, 0, stream>>>(hash_view(d), d.counters, rs.gathered,
                                                                                     rs.counts, nranks, rank);
      count_launch();
    }
    // 3. the canonical rank's brick order (its pool order after step 2) is the order of the exchange
    GSB_NCCL_OK(nccl().GroupStart());
    GSB_NCCL_OK(nccl().Broadcast(d.counters + kCntPool, rs.n_union, 1, ncclUint32, canon_rank, comm, stream));
    GSB_NCCL_OK(nccl().Broadcast(index, canonical ? index : rs.canon, (size_t)pool * 4, ncclInt32, canon_rank, comm, stream));
    GSB_NCCL_OK(nccl().GroupEnd());
    GSB_CUDA_OK(cudaMemcpyAsync(&n_union, rs.n_union, sizeof(uint32_t), cudaMemcpyDeviceToHost, stream));
    GSB_CUDA_OK(cudaStreamSynchronize(stream));
  }
  if (n_union > pool) n_union = pool;
  if (n_union == 0) return GSB_OK;
  rs = carve_reduce(scratch, pool, nranks, canonical ? 0 : n_union, with_color);
  const size_t need = carve_reduce(nullptr, pool, nranks, n_union, with_color).total;  // same on every rank
  if (need > scratch_bytes) {
    if (required_bytes) *required_bytes = need;
    return fail(GSB_ERR_WORKSPACE, "tsdf_reduce: scratch has %zu bytes, %zu needed for %u bricks", scratch_bytes, need, n_union);
  }
  const size_t pairs = (size_t)n_union * (GSB_BRICK_VOXELS / 2);
  const unsigned pgrid = (unsigned)((pairs + 255) / 256);
  const float* send_tw;
  const float* send_color = nullptr;
  float* recv_tw;
  float* recv_color = nullptr;
  int rc;
  {
    StageTimer tm(kStMergePack, stream);
    if (canonical) {  // the pool prefix [0, n_union) IS the payload: convert and exchange it in place
      if ((rc = tsdf_sums(vol, true, n_union, stream))) return rc;
      send_tw = recv_tw = d.tsdf_weight;
      send_color = recv_color = d.color;
    } else {
      map_canonical_kernel<<<(n_union + 255) / 256, 256, 0, stream>>>(keys, d.hash_vals, mask, pool, rs.canon, rs.n_union, rs.slot_of);
      move_sums_kernel<true><<<pgrid, 256, 0, stream>>>(tw, color, rs.slot_of, n_union, rs.ptw, rs.pcolor);
      count_launch(2);
      send_tw = recv_tw = reinterpret_cast<float*>(rs.ptw);
      send_color = recv_color = reinterpret_cast<float*>(rs.pcolor);
    }
  }
  if ((rc = check_launch("tsdf_reduce pack", stream, false))) return rc;
  // 5. ONE reduce of the payload (two buffers in one NCCL group)
  {
    StageTimer tm(kStMergeReduce, stream);
    GSB_NCCL_OK(nccl().GroupStart());
    if (all) {
      GSB_NCCL_OK(nccl().AllReduce(send_tw, recv_tw, pairs * 4, ncclFloat32, ncclSum, comm, stream));
      if (with_color) GSB_NCCL_OK(nccl().AllReduce(send_color, recv_color, pairs * 8, ncclFloat32, ncclSum, comm, stream));
    } else {
      GSB_NCCL_OK(nccl().Reduce(send_tw, recv_tw, pairs * 4, ncclFloat32, ncclSum, root, comm, stream));
      if (with_color) GSB_NCCL_OK(nccl().Reduce(send_color, recv_color, pairs * 8, ncclFloat32, ncclSum, root, comm, stream));
    }
    GSB_NCCL_OK(nccl().GroupEnd());
  }
  // 6. back to (mean, weight) where the result lives
  {
    StageTimer tm(kStMergeUnpack, stream);
    if (canonical) {
      if ((rc = tsdf_sums(vol, false, n_union, stream))) return rc;
    } else if (all) {
      move_sums_kernel<false><<<pgrid, 256, 0, stream>>>(tw, color, rs.slot_of, n_union, rs.ptw, rs.pcolor);
      count_launch();
    }
  }
  return check_launch("tsdf_reduce unpack", stream, false);
}

}  // extern "C"
