// Mesh-quality evaluation: the DTU evaluator's surface sampling (evaluation/DTU/eval_code/eval.py:48-71) and exact
// nearest-neighbour distances (eval.py:119-120,132-133; MobileBrick evaluate.py:47-54) without Open3D or sklearn.
//
// Every floating-point operation is fp64 with an explicit rounding intrinsic, so nvcc cannot contract a multiply and an
// add into an FMA: the reference computes in numpy / sklearn float64 without FMA and the results compare bit for bit.
#include <cub/cub.cuh>

#include "gs2mesh_b200.h"
#include "gsb_common.h"

namespace gsb {
namespace {

// ---------------------------------------------------------------------------------------------------------------------
// Surface sampling.  Per triangle (a, b, c), in numpy's operation order (eval.py:54-65):
//   v1 = b - a, v2 = c - a, l = sqrt((x*x + y*y) + z*z), area2 = |cross(v1, v2)|, thr = thresh * sqrt(l1*l2/area2),
//   n1 = floor(l1/thr), n2 = floor(l2/thr); grid point (i, j), i in 0..n1, j in 0..n2 (i-major, np.mgrid) is kept when
//   (i+0.5)/max(n1,1e-7) + (j+0.5)/max(n2,1e-7) < 1 (eval.py:12-17) and emitted as (v1*k0 + v2*k1) + a (eval.py:18).
// One warp per triangle, one lane per row i: a sliver or a large triangle spreads over the lanes instead of serialising
// one thread.
// ---------------------------------------------------------------------------------------------------------------------
struct Tri {
  double a[3], v1[3], v2[3];
  double n1, n2;  // 0 when the triangle has zero area (eval.py:59-62 drops it)
};

__device__ __forceinline__ double norm3(const double* v) {
  return __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(v[0], v[0]), __dmul_rn(v[1], v[1])), __dmul_rn(v[2], v[2])));
}

__device__ Tri load_tri(const double* __restrict__ xyz, const long long* __restrict__ tris, long long t, double thresh) {
  Tri r;
  const long long i0 = tris[3 * t], i1 = tris[3 * t + 1], i2 = tris[3 * t + 2];
  double b[3], c[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    r.a[k] = xyz[3 * i0 + k];
    b[k] = xyz[3 * i1 + k];
    c[k] = xyz[3 * i2 + k];
    r.v1[k] = __dsub_rn(b[k], r.a[k]);
    r.v2[k] = __dsub_rn(c[k], r.a[k]);
  }
  const double l1 = norm3(r.v1), l2 = norm3(r.v2);
  // np.cross: cp0 = a1*b2 - a2*b1, cp1 = a2*b0 - a0*b2, cp2 = a0*b1 - a1*b0
  double cr[3];
  cr[0] = __dsub_rn(__dmul_rn(r.v1[1], r.v2[2]), __dmul_rn(r.v1[2], r.v2[1]));
  cr[1] = __dsub_rn(__dmul_rn(r.v1[2], r.v2[0]), __dmul_rn(r.v1[0], r.v2[2]));
  cr[2] = __dsub_rn(__dmul_rn(r.v1[0], r.v2[1]), __dmul_rn(r.v1[1], r.v2[0]));
  const double area2 = norm3(cr);
  if (!(area2 > 0.0)) {
    r.n1 = r.n2 = -1.0;
    return r;
  }
  const double thr = __dmul_rn(thresh, __dsqrt_rn(__ddiv_rn(__dmul_rn(l1, l2), area2)));
  r.n1 = floor(__ddiv_rn(l1, thr));
  r.n2 = floor(__ddiv_rn(l2, thr));
  return r;
}

__device__ __forceinline__ double grid_coord(long long i, double n) { return __ddiv_rn(__dadd_rn((double)i, 0.5), fmax(n, 1e-7)); }

// number of j in [0, n2] with k0 + k1(j) < 1; the predicate is monotone in j, so an estimate is fixed up at its boundary
__device__ long long row_count(double k0, double n2) {
  const long long jmax = (long long)n2;
  const double est = (1.0 - k0) * fmax(n2, 1e-7) - 0.5;  // approximately the last j that passes
  long long j = est < -1.0 ? -1 : (est > (double)jmax ? jmax : (long long)floor(est));
  while (j + 1 <= jmax && __dadd_rn(k0, grid_coord(j + 1, n2)) < 1.0) ++j;
  while (j >= 0 && !(__dadd_rn(k0, grid_coord(j, n2)) < 1.0)) --j;
  return j + 1;
}

__global__ void __launch_bounds__(256) sample_count_kernel(const double* __restrict__ xyz, const long long* __restrict__ tris,
                                                           long long nt, double thresh, long long* __restrict__ counts) {
  const long long t = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (t >= nt) return;
  const Tri tr = load_tri(xyz, tris, t, thresh);
  long long total = 0;
  if (tr.n1 >= 0.0)
    for (long long i = lane; i <= (long long)tr.n1; i += 32) total += row_count(grid_coord(i, tr.n1), tr.n2);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) total += __shfl_xor_sync(0xffffffffu, total, o);
  if (lane == 0) counts[t] = total;
}

__global__ void __launch_bounds__(256) sample_emit_kernel(const double* __restrict__ xyz, const long long* __restrict__ tris,
                                                          long long nt, double thresh, const long long* __restrict__ offsets,
                                                          double* __restrict__ out) {
  const long long t = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (t >= nt) return;
  const Tri tr = load_tri(xyz, tris, t, thresh);
  if (tr.n1 < 0.0) return;
  long long base = offsets[t];
  const long long rows = (long long)tr.n1 + 1;
  for (long long r0 = 0; r0 < rows; r0 += 32) {  // 32 rows at a time; a warp scan orders their outputs
    const long long i = r0 + lane;
    const double k0 = grid_coord(i, tr.n1);
    const long long m = i < rows ? row_count(k0, tr.n2) : 0;
    long long incl = m;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const long long v = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += v;
    }
    double* dst = out + 3 * (base + incl - m);
    for (long long j = 0; j < m; ++j) {
      const double k1 = grid_coord(j, tr.n2);
#pragma unroll
      for (int k = 0; k < 3; ++k) dst[3 * j + k] = __dadd_rn(__dadd_rn(__dmul_rn(tr.v1[k], k0), __dmul_rn(tr.v2[k], k1)), tr.a[k]);
    }
    base += __shfl_sync(0xffffffffu, incl, 31);
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// Uniform grid of reference points (counting sort of point ids by cell) and the exact 1-NN ring search over it.
// ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ int cell_axis(double p, double o, double h, int dim) {
  const double c = floor((p - o) / h);
  return c < 0.0 ? 0 : (c >= (double)dim ? dim - 1 : (int)c);
}

__global__ void __launch_bounds__(256) grid_count_kernel(const GsbPointGrid g, int* __restrict__ cell_of,
                                                         unsigned long long* __restrict__ counts) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= g.n_points) return;
  const double* p = g.points + 3 * i;
  const int cx = cell_axis(p[0], g.origin[0], g.cell, g.dims[0]), cy = cell_axis(p[1], g.origin[1], g.cell, g.dims[1]),
            cz = cell_axis(p[2], g.origin[2], g.cell, g.dims[2]);
  const int c = (cx * g.dims[1] + cy) * g.dims[2] + cz;
  cell_of[i] = c;
  atomicAdd(&counts[c + 1], 1ull);
}

__global__ void __launch_bounds__(256) grid_scatter_kernel(const GsbPointGrid g, const int* __restrict__ cell_of,
                                                           unsigned int* __restrict__ fill) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= g.n_points) return;
  const int c = cell_of[i];
  g.ids[g.cell_start[c] + atomicAdd(&fill[c], 1u)] = i;
}

// Rings of cells at Chebyshev distance k around the query's (unclamped) cell.  Every point in a ring > k lies at least
// k*h away, so the search stops once the best distance is below that bound (with a relative margin far above the
// rounding error of the distance expression), or once k*h reaches max_dist.
__global__ void __launch_bounds__(128) nearest_kernel(const GsbPointGrid g, const double* __restrict__ q, long long nq,
                                                      double max_dist, double* __restrict__ out_dist,
                                                      long long* __restrict__ out_idx) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nq) return;
  const double qx = q[3 * t], qy = q[3 * t + 1], qz = q[3 * t + 2];
  const long long qc[3] = {(long long)floor((qx - g.origin[0]) / g.cell), (long long)floor((qy - g.origin[1]) / g.cell),
                           (long long)floor((qz - g.origin[2]) / g.cell)};
  // first ring that can reach the grid, last ring that still meets it
  long long k0 = 0, k1 = 0;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const long long below = -qc[a], above = qc[a] - (g.dims[a] - 1);
    k0 = max(k0, max(below, above));
    k1 = max(k1, max(qc[a], (long long)(g.dims[a] - 1) - qc[a]));
  }
  double best2 = INFINITY;
  long long best = -1;
  const double margin = 1.0 - 1e-9;
  for (long long k = k0; k <= k1; ++k) {
    const double lb = (double)(k > 0 ? k - 1 : 0) * g.cell * margin;  // every point of ring k is at least this far away
    if (lb >= max_dist) break;
    if (best >= 0 && best2 < lb * lb) break;
    const long long xl = max(qc[0] - k, 0ll), xh = min(qc[0] + k, (long long)g.dims[0] - 1);
    const long long yl = max(qc[1] - k, 0ll), yh = min(qc[1] + k, (long long)g.dims[1] - 1);
    for (long long x = xl; x <= xh; ++x) {
      const bool xedge = (x == qc[0] - k) || (x == qc[0] + k);
      for (long long y = yl; y <= yh; ++y) {
        const bool yedge = xedge || (y == qc[1] - k) || (y == qc[1] + k);
        // edge rows of the ring are whole z runs (clamped to the grid); inner rows only touch its two z faces
        const long long zl = yedge ? max(qc[2] - k, 0ll) : qc[2] - k;
        const long long zh = yedge ? min(qc[2] + k, (long long)g.dims[2] - 1) : qc[2] + k;
        for (long long zz = zl; zz <= zh; zz += (yedge ? 1 : 2 * k)) {
          if (zz < 0 || zz >= g.dims[2]) continue;
          const long long c = (x * g.dims[1] + y) * g.dims[2] + zz;
          for (long long s = g.cell_start[c], e = g.cell_start[c + 1]; s < e; ++s) {
            const long long id = g.ids[s];
            const double* p = g.points + 3 * id;
            const double dx = __dsub_rn(qx, p[0]), dy = __dsub_rn(qy, p[1]), dz = __dsub_rn(qz, p[2]);
            const double d2 = __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
            if (d2 < best2 || (d2 == best2 && id < best)) {
              best2 = d2;
              best = id;
            }
          }
        }
      }
    }
  }
  const double d = best >= 0 ? __dsqrt_rn(best2) : INFINITY;
  const bool hit = d < max_dist;
  out_dist[t] = hit ? d : INFINITY;
  out_idx[t] = hit ? best : -1;
}

// ---------------------------------------------------------------------------------------------------------------------
// Greedy radius downsampling (eval.py:88-93): point p is kept iff no earlier kept point q (q < p) has
// ((dx*dx)+dy*dy)+dz*dz <= r*r (sklearn's radius_neighbors test on reduced distances, inclusive).  Parallel form of the
// sequential loop (Blelloch, Fineman, Shun, SPAA 2012): in each round an undecided point with a kept earlier neighbour is
// dropped, one whose earlier neighbours are all dropped is kept.  Decided states never change, so a round may read states
// written in the same round.  The earliest undecided point is decided in every round.
// state: 0 undecided, 1 kept, 2 dropped.  The grid's cell is >= r, so the neighbours lie in the 27 surrounding cells.
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) downsample_round_kernel(const GsbPointGrid g, double r2, unsigned char* state,
                                                               unsigned int* __restrict__ undecided) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= g.n_points || state[p] != 0) return;
  const double px = g.points[3 * p], py = g.points[3 * p + 1], pz = g.points[3 * p + 2];
  const int cx = cell_axis(px, g.origin[0], g.cell, g.dims[0]), cy = cell_axis(py, g.origin[1], g.cell, g.dims[1]),
            cz = cell_axis(pz, g.origin[2], g.cell, g.dims[2]);
  const double* __restrict__ pts = g.points;
  const int64_t* __restrict__ start = g.cell_start;
  const int64_t* __restrict__ ids = g.ids;
  bool pending = false;
  for (int nb = 0; nb < 27; ++nb) {
    const int x = cx + nb / 9 - 1, y = cy + (nb / 3) % 3 - 1, z = cz + nb % 3 - 1;
    if (x < 0 || x >= g.dims[0] || y < 0 || y >= g.dims[1] || z < 0 || z >= g.dims[2]) continue;
    const long long c = ((long long)x * g.dims[1] + y) * g.dims[2] + z;
    for (long long s = start[c], e = start[c + 1]; s < e; ++s) {
      const long long q = ids[s];
      if (q >= p) continue;
      const double dx = __dsub_rn(px, pts[3 * q]), dy = __dsub_rn(py, pts[3 * q + 1]), dz = __dsub_rn(pz, pts[3 * q + 2]);
      if (!(__dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz)) <= r2)) continue;
      const unsigned char sq = *((volatile unsigned char*)state + q);
      if (sq == 1) {
        state[p] = 2;
        return;
      }
      if (sq == 0) pending = true;
    }
  }
  if (!pending) {
    state[p] = 1;
    return;
  }
  atomicAdd(undecided, 1u);
}

__global__ void __launch_bounds__(256) downsample_finish_kernel(unsigned char* __restrict__ state, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) state[i] = state[i] == 1;
}

bool grid_ok(const GsbPointGrid* g) {
  if (!g || g->n_points < 0 || (g->n_points && !g->points) || !g->cell_start || !(g->cell > 0.0)) return false;
  double cells = 1.0;
  for (int a = 0; a < 3; ++a) {
    if (g->dims[a] <= 0) return false;
    cells *= g->dims[a];
  }
  return cells < 2147483647.0;
}

long long grid_cells(const GsbPointGrid* g) { return (long long)g->dims[0] * g->dims[1] * g->dims[2]; }

size_t scan_bytes(long long cells) {
  size_t b = 0;
  cub::DeviceScan::InclusiveSum(nullptr, b, (unsigned long long*)nullptr, (unsigned long long*)nullptr, (int)(cells + 1));
  return b;
}

}  // namespace
}  // namespace gsb

using namespace gsb;

extern "C" {

int gsb_eval_sample_count(const double* vertices, int64_t n_vertices, const int64_t* triangles, int64_t n_triangles, double thresh,
                          int64_t* tri_counts, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (n_vertices < 0 || n_triangles < 0 || !(thresh > 0.0) || (n_triangles && (!vertices || !triangles || !tri_counts)))
    return fail(GSB_ERR_INVALID, "eval_sample_count: bad arguments");
  if (n_triangles == 0) return GSB_OK;
  sample_count_kernel<<<(unsigned)((n_triangles * 32 + 255) / 256), 256, 0, stream>>>(
      vertices, reinterpret_cast<const long long*>(triangles), n_triangles, thresh, reinterpret_cast<long long*>(tri_counts));
  count_launch();
  return check_launch("sample_count_kernel", stream, false);
}

int gsb_eval_sample_emit(const double* vertices, int64_t n_vertices, const int64_t* triangles, int64_t n_triangles, double thresh,
                         const int64_t* tri_offsets, double* samples, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (n_vertices < 0 || n_triangles < 0 || !(thresh > 0.0) ||
      (n_triangles && (!vertices || !triangles || !tri_offsets || !samples)))
    return fail(GSB_ERR_INVALID, "eval_sample_emit: bad arguments");
  if (n_triangles == 0) return GSB_OK;
  sample_emit_kernel<<<(unsigned)((n_triangles * 32 + 255) / 256), 256, 0, stream>>>(
      vertices, reinterpret_cast<const long long*>(triangles), n_triangles, thresh,
      reinterpret_cast<const long long*>(tri_offsets), samples);
  count_launch();
  return check_launch("sample_emit_kernel", stream, false);
}

size_t gsb_eval_grid_workspace_bytes(int64_t n_points, int64_t n_cells) {
  if (n_points < 0 || n_cells <= 0 || n_cells >= 2147483647) return 0;
  Carver c(nullptr);
  c.take<int>((size_t)n_points);
  c.take<unsigned int>((size_t)n_cells);
  c.take<char>(scan_bytes(n_cells));
  return c.total();
}

int gsb_eval_grid_build(const GsbPointGrid* grid, void* workspace, size_t workspace_bytes, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (!grid_ok(grid) || (grid->n_points && !grid->ids) || !workspace) return fail(GSB_ERR_INVALID, "eval_grid_build: bad arguments");
  const long long cells = grid_cells(grid), n = grid->n_points;
  if (workspace_bytes < gsb_eval_grid_workspace_bytes(n, cells))
    return fail(GSB_ERR_WORKSPACE, "eval_grid_build: workspace %zu < %zu bytes", workspace_bytes,
                gsb_eval_grid_workspace_bytes(n, cells));
  Carver c(workspace);
  int* cell_of = c.take<int>((size_t)n);
  unsigned int* fill = c.take<unsigned int>((size_t)cells);
  size_t tmp_bytes = scan_bytes(cells);
  void* tmp = c.take<char>(tmp_bytes);
  auto* start = reinterpret_cast<unsigned long long*>(grid->cell_start);
  GSB_CUDA_OK(cudaMemsetAsync(start, 0, sizeof(long long) * (size_t)(cells + 1), stream));
  GSB_CUDA_OK(cudaMemsetAsync(fill, 0, sizeof(unsigned int) * (size_t)cells, stream));
  if (n == 0) return GSB_OK;
  const unsigned blocks = (unsigned)((n + 255) / 256);
  grid_count_kernel<<<blocks, 256, 0, stream>>>(*grid, cell_of, start);
  count_launch();
  GSB_CUDA_OK(cub::DeviceScan::InclusiveSum(tmp, tmp_bytes, start, start, (int)(cells + 1), stream));
  grid_scatter_kernel<<<blocks, 256, 0, stream>>>(*grid, cell_of, fill);
  count_launch();
  return check_launch("grid build", stream, false);
}

int gsb_eval_nearest(const GsbPointGrid* grid, const double* queries, int64_t n_queries, double max_dist, double* dist,
                     int64_t* index, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (!grid_ok(grid) || (grid->n_points && !grid->ids) || n_queries < 0 || (n_queries && (!queries || !dist || !index)) ||
      !(max_dist > 0.0))
    return fail(GSB_ERR_INVALID, "eval_nearest: bad arguments");
  if (n_queries == 0) return GSB_OK;
  nearest_kernel<<<(unsigned)((n_queries + 127) / 128), 128, 0, stream>>>(*grid, queries, n_queries, max_dist, dist,
                                                                          reinterpret_cast<long long*>(index));
  count_launch();
  return check_launch("nearest_kernel", stream, false);
}

int gsb_eval_radius_downsample(const GsbPointGrid* grid, double radius, uint8_t* keep, uint32_t* counters,
                               uint32_t* host_undecided, int32_t* rounds, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (!grid_ok(grid) || (grid->n_points && (!grid->ids || !keep || !counters || !host_undecided)) || !(radius >= 0.0) ||
      !(grid->cell >= radius * 1.0000001))
    return fail(GSB_ERR_INVALID, "eval_radius_downsample: bad arguments (the grid cell must exceed the radius)");
  const long long n = grid->n_points;
  if (rounds) *rounds = 0;
  if (n == 0) return GSB_OK;
  GSB_CUDA_OK(cudaMemsetAsync(keep, 0, (size_t)n, stream));
  const double r2 = radius * radius;  // sklearn: _dist_to_rdist(r)
  const unsigned blocks = (unsigned)((n + 127) / 128);
  constexpr int kBatch = 4;  // rounds between two reads of the undecided count
  for (int done = 0;;) {
    GSB_CUDA_OK(cudaMemsetAsync(counters, 0, sizeof(uint32_t) * kBatch, stream));
    for (int b = 0; b < kBatch; ++b) {
      downsample_round_kernel<<<blocks, 128, 0, stream>>>(*grid, r2, keep, counters + b);
      count_launch();
    }
    done += kBatch;
    GSB_CUDA_OK(cudaMemcpyAsync(host_undecided, counters + kBatch - 1, sizeof(uint32_t), cudaMemcpyDeviceToHost, stream));
    GSB_CUDA_OK(cudaStreamSynchronize(stream));
    if (*host_undecided == 0) {
      if (rounds) *rounds = done;
      break;
    }
    if (done > n + kBatch) return fail(GSB_ERR_CUDA, "eval_radius_downsample: no progress after %d rounds", done);
  }
  downsample_finish_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(keep, n);
  count_launch();
  return check_launch("radius downsample", stream, false);
}

}  // extern "C"
