// MobileBrick evaluation (evaluation/MobileBrick/eval_code/evaluate.py:34-108) without Open3D: Open3D 0.17's
// TriangleMesh::GetSurfaceArea, SamplePointsUniformlyImpl and SamplePointsPoissonDisk (weighted sample elimination,
// Yuksel 2015), and the reference's grid_sample visibility lookup.  DESIGN.md section 7e gives the operation orders and
// the argument that the round-based elimination keeps exactly the points Open3D's sequential heap loop keeps.
//
// Like gsb_eval.cu, every fp64 operation carries an explicit rounding intrinsic, so nvcc cannot contract a multiply and
// an add into an FMA.
#include "gs2mesh_b200.h"
#include "gsb_common.h"
#include "gsb_grid.cuh"

namespace gsb {
namespace {

// GetSurfaceArea's per-triangle term: 0.5 * ((p0 - p1).cross(p0 - p2)).norm()
__global__ void __launch_bounds__(256) triangle_area_kernel(const double* __restrict__ v, const long long* __restrict__ tris,
                                                            long long nt, double* __restrict__ areas) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nt) return;
  const double* p0 = v + 3 * tris[3 * t];
  const double* p1 = v + 3 * tris[3 * t + 1];
  const double* p2 = v + 3 * tris[3 * t + 2];
  double a[3], b[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    a[k] = __dsub_rn(p0[k], p1[k]);
    b[k] = __dsub_rn(p0[k], p2[k]);
  }
  const double cx = __dsub_rn(__dmul_rn(a[1], b[2]), __dmul_rn(a[2], b[1]));
  const double cy = __dsub_rn(__dmul_rn(a[2], b[0]), __dmul_rn(a[0], b[2]));
  const double cz = __dsub_rn(__dmul_rn(a[0], b[1]), __dmul_rn(a[1], b[0]));
  areas[t] = __dmul_rn(0.5, __dsqrt_rn(sq_norm3(cx, cy, cz)));
}

// SamplePointsUniformlyImpl, one thread per sample j: its triangle is the t with bounds[t] <= j < bounds[t+1] (binary
// search over the nondecreasing bounds), r1 = variates[2j], r2 = variates[2j+1], a = 1 - sqrt(r1), b = sqrt(r1) * (1 - r2),
// c = sqrt(r1) * r2, point = (a*v0 + b*v1) + c*v2 per component.  Samples past bounds[nt] stay (0, 0, 0) as in Open3D.
__global__ void __launch_bounds__(256) sample_uniform_kernel(const double* __restrict__ v, const long long* __restrict__ tris,
                                                             long long nt, const long long* __restrict__ bounds,
                                                             const double* __restrict__ variates, long long ns,
                                                             double* __restrict__ out) {
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= ns) return;
  if (j >= bounds[nt]) {
    out[3 * j] = out[3 * j + 1] = out[3 * j + 2] = 0.0;
    return;
  }
  long long lo = 0, hi = nt;  // bounds[lo] <= j < bounds[hi]
  while (hi - lo > 1) {
    const long long mid = (lo + hi) >> 1;
    if (bounds[mid] <= j) lo = mid;
    else hi = mid;
  }
  const double r1 = variates[2 * j], r2 = variates[2 * j + 1];
  const double s = __dsqrt_rn(r1);
  const double a = __dsub_rn(1.0, s), b = __dmul_rn(s, __dsub_rn(1.0, r2)), c = __dmul_rn(s, r2);
  const double* p0 = v + 3 * tris[3 * lo];
  const double* p1 = v + 3 * tris[3 * lo + 1];
  const double* p2 = v + 3 * tris[3 * lo + 2];
#pragma unroll
  for (int k = 0; k < 3; ++k)
    out[3 * j + k] = __dadd_rn(__dadd_rn(__dmul_rn(a, p0[k]), __dmul_rn(b, p1[k])), __dmul_rn(c, p2[k]));
}

// ---------------------------------------------------------------------------------------------------------------------
// Poisson-disk elimination.  Neighbours of p: every q != p with ((dx*dx)+dy*dy)+dz*dz < r_max^2 (nanoflann's radius
// search, strict), dx = p.x - q.x.  The grid's cell is >= r_max, so they lie in the 27 cells around p's cell.
// ---------------------------------------------------------------------------------------------------------------------
template <bool kEmit>
__global__ void __launch_bounds__(128) neighbour_kernel(const GsbPointGrid g, double r2, long long* __restrict__ counts,
                                                        const long long* __restrict__ offsets, int* __restrict__ nbr,
                                                        double* __restrict__ d2_out) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= g.n_points) return;
  const double px = g.points[3 * p], py = g.points[3 * p + 1], pz = g.points[3 * p + 2];
  long long n = 0;
  const long long base = kEmit ? offsets[p] : 0;
  visit_27_cells(g, px, py, pz, [&](long long q) {
    if (q == p) return true;
    const double d2 = sq_dist(px, py, pz, g.points + 3 * q);
    if (!(d2 < r2)) return true;
    if (kEmit) {  // insertion into the (d2, q)-sorted list of this point's slice
      long long k = n;
      while (k > 0) {
        const double dk = d2_out[base + k - 1];
        const int qk = nbr[base + k - 1];
        if (dk < d2 || (dk == d2 && qk < q)) break;
        d2_out[base + k] = dk;
        nbr[base + k] = qk;
        --k;
      }
      d2_out[base + k] = d2;
      nbr[base + k] = (int)q;
    }
    ++n;
    return true;
  });
  if (!kEmit) counts[p] = n;
}

// term = (1 - max(sqrt(d2), r_min) / r_max)^8 with the power as three squarings (DESIGN.md section 7e, DOUBT 1)
__global__ void __launch_bounds__(256) weight_term_kernel(double* __restrict__ term, long long n, double r_min, double r_max) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double d = __dsqrt_rn(term[i]);
  if (d < r_min) d = r_min;
  const double t = __dsub_rn(1.0, __ddiv_rn(d, r_max));
  const double s = __dmul_rn(t, t), q = __dmul_rn(s, s);
  term[i] = __dmul_rn(q, q);
}

// weight[p] of every live point (round_of[p] == 0): the terms of its live neighbours summed from 0.0 in CSR order
__global__ void __launch_bounds__(128) weight_kernel(const long long* __restrict__ offsets, const int* __restrict__ nbr,
                                                     const double* __restrict__ term, long long n,
                                                     const int* __restrict__ round_of, double* __restrict__ weight) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n || round_of[p] != 0) return;
  double w = 0.0;
  for (long long k = offsets[p], e = offsets[p + 1]; k < e; ++k)
    if (round_of[nbr[k]] == 0) w = __dadd_rn(w, term[k]);
  weight[p] = w;
}

// Round r: a point live at the start of the round whose key (weight, index) exceeds the key of every neighbour live at
// the start of the round is deleted (round_of = r); its weight stays as its removal key.  A neighbour marked in this same
// round reads round_of == r and still counts as live.  live counts the points left.
__global__ void __launch_bounds__(128) round_kernel(const long long* __restrict__ offsets, const int* __restrict__ nbr,
                                                    long long n, int r, const double* __restrict__ weight, int* round_of,
                                                    unsigned int* __restrict__ live) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n || round_of[p] != 0) return;
  const double w = weight[p];
  for (long long k = offsets[p], e = offsets[p + 1]; k < e; ++k) {
    const int q = nbr[k];
    const int rq = *((volatile int*)round_of + q);
    if (rq != 0 && rq != r) continue;
    const double wq = weight[q];
    if (wq > w || (wq == w && q > p)) {
      atomicAdd(live, 1u);
      return;
    }
  }
  round_of[p] = r;
}

// grid_sample(volume, g, mode="nearest", padding_mode="zeros", align_corners=True) > 0 at the reference's coordinates
__global__ void __launch_bounds__(256) visibility_kernel(const double* __restrict__ v, long long n, double m0, double m1,
                                                         double m2, double vs, int r0, int r1, int r2,
                                                         const uint8_t* __restrict__ volume, uint8_t* __restrict__ keep) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double mins[3] = {m0, m1, m2};
  const int res[3] = {r0, r1, r2};
  int idx[3];
  bool inside = true;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const double u = __ddiv_rn(__dsub_rn(v[3 * i + a], mins[a]), vs);
    const double gd = __dsub_rn(__dmul_rn(__ddiv_rn(u, (double)(res[a] - 1)), 2.0), 1.0);
    const float g = __double2float_rn(gd);
    // grid_sampler_compute_source_index (align_corners), whose safe_downgrade_to_int_range sends a non-finite coordinate
    // outside the volume; then nearbyint and the cast to int (saturating: finite values beyond int fall outside too)
    const float x = __fmul_rn(__fdiv_rn(__fadd_rn(g, 1.0f), 2.0f), (float)(res[a] - 1));
    idx[a] = isfinite(x) ? __float2int_rn(x) : -1;
    inside = inside && idx[a] >= 0 && idx[a] < res[a];
  }
  keep[i] = inside && volume[((long long)idx[0] * r1 + idx[1]) * r2 + idx[2]] != 0;
}

}  // namespace
}  // namespace gsb

using namespace gsb;

extern "C" {

int gsb_eval_triangle_areas(const double* vertices, int64_t n_vertices, const int64_t* triangles, int64_t n_triangles,
                            double* areas, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (n_vertices < 0 || n_triangles < 0 || (n_triangles && (!vertices || !triangles || !areas)))
    return fail(GSB_ERR_INVALID, "eval_triangle_areas: bad arguments");
  if (n_triangles == 0) return GSB_OK;
  triangle_area_kernel<<<(unsigned)((n_triangles + 255) / 256), 256, 0, stream>>>(
      vertices, reinterpret_cast<const long long*>(triangles), n_triangles, areas);
  count_launch();
  return check_launch("triangle_area_kernel", stream, false);
}

int gsb_eval_sample_uniform(const double* vertices, int64_t n_vertices, const int64_t* triangles, int64_t n_triangles,
                            const int64_t* bounds, const double* variates, int64_t n_samples, double* samples,
                            void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (n_vertices < 0 || n_triangles <= 0 || n_samples < 0 ||
      (n_samples && (!vertices || !triangles || !bounds || !variates || !samples)))
    return fail(GSB_ERR_INVALID, "eval_sample_uniform: bad arguments (at least one triangle)");
  if (n_samples == 0) return GSB_OK;
  sample_uniform_kernel<<<(unsigned)((n_samples + 255) / 256), 256, 0, stream>>>(
      vertices, reinterpret_cast<const long long*>(triangles), n_triangles, reinterpret_cast<const long long*>(bounds),
      variates, n_samples, samples);
  count_launch();
  return check_launch("sample_uniform_kernel", stream, false);
}

int gsb_eval_poisson_neighbours(const GsbPointGrid* grid, double r_max, double r_min, int64_t* counts,
                                const int64_t* offsets, int32_t* neighbours, double* terms, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  const bool emit = offsets != nullptr;
  if (!grid_ok(grid) || grid->n_points >= 2147483647 ||  // the neighbour ids are int32
      !(r_max > 0.0) || !(r_max < INFINITY) || !(r_min >= 0.0) || !(r_min <= r_max) || !(grid->cell >= r_max * 1.0000001) ||
      (grid->n_points && (emit ? (!neighbours || !terms) : !counts)))
    return fail(GSB_ERR_INVALID,
                "eval_poisson_neighbours: bad arguments (0 <= r_min <= r_max finite, the grid cell must exceed r_max, "
                "fewer than 2^31 points)");
  const long long n = grid->n_points;
  if (n == 0) return GSB_OK;
  const unsigned blocks = (unsigned)((n + 127) / 128);
  const double r2 = r_max * r_max;  // KDTreeFlann::SearchRadius passes radius * radius to nanoflann
  if (!emit) {
    neighbour_kernel<false><<<blocks, 128, 0, stream>>>(*grid, r2, reinterpret_cast<long long*>(counts), nullptr, nullptr,
                                                        nullptr);
    count_launch();
    return check_launch("neighbour count", stream, false);
  }
  neighbour_kernel<true><<<blocks, 128, 0, stream>>>(*grid, r2, nullptr, reinterpret_cast<const long long*>(offsets),
                                                     neighbours, terms);
  count_launch();
  long long total = 0;
  GSB_CUDA_OK(cudaMemcpyAsync(&total, offsets + n, sizeof(long long), cudaMemcpyDeviceToHost, stream));
  GSB_CUDA_OK(cudaStreamSynchronize(stream));
  if (total) {
    weight_term_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(terms, total, r_min, r_max);
    count_launch();
  }
  return check_launch("neighbour emit", stream, false);
}

int gsb_eval_poisson_eliminate(const int64_t* offsets, const int32_t* neighbours, const double* terms, int64_t n_points,
                               double* weight, int32_t* round_of, uint32_t* counters, uint32_t* host_live, int32_t* rounds,
                               void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (n_points < 0 || n_points >= 2147483647 ||
      (n_points && (!offsets || !neighbours || !terms || !weight || !round_of || !counters || !host_live)))
    return fail(GSB_ERR_INVALID, "eval_poisson_eliminate: bad arguments");
  if (rounds) *rounds = 0;
  const long long n = n_points;
  if (n == 0) return GSB_OK;
  const auto* off = reinterpret_cast<const long long*>(offsets);
  const unsigned blocks = (unsigned)((n + 127) / 128);
  GSB_CUDA_OK(cudaMemsetAsync(round_of, 0, sizeof(int32_t) * (size_t)n, stream));
  weight_kernel<<<blocks, 128, 0, stream>>>(off, neighbours, terms, n, round_of, weight);
  count_launch();
  constexpr int kBatch = 4;  // rounds between two reads of the live count
  for (int done = 0;;) {
    GSB_CUDA_OK(cudaMemsetAsync(counters, 0, sizeof(uint32_t) * kBatch, stream));
    for (int b = 0; b < kBatch; ++b) {
      round_kernel<<<blocks, 128, 0, stream>>>(off, neighbours, n, done + b + 1, weight, round_of, counters + b);
      weight_kernel<<<blocks, 128, 0, stream>>>(off, neighbours, terms, n, round_of, weight);
      count_launch(2);
    }
    GSB_CUDA_OK(cudaMemcpyAsync(host_live, counters, sizeof(uint32_t) * kBatch, cudaMemcpyDeviceToHost, stream));
    GSB_CUDA_OK(cudaStreamSynchronize(stream));
    for (int b = 0; b < kBatch; ++b)
      if (host_live[b] == 0) {
        if (rounds) *rounds = done + b + 1;
        return check_launch("poisson eliminate", stream, false);
      }
    done += kBatch;
    // every round deletes the live point of largest key, so n rounds always suffice
    if (done > n + kBatch) return fail(GSB_ERR_CUDA, "eval_poisson_eliminate: no progress after %d rounds", done);
  }
}

int gsb_eval_visibility(const double* vertices, int64_t n_vertices, const double* min_pts, double voxel_size,
                        const int32_t* resolution, const uint8_t* volume, uint8_t* keep, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  // a non-finite or non-positive voxel size, or a non-finite min_pts, would map every vertex to voxel 0 or to none
  if (n_vertices < 0 || !min_pts || !resolution || resolution[0] < 2 || resolution[1] < 2 || resolution[2] < 2 ||
      (double)resolution[0] * resolution[1] * resolution[2] > 9e15 || !(voxel_size > 0.0) || !(voxel_size < INFINITY) ||
      !isfinite(min_pts[0]) || !isfinite(min_pts[1]) || !isfinite(min_pts[2]) ||
      (n_vertices && (!vertices || !volume || !keep)))
    return fail(GSB_ERR_INVALID,
                "eval_visibility: bad arguments (every resolution must be >= 2, voxel_size finite and > 0, min_pts "
                "finite)");
  if (n_vertices == 0) return GSB_OK;
  visibility_kernel<<<(unsigned)((n_vertices + 255) / 256), 256, 0, stream>>>(vertices, n_vertices, min_pts[0], min_pts[1],
                                                                              min_pts[2], voxel_size, resolution[0],
                                                                              resolution[1], resolution[2], volume, keep);
  count_launch();
  return check_launch("visibility_kernel", stream, false);
}

}  // extern "C"
