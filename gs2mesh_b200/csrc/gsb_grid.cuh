// GsbPointGrid (include/gs2mesh_b200.h) as gsb_eval.cu's searches, gsb_mobilebrick.cu's Poisson-disk neighbours and
// gsb_normals.cu's k nearest neighbours read it.  Every fp64 operation carries an explicit rounding intrinsic, so nvcc cannot contract a multiply-add into an FMA.
#pragma once

#include "gs2mesh_b200.h"

namespace gsb {

constexpr int kMaxAxisCells = 1 << 21;  // the ring walk's margin (kRingMargin, below) covers axes up to this size

// cell > 0, 1..kMaxAxisCells cells per axis, fewer than 2^31 cells, and the point, id and cell-start arrays present
inline bool grid_ok(const GsbPointGrid* g) {
  if (!g || g->n_points < 0 || (g->n_points && (!g->points || !g->ids)) || !g->cell_start || !(g->cell > 0.0)) return false;
  double cells = 1.0;
  for (int a = 0; a < 3; ++a) {
    if (g->dims[a] <= 0 || g->dims[a] > kMaxAxisCells) return false;
    cells *= g->dims[a];
  }
  return cells < 2147483647.0;
}

// the cell of coordinate p on an axis with origin o, cell h and dim cells, clamped into the grid
__device__ __forceinline__ int cell_axis(double p, double o, double h, int dim) {
  const double c = floor((p - o) / h);
  return c < 0.0 ? 0 : (c >= (double)dim ? dim - 1 : (int)c);
}

// ((x*x) + y*y) + z*z
__device__ __forceinline__ double sq_norm3(double x, double y, double z) {
  return __dadd_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)), __dmul_rn(z, z));
}

// ((dx*dx) + dy*dy) + dz*dz with d = (x, y, z) - p.  Swapping the two points negates d exactly, so the result is the same.
__device__ __forceinline__ double sq_dist(double x, double y, double z, const double* p) {
  return sq_norm3(__dsub_rn(x, p[0]), __dsub_rn(y, p[1]), __dsub_rn(z, p[2]));
}

// Calls visit(q) for every point id q in the 27 cells around (x, y, z)'s cell that lie in the grid, x-major, until visit
// returns false (and then returns false).  With a cell >= r, these cells hold every point within r of (x, y, z).
template <typename Visit>
__device__ __forceinline__ bool visit_27_cells(const GsbPointGrid& g, double x, double y, double z, Visit&& visit) {
  const int cx = cell_axis(x, g.origin[0], g.cell, g.dims[0]), cy = cell_axis(y, g.origin[1], g.cell, g.dims[1]),
            cz = cell_axis(z, g.origin[2], g.cell, g.dims[2]);
  const int64_t* __restrict__ start = g.cell_start;
  const int64_t* __restrict__ ids = g.ids;
  for (int nb = 0; nb < 27; ++nb) {
    const int cx1 = cx + nb / 9 - 1, cy1 = cy + (nb / 3) % 3 - 1, cz1 = cz + nb % 3 - 1;
    if (cx1 < 0 || cx1 >= g.dims[0] || cy1 < 0 || cy1 >= g.dims[1] || cz1 < 0 || cz1 >= g.dims[2]) continue;
    const long long c = ((long long)cx1 * g.dims[1] + cy1) * g.dims[2] + cz1;
    for (long long s = start[c], e = start[c + 1]; s < e; ++s)
      if (!visit((long long)ids[s])) return false;
  }
  return true;
}

// Rings of cells at Chebyshev distance k around a query's cell, for the exact nearest-neighbour searches
// (gsb_eval.cu's ring_nearest, gsb_normals.cu's ring_knn).  Every point in a ring > k lies at least k*h away.
//
// The query's cell is clamped, in double, to [-kFarCells, dims-1 + kFarCells] per axis: a query farther out gets a cell
// nearer the grid, which only shrinks the ring bounds (k-1)*h, so they stay lower bounds; k and qc +- k stay far from
// int64 overflow, and the rings walked stay within kFarCells + dims.
//
// The ring bound's relative margin kRingMargin must exceed the rounding error of the cell indices.  A query's or a
// point's index (p - o) / h rounds twice, so it is off by at most 2^-52 * |index| cells.  A point in ring k of a query
// has |index| < dims and the query |index| <= k + dims, so the two are off by at most 2^-52 * (k + 2*dims) cells, which
// stays below kRingMargin * (k - 1) for every k >= 2 while dims <= kMaxAxisCells (9.3e-10 at k = 2; grid_ok refuses
// larger axes).  The distance expression's own rounding (a few ulp) is far below the margin.  PointGrid's cell floor of
// (hi - lo) / 1e6 keeps every axis at about 1e6 cells: a change to that floor must keep it within the limit.
constexpr double kFarCells = 1099511627776.0;  // 2^40
constexpr double kRingMargin = 1e-9;

__device__ __forceinline__ long long query_cell(double p, double o, double h, int dim) {
  return (long long)fmin(fmax(floor((p - o) / h), -kFarCells), (double)(dim - 1) + kFarCells);
}

// Walks the rings around finite (qx, qy, qz) outward, from the first ring that reaches the grid to the last that meets
// it, calling visit(id) for every point id of each ring's cells.  Before ring k it stops when the ring's lower bound lb
// (every point of ring k and beyond is at least lb away) reaches max_dist, or when done(lb) returns true.
template <typename Done, typename Visit>
__device__ __forceinline__ void walk_rings(const GsbPointGrid& g, double qx, double qy, double qz, double max_dist,
                                           Done&& done, Visit&& visit) {
  const long long qc[3] = {query_cell(qx, g.origin[0], g.cell, g.dims[0]), query_cell(qy, g.origin[1], g.cell, g.dims[1]),
                           query_cell(qz, g.origin[2], g.cell, g.dims[2])};
  // first ring that can reach the grid, last ring that still meets it
  long long k0 = 0, k1 = 0;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const long long below = -qc[a], above = qc[a] - (g.dims[a] - 1);
    k0 = max(k0, max(below, above));
    k1 = max(k1, max(qc[a], (long long)(g.dims[a] - 1) - qc[a]));
  }
  const double margin = 1.0 - kRingMargin;
  for (long long k = k0; k <= k1; ++k) {
    const double lb = (double)(k > 0 ? k - 1 : 0) * g.cell * margin;  // every point of ring k is at least this far away
    if (lb >= max_dist) break;
    if (done(lb)) break;
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
          for (long long s = g.cell_start[c], e = g.cell_start[c + 1]; s < e; ++s) visit((long long)g.ids[s]);
        }
      }
    }
  }
}

}  // namespace gsb
