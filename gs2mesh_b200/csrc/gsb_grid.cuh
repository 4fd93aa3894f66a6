// GsbPointGrid (include/gs2mesh_b200.h) as gsb_eval.cu's searches and gsb_mobilebrick.cu's Poisson-disk neighbours read
// it.  Every fp64 operation carries an explicit rounding intrinsic, so nvcc cannot contract a multiply-add into an FMA.
#pragma once

#include "gs2mesh_b200.h"

namespace gsb {

constexpr int kMaxAxisCells = 1 << 21;  // gsb_eval.cu's ring-search margin (kRingMargin) covers axes up to this size

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

}  // namespace gsb
