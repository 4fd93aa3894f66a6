// Vertex-clustering simplification: Open3D 0.17.0 TriangleMesh::SimplifyVertexClustering with average and quadric
// contraction (DESIGN.md section 7, "Simplification"; restated in tests/simplify_oracle.py).
//
// Each vertex gets the cell floor((v - m) / s) of a grid anchored half a cell below the vertices' minimum, packed into
// one 63-bit key over the cell box.  A stable radix sort of (key, vertex id) groups the cells with their vertices in
// ascending id; cells are numbered in the order of their smallest vertex id (an exclusive scan over the "first of its
// cell" flags, indexed by vertex id), Open3D's numbering.  One thread per cell sums its vertices sequentially in
// ascending id, and for the quadric contraction the plane quadrics of each vertex's distinct triangles in ascending
// triangle id, then solves -A^-1 b with Eigen's pivoted LDLT when |det A| > 1e-4.  Triangles are mapped through the
// cell numbering, dropped when two corners share a cell, rotated to start at their smallest id, stably sorted as triples
// (two LSD radix passes) and de-duplicated by keeping the head of each run, then compacted in input order.
//
// Every fp64 operation is an explicit __d*_rn in the restatement's order, so nvcc contracts nothing.  No floating-point
// atomics; integer atomics only count (incidences per vertex, quadric cells), so every run writes the same bytes.
#include <cub/cub.cuh>

#include <cmath>

#include "gs2mesh_b200.h"
#include "gsb_common.h"

namespace gsb {
namespace {

constexpr double kDetThreshold = 1e-4;            // Quadric::IsInvertible
constexpr double kDblMin = 2.2250738585072014e-308;  // std::numeric_limits<double>::min(), LDLT's pivot tolerance

struct CellGrid {
  double m[3];  // min bound - s/2
  double s;
  unsigned long long dims[3];  // cells per axis
};

__device__ __forceinline__ long long cell_index(double v, double m, double s) {
  return (long long)floor(__ddiv_rn(__dsub_rn(v, m), s));
}

// key = (c0 * d1 + c1) * d2 + c2 over the cell box; the host has checked d0 * d1 * d2 <= 2^63
__global__ void __launch_bounds__(256) simplify_key_kernel(const double* __restrict__ xyz, int n, CellGrid g,
                                                           unsigned long long* __restrict__ keys, uint32_t* __restrict__ ids) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  unsigned long long c[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) c[a] = (unsigned long long)cell_index(xyz[3 * (size_t)i + a], g.m[a], g.s);
  keys[i] = (c[0] * g.dims[1] + c[1]) * g.dims[2] + c[2];
  ids[i] = (uint32_t)i;
}

// Per sorted position j: head[j] = j starts a cell; first[v] = vertex v is its cell's smallest id (the stable sort
// keeps ids ascending inside a cell, so the head is the smallest).
__global__ void __launch_bounds__(256) simplify_head_kernel(const unsigned long long* __restrict__ keys,
                                                            const uint32_t* __restrict__ ids, int n, int* __restrict__ head,
                                                            int* __restrict__ first) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const int h = j == 0 || keys[j] != keys[j - 1];
  head[j] = h;
  first[ids[j]] = h;
}

// For each head j (segment seg = segid[j], cell c = rank[ids[j]]): where the segment begins and which cell it is.
__global__ void __launch_bounds__(256) simplify_segment_kernel(const uint32_t* __restrict__ ids, const int* __restrict__ head,
                                                               const int* __restrict__ segid, const int* __restrict__ rank, int n,
                                                               int* __restrict__ seg_begin, int* __restrict__ seg_cell,
                                                               int* __restrict__ cell_seg) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  if (j == n - 1) seg_begin[segid[j] + head[j]] = n;  // one past the last segment
  if (!head[j]) return;
  const int seg = segid[j], c = rank[ids[j]];
  seg_begin[seg] = j;
  seg_cell[seg] = c;
  cell_seg[c] = seg;
}

__global__ void __launch_bounds__(256) simplify_vertex_cell_kernel(const uint32_t* __restrict__ ids, const int* __restrict__ head,
                                                                   const int* __restrict__ segid, const int* __restrict__ seg_cell,
                                                                   int n, int* __restrict__ vcell) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  // segid is the exclusive scan of head: a head's segment is segid[j], a non-head's is segid[j] - 1
  vcell[ids[j]] = seg_cell[segid[j] + head[j] - 1];
}

// Vertex -> triangle incidence: (vertex, triangle) pairs of the flattened triangle array, sorted stably by vertex so
// each vertex's triangles come in ascending id, and integer counts per vertex for the offsets.
__global__ void __launch_bounds__(256) simplify_incidence_kernel(const long long* __restrict__ tris, long long n3,
                                                                 uint32_t* __restrict__ vkey, uint32_t* __restrict__ tid,
                                                                 unsigned long long* __restrict__ count) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n3) return;
  const uint32_t v = (uint32_t)tris[p];
  vkey[p] = v;
  tid[p] = (uint32_t)(p / 3);
  atomicAdd(&count[v], 1ull);
}

// Open3D's ComputeTrianglePlane and GetTriangleArea folded into Quadric(plane, area): e0 = p1 - p0, e1 = p2 - p0,
// c = e0 x e1, |c| = sqrt((cx^2 + cy^2) + cz^2); n = c / |c| and d = -((n.x p0.x + n.y p0.y) + n.z p0.z), or the plane
// (0,0,0,0) when |c| == 0; w = 0.5 |c|; A_ij = (w n_i) n_j (all nine, not symmetrised), b_i = (w d) n_i.
__device__ __forceinline__ void triangle_quadric(const double* __restrict__ xyz, const long long* __restrict__ tris, uint32_t t,
                                                 double (&q)[12]) {
  const long long i0 = tris[3 * (size_t)t], i1 = tris[3 * (size_t)t + 1], i2 = tris[3 * (size_t)t + 2];
  const double x0 = xyz[3 * i0], y0 = xyz[3 * i0 + 1], z0 = xyz[3 * i0 + 2];
  const double ax = __dsub_rn(xyz[3 * i1], x0), ay = __dsub_rn(xyz[3 * i1 + 1], y0), az = __dsub_rn(xyz[3 * i1 + 2], z0);
  const double bx = __dsub_rn(xyz[3 * i2], x0), by = __dsub_rn(xyz[3 * i2 + 1], y0), bz = __dsub_rn(xyz[3 * i2 + 2], z0);
  const double cx = __dsub_rn(__dmul_rn(ay, bz), __dmul_rn(az, by));
  const double cy = __dsub_rn(__dmul_rn(az, bx), __dmul_rn(ax, bz));
  const double cz = __dsub_rn(__dmul_rn(ax, by), __dmul_rn(ay, bx));
  const double norm = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(cx, cx), __dmul_rn(cy, cy)), __dmul_rn(cz, cz)));
  double n[3] = {0.0, 0.0, 0.0}, d = 0.0;
  if (norm != 0.0) {
    n[0] = __ddiv_rn(cx, norm);
    n[1] = __ddiv_rn(cy, norm);
    n[2] = __ddiv_rn(cz, norm);
    d = -__dadd_rn(__dadd_rn(__dmul_rn(n[0], x0), __dmul_rn(n[1], y0)), __dmul_rn(n[2], z0));
  }
  const double w = __dmul_rn(0.5, norm);
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const double wn = __dmul_rn(w, n[i]);
#pragma unroll
    for (int j = 0; j < 3; ++j) q[3 * i + j] = __dmul_rn(wn, n[j]);
  }
  const double wd = __dmul_rn(w, d);
#pragma unroll
  for (int i = 0; i < 3; ++i) q[9 + i] = __dmul_rn(wd, n[i]);
}

// Eigen's 3x3 determinant: (m00 (m11 m22 - m12 m21) - m01 (m10 m22 - m12 m20)) + m02 (m10 m21 - m11 m20)
__device__ __forceinline__ double det3(const double (&a)[12]) {
  const double h0 = __dmul_rn(a[0], __dsub_rn(__dmul_rn(a[4], a[8]), __dmul_rn(a[5], a[7])));
  const double h1 = __dmul_rn(a[1], __dsub_rn(__dmul_rn(a[3], a[8]), __dmul_rn(a[5], a[6])));
  const double h2 = __dmul_rn(a[2], __dsub_rn(__dmul_rn(a[3], a[7]), __dmul_rn(a[4], a[6])));
  return __dadd_rn(__dsub_rn(h0, h1), h2);
}

__device__ __forceinline__ void swap_d(double& a, double& b) {
  const double t = a;
  a = b;
  b = t;
}

// x = A^-1 b by Eigen's LDLT<Matrix3d> (lower, pivoted on the largest remaining |diagonal|, first on ties; only the
// lower triangle of A is read), then the solve with Eigen's unrolled triangular solves and its pseudo-inverse of D
// (a component whose |D_i| <= DBL_MIN becomes 0).  tests/simplify_oracle.py::ldlt_solve states the same steps.
__device__ void ldlt_solve3(const double (&a)[12], double (&y)[3]) {
  double m[3][3];
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) m[i][j] = a[3 * i + j];
  int tr[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    int p = k;
#pragma unroll
    for (int i = k + 1; i < 3; ++i)
      if (fabs(m[i][i]) > fabs(m[p][p])) p = i;
    tr[k] = p;
    if (p != k) {
      for (int j = 0; j < k; ++j) swap_d(m[k][j], m[p][j]);
      for (int i = p + 1; i < 3; ++i) swap_d(m[i][k], m[i][p]);
      swap_d(m[k][k], m[p][p]);
      for (int i = k + 1; i < p; ++i) {
        const double t = m[i][k];
        m[i][k] = m[p][i];
        m[p][i] = t;
      }
    }
    if (k == 1) {
      const double t0 = __dmul_rn(m[0][0], m[1][0]);
      m[1][1] = __dsub_rn(m[1][1], __dmul_rn(m[1][0], t0));
      m[2][1] = __dsub_rn(m[2][1], __dmul_rn(m[2][0], t0));
    } else if (k == 2) {
      const double t0 = __dmul_rn(m[0][0], m[2][0]), t1 = __dmul_rn(m[1][1], m[2][1]);
      m[2][2] = __dsub_rn(m[2][2], __dadd_rn(__dmul_rn(m[2][0], t0), __dmul_rn(m[2][1], t1)));
    }
    if (fabs(m[k][k]) > 0.0)
      for (int i = k + 1; i < 3; ++i) m[i][k] = __ddiv_rn(m[i][k], m[k][k]);
  }
  y[0] = a[9];
  y[1] = a[10];
  y[2] = a[11];
#pragma unroll
  for (int k = 0; k < 3; ++k)
    if (tr[k] != k) swap_d(y[k], y[tr[k]]);
  y[1] = __dsub_rn(y[1], __dmul_rn(m[1][0], y[0]));
  y[2] = __dsub_rn(y[2], __dadd_rn(__dmul_rn(m[2][0], y[0]), __dmul_rn(m[2][1], y[1])));
#pragma unroll
  for (int i = 0; i < 3; ++i) y[i] = fabs(m[i][i]) > kDblMin ? __ddiv_rn(y[i], m[i][i]) : 0.0;
  y[1] = __dsub_rn(y[1], __dmul_rn(m[2][1], y[2]));
  y[0] = __dsub_rn(y[0], __dadd_rn(__dmul_rn(m[1][0], y[1]), __dmul_rn(m[2][0], y[2])));
#pragma unroll
  for (int k = 2; k >= 0; --k)
    if (tr[k] != k) swap_d(y[k], y[tr[k]]);
}

// One thread per cell: sequential sums in ascending vertex id from 0.0, divided by double(count); with `quadric`, the
// quadric of every (vertex, distinct incident triangle) pair in (vertex, triangle) order, and -A^-1 b when
// |det A| > 1e-4.
__global__ void __launch_bounds__(128) simplify_cell_kernel(const double* __restrict__ xyz, const double* __restrict__ rgb,
                                                            const double* __restrict__ nrm, const uint32_t* __restrict__ ids,
                                                            const int* __restrict__ seg_begin, const int* __restrict__ cell_seg,
                                                            const int* __restrict__ n_cells_of, const long long* __restrict__ tris,
                                                            const long long* __restrict__ inc_off, const uint32_t* __restrict__ inc_tid,
                                                            double* __restrict__ out_xyz, double* __restrict__ out_rgb,
                                                            double* __restrict__ out_nrm, unsigned long long* __restrict__ n_quadric) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= *n_cells_of) return;
  const int seg = cell_seg[c], begin = seg_begin[seg], end = seg_begin[seg + 1];
  const double cnt = (double)(end - begin);
  double sp[3] = {0.0, 0.0, 0.0}, sc[3] = {0.0, 0.0, 0.0}, sn[3] = {0.0, 0.0, 0.0};
  for (int j = begin; j < end; ++j) {
    const size_t v = ids[j];
#pragma unroll
    for (int a = 0; a < 3; ++a) sp[a] = __dadd_rn(sp[a], xyz[3 * v + a]);
    if (rgb)
#pragma unroll
      for (int a = 0; a < 3; ++a) sc[a] = __dadd_rn(sc[a], rgb[3 * v + a]);
    if (nrm)
#pragma unroll
      for (int a = 0; a < 3; ++a) sn[a] = __dadd_rn(sn[a], nrm[3 * v + a]);
  }
  double pos[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) pos[a] = __ddiv_rn(sp[a], cnt);
  if (inc_off) {
    double q[12];
#pragma unroll
    for (int k = 0; k < 12; ++k) q[k] = 0.0;
    for (int j = begin; j < end; ++j) {
      const uint32_t v = ids[j];
      uint32_t prev = 0xffffffffu;
      for (long long k = inc_off[v]; k < inc_off[v + 1]; ++k) {
        const uint32_t t = inc_tid[k];
        if (t == prev) continue;  // (a, a, b): once for a
        prev = t;
        double qt[12];
        triangle_quadric(xyz, tris, t, qt);
#pragma unroll
        for (int e = 0; e < 12; ++e) q[e] = __dadd_rn(q[e], qt[e]);
      }
    }
    if (fabs(det3(q)) > kDetThreshold) {
      double y[3];
      ldlt_solve3(q, y);
#pragma unroll
      for (int a = 0; a < 3; ++a) pos[a] = -y[a];
      atomicAdd(n_quadric, 1ull);
    }
  }
#pragma unroll
  for (int a = 0; a < 3; ++a) out_xyz[3 * (size_t)c + a] = pos[a];
  if (rgb)
#pragma unroll
    for (int a = 0; a < 3; ++a) out_rgb[3 * (size_t)c + a] = __ddiv_rn(sc[a], cnt);
  if (nrm)
#pragma unroll
    for (int a = 0; a < 3; ++a) out_nrm[3 * (size_t)c + a] = __ddiv_rn(sn[a], cnt);
}

// Triangle t -> its cells (a, b, c), rotated so the smallest comes first (Open3D: (b, c, a) if b is smallest, (c, a, b)
// if c is); a triangle with two corners in one cell is dropped (tri3 a = -1) and sorts last in the second pass.
__global__ void __launch_bounds__(256) simplify_triangle_kernel(const long long* __restrict__ tris, const int* __restrict__ vcell,
                                                                int nt, int* __restrict__ tri3, uint32_t* __restrict__ lo_key,
                                                                uint32_t* __restrict__ tid) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nt) return;
  int a = vcell[tris[3 * (size_t)t]], b = vcell[tris[3 * (size_t)t + 1]], c = vcell[tris[3 * (size_t)t + 2]];
  const bool drop = a == b || a == c || b == c;
  if (b < a && b < c) {
    const int x = a;
    a = b;
    b = c;
    c = x;
  } else if (c < a && c < b) {
    const int x = b;
    b = a;
    a = c;
    c = x;
  }
  tri3[3 * (size_t)t] = a;
  tri3[3 * (size_t)t + 1] = b;
  tri3[3 * (size_t)t + 2] = c;
  if (drop) tri3[3 * (size_t)t] = -1;
  lo_key[t] = (uint32_t)c;
  tid[t] = (uint32_t)t;
}

// The second pass's keys in the order the first pass left: (a * nv + b), or nv * nv for a dropped triangle.
__global__ void __launch_bounds__(256) simplify_hi_key_kernel(const int* __restrict__ tri3, const uint32_t* __restrict__ tid,
                                                              int nt, unsigned long long nv, unsigned long long* __restrict__ hi_key) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= nt) return;
  const size_t t = tid[j];
  const int a = tri3[3 * t];
  hi_key[j] = a < 0 ? nv * nv : (unsigned long long)a * nv + (unsigned long long)tri3[3 * t + 1];
}

// keep[t] = t heads its run of equal rotated triples in the sorted order (the smallest id of the run: both passes are
// stable over ascending ids) and is not dropped.
__global__ void __launch_bounds__(256) simplify_unique_kernel(const int* __restrict__ tri3, const uint32_t* __restrict__ tid,
                                                              const unsigned long long* __restrict__ hi_key, int nt,
                                                              unsigned long long dropped_key, int* __restrict__ keep) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= nt) return;
  const uint32_t t = tid[j];
  int k = hi_key[j] != dropped_key;
  if (k && j > 0 && hi_key[j] == hi_key[j - 1]) k = tri3[3 * (size_t)t + 2] != tri3[3 * (size_t)tid[j - 1] + 2];
  keep[t] = k;
}

__global__ void __launch_bounds__(256) simplify_compact_kernel(const int* __restrict__ tri3, const int* __restrict__ keep,
                                                               const int* __restrict__ pos, int nt, long long* __restrict__ out) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nt || !keep[t]) return;
  const size_t o = 3 * (size_t)pos[t];
#pragma unroll
  for (int k = 0; k < 3; ++k) out[o + k] = tri3[3 * (size_t)t + k];
}

// sizes[0] = cells (the rank after the last vertex), sizes[1] = kept triangles; sizes[2] was zeroed and counted.
__global__ void simplify_sizes_kernel(const int* __restrict__ first, const int* __restrict__ rank, int nv,
                                      const int* __restrict__ keep, const int* __restrict__ pos, int nt, int* __restrict__ n_cells,
                                      long long* __restrict__ sizes) {
  const int cells = nv ? rank[nv - 1] + first[nv - 1] : 0;
  *n_cells = cells;
  sizes[0] = cells;
  sizes[1] = nt ? (long long)pos[nt - 1] + keep[nt - 1] : 0;
}

// key bits a radix sort needs for keys <= max_value (at least one)
inline int sort_bits(unsigned long long max_value) {
  int b = 1;
  while (b < 64 && (max_value >> b) != 0) ++b;
  return b;
}

struct SimplifyWork {
  unsigned long long* vkeys;  // [2 nv] cell keys (DoubleBuffer)
  uint32_t* vids;             // [2 nv] vertex ids (DoubleBuffer)
  int *head, *first, *segid, *rank, *seg_begin, *seg_cell, *cell_seg, *vcell;  // [nv] each, seg_begin [nv + 1]
  int* n_cells;                                                                // [1]
  uint32_t *inc_v, *inc_t;                                                     // [2 * 3 nt] each (DoubleBuffer)
  unsigned long long* inc_count;                                               // [nv + 1] incidences per vertex
  long long* inc_off;                                                          // [nv + 1] their exclusive scan
  int* tri3;                                                                   // [3 nt]
  uint32_t *lo_key, *tid;                                                      // [2 nt] each (DoubleBuffer)
  unsigned long long* hi_key;                                                  // [2 nt] (DoubleBuffer)
  int *keep, *pos;                                                             // [nt] each
  void* tmp;
  size_t tmp_bytes, total;
};

size_t simplify_cub_bytes(int64_t nv, int64_t nt) {
  size_t a = 0, b = 0, c = 0, d = 0, e = 0, f = 0;
  cub::DoubleBuffer<unsigned long long> k64(nullptr, nullptr);
  cub::DoubleBuffer<uint32_t> v32(nullptr, nullptr), k32(nullptr, nullptr);
  cub::DeviceRadixSort::SortPairs(nullptr, a, k64, v32, (int)nv);
  cub::DeviceRadixSort::SortPairs(nullptr, b, k32, v32, 3 * (long long)nt);
  cub::DeviceRadixSort::SortPairs(nullptr, c, k32, v32, (int)nt);
  cub::DeviceRadixSort::SortPairs(nullptr, d, k64, v32, (int)nt);
  cub::DeviceScan::ExclusiveSum(nullptr, e, (int*)nullptr, (int*)nullptr, (int)(nv > nt ? nv : nt));
  cub::DeviceScan::ExclusiveSum(nullptr, f, (unsigned long long*)nullptr, (long long*)nullptr, (long long)nv + 1);
  size_t m = a;
  for (size_t x : {b, c, d, e, f}) m = x > m ? x : m;
  return m;
}

SimplifyWork carve_simplify(void* base, int64_t nv, int64_t nt) {
  Carver c(base);
  SimplifyWork w;
  w.vkeys = c.take<unsigned long long>(2 * (size_t)nv);
  w.vids = c.take<uint32_t>(2 * (size_t)nv);
  w.head = c.take<int>((size_t)nv);
  w.first = c.take<int>((size_t)nv);
  w.segid = c.take<int>((size_t)nv);
  w.rank = c.take<int>((size_t)nv);
  w.seg_begin = c.take<int>((size_t)nv + 1);
  w.seg_cell = c.take<int>((size_t)nv);
  w.cell_seg = c.take<int>((size_t)nv);
  w.vcell = c.take<int>((size_t)nv);
  w.n_cells = c.take<int>(1);
  w.inc_v = c.take<uint32_t>(6 * (size_t)nt);
  w.inc_t = c.take<uint32_t>(6 * (size_t)nt);
  w.inc_count = c.take<unsigned long long>((size_t)nv + 1);
  w.inc_off = c.take<long long>((size_t)nv + 1);
  w.tri3 = c.take<int>(3 * (size_t)nt);
  w.lo_key = c.take<uint32_t>(2 * (size_t)nt);
  w.tid = c.take<uint32_t>(2 * (size_t)nt);
  w.hi_key = c.take<unsigned long long>(2 * (size_t)nt);
  w.keep = c.take<int>((size_t)nt);
  w.pos = c.take<int>((size_t)nt);
  w.tmp_bytes = simplify_cub_bytes(nv, nt);
  w.tmp = c.take<char>(w.tmp_bytes);
  w.total = c.total();
  return w;
}

bool finite3(const double* v) { return std::isfinite(v[0]) && std::isfinite(v[1]) && std::isfinite(v[2]); }

}  // namespace
}  // namespace gsb

using namespace gsb;

extern "C" {

size_t gsb_mesh_simplify_workspace_bytes(int64_t n_vertices, int64_t n_triangles) {
  if (!mesh_sizes_ok(n_triangles, n_vertices, kMaxMeshIds)) return 0;
  return carve_simplify(nullptr, n_vertices, n_triangles).total;
}

int gsb_mesh_simplify(const double* vertices, const double* colors, const double* normals, int64_t n_vertices,
                      const int64_t* triangles, int64_t n_triangles, const double* min_bound, const double* max_bound,
                      double voxel_size, int contraction, void* workspace, size_t workspace_bytes, double* out_vertices,
                      double* out_colors, double* out_normals, int64_t* out_triangles, int64_t* sizes, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (!mesh_sizes_ok(n_triangles, n_vertices, kMaxMeshIds))
    return mesh_size_error("mesh_simplify", n_triangles, n_vertices, kMaxMeshIds);
  if (contraction != GSB_SIMPLIFY_AVERAGE && contraction != GSB_SIMPLIFY_QUADRIC)
    return fail(GSB_ERR_INVALID, "mesh_simplify: unknown contraction %d", contraction);
  if (!sizes || !min_bound || !max_bound ||
      (n_vertices && (!vertices || !workspace || !out_vertices || (colors && !out_colors) || (normals && !out_normals))) ||
      (n_triangles && (!triangles || !out_triangles)))
    return fail(GSB_ERR_INVALID, "mesh_simplify: bad arguments");
  if (!(voxel_size > 0.0)) return fail(GSB_ERR_INVALID, "mesh_simplify: voxel_size <= 0.0");
  if (!std::isfinite(voxel_size)) return fail(GSB_ERR_INVALID, "mesh_simplify: voxel_size is not finite");
  if (!finite3(min_bound) || !finite3(max_bound)) return fail(GSB_ERR_INVALID, "mesh_simplify: the vertices are not finite");
  // Open3D: voxel_min_bound = min - s/2, voxel_max_bound = max + s/2, s * INT_MAX < (max_bound - min_bound).maxCoeff()
  CellGrid g;
  g.s = voxel_size;
  const double half = voxel_size * 0.5;
  double span = 0.0;
  for (int a = 0; a < 3; ++a) {
    g.m[a] = min_bound[a] - half;
    const double e = (max_bound[a] + half) - g.m[a];
    span = a == 0 || e > span ? e : span;
  }
  if (voxel_size * 2147483647.0 < span) return fail(GSB_ERR_INVALID, "mesh_simplify: voxel_size is too small.");
  // cells per axis: the cell of the maximum (the largest any vertex gets; the minimum's cell is 0) + 1, <= 2^31
  unsigned __int128 cells = 1;
  for (int a = 0; a < 3; ++a) {
    g.dims[a] = (unsigned long long)std::floor((max_bound[a] - g.m[a]) / voxel_size) + 1;
    cells *= g.dims[a];
  }
  if (cells > ((unsigned __int128)1 << 63))
    return fail(GSB_ERR_INVALID,
                "mesh_simplify: %llu x %llu x %llu cells; cell keys are limited to 63 bits (at most 2^63 cells in the box)",
                g.dims[0], g.dims[1], g.dims[2]);
  const size_t need = gsb_mesh_simplify_workspace_bytes(n_vertices, n_triangles);
  if (n_vertices && workspace_bytes < need)
    return fail(GSB_ERR_WORKSPACE, "mesh_simplify: workspace %zu < %zu bytes", workspace_bytes, need);
  GSB_CUDA_OK(cudaMemsetAsync(sizes, 0, 3 * sizeof(int64_t), stream));
  if (n_vertices == 0) return GSB_OK;

  const int nv = (int)n_vertices, nt = (int)n_triangles;
  const SimplifyWork w = carve_simplify(workspace, n_vertices, n_triangles);
  const auto* tris = reinterpret_cast<const long long*>(triangles);
  size_t tmp_bytes;

  // cells and their numbering
  simplify_key_kernel<<<blocks_for(nv), 256, 0, stream>>>(vertices, nv, g, w.vkeys, w.vids);
  count_launch();
  cub::DoubleBuffer<unsigned long long> vk(w.vkeys, w.vkeys + nv);
  cub::DoubleBuffer<uint32_t> vi(w.vids, w.vids + nv);
  tmp_bytes = w.tmp_bytes;
  GSB_CUDA_OK(cub::DeviceRadixSort::SortPairs(w.tmp, tmp_bytes, vk, vi, nv, 0, sort_bits((unsigned long long)(cells - 1)), stream));
  const uint32_t* ids = vi.Current();
  simplify_head_kernel<<<blocks_for(nv), 256, 0, stream>>>(vk.Current(), ids, nv, w.head, w.first);
  count_launch();
  tmp_bytes = w.tmp_bytes;
  GSB_CUDA_OK(cub::DeviceScan::ExclusiveSum(w.tmp, tmp_bytes, w.head, w.segid, nv, stream));
  tmp_bytes = w.tmp_bytes;
  GSB_CUDA_OK(cub::DeviceScan::ExclusiveSum(w.tmp, tmp_bytes, w.first, w.rank, nv, stream));
  simplify_segment_kernel<<<blocks_for(nv), 256, 0, stream>>>(ids, w.head, w.segid, w.rank, nv, w.seg_begin, w.seg_cell,
                                                              w.cell_seg);
  simplify_vertex_cell_kernel<<<blocks_for(nv), 256, 0, stream>>>(ids, w.head, w.segid, w.seg_cell, nv, w.vcell);
  count_launch(2);

  // triangles: remap, two stable passes (c, then a * nv + b), run heads, compaction in input order
  int* keep = w.keep;
  if (nt) {
    const unsigned long long unv = (unsigned long long)nv, dropped = unv * unv;
    simplify_triangle_kernel<<<blocks_for(nt), 256, 0, stream>>>(tris, w.vcell, nt, w.tri3, w.lo_key, w.tid);
    count_launch();
    cub::DoubleBuffer<uint32_t> lk(w.lo_key, w.lo_key + nt), ti(w.tid, w.tid + nt);
    tmp_bytes = w.tmp_bytes;
    GSB_CUDA_OK(cub::DeviceRadixSort::SortPairs(w.tmp, tmp_bytes, lk, ti, nt, 0, sort_bits(unv - 1), stream));
    cub::DoubleBuffer<unsigned long long> hk(w.hi_key, w.hi_key + nt);
    uint32_t* ti_alt = ti.Alternate();
    simplify_hi_key_kernel<<<blocks_for(nt), 256, 0, stream>>>(w.tri3, ti.Current(), nt, unv, hk.Current());
    count_launch();
    cub::DoubleBuffer<uint32_t> ti2(ti.Current(), ti_alt);
    tmp_bytes = w.tmp_bytes;
    GSB_CUDA_OK(cub::DeviceRadixSort::SortPairs(w.tmp, tmp_bytes, hk, ti2, nt, 0, sort_bits(dropped), stream));
    simplify_unique_kernel<<<blocks_for(nt), 256, 0, stream>>>(w.tri3, ti2.Current(), hk.Current(), nt, dropped, keep);
    count_launch();
    tmp_bytes = w.tmp_bytes;
    GSB_CUDA_OK(cub::DeviceScan::ExclusiveSum(w.tmp, tmp_bytes, keep, w.pos, nt, stream));
    simplify_compact_kernel<<<blocks_for(nt), 256, 0, stream>>>(w.tri3, keep, w.pos, nt, reinterpret_cast<long long*>(out_triangles));
    count_launch();
  }
  simplify_sizes_kernel<<<1, 1, 0, stream>>>(w.first, w.rank, nv, keep, w.pos, nt, w.n_cells, reinterpret_cast<long long*>(sizes));
  count_launch();

  // vertex -> triangle incidence for the quadrics
  const long long* inc_off = nullptr;
  const uint32_t* inc_tid = nullptr;
  if (contraction == GSB_SIMPLIFY_QUADRIC) {
    GSB_CUDA_OK(cudaMemsetAsync(w.inc_count, 0, sizeof(unsigned long long) * ((size_t)nv + 1), stream));
    if (nt) {
      const long long n3 = 3 * (long long)nt;
      simplify_incidence_kernel<<<blocks_for(n3), 256, 0, stream>>>(tris, n3, w.inc_v, w.inc_t, w.inc_count);
      count_launch();
      cub::DoubleBuffer<uint32_t> iv(w.inc_v, w.inc_v + n3), it(w.inc_t, w.inc_t + n3);
      tmp_bytes = w.tmp_bytes;
      GSB_CUDA_OK(cub::DeviceRadixSort::SortPairs(w.tmp, tmp_bytes, iv, it, n3, 0, sort_bits((unsigned long long)nv - 1), stream));
      inc_tid = it.Current();
    } else {
      inc_tid = w.inc_t;
    }
    tmp_bytes = w.tmp_bytes;
    GSB_CUDA_OK(cub::DeviceScan::ExclusiveSum(w.tmp, tmp_bytes, w.inc_count, w.inc_off, (long long)nv + 1, stream));
    inc_off = w.inc_off;
  }
  simplify_cell_kernel<<<blocks_for(nv, 128), 128, 0, stream>>>(
      vertices, colors, normals, ids, w.seg_begin, w.cell_seg, w.n_cells, tris, inc_off, inc_tid, out_vertices,
      colors ? out_colors : nullptr, normals ? out_normals : nullptr, reinterpret_cast<unsigned long long*>(sizes + 2));
  count_launch();
  return check_launch("mesh_simplify", stream, false);
}

}  // extern "C"
