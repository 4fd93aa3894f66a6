// Mesh topology queries: Open3D 0.17.0 TriangleMesh::GetNonManifoldEdges / IsOrientable / EulerPoincareCharacteristic,
// GetNonManifoldVertices, GetSelfIntersectingTriangles, GetSurfaceArea and GetVolume (DESIGN.md section 7, "Topology
// queries"; restated in tests/topology_oracle.py).
//
// Edges: the 3 n_triangles edge incidences are radix-sorted by edge key (gsb_union_find.cuh's edge_key, the key of the
// cluster kernels) in triangle-major order, so each edge's incidences form one run in ascending (triangle, corner).
// Run lengths give the non-manifold edges; orientability is a union-find over the double cover (t, unflipped) /
// (t, flipped), one constraint per incidence against its run's first incidence.
// Vertices: one global union-find over the nodes (v, link vertex) of every vertex's link graph.
// Self-intersection: a uniform grid over the triangles' boxes, each pair tested once in the cell holding the minimum
// corner of the two boxes' intersection, one thread per candidate pair, with Moeller's NoDivTriTriIsect in fp64.
// Area and volume: per-triangle terms summed by a fixed-shape two-stage reduction.
//
// Every fp64 operation is an explicit __d*_rn, so nvcc contracts nothing; there are no floating-point atomics, so every
// run writes the same bytes.  The library allocates nothing and does not synchronise.
#include <cub/cub.cuh>

#include "gs2mesh_b200.h"
#include "gsb_common.h"
#include "gsb_union_find.cuh"

namespace gsb {
namespace {

// 6 n_triangles link-graph slots (two nodes per (triangle, corner)) are int ids: n_triangles <= (2^31 - 1) / 6.
constexpr int64_t kMaxTopoTriangles = 357913941;
constexpr int kLevels = 22;         // grid levels: 2^(20-L) + 1 cells per axis, L = 0 .. 21 (one cell)
constexpr int kRegsPerTriangle = 4;  // the chosen level registers at most 4 n_triangles (triangle, cell) pairs
constexpr int kNarrowBlocks = 132 * 8;  // grid-stride over the candidates: 8 blocks per SM of an H100 SXM
constexpr double kEps = 1e-6;        // Moeller's EPSILON with USE_EPSILON_TEST

template <typename T>
__device__ __forceinline__ long long upper_bound(const T* a, long long n, T x) {  // first index with a[i] > x
  long long lo = 0, hi = n;
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if (a[mid] <= x) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

// ---------------------------------------------------------------------------------------------------------------------
// Edges and orientability
// ---------------------------------------------------------------------------------------------------------------------

// Incidence i = 3t + k is edge (v[k], v[k+1 mod 3]) of triangle t: key edge_key, value 2t + (v[k] > v[k+1]) (the
// direction bit: 0 from the smaller id to the larger).  Double-cover nodes 2t (t as given) and 2t + 1 (t flipped).
__global__ void __launch_bounds__(256) edge_incidence_kernel(const long long* __restrict__ tris, int nt, unsigned long long stride,
                                                             unsigned long long* __restrict__ keys, int* __restrict__ val,
                                                             int* __restrict__ parent) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nt) return;
  const long long v[3] = {tris[3 * (size_t)t], tris[3 * (size_t)t + 1], tris[3 * (size_t)t + 2]};
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const long long a = v[k], b = v[(k + 1) % 3];
    keys[3 * (size_t)t + k] = edge_key(a, b, stride);
    val[3 * (size_t)t + k] = 2 * t + (a > b);
  }
  parent[2 * t] = 2 * t;
  parent[2 * t + 1] = 2 * t + 1;
}

// head[i] = 1 where a run of equal keys starts.
__global__ void __launch_bounds__(256) run_head_kernel(const unsigned long long* __restrict__ keys, long long n,
                                                       unsigned long long sentinel, int* __restrict__ head) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  head[i] = keys[i] != sentinel && (i == 0 || keys[i] != keys[i - 1]);
}

// run_id = inclusive scan of head; start[run] = its first position and start[n_runs] = the end of the last run (start
// may be NULL: only the count is wanted).
__global__ void __launch_bounds__(256) run_start_kernel(const int* __restrict__ head, const int* __restrict__ run_id, long long n,
                                                        const unsigned long long* __restrict__ keys, unsigned long long sentinel,
                                                        int* __restrict__ start, int* __restrict__ n_runs) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (start && head[i]) start[run_id[i] - 1] = (int)i;
  const bool valid = keys[i] != sentinel;  // sentinels sort last
  if (valid && (i == n - 1 || keys[i + 1] == sentinel)) {
    if (start) start[run_id[i]] = (int)(i + 1);
    *n_runs = run_id[i];
  }
  if (i == 0 && !valid) *n_runs = 0;
}

// Orientation constraints: every incidence of an edge (a, b), a != b, other than the run's first (the centre c)
// requires flip(u) xor flip(c) = [direction(u) == direction(c)].
__global__ void __launch_bounds__(256) orient_union_kernel(const unsigned long long* __restrict__ keys, const int* __restrict__ val,
                                                           const int* __restrict__ head, const int* __restrict__ run_id,
                                                           const int* __restrict__ start, long long n, unsigned long long stride,
                                                           int* parent) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || head[i]) return;
  const unsigned long long key = keys[i];
  if (key / stride == key % stride) return;  // (a, a) has no direction
  const int c = start[run_id[i] - 1];
  const int u = val[i] >> 1, cu = val[c] >> 1;
  if ((val[i] & 1) == (val[c] & 1)) {
    uf_union(parent, 2 * u, 2 * cu + 1);
    uf_union(parent, 2 * u + 1, 2 * cu);
  } else {
    uf_union(parent, 2 * u, 2 * cu);
    uf_union(parent, 2 * u + 1, 2 * cu + 1);
  }
}

__global__ void __launch_bounds__(256) orient_check_kernel(const int* __restrict__ parent, int nt, int* __restrict__ conflict) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nt) return;
  if (uf_root(parent, 2 * t) == uf_root(parent, 2 * t + 1)) *conflict = 1;  // every writer stores the same value
}

// bad[r] = 1 for a non-manifold edge run: more than two incidences, or (allow_boundary == 0) any count but two.
__global__ void __launch_bounds__(256) edge_flag_kernel(const int* __restrict__ start, const int* __restrict__ n_runs, long long n,
                                                        int allow_boundary, int* __restrict__ bad) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  if (r >= *n_runs) {
    bad[r] = 0;
    return;
  }
  const int len = start[r + 1] - start[r];
  bad[r] = allow_boundary ? len > 2 : len != 2;
}

__global__ void __launch_bounds__(256) edge_emit_kernel(const unsigned long long* __restrict__ keys, const int* __restrict__ start,
                                                        const int* __restrict__ n_runs, const int* __restrict__ bad,
                                                        const int* __restrict__ pos, long long n, unsigned long long stride,
                                                        long long* __restrict__ out_edges) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n || r >= *n_runs || !bad[r]) return;
  const unsigned long long key = keys[start[r]];
  out_edges[2 * (size_t)pos[r]] = (long long)(key / stride);
  out_edges[2 * (size_t)pos[r] + 1] = (long long)(key % stride);
}

__global__ void edge_sizes_kernel(const int* __restrict__ bad, const int* __restrict__ pos, const int* __restrict__ n_runs,
                                  const int* __restrict__ conflict, long long* __restrict__ sizes) {
  const int e = *n_runs;
  sizes[0] = e ? (long long)pos[e - 1] + bad[e - 1] : 0;
  sizes[1] = e;
  sizes[2] = !*conflict;
}

__global__ void edge_sizes_empty_kernel(long long* __restrict__ sizes) {
  sizes[0] = 0;
  sizes[1] = 0;
  sizes[2] = 1;
}

// ---------------------------------------------------------------------------------------------------------------------
// Vertex manifoldness
// ---------------------------------------------------------------------------------------------------------------------

// Slot s = 3t + k for the k-th distinct vertex v of triangle t: the link edge Open3D's if/else chain adds for (v, t), as
// the two node keys v * nv + x and v * nv + y (the sentinel nv^2 where the chain adds none).
__global__ void __launch_bounds__(256) link_edge_kernel(const long long* __restrict__ tris, int nt, unsigned long long nv,
                                                        unsigned long long* __restrict__ keys, int* __restrict__ slot) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nt) return;
  const long long v[3] = {tris[3 * (size_t)t], tris[3 * (size_t)t + 1], tris[3 * (size_t)t + 2]};
  const unsigned long long sentinel = nv * nv;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const size_t s = 3 * (size_t)t + k;
    unsigned long long k0 = sentinel, k1 = sentinel;
    const long long c = v[k];
    const bool repeat = (k > 0 && v[0] == c) || (k > 1 && v[1] == c);  // the triangle counts once per vertex
    if (!repeat) {
      long long x = -1, y = -1;
      if (v[0] != c && v[1] != c) x = v[0], y = v[1];
      else if (v[0] != c && v[2] != c) x = v[0], y = v[2];
      else if (v[1] != c && v[2] != c) x = v[1], y = v[2];
      if (x >= 0) {
        k0 = (unsigned long long)c * nv + (unsigned long long)x;
        k1 = (unsigned long long)c * nv + (unsigned long long)y;
      }
    }
    keys[2 * s] = k0;
    keys[2 * s + 1] = k1;
    slot[2 * s] = (int)(2 * s);
    slot[2 * s + 1] = (int)(2 * s + 1);
  }
}

// node_of[slot] = the node id (rank of its key among the distinct keys) or -1; node_vertex / parent per node.
__global__ void __launch_bounds__(256) link_nodes_kernel(const unsigned long long* __restrict__ keys, const int* __restrict__ slot,
                                                         const int* __restrict__ head, const int* __restrict__ rank, long long n,
                                                         unsigned long long nv, int* __restrict__ node_of, int* __restrict__ node_vertex,
                                                         int* __restrict__ parent) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned long long key = keys[i];
  if (key == nv * nv) {
    node_of[slot[i]] = -1;
    return;
  }
  const int node = rank[i] - 1;
  node_of[slot[i]] = node;
  if (head[i]) {
    node_vertex[node] = (int)(key / nv);
    parent[node] = node;
  }
}

__global__ void __launch_bounds__(256) link_union_kernel(const int* __restrict__ node_of, long long n_slots, int* parent) {
  const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n_slots) return;
  const int a = node_of[2 * s], b = node_of[2 * s + 1];
  if (a >= 0) uf_union(parent, a, b);
}

// roots[v] = the number of components of v's link graph (integer atomics: exact).
__global__ void __launch_bounds__(256) link_roots_kernel(const int* __restrict__ parent, const int* __restrict__ node_vertex,
                                                         const int* __restrict__ n_nodes, long long n, int* roots) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || i >= *n_nodes) return;
  if (parent[i] == i) atomicAdd(&roots[node_vertex[i]], 1);
}

__global__ void __launch_bounds__(256) vertex_flag_kernel(const int* __restrict__ roots, int nv, int* __restrict__ bad) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v < nv) bad[v] = roots[v] > 1;
}

__global__ void __launch_bounds__(256) vertex_emit_kernel(const int* __restrict__ bad, const int* __restrict__ pos, int nv,
                                                          long long* __restrict__ out, long long* __restrict__ count) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= nv) return;
  if (out && bad[v]) out[pos[v]] = v;  // out == NULL: the count only
  if (v == nv - 1) *count = (long long)pos[v] + bad[v];
}

// ---------------------------------------------------------------------------------------------------------------------
// Self-intersection: grid broad phase
// ---------------------------------------------------------------------------------------------------------------------

// Grid coordinate of x on one axis at level L: u = (x - o) / E clamped to [0, 1], floor(u * 2^(20-L)).  Monotone in x,
// so the cell of max(lo0, lo1) is the larger of the two boxes' lower cells.
__device__ __forceinline__ int cell_of(double x, double o, double extent, int level) {
  double u = __ddiv_rn(__dsub_rn(x, o), extent);
  u = u < 0.0 ? 0.0 : (u > 1.0 ? 1.0 : u);
  return (int)floor(ldexp(u, 20 - level));
}

struct Grid {
  double o[3];
  double extent;
};

__device__ __forceinline__ void load_box(const double* __restrict__ box, int t, double lo[3], double hi[3]) {
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    lo[a] = box[6 * (size_t)t + a];
    hi[a] = box[6 * (size_t)t + 3 + a];
  }
}

// Triangle boxes (min / max of the corners, Open3D's cwiseMin / cwiseMax), and the registrations every level would make
// (cells per triangle, capped at 2^32 so the sums cannot overflow), summed per level with integer atomics.
__global__ void __launch_bounds__(256) box_kernel(const double* __restrict__ xyz, const long long* __restrict__ tris, int nt,
                                                  Grid g, double* __restrict__ box, unsigned long long* __restrict__ level_regs) {
  using Reduce = cub::BlockReduce<unsigned long long, 256>;
  __shared__ typename Reduce::TempStorage tmp;
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  double lo[3] = {0, 0, 0}, hi[3] = {0, 0, 0};
  if (t < nt) {
    const long long i0 = tris[3 * (size_t)t], i1 = tris[3 * (size_t)t + 1], i2 = tris[3 * (size_t)t + 2];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const double p0 = xyz[3 * i0 + a], p1 = xyz[3 * i1 + a], p2 = xyz[3 * i2 + a];
      lo[a] = fmin(p0, fmin(p1, p2));
      hi[a] = fmax(p0, fmax(p1, p2));
      box[6 * (size_t)t + a] = lo[a];
      box[6 * (size_t)t + 3 + a] = hi[a];
    }
  }
  for (int L = 0; L < kLevels; ++L) {
    unsigned long long n = 0;
    if (t < nt) {
      n = 1;
#pragma unroll
      for (int a = 0; a < 3; ++a)
        n *= (unsigned long long)(cell_of(hi[a], g.o[a], g.extent, L) - cell_of(lo[a], g.o[a], g.extent, L) + 1);
      n = n < (1ull << 32) ? n : (1ull << 32);
    }
    const unsigned long long s = Reduce(tmp).Sum(n);
    if (threadIdx.x == 0 && s) atomicAdd(&level_regs[L], s);
    __syncthreads();
  }
}

// The finest level whose registrations fit kRegsPerTriangle * n_triangles (the coarsest, one cell, always does).
__global__ void choose_level_kernel(const unsigned long long* __restrict__ level_regs, int nt, int* __restrict__ level,
                                    long long* __restrict__ stats) {
  int L = 0;
  while (L < kLevels - 1 && level_regs[L] > (unsigned long long)kRegsPerTriangle * nt) ++L;
  *level = L;
  stats[2] = (long long)level_regs[L];
  stats[3] = L;
}

__device__ __forceinline__ void cell_span(const double* __restrict__ box, int t, const Grid& g, int L, int c0[3], int n[3]) {
  double lo[3], hi[3];
  load_box(box, t, lo, hi);
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    c0[a] = cell_of(lo[a], g.o[a], g.extent, L);
    n[a] = cell_of(hi[a], g.o[a], g.extent, L) - c0[a] + 1;
  }
}

__device__ __forceinline__ unsigned long long cell_key(int x, int y, int z) {
  return ((unsigned long long)x << 42) | ((unsigned long long)y << 21) | (unsigned long long)z;
}

__global__ void __launch_bounds__(256) reg_count_kernel(const double* __restrict__ box, int nt, Grid g, const int* __restrict__ level,
                                                        int* __restrict__ count) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nt) return;
  int c0[3], n[3];
  cell_span(box, t, g, *level, c0, n);
  count[t] = n[0] * n[1] * n[2];
}

// One thread per registration slot r < cap: the triangle owning r (upper bound in the offsets) and its cell; slots past
// the registrations get the sentinel key.  Registrations come in ascending triangle order, which the stable sort keeps
// inside each cell.
__global__ void __launch_bounds__(256) reg_fill_kernel(const double* __restrict__ box, int nt, Grid g, const int* __restrict__ level,
                                                       const int* __restrict__ offset, const int* __restrict__ count, long long cap,
                                                       unsigned long long* __restrict__ keys, int* __restrict__ ids) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= cap) return;
  const long long total = (long long)offset[nt - 1] + count[nt - 1];
  if (r >= total) {
    keys[r] = ~0ull;
    ids[r] = 0;
    return;
  }
  const int t = (int)upper_bound(offset, nt, (int)r) - 1;
  int c0[3], n[3];
  cell_span(box, t, g, *level, c0, n);
  const int j = (int)(r - offset[t]);
  const int dz = j % n[2], dy = (j / n[2]) % n[1], dx = j / (n[2] * n[1]);
  keys[r] = cell_key(c0[0] + dx, c0[1] + dy, c0[2] + dz);
  ids[r] = t;
}

// Per cell (run of equal keys) its start and k(k-1)/2 candidate pairs; cells past the last get 0 pairs.
__global__ void __launch_bounds__(256) cell_pairs_kernel(const int* __restrict__ start, const int* __restrict__ n_cells, long long cap,
                                                         long long* __restrict__ pairs) {
  const long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= cap) return;
  if (c >= *n_cells) {
    pairs[c] = 0;
    return;
  }
  const long long k = start[c + 1] - start[c];
  pairs[c] = k * (k - 1) / 2;
}

__global__ void pair_total_kernel(const long long* __restrict__ pair_off, const long long* __restrict__ pairs,
                                  const int* __restrict__ n_cells, long long* __restrict__ stats, long long* __restrict__ total) {
  const int c = *n_cells;
  *total = c ? pair_off[c - 1] + pairs[c - 1] : 0;
  stats[1] = *total;
}

// ---------------------------------------------------------------------------------------------------------------------
// Self-intersection: narrow phase (Open3D's IntersectionTest::TriangleTriangle3d)
// ---------------------------------------------------------------------------------------------------------------------
#define DADD __dadd_rn
#define DSUB __dsub_rn
#define DMUL __dmul_rn

__device__ __forceinline__ double dot3(const double* a, const double* b) {
  return DADD(DADD(DMUL(a[0], b[0]), DMUL(a[1], b[1])), DMUL(a[2], b[2]));
}
__device__ __forceinline__ void cross3(double* d, const double* a, const double* b) {
  d[0] = DSUB(DMUL(a[1], b[2]), DMUL(a[2], b[1]));
  d[1] = DSUB(DMUL(a[2], b[0]), DMUL(a[0], b[2]));
  d[2] = DSUB(DMUL(a[0], b[1]), DMUL(a[1], b[0]));
}

// EDGE_EDGE_TEST(V0, U0, U1) with A = V1 - V0 projected on (i0, i1)
__device__ __forceinline__ bool edge_edge(double Ax, double Ay, const double* V0, const double* U0, const double* U1, int i0, int i1) {
  const double Bx = DSUB(U0[i0], U1[i0]), By = DSUB(U0[i1], U1[i1]);
  const double Cx = DSUB(V0[i0], U0[i0]), Cy = DSUB(V0[i1], U0[i1]);
  const double f = DSUB(DMUL(Ay, Bx), DMUL(Ax, By));
  const double d = DSUB(DMUL(By, Cx), DMUL(Bx, Cy));
  if ((f > 0.0 && d >= 0.0 && d <= f) || (f < 0.0 && d <= 0.0 && d >= f)) {
    const double e = DSUB(DMUL(Ax, Cy), DMUL(Ay, Cx));
    if (f > 0.0) {
      if (e >= 0.0 && e <= f) return true;
    } else {
      if (e <= 0.0 && e >= f) return true;
    }
  }
  return false;
}

__device__ __forceinline__ bool edge_against_tri(const double* V0, const double* V1, const double* U0, const double* U1,
                                                 const double* U2, int i0, int i1) {
  const double Ax = DSUB(V1[i0], V0[i0]), Ay = DSUB(V1[i1], V0[i1]);
  return edge_edge(Ax, Ay, V0, U0, U1, i0, i1) || edge_edge(Ax, Ay, V0, U1, U2, i0, i1) || edge_edge(Ax, Ay, V0, U2, U0, i0, i1);
}

// one line of POINT_IN_TRI: a = P[i1] - Q[i1], b = -(P[i0] - Q[i0]), c = -a*Q[i0] - b*Q[i1], d = a*V[i0] + b*V[i1] + c
__device__ __forceinline__ double side(const double* V, const double* Q, const double* P, int i0, int i1) {
  const double a = DSUB(P[i1], Q[i1]);
  const double b = -DSUB(P[i0], Q[i0]);
  const double c = DSUB(DMUL(-a, Q[i0]), DMUL(b, Q[i1]));
  return DADD(DADD(DMUL(a, V[i0]), DMUL(b, V[i1])), c);
}

__device__ __forceinline__ bool point_in_tri(const double* V0, const double* U0, const double* U1, const double* U2, int i0, int i1) {
  const double d0 = side(V0, U0, U1, i0, i1), d1 = side(V0, U1, U2, i0, i1), d2 = side(V0, U2, U0, i0, i1);
  return DMUL(d0, d1) > 0.0 && DMUL(d0, d2) > 0.0;
}

__device__ bool coplanar_tri_tri(const double* N, const double* V0, const double* V1, const double* V2, const double* U0,
                                 const double* U1, const double* U2) {
  const double A0 = fabs(N[0]), A1 = fabs(N[1]), A2 = fabs(N[2]);
  int i0, i1;
  if (A0 > A1) {
    if (A0 > A2) i0 = 1, i1 = 2;
    else i0 = 0, i1 = 1;
  } else {
    if (A2 > A1) i0 = 0, i1 = 1;
    else i0 = 0, i1 = 2;
  }
  if (edge_against_tri(V0, V1, U0, U1, U2, i0, i1)) return true;
  if (edge_against_tri(V1, V2, U0, U1, U2, i0, i1)) return true;
  if (edge_against_tri(V2, V0, U0, U1, U2, i0, i1)) return true;
  if (point_in_tri(V0, U0, U1, U2, i0, i1)) return true;
  if (point_in_tri(U0, V0, V1, V2, i0, i1)) return true;
  return false;
}

// NEWCOMPUTE_INTERVALS: false when the triangles are coplanar (the caller then runs the coplanar test)
__device__ __forceinline__ bool intervals(double VV0, double VV1, double VV2, double D0, double D1, double D2, double D0D1,
                                          double D0D2, double& A, double& B, double& C, double& X0, double& X1) {
  if (D0D1 > 0.0) {
    A = VV2, B = DMUL(DSUB(VV0, VV2), D2), C = DMUL(DSUB(VV1, VV2), D2), X0 = DSUB(D2, D0), X1 = DSUB(D2, D1);
  } else if (D0D2 > 0.0) {
    A = VV1, B = DMUL(DSUB(VV0, VV1), D1), C = DMUL(DSUB(VV2, VV1), D1), X0 = DSUB(D1, D0), X1 = DSUB(D1, D2);
  } else if (DMUL(D1, D2) > 0.0 || D0 != 0.0) {
    A = VV0, B = DMUL(DSUB(VV1, VV0), D0), C = DMUL(DSUB(VV2, VV0), D0), X0 = DSUB(D0, D1), X1 = DSUB(D0, D2);
  } else if (D1 != 0.0) {
    A = VV1, B = DMUL(DSUB(VV0, VV1), D1), C = DMUL(DSUB(VV2, VV1), D1), X0 = DSUB(D1, D0), X1 = DSUB(D1, D2);
  } else if (D2 != 0.0) {
    A = VV2, B = DMUL(DSUB(VV0, VV2), D2), C = DMUL(DSUB(VV1, VV2), D2), X0 = DSUB(D2, D0), X1 = DSUB(D2, D1);
  } else {
    return false;
  }
  return true;
}

__device__ bool no_div_tri_tri(const double* V0, const double* V1, const double* V2, const double* U0, const double* U1,
                               const double* U2) {
  double E1[3], E2[3], N1[3], N2[3], D[3];
  for (int a = 0; a < 3; ++a) E1[a] = DSUB(V1[a], V0[a]), E2[a] = DSUB(V2[a], V0[a]);
  cross3(N1, E1, E2);
  const double d1 = -dot3(N1, V0);
  double du0 = DADD(dot3(N1, U0), d1), du1 = DADD(dot3(N1, U1), d1), du2 = DADD(dot3(N1, U2), d1);
  if (fabs(du0) < kEps) du0 = 0.0;
  if (fabs(du1) < kEps) du1 = 0.0;
  if (fabs(du2) < kEps) du2 = 0.0;
  const double du0du1 = DMUL(du0, du1), du0du2 = DMUL(du0, du2);
  if (du0du1 > 0.0 && du0du2 > 0.0) return false;

  for (int a = 0; a < 3; ++a) E1[a] = DSUB(U1[a], U0[a]), E2[a] = DSUB(U2[a], U0[a]);
  cross3(N2, E1, E2);
  const double d2 = -dot3(N2, U0);
  double dv0 = DADD(dot3(N2, V0), d2), dv1 = DADD(dot3(N2, V1), d2), dv2 = DADD(dot3(N2, V2), d2);
  if (fabs(dv0) < kEps) dv0 = 0.0;
  if (fabs(dv1) < kEps) dv1 = 0.0;
  if (fabs(dv2) < kEps) dv2 = 0.0;
  const double dv0dv1 = DMUL(dv0, dv1), dv0dv2 = DMUL(dv0, dv2);
  if (dv0dv1 > 0.0 && dv0dv2 > 0.0) return false;

  cross3(D, N1, N2);
  double mx = fabs(D[0]);
  int index = 0;
  const double bb = fabs(D[1]), cc = fabs(D[2]);
  if (bb > mx) mx = bb, index = 1;
  if (cc > mx) mx = cc, index = 2;
  const double vp0 = V0[index], vp1 = V1[index], vp2 = V2[index];
  const double up0 = U0[index], up1 = U1[index], up2 = U2[index];

  double a, b, c, x0, x1, d, e, f, y0, y1;
  if (!intervals(vp0, vp1, vp2, dv0, dv1, dv2, dv0dv1, dv0dv2, a, b, c, x0, x1)) return coplanar_tri_tri(N1, V0, V1, V2, U0, U1, U2);
  if (!intervals(up0, up1, up2, du0, du1, du2, du0du1, du0du2, d, e, f, y0, y1)) return coplanar_tri_tri(N1, V0, V1, V2, U0, U1, U2);
  const double xx = DMUL(x0, x1), yy = DMUL(y0, y1), xxyy = DMUL(xx, yy);
  double tmp = DMUL(a, xxyy);
  double s10 = DADD(tmp, DMUL(DMUL(b, x1), yy)), s11 = DADD(tmp, DMUL(DMUL(c, x0), yy));
  tmp = DMUL(d, xxyy);
  double s20 = DADD(tmp, DMUL(DMUL(e, xx), y1)), s21 = DADD(tmp, DMUL(DMUL(f, xx), y0));
  if (s10 > s11) tmp = s10, s10 = s11, s11 = tmp;
  if (s20 > s21) tmp = s20, s20 = s21, s21 = tmp;
  return !(s11 < s20 || s21 < s10);
}

// TriangleTriangle3d: the six points less their mean, divided per axis by sqrt(sum of squares / 5) + 1e-12.
__device__ bool tri_tri_3d(const double (&p)[6][3]) {
  double q[6][3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    double s = p[0][a];
    for (int k = 1; k < 6; ++k) s = DADD(s, p[k][a]);
    const double mu = __ddiv_rn(s, 6.0);
    double ss = 0.0;
    for (int k = 0; k < 6; ++k) {
      const double d = DSUB(p[k][a], mu);
      ss = k ? DADD(ss, DMUL(d, d)) : DMUL(d, d);
    }
    const double sigma = DADD(__dsqrt_rn(__ddiv_rn(ss, 5.0)), 1e-12);
    for (int k = 0; k < 6; ++k) q[k][a] = __ddiv_rn(DSUB(p[k][a], mu), sigma);
  }
  return no_div_tri_tri(q[0], q[1], q[2], q[3], q[4], q[5]);
}

// One thread per candidate pair p (grid-stride over the device-side total): its cell by an upper bound in the cells'
// pair offsets, its (i < j) inside the cell by the triangular decode, then the tests.  The pair counts only in the cell
// of the minimum corner of the boxes' intersection; out == NULL counts, else keys t0 * nt + t1 go to free slots below
// capacity.
__global__ void __launch_bounds__(256) narrow_kernel(const double* __restrict__ xyz, const long long* __restrict__ tris, int nt,
                                                     const double* __restrict__ box, Grid g, const int* __restrict__ level,
                                                     const unsigned long long* __restrict__ cell_keys, const int* __restrict__ ids,
                                                     const int* __restrict__ start, const long long* __restrict__ pair_off,
                                                     const int* __restrict__ n_cells, const long long* __restrict__ total,
                                                     unsigned long long* __restrict__ found, unsigned long long* __restrict__ out,
                                                     long long capacity) {
  const long long P = *total;
  const int nc = *n_cells, L = *level;
  unsigned long long mine = 0;
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < P; p += (long long)gridDim.x * blockDim.x) {
    const long long c = upper_bound(pair_off, nc, p) - 1;
    const long long q = p - pair_off[c];
    long long j = (long long)((1.0 + sqrt(1.0 + 8.0 * (double)q)) * 0.5);
    while (j * (j - 1) / 2 > q) --j;
    while ((j + 1) * j / 2 <= q) ++j;
    const long long i = q - j * (j - 1) / 2;
    const int s = start[c];
    const int t0 = ids[s + i], t1 = ids[s + j];
    double lo0[3], hi0[3], lo1[3], hi1[3];
    load_box(box, t0, lo0, hi0);
    load_box(box, t1, lo1, hi1);
    bool hit = true;
#pragma unroll
    for (int a = 0; a < 3; ++a) hit = hit && !(hi0[a] < lo1[a] || lo0[a] > hi1[a]);  // Open3D's AABBAABB
    if (!hit) continue;
    const unsigned long long key = cell_keys[s];
    const int cell[3] = {(int)(key >> 42), (int)((key >> 21) & 0x1fffff), (int)(key & 0x1fffff)};
#pragma unroll
    for (int a = 0; a < 3; ++a) hit = hit && cell_of(fmax(lo0[a], lo1[a]), g.o[a], g.extent, L) == cell[a];
    if (!hit) continue;
    long long v0[3], v1[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) v0[k] = tris[3 * (size_t)t0 + k], v1[k] = tris[3 * (size_t)t1 + k];
#pragma unroll
    for (int k = 0; k < 3; ++k) hit = hit && v0[k] != v1[0] && v0[k] != v1[1] && v0[k] != v1[2];
    if (!hit) continue;
    double pts[6][3];
#pragma unroll
    for (int k = 0; k < 3; ++k)
#pragma unroll
      for (int a = 0; a < 3; ++a) pts[k][a] = xyz[3 * v0[k] + a], pts[3 + k][a] = xyz[3 * v1[k] + a];
    if (!tri_tri_3d(pts)) continue;
    if (out) {
      const unsigned long long slot = atomicAdd(found, 1ull);
      if ((long long)slot < capacity) out[slot] = (unsigned long long)t0 * (unsigned long long)nt + (unsigned long long)t1;
    } else {
      ++mine;
    }
  }
  if (!out) {
    using Reduce = cub::BlockReduce<unsigned long long, 256>;
    __shared__ typename Reduce::TempStorage tmp;
    const unsigned long long s = Reduce(tmp).Sum(mine);
    if (threadIdx.x == 0 && s) atomicAdd(found, s);
  }
}

__global__ void __launch_bounds__(256) pairs_expand_kernel(const unsigned long long* __restrict__ keys, long long n, int nt,
                                                           long long* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned long long k = keys[i];
  const bool valid = k < (unsigned long long)nt * (unsigned long long)nt;  // the sentinel marks unfilled slots
  out[2 * i] = valid ? (long long)(k / (unsigned long long)nt) : -1;
  out[2 * i + 1] = valid ? (long long)(k % (unsigned long long)nt) : -1;
}

__global__ void found_kernel(const unsigned long long* __restrict__ found, long long* __restrict__ stats) { stats[0] = (long long)*found; }

// ---------------------------------------------------------------------------------------------------------------------
// Area and volume
// ---------------------------------------------------------------------------------------------------------------------
constexpr int kSumThreads = 256;

// s[0..255] -> s[0]: s[i] = s[i] + s[i + w] for w = 128, 64, ..., 1.
__device__ __forceinline__ void tree_sum(double* s) {
#pragma unroll
  for (int w = kSumThreads / 2; w > 0; w >>= 1) {
    if (threadIdx.x < w) s[threadIdx.x] = DADD(s[threadIdx.x], s[threadIdx.x + w]);
    __syncthreads();
  }
}

// Per triangle: area 0.5 * ||(p0 - p1) x (p0 - p2)||, signed volume p0 . (p1 x p2) / 6 (Eigen's cross and dot); one
// block's 256 terms (0.0 past the last triangle) summed by tree_sum.
__global__ void __launch_bounds__(kSumThreads) area_volume_terms_kernel(const double* __restrict__ xyz, const long long* __restrict__ tris,
                                                                         int nt, double* __restrict__ partial) {
  __shared__ double sa[kSumThreads], sv[kSumThreads];
  const int t = blockIdx.x * kSumThreads + threadIdx.x;
  double area = 0.0, vol = 0.0;
  if (t < nt) {
    const long long i0 = tris[3 * (size_t)t], i1 = tris[3 * (size_t)t + 1], i2 = tris[3 * (size_t)t + 2];
    double p0[3], p1[3], p2[3], x[3], y[3], c[3];
    for (int a = 0; a < 3; ++a) p0[a] = xyz[3 * i0 + a], p1[a] = xyz[3 * i1 + a], p2[a] = xyz[3 * i2 + a];
    for (int a = 0; a < 3; ++a) x[a] = DSUB(p0[a], p1[a]), y[a] = DSUB(p0[a], p2[a]);
    cross3(c, x, y);
    area = DMUL(0.5, __dsqrt_rn(dot3(c, c)));
    cross3(c, p1, p2);
    vol = __ddiv_rn(dot3(p0, c), 6.0);
  }
  sa[threadIdx.x] = area;
  sv[threadIdx.x] = vol;
  __syncthreads();
  tree_sum(sa);
  tree_sum(sv);
  if (threadIdx.x == 0) {
    partial[2 * (size_t)blockIdx.x] = sa[0];
    partial[2 * (size_t)blockIdx.x + 1] = sv[0];
  }
}

// One block: thread i adds partials i, i + 256, ... from 0.0 in order, then tree_sum.
__global__ void __launch_bounds__(kSumThreads) area_volume_final_kernel(const double* __restrict__ partial, int n_blocks,
                                                                         double* __restrict__ out) {
  __shared__ double sa[kSumThreads], sv[kSumThreads];
  double a = 0.0, v = 0.0;
  for (int i = threadIdx.x; i < n_blocks; i += kSumThreads) {
    a = DADD(a, partial[2 * (size_t)i]);
    v = DADD(v, partial[2 * (size_t)i + 1]);
  }
  sa[threadIdx.x] = a;
  sv[threadIdx.x] = v;
  __syncthreads();
  tree_sum(sa);
  tree_sum(sv);
  if (threadIdx.x == 0) out[0] = sa[0], out[1] = sv[0];
}

// ---------------------------------------------------------------------------------------------------------------------
// Workspaces (a NULL base gives only `total`)
// ---------------------------------------------------------------------------------------------------------------------
struct EdgeWork {
  unsigned long long* keys;  // [2][3 nt]
  int* val;                  // [2][3 nt]
  int *parent, *head, *run_id, *start, *bad, *pos, *n_runs, *conflict;  // [2 nt], [3 nt] x2, [3 nt + 1], [3 nt] x2, [1], [1]
  void* tmp;
  size_t tmp_bytes, total;
};

EdgeWork carve_edges(void* base, int64_t nt) {
  const long long n3 = 3 * nt;
  size_t a = 0, b = 0;
  cub::DoubleBuffer<unsigned long long> k(nullptr, nullptr);
  cub::DoubleBuffer<int> v(nullptr, nullptr);
  cub::DeviceRadixSort::SortPairs(nullptr, a, k, v, n3);
  cub::DeviceScan::InclusiveSum(nullptr, b, (int*)nullptr, (int*)nullptr, n3);
  Carver c(base);
  EdgeWork w;
  w.keys = c.take<unsigned long long>(2 * (size_t)n3);
  w.val = c.take<int>(2 * (size_t)n3);
  w.parent = c.take<int>(2 * (size_t)nt);
  w.head = c.take<int>((size_t)n3);
  w.run_id = c.take<int>((size_t)n3);
  w.start = c.take<int>((size_t)n3 + 1);
  w.bad = c.take<int>((size_t)n3);
  w.pos = c.take<int>((size_t)n3);
  w.n_runs = c.take<int>(1);
  w.conflict = c.take<int>(1);
  w.tmp_bytes = a > b ? a : b;
  w.tmp = c.take<char>(w.tmp_bytes);
  w.total = c.total();
  return w;
}

struct VertexWork {
  unsigned long long* keys;  // [2][6 nt]
  int* slot;                 // [2][6 nt]
  int *head, *rank, *node_of, *node_vertex, *parent, *n_nodes;  // [6 nt] x5, [1]
  int *roots, *bad, *pos;                                        // [nv] x3
  void* tmp;
  size_t tmp_bytes, total;
};

VertexWork carve_vertices(void* base, int64_t nt, int64_t nv) {
  const long long n6 = 6 * nt;
  size_t a = 0, b = 0, d = 0;
  cub::DoubleBuffer<unsigned long long> k(nullptr, nullptr);
  cub::DoubleBuffer<int> v(nullptr, nullptr);
  cub::DeviceRadixSort::SortPairs(nullptr, a, k, v, n6);
  cub::DeviceScan::InclusiveSum(nullptr, b, (int*)nullptr, (int*)nullptr, n6);
  cub::DeviceScan::ExclusiveSum(nullptr, d, (int*)nullptr, (int*)nullptr, (long long)nv);
  Carver c(base);
  VertexWork w;
  w.keys = c.take<unsigned long long>(2 * (size_t)n6);
  w.slot = c.take<int>(2 * (size_t)n6);
  w.head = c.take<int>((size_t)n6);
  w.rank = c.take<int>((size_t)n6);
  w.node_of = c.take<int>((size_t)n6);
  w.node_vertex = c.take<int>((size_t)n6);
  w.parent = c.take<int>((size_t)n6);
  w.n_nodes = c.take<int>(1);
  w.roots = c.take<int>((size_t)nv);
  w.bad = c.take<int>((size_t)nv);
  w.pos = c.take<int>((size_t)nv);
  w.tmp_bytes = a > b ? a : b;
  w.tmp_bytes = d > w.tmp_bytes ? d : w.tmp_bytes;
  w.tmp = c.take<char>(w.tmp_bytes);
  w.total = c.total();
  return w;
}

struct IsectWork {
  double* box;                      // [6 nt]
  unsigned long long* level_regs;   // [kLevels]
  int *level, *reg_count, *reg_off;  // [1], [nt], [nt]
  unsigned long long* cell_keys;    // [2][cap]
  int *ids, *head, *cell_id, *start, *n_cells;  // [2][cap], [cap], [cap], [cap + 1], [1]
  long long *pairs, *pair_off, *total;           // [cap], [cap], [1]
  unsigned long long* found;                     // [1]
  unsigned long long* out_keys;                  // [2][capacity]
  void* tmp;
  size_t tmp_bytes, total_bytes;
};

IsectWork carve_isect(void* base, int64_t nt, int64_t capacity) {
  const long long cap = kRegsPerTriangle * nt;
  size_t a = 0, b = 0, d = 0, e = 0, f = 0;
  cub::DoubleBuffer<unsigned long long> k(nullptr, nullptr);
  cub::DoubleBuffer<int> v(nullptr, nullptr);
  cub::DeviceRadixSort::SortPairs(nullptr, a, k, v, cap);
  cub::DeviceScan::ExclusiveSum(nullptr, b, (int*)nullptr, (int*)nullptr, (long long)nt);
  cub::DeviceScan::InclusiveSum(nullptr, d, (int*)nullptr, (int*)nullptr, cap);
  cub::DeviceScan::ExclusiveSum(nullptr, e, (long long*)nullptr, (long long*)nullptr, cap);
  cub::DeviceRadixSort::SortKeys(nullptr, f, k, (long long)capacity);
  Carver c(base);
  IsectWork w;
  w.box = c.take<double>(6 * (size_t)nt);
  w.level_regs = c.take<unsigned long long>(kLevels);
  w.level = c.take<int>(1);
  w.reg_count = c.take<int>((size_t)nt);
  w.reg_off = c.take<int>((size_t)nt);
  w.cell_keys = c.take<unsigned long long>(2 * (size_t)cap);
  w.ids = c.take<int>(2 * (size_t)cap);
  w.head = c.take<int>((size_t)cap);
  w.cell_id = c.take<int>((size_t)cap);
  w.start = c.take<int>((size_t)cap + 1);
  w.n_cells = c.take<int>(1);
  w.pairs = c.take<long long>((size_t)cap);
  w.pair_off = c.take<long long>((size_t)cap);
  w.total = c.take<long long>(1);
  w.found = c.take<unsigned long long>(1);
  w.out_keys = c.take<unsigned long long>(2 * (size_t)capacity);
  w.tmp_bytes = a;
  for (size_t x : {b, d, e, f}) w.tmp_bytes = x > w.tmp_bytes ? x : w.tmp_bytes;
  w.tmp = c.take<char>(w.tmp_bytes);
  w.total_bytes = c.total();
  return w;
}

size_t area_volume_bytes(int64_t nt) { return align_up(2 * sizeof(double) * (size_t)blocks_for(nt, kSumThreads), 256); }

}  // namespace
}  // namespace gsb

using namespace gsb;

extern "C" {

size_t gsb_mesh_edge_topology_workspace_bytes(int64_t n_triangles, int64_t n_vertices) {
  if (!mesh_sizes_ok(n_triangles, n_vertices, kMaxTopoTriangles)) return 0;
  return carve_edges(nullptr, n_triangles).total;
}

int gsb_mesh_edge_topology(const int64_t* triangles, int64_t n_triangles, int64_t n_vertices, int allow_boundary_edges,
                           void* workspace, size_t workspace_bytes, int64_t* out_edges, int64_t* sizes, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (!mesh_sizes_ok(n_triangles, n_vertices, kMaxTopoTriangles))
    return mesh_size_error("mesh_edge_topology", n_triangles, n_vertices, kMaxTopoTriangles);
  if (!sizes || (n_triangles && (!triangles || !workspace))) return fail(GSB_ERR_INVALID, "mesh_edge_topology: bad arguments");
  const size_t need = gsb_mesh_edge_topology_workspace_bytes(n_triangles, n_vertices);
  if (n_triangles && workspace_bytes < need)
    return fail(GSB_ERR_WORKSPACE, "mesh_edge_topology: workspace %zu < %zu bytes", workspace_bytes, need);
  if (n_triangles == 0) {  // no edges, orientable
    edge_sizes_empty_kernel<<<1, 1, 0, stream>>>(reinterpret_cast<long long*>(sizes));
    count_launch();
    return check_launch("mesh_edge_topology", stream, false);
  }
  const int nt = (int)n_triangles;
  const long long n3 = 3 * (long long)nt;
  const EdgeWork w = carve_edges(workspace, n_triangles);
  const auto* tris = reinterpret_cast<const long long*>(triangles);
  const unsigned long long stride = (unsigned long long)n_vertices + 1;
  const unsigned long long sentinel = stride * stride;  // above every key; never produced here
  GSB_CUDA_OK(cudaMemsetAsync(w.conflict, 0, sizeof(int), stream));
  edge_incidence_kernel<<<blocks_for(nt), 256, 0, stream>>>(tris, nt, stride, w.keys, w.val, w.parent);
  count_launch();
  cub::DoubleBuffer<unsigned long long> keys(w.keys, w.keys + n3);
  cub::DoubleBuffer<int> val(w.val, w.val + n3);
  size_t tmp_bytes = w.tmp_bytes;
  GSB_CUDA_OK(cub::DeviceRadixSort::SortPairs(w.tmp, tmp_bytes, keys, val, n3, 0, bits_of(stride * stride - 1), stream));
  run_head_kernel<<<blocks_for(n3), 256, 0, stream>>>(keys.Current(), n3, sentinel, w.head);
  count_launch();
  tmp_bytes = w.tmp_bytes;
  GSB_CUDA_OK(cub::DeviceScan::InclusiveSum(w.tmp, tmp_bytes, w.head, w.run_id, n3, stream));
  run_start_kernel<<<blocks_for(n3), 256, 0, stream>>>(w.head, w.run_id, n3, keys.Current(), sentinel, w.start, w.n_runs);
  count_launch();
  orient_union_kernel<<<blocks_for(n3), 256, 0, stream>>>(keys.Current(), val.Current(), w.head, w.run_id, w.start, n3, stride,
                                                          w.parent);
  count_launch();
  orient_check_kernel<<<blocks_for(nt), 256, 0, stream>>>(w.parent, nt, w.conflict);
  count_launch();
  edge_flag_kernel<<<blocks_for(n3), 256, 0, stream>>>(w.start, w.n_runs, n3, allow_boundary_edges != 0, w.bad);
  count_launch();
  tmp_bytes = w.tmp_bytes;
  GSB_CUDA_OK(cub::DeviceScan::ExclusiveSum(w.tmp, tmp_bytes, w.bad, w.pos, n3, stream));
  if (out_edges) {
    edge_emit_kernel<<<blocks_for(n3), 256, 0, stream>>>(keys.Current(), w.start, w.n_runs, w.bad, w.pos, n3, stride,
                                                         reinterpret_cast<long long*>(out_edges));
    count_launch();
  }
  edge_sizes_kernel<<<1, 1, 0, stream>>>(w.bad, w.pos, w.n_runs, w.conflict, reinterpret_cast<long long*>(sizes));
  count_launch();
  return check_launch("mesh_edge_topology", stream, false);
}

size_t gsb_mesh_vertex_topology_workspace_bytes(int64_t n_triangles, int64_t n_vertices) {
  if (!mesh_sizes_ok(n_triangles, n_vertices, kMaxTopoTriangles)) return 0;
  return carve_vertices(nullptr, n_triangles, n_vertices).total;
}

int gsb_mesh_non_manifold_vertices(const int64_t* triangles, int64_t n_triangles, int64_t n_vertices, void* workspace,
                                   size_t workspace_bytes, int64_t* out_vertices, int64_t* count, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (!mesh_sizes_ok(n_triangles, n_vertices, kMaxTopoTriangles))
    return mesh_size_error("mesh_non_manifold_vertices", n_triangles, n_vertices, kMaxTopoTriangles);
  if (!count || (n_triangles && (!triangles || !workspace)))
    return fail(GSB_ERR_INVALID, "mesh_non_manifold_vertices: bad arguments");
  const size_t need = gsb_mesh_vertex_topology_workspace_bytes(n_triangles, n_vertices);
  if (n_triangles && workspace_bytes < need)
    return fail(GSB_ERR_WORKSPACE, "mesh_non_manifold_vertices: workspace %zu < %zu bytes", workspace_bytes, need);
  if (n_triangles == 0) {
    GSB_CUDA_OK(cudaMemsetAsync(count, 0, sizeof(int64_t), stream));
    return GSB_OK;
  }
  const int nt = (int)n_triangles, nv = (int)n_vertices;
  const long long n6 = 6 * (long long)nt;
  const VertexWork w = carve_vertices(workspace, n_triangles, n_vertices);
  const auto* tris = reinterpret_cast<const long long*>(triangles);
  const unsigned long long unv = (unsigned long long)nv, sentinel = unv * unv;
  link_edge_kernel<<<blocks_for(nt), 256, 0, stream>>>(tris, nt, unv, w.keys, w.slot);
  count_launch();
  cub::DoubleBuffer<unsigned long long> keys(w.keys, w.keys + n6);
  cub::DoubleBuffer<int> slot(w.slot, w.slot + n6);
  size_t tmp_bytes = w.tmp_bytes;
  GSB_CUDA_OK(cub::DeviceRadixSort::SortPairs(w.tmp, tmp_bytes, keys, slot, n6, 0, bits_of(sentinel), stream));
  run_head_kernel<<<blocks_for(n6), 256, 0, stream>>>(keys.Current(), n6, sentinel, w.head);
  count_launch();
  tmp_bytes = w.tmp_bytes;
  GSB_CUDA_OK(cub::DeviceScan::InclusiveSum(w.tmp, tmp_bytes, w.head, w.rank, n6, stream));
  run_start_kernel<<<blocks_for(n6), 256, 0, stream>>>(w.head, w.rank, n6, keys.Current(), sentinel, nullptr, w.n_nodes);
  count_launch();
  link_nodes_kernel<<<blocks_for(n6), 256, 0, stream>>>(keys.Current(), slot.Current(), w.head, w.rank, n6, unv, w.node_of,
                                                        w.node_vertex, w.parent);
  count_launch();
  link_union_kernel<<<blocks_for(3 * (long long)nt), 256, 0, stream>>>(w.node_of, 3 * (long long)nt, w.parent);
  count_launch();
  GSB_CUDA_OK(cudaMemsetAsync(w.roots, 0, sizeof(int) * (size_t)nv, stream));
  link_roots_kernel<<<blocks_for(n6), 256, 0, stream>>>(w.parent, w.node_vertex, w.n_nodes, n6, w.roots);
  count_launch();
  vertex_flag_kernel<<<blocks_for(nv), 256, 0, stream>>>(w.roots, nv, w.bad);
  count_launch();
  tmp_bytes = w.tmp_bytes;
  GSB_CUDA_OK(cub::DeviceScan::ExclusiveSum(w.tmp, tmp_bytes, w.bad, w.pos, (long long)nv, stream));
  vertex_emit_kernel<<<blocks_for(nv), 256, 0, stream>>>(w.bad, w.pos, nv, reinterpret_cast<long long*>(out_vertices),
                                                         reinterpret_cast<long long*>(count));
  count_launch();
  return check_launch("mesh_non_manifold_vertices", stream, false);
}

size_t gsb_mesh_self_intersections_workspace_bytes(int64_t n_triangles, int64_t n_vertices, int64_t capacity) {
  if (!mesh_sizes_ok(n_triangles, n_vertices, kMaxTopoTriangles) || capacity < 0 || capacity > n_triangles * (n_triangles - 1) / 2)
    return 0;
  return carve_isect(nullptr, n_triangles, capacity).total_bytes;
}

int gsb_mesh_self_intersections(const double* vertices, int64_t n_vertices, const int64_t* triangles, int64_t n_triangles,
                                const double* min_bound, const double* max_bound, void* workspace, size_t workspace_bytes,
                                int64_t* out_pairs, int64_t capacity, int64_t* stats, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  const char* who = "mesh_self_intersections";
  if (!mesh_sizes_ok(n_triangles, n_vertices, kMaxTopoTriangles))
    return mesh_size_error(who, n_triangles, n_vertices, kMaxTopoTriangles);
  if (capacity < 0 || capacity > n_triangles * (n_triangles - 1) / 2)
    return fail(GSB_ERR_INVALID, "%s: capacity %lld outside [0, n_triangles (n_triangles - 1) / 2]", who, (long long)capacity);
  if (!stats || (n_triangles && (!vertices || !triangles || !workspace || !min_bound || !max_bound)) || (capacity && !out_pairs))
    return fail(GSB_ERR_INVALID, "%s: bad arguments", who);
  for (int a = 0; a < 3 && n_triangles; ++a)
    if (!isfinite(min_bound[a]) || !isfinite(max_bound[a]) || !(min_bound[a] <= max_bound[a]))
      return fail(GSB_ERR_INVALID, "%s: the vertex bounds are not finite", who);
  const size_t need = gsb_mesh_self_intersections_workspace_bytes(n_triangles, n_vertices, capacity);
  if (n_triangles && workspace_bytes < need) return fail(GSB_ERR_WORKSPACE, "%s: workspace %zu < %zu bytes", who, workspace_bytes, need);
  if (n_triangles == 0) {
    GSB_CUDA_OK(cudaMemsetAsync(stats, 0, 4 * sizeof(int64_t), stream));
    return GSB_OK;
  }
  const int nt = (int)n_triangles;
  const long long cap = kRegsPerTriangle * (long long)nt;
  const IsectWork w = carve_isect(workspace, n_triangles, capacity);
  const auto* tris = reinterpret_cast<const long long*>(triangles);
  auto* st = reinterpret_cast<long long*>(stats);
  Grid g;
  g.extent = 0.0;
  for (int a = 0; a < 3; ++a) {
    g.o[a] = min_bound[a];
    const double e = max_bound[a] - min_bound[a];
    g.extent = e > g.extent ? e : g.extent;
  }
  if (!(g.extent > 0.0) || !isfinite(g.extent)) g.extent = 1.0;

  GSB_CUDA_OK(cudaMemsetAsync(w.level_regs, 0, kLevels * sizeof(unsigned long long), stream));
  GSB_CUDA_OK(cudaMemsetAsync(w.found, 0, sizeof(unsigned long long), stream));
  box_kernel<<<blocks_for(nt), 256, 0, stream>>>(vertices, tris, nt, g, w.box, w.level_regs);
  count_launch();
  choose_level_kernel<<<1, 1, 0, stream>>>(w.level_regs, nt, w.level, st);
  count_launch();
  reg_count_kernel<<<blocks_for(nt), 256, 0, stream>>>(w.box, nt, g, w.level, w.reg_count);
  count_launch();
  size_t tmp_bytes = w.tmp_bytes;
  GSB_CUDA_OK(cub::DeviceScan::ExclusiveSum(w.tmp, tmp_bytes, w.reg_count, w.reg_off, (long long)nt, stream));
  reg_fill_kernel<<<blocks_for(cap), 256, 0, stream>>>(w.box, nt, g, w.level, w.reg_off, w.reg_count, cap, w.cell_keys, w.ids);
  count_launch();
  cub::DoubleBuffer<unsigned long long> keys(w.cell_keys, w.cell_keys + cap);
  cub::DoubleBuffer<int> ids(w.ids, w.ids + cap);
  tmp_bytes = w.tmp_bytes;
  GSB_CUDA_OK(cub::DeviceRadixSort::SortPairs(w.tmp, tmp_bytes, keys, ids, cap, 0, 64, stream));
  run_head_kernel<<<blocks_for(cap), 256, 0, stream>>>(keys.Current(), cap, ~0ull, w.head);
  count_launch();
  tmp_bytes = w.tmp_bytes;
  GSB_CUDA_OK(cub::DeviceScan::InclusiveSum(w.tmp, tmp_bytes, w.head, w.cell_id, cap, stream));
  run_start_kernel<<<blocks_for(cap), 256, 0, stream>>>(w.head, w.cell_id, cap, keys.Current(), ~0ull, w.start, w.n_cells);
  count_launch();
  cell_pairs_kernel<<<blocks_for(cap), 256, 0, stream>>>(w.start, w.n_cells, cap, w.pairs);
  count_launch();
  tmp_bytes = w.tmp_bytes;
  GSB_CUDA_OK(cub::DeviceScan::ExclusiveSum(w.tmp, tmp_bytes, w.pairs, w.pair_off, cap, stream));
  pair_total_kernel<<<1, 1, 0, stream>>>(w.pair_off, w.pairs, w.n_cells, st, w.total);
  count_launch();
  unsigned long long* out_keys = out_pairs ? w.out_keys : nullptr;
  if (out_keys) {
    // unfilled slots keep a key above every pair's, so they sort last
    GSB_CUDA_OK(cudaMemsetAsync(out_keys, 0xff, (size_t)capacity * sizeof(unsigned long long), stream));
  }
  narrow_kernel<<<kNarrowBlocks, 256, 0, stream>>>(vertices, tris, nt, w.box, g, w.level, keys.Current(), ids.Current(), w.start,
                                                   w.pair_off, w.n_cells, w.total, w.found, out_keys, capacity);
  count_launch();
  found_kernel<<<1, 1, 0, stream>>>(w.found, st);
  count_launch();
  if (out_keys) {
    cub::DoubleBuffer<unsigned long long> pk(out_keys, out_keys + capacity);
    tmp_bytes = w.tmp_bytes;
    GSB_CUDA_OK(cub::DeviceRadixSort::SortKeys(w.tmp, tmp_bytes, pk, capacity, 0, 64, stream));
    pairs_expand_kernel<<<blocks_for(capacity), 256, 0, stream>>>(pk.Current(), capacity, nt, reinterpret_cast<long long*>(out_pairs));
    count_launch();
  }
  return check_launch(who, stream, false);
}

size_t gsb_mesh_area_volume_workspace_bytes(int64_t n_triangles, int64_t n_vertices) {
  if (!mesh_sizes_ok(n_triangles, n_vertices, kMaxTopoTriangles)) return 0;
  return area_volume_bytes(n_triangles);
}

int gsb_mesh_area_volume(const double* vertices, int64_t n_vertices, const int64_t* triangles, int64_t n_triangles,
                         void* workspace, size_t workspace_bytes, double* out, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (!mesh_sizes_ok(n_triangles, n_vertices, kMaxTopoTriangles))
    return mesh_size_error("mesh_area_volume", n_triangles, n_vertices, kMaxTopoTriangles);
  if (!out || (n_triangles && (!vertices || !triangles || !workspace))) return fail(GSB_ERR_INVALID, "mesh_area_volume: bad arguments");
  const size_t need = gsb_mesh_area_volume_workspace_bytes(n_triangles, n_vertices);
  if (n_triangles && workspace_bytes < need)
    return fail(GSB_ERR_WORKSPACE, "mesh_area_volume: workspace %zu < %zu bytes", workspace_bytes, need);
  if (n_triangles == 0) {
    GSB_CUDA_OK(cudaMemsetAsync(out, 0, 2 * sizeof(double), stream));
    return GSB_OK;
  }
  const int nt = (int)n_triangles;
  const int nb = (int)blocks_for(nt, kSumThreads);
  auto* partial = static_cast<double*>(workspace);
  area_volume_terms_kernel<<<nb, kSumThreads, 0, stream>>>(vertices, reinterpret_cast<const long long*>(triangles), nt, partial);
  count_launch();
  area_volume_final_kernel<<<1, kSumThreads, 0, stream>>>(partial, nb, out);
  count_launch();
  return check_launch("mesh_area_volume", stream, false);
}

}  // extern "C"
