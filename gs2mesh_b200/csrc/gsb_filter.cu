// Mesh smoothing and sharpening: Open3D 0.17.0 TriangleMesh::FilterSmoothSimple, FilterSmoothLaplacian,
// FilterSmoothTaubin and FilterSharpen (DESIGN.md section 7, "Smoothing and sharpening"; restated in
// tests/filter_oracle.py).
//
// One thread per vertex walks its CSR run of neighbours in ascending id and filters every attribute of the pass in one
// sweep (the Laplacian weights are computed once and shared).  Passes are Jacobi style: each reads only the previous
// pass's arrays.  The entry enqueues every pass, ping-ponging between the caller's output arrays and one workspace copy
// per attribute so that the last pass lands in the output; the inputs are never written.
//
// Every fp64 operation is an explicit __d*_rn in the restatement's order, so nvcc contracts nothing.  No atomics: every
// run writes the same bytes.
#include "gs2mesh_b200.h"
#include "gsb_common.h"

namespace gsb {
namespace {

constexpr double kWeightEps = 1e-12;  // Open3D's 1 / (|p_v - p_u| + 1e-12)

enum FilterOp { kOpSimple = 0, kOpLaplacian = 1, kOpSharpen = 2 };

// The attributes one pass filters: position, colour, normal.  src[a] == NULL: attribute a is not filtered.
struct FilterPass {
  const double* src[3];
  double* dst[3];
  const double* weight_xyz;  // the positions the Laplacian weights come from: this pass's input positions
};

// One pass over vertex v's neighbours N(v) (CSR run [off[v], off[v+1]), ascending ids):
//   simple     x' = (x + sum_u x_u) / double(1 + deg)
//   laplacian  w_u = 1 / (sqrt((dx^2 + dy^2) + dz^2) + 1e-12), d = p_v - p_u; x' = x + param * (sum_u (w_u x_u) / sum_u w_u - x);
//              a vertex without neighbours keeps x
//   sharpen    x' = x + param * sum_u (x - x_u)
// Sums start from 0.0 and add in ascending neighbour id.
template <int Op>
__global__ void __launch_bounds__(256) filter_pass_kernel(const long long* __restrict__ off, const long long* __restrict__ nb,
                                                          int nv, FilterPass f, double param) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= nv) return;
  const long long begin = off[v], end = off[v + 1];
  double x[3][3], s[3][3];
#pragma unroll
  for (int a = 0; a < 3; ++a)
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      x[a][c] = f.src[a] ? f.src[a][3 * (size_t)v + c] : 0.0;
      s[a][c] = 0.0;
    }
  double p[3] = {0.0, 0.0, 0.0}, wsum = 0.0;
  if (Op == kOpLaplacian)
#pragma unroll
    for (int c = 0; c < 3; ++c) p[c] = f.weight_xyz[3 * (size_t)v + c];
  for (long long k = begin; k < end; ++k) {
    const size_t u = (size_t)nb[k];
    double w = 0.0;
    if (Op == kOpLaplacian) {
      const double dx = __dsub_rn(p[0], f.weight_xyz[3 * u]), dy = __dsub_rn(p[1], f.weight_xyz[3 * u + 1]),
                   dz = __dsub_rn(p[2], f.weight_xyz[3 * u + 2]);
      const double dist = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz)));
      w = __ddiv_rn(1.0, __dadd_rn(dist, kWeightEps));
      wsum = __dadd_rn(wsum, w);
    }
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      if (!f.src[a]) continue;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const double xu = f.src[a][3 * u + c];
        const double term = Op == kOpSimple ? xu : Op == kOpLaplacian ? __dmul_rn(w, xu) : __dsub_rn(x[a][c], xu);
        s[a][c] = __dadd_rn(s[a][c], term);
      }
    }
  }
  const double count = (double)(1 + (end - begin));
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    if (!f.src[a]) continue;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      double y;
      if (Op == kOpSimple)
        y = __ddiv_rn(__dadd_rn(x[a][c], s[a][c]), count);
      else if (Op == kOpLaplacian)
        y = end == begin ? x[a][c] : __dadd_rn(x[a][c], __dmul_rn(param, __dsub_rn(__ddiv_rn(s[a][c], wsum), x[a][c])));
      else
        y = __dadd_rn(x[a][c], __dmul_rn(param, s[a][c]));
      f.dst[a][3 * (size_t)v + c] = y;
    }
  }
}

bool filter_sizes_ok(int64_t nv) { return nv >= 0 && nv <= kMaxMeshIds; }

struct FilterWork {
  double* xyz[3];  // [3 nv] per attribute (position, colour, normal), NULL for an absent colour or normal
  size_t total;
};

FilterWork carve_filter(void* base, int64_t nv, bool with_colors, bool with_normals) {
  Carver c(base);
  FilterWork w;
  w.xyz[0] = c.take<double>(3 * (size_t)nv);
  w.xyz[1] = with_colors ? c.take<double>(3 * (size_t)nv) : nullptr;
  w.xyz[2] = with_normals ? c.take<double>(3 * (size_t)nv) : nullptr;
  w.total = c.total();
  return w;
}

}  // namespace
}  // namespace gsb

using namespace gsb;

extern "C" {

size_t gsb_mesh_filter_workspace_bytes(int64_t n_vertices, int with_colors, int with_normals) {
  if (!filter_sizes_ok(n_vertices)) return 0;
  return carve_filter(nullptr, n_vertices, with_colors != 0, with_normals != 0).total;
}

int gsb_mesh_filter(int kind, const double* vertices, const double* colors, const double* normals, int64_t n_vertices,
                    const int64_t* adjacency_offsets, const int64_t* neighbours, int32_t iterations, double param0,
                    double param1, int scope, void* workspace, size_t workspace_bytes, double* out_vertices, double* out_colors,
                    double* out_normals, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (kind < GSB_FILTER_SIMPLE || kind > GSB_FILTER_SHARPEN) return fail(GSB_ERR_INVALID, "mesh_filter: unknown kind %d", kind);
  if (scope < GSB_FILTER_SCOPE_ALL || scope > GSB_FILTER_SCOPE_VERTEX)
    return fail(GSB_ERR_INVALID, "mesh_filter: unknown scope %d", scope);
  if (iterations < 0) return fail(GSB_ERR_INVALID, "mesh_filter: iterations %d < 0", (int)iterations);
  if (!filter_sizes_ok(n_vertices))
    return fail(GSB_ERR_INVALID, "mesh_filter: %lld vertices; ids are 32-bit (at least 0 and at most %lld)",
                (long long)n_vertices, (long long)kMaxMeshIds);
  if ((!colors && out_colors) || (!normals && out_normals))
    return fail(GSB_ERR_INVALID, "mesh_filter: an output colour or normal array without its input");
  // neighbours may be NULL: a mesh without triangles has none, and only the offsets say so
  if (n_vertices && (!vertices || !out_vertices || !adjacency_offsets || !workspace || (colors && !out_colors) ||
                     (normals && !out_normals)))
    return fail(GSB_ERR_INVALID, "mesh_filter: bad arguments");
  const size_t need = gsb_mesh_filter_workspace_bytes(n_vertices, colors != nullptr, normals != nullptr);
  if (n_vertices && workspace_bytes < need)
    return fail(GSB_ERR_WORKSPACE, "mesh_filter: workspace %zu < %zu bytes", workspace_bytes, need);
  if (n_vertices == 0) return GSB_OK;

  const int nv = (int)n_vertices;
  const size_t bytes = 3 * sizeof(double) * (size_t)nv;
  const FilterWork w = carve_filter(workspace, n_vertices, colors != nullptr, normals != nullptr);
  const double* in[3] = {vertices, colors, normals};
  double* out[3] = {out_vertices, out_colors, out_normals};
  // FilterScope: positions for All and Vertex, colours for All and Color, normals for All and Normal
  const bool filtered[3] = {scope == GSB_FILTER_SCOPE_ALL || scope == GSB_FILTER_SCOPE_VERTEX,
                            colors && (scope == GSB_FILTER_SCOPE_ALL || scope == GSB_FILTER_SCOPE_COLOR),
                            normals && (scope == GSB_FILTER_SCOPE_ALL || scope == GSB_FILTER_SCOPE_NORMAL)};
  const long long passes = (long long)iterations * (kind == GSB_FILTER_TAUBIN ? 2 : 1);
  for (int a = 0; a < 3; ++a)
    if (in[a] && (!filtered[a] || passes == 0)) GSB_CUDA_OK(cudaMemcpyAsync(out[a], in[a], bytes, cudaMemcpyDeviceToDevice, stream));

  const auto* off = reinterpret_cast<const long long*>(adjacency_offsets);
  const auto* nb = reinterpret_cast<const long long*>(neighbours);
  const double* cur[3] = {vertices, colors, normals};
  for (long long k = 0; k < passes; ++k) {
    // pass k writes the output when passes - 1 - k is even, so the last pass always does
    const bool to_out = (passes - 1 - k) % 2 == 0;
    FilterPass f;
    for (int a = 0; a < 3; ++a) {
      f.src[a] = filtered[a] ? cur[a] : nullptr;
      f.dst[a] = filtered[a] ? (to_out ? out[a] : w.xyz[a]) : nullptr;
    }
    f.weight_xyz = cur[0];  // the input positions when positions are not filtered
    if (kind == GSB_FILTER_SIMPLE)
      filter_pass_kernel<kOpSimple><<<blocks_for(nv), 256, 0, stream>>>(off, nb, nv, f, 0.0);
    else if (kind == GSB_FILTER_SHARPEN)
      filter_pass_kernel<kOpSharpen><<<blocks_for(nv), 256, 0, stream>>>(off, nb, nv, f, param0);
    else  // Laplacian with param0; Taubin alternates param0 (lambda) and param1 (mu)
      filter_pass_kernel<kOpLaplacian><<<blocks_for(nv), 256, 0, stream>>>(off, nb, nv, f,
                                                                          kind == GSB_FILTER_TAUBIN && k % 2 ? param1 : param0);
    count_launch();
    for (int a = 0; a < 3; ++a)
      if (filtered[a]) cur[a] = f.dst[a];
  }
  return check_launch("mesh_filter", stream, false);
}

}  // extern "C"
