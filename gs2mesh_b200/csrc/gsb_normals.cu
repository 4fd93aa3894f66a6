// Exact k nearest neighbours on the shared point grid, and Open3D 0.17's PointCloud::EstimateNormals with
// KDTreeSearchParamKNN(k) and fast_normal_computation (ComputeCovariance, FastEigen3x3) for a cloud without normals: the
// Tanks and Temples toolbox's estimate_normals (evaluation.py:60-84).  Open3D 0.17's PointCloud::RemoveStatisticalOutliers
// and RemoveRadiusOutliers on the same grid (DESIGN.md section 7, "Point-cloud cleaning and downsampling"), and its
// PointCloud::ClusterDBSCAN (DESIGN.md section 7, "Density clustering").
//
// Every fp64 operation carries an explicit rounding intrinsic, so nvcc cannot contract a multiply-add into an FMA, and
// acos / cos are fdlibm's algorithms in those operations rather than the device's libm: tests/normals_oracle.py restates
// the same operations in numpy and the results compare bit for bit.
#include <cub/cub.cuh>

#include "gs2mesh_b200.h"
#include "gsb_common.h"
#include "gsb_grid.cuh"
#include "gsb_union_find.cuh"

namespace gsb {
namespace {

constexpr int kMaxK = GSB_KNN_MAX_K;

__device__ __forceinline__ double add(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double sub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double mul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double quo(double a, double b) { return __ddiv_rn(a, b); }

// (d2, id) before (d2b, idb) in ascending (d2, index) order
__device__ __forceinline__ bool before(double d2, long long id, double d2b, long long idb) {
  return d2 < d2b || (d2 == d2b && id < idb);
}

// The k nearest grid points of (qx, qy, qz) in ascending (d2, index) order into d2s / ids; returns how many (min(k,
// n_points), 0 for a query with a non-finite coordinate).  The rings of walk_rings stop once k points are held and the
// k-th d2 is below the next ring's bound: every later point is then strictly farther, so no tie at the k-th place is
// missed.
__device__ __forceinline__ int ring_knn(const GsbPointGrid& g, double qx, double qy, double qz, int k, double* d2s,
                                        long long* ids) {
  if (!(isfinite(qx) && isfinite(qy) && isfinite(qz))) return 0;
  int n = 0;
  walk_rings(
      g, qx, qy, qz, INFINITY, [&](double lb) { return n == k && d2s[k - 1] < lb * lb; },
      [&](long long id) {
        const double d2 = sq_dist(qx, qy, qz, g.points + 3 * id);
        if (n == k && !before(d2, id, d2s[k - 1], ids[k - 1])) return;
        int j = n < k ? n++ : k - 1;
        for (; j > 0 && before(d2, id, d2s[j - 1], ids[j - 1]); --j) {
          d2s[j] = d2s[j - 1];
          ids[j] = ids[j - 1];
        }
        d2s[j] = d2;
        ids[j] = id;
      });
  return n;
}

__global__ void __launch_bounds__(128, 4) knn_kernel(const GsbPointGrid g, const double* __restrict__ q, long long nq, int k,
                                                  double* __restrict__ out_d2, long long* __restrict__ out_idx) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nq) return;
  double d2s[kMaxK];
  long long ids[kMaxK];
  const int n = ring_knn(g, q[3 * t], q[3 * t + 1], q[3 * t + 2], k, d2s, ids);
  for (int j = 0; j < k; ++j) {
    out_d2[t * k + j] = j < n ? d2s[j] : INFINITY;
    out_idx[t * k + j] = j < n ? ids[j] : -1;
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// fdlibm's acos and cos (Sun Microsystems, freely redistributable), for the arguments FastEigen3x3 passes: acos on
// [-1, 1] without the tiny-argument shortcut, cos on [0, 4] with __ieee754_rem_pio2's three-part pi/2 always.  Within an
// ulp of a correctly rounded result; Open3D calls the host libm, which may differ from these in the last bit.
// ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ double bits(unsigned long long b) { return __longlong_as_double((long long)b); }
__device__ __forceinline__ int hi_abs(double x) { return __double2hiint(x) & 0x7fffffff; }

__device__ __forceinline__ double acos_rational(double z) {  // z * P(z) / Q(z)
  const double p = mul(z, add(bits(0x3FC5555555555555ull),
                              mul(z, add(bits(0xBFD4D61203EB6F7Dull),
                                         mul(z, add(bits(0x3FC9C1550E884455ull),
                                                    mul(z, add(bits(0xBFA48228B5688F3Bull),
                                                               mul(z, add(bits(0x3F49EFE07501B288ull),
                                                                          mul(z, bits(0x3F023DE10DFDF709ull))))))))))));
  const double qq = add(1.0, mul(z, add(bits(0xC0033A271C8A2D4Bull),
                                       mul(z, add(bits(0x40002AE59C598AC8ull),
                                                  mul(z, add(bits(0xBFE6066C1B8D0159ull),
                                                             mul(z, bits(0x3FB3B8C5B12E9282ull)))))))));
  return quo(p, qq);
}

__device__ __forceinline__ double fd_acos(double x) {
  const double pi = bits(0x400921FB54442D18ull), pio2_hi = bits(0x3FF921FB54442D18ull),
               pio2_lo = bits(0x3C91A62633145C07ull);
  if (x == 1.0) return 0.0;
  if (x == -1.0) return add(pi, mul(2.0, pio2_lo));
  if (fabs(x) < 0.5) return sub(pio2_hi, sub(x, sub(pio2_lo, mul(x, acos_rational(mul(x, x))))));
  if (x < 0.0) {
    const double z = mul(add(1.0, x), 0.5);
    const double s = __dsqrt_rn(z);
    return sub(pi, mul(2.0, add(s, sub(mul(acos_rational(z), s), pio2_lo))));
  }
  const double z = mul(sub(1.0, x), 0.5);  // x > 0.5, or NaN
  const double s = __dsqrt_rn(z);
  const double df = __hiloint2double(__double2hiint(s), 0);
  const double c = quo(sub(z, mul(df, df)), add(s, df));
  return mul(2.0, add(df, add(mul(acos_rational(z), s), c)));
}

__device__ __forceinline__ double kernel_cos(double x, double y) {
  const double z = mul(x, x);
  const double r = mul(z, add(bits(0x3FA555555555554Cull),
                              mul(z, add(bits(0xBF56C16C16C15177ull),
                                         mul(z, add(bits(0x3EFA01A019CB1590ull),
                                                    mul(z, add(bits(0xBE927E4F809C52ADull),
                                                               mul(z, add(bits(0x3E21EE9EBDB4B1C4ull),
                                                                          mul(z, bits(0xBDA8FAE9BE8838D4ull))))))))))));
  const int ix = hi_abs(x);
  const double zr_xy = sub(mul(z, r), mul(x, y));
  if (ix < 0x3FD33333) return sub(1.0, sub(mul(0.5, z), zr_xy));
  const double qx = ix > 0x3FE90000 ? 0.28125 : __hiloint2double(ix - 0x00200000, 0);
  return sub(sub(1.0, qx), sub(sub(mul(0.5, z), qx), zr_xy));
}

__device__ __forceinline__ double kernel_sin(double x, double y) {
  const double z = mul(x, x), v = mul(z, x);
  const double r = add(bits(0x3F8111111110F8A6ull),
                       mul(z, add(bits(0xBF2A01A019C161D5ull),
                                  mul(z, add(bits(0x3EC71DE357B1FE7Dull),
                                             mul(z, add(bits(0xBE5AE5E68A2B9CEBull), mul(z, bits(0x3DE5D93A5ACFD57Cull)))))))));
  return sub(x, sub(sub(mul(z, sub(mul(0.5, y), mul(v, r))), y), mul(v, bits(0xBFC5555555555549ull))));
}

__device__ __forceinline__ double fd_cos(double x) {
  const double fn = floor(add(mul(x, bits(0x3FE45F306DC9C883ull)), 0.5));
  const double t = sub(x, mul(fn, bits(0x3FF921FB54400000ull)));
  double w = mul(fn, bits(0x3DD0B4611A600000ull));
  const double r = sub(t, w);
  w = sub(mul(fn, bits(0x3BA3198A2E037073ull)), sub(sub(t, r), w));
  const double y0 = sub(r, w), y1 = sub(sub(r, y0), w);
  if (fn == 1.0) return -kernel_sin(y0, y1);
  if (fn == 2.0) return -kernel_cos(y0, y1);
  return kernel_cos(y0, y1);
}

// ---------------------------------------------------------------------------------------------------------------------
// FastEigen3x3 (Open3D 0.17 EstimateNormals.cpp, after Eberly, "A Robust Eigensolver for 3x3 Symmetric Matrices"), with
// C++'s left-to-right sums, Eigen's cross product and ((x0*y0 + x1*y1) + x2*y2) dot product, and std::max / std::min.
// The symmetric matrix is a[6] = (A00, A01, A02, A11, A12, A22).
// ---------------------------------------------------------------------------------------------------------------------
struct V3 {
  double x, y, z;
};

__device__ __forceinline__ V3 cross(V3 a, V3 b) {
  return {sub(mul(a.y, b.z), mul(a.z, b.y)), sub(mul(a.z, b.x), mul(a.x, b.z)), sub(mul(a.x, b.y), mul(a.y, b.x))};
}
__device__ __forceinline__ double dot(V3 a, V3 b) { return add(add(mul(a.x, b.x), mul(a.y, b.y)), mul(a.z, b.z)); }
__device__ __forceinline__ V3 scaled(V3 a, double d) { return {quo(a.x, d), quo(a.y, d), quo(a.z, d)}; }

__device__ __forceinline__ V3 eigenvector0(const double* a, double ev) {
  const V3 r0 = {sub(a[0], ev), a[1], a[2]}, r1 = {a[1], sub(a[3], ev), a[4]}, r2 = {a[2], a[4], sub(a[5], ev)};
  const V3 c01 = cross(r0, r1), c02 = cross(r0, r2), c12 = cross(r1, r2);
  const double d0 = dot(c01, c01), d1 = dot(c02, c02), d2 = dot(c12, c12);
  double dmax = d0;
  int imax = 0;
  if (d1 > dmax) {
    dmax = d1;
    imax = 1;
  }
  if (d2 > dmax) imax = 2;
  return imax == 0 ? scaled(c01, __dsqrt_rn(d0)) : imax == 1 ? scaled(c02, __dsqrt_rn(d1)) : scaled(c12, __dsqrt_rn(d2));
}

__device__ __forceinline__ V3 eigenvector1(const double* a, V3 e0, double ev) {
  V3 u;
  if (fabs(e0.x) > fabs(e0.y)) {
    const double inv = quo(1.0, __dsqrt_rn(add(mul(e0.x, e0.x), mul(e0.z, e0.z))));
    u = {mul(-e0.z, inv), 0.0, mul(e0.x, inv)};
  } else {
    const double inv = quo(1.0, __dsqrt_rn(add(mul(e0.y, e0.y), mul(e0.z, e0.z))));
    u = {0.0, mul(e0.z, inv), mul(-e0.y, inv)};
  }
  const V3 v = cross(e0, u);
  const V3 row0 = {a[0], a[1], a[2]}, row1 = {a[1], a[3], a[4]}, row2 = {a[2], a[4], a[5]};
  const V3 au = {dot(row0, u), dot(row1, u), dot(row2, u)}, av = {dot(row0, v), dot(row1, v), dot(row2, v)};
  double m00 = sub(dot(u, au), ev), m01 = dot(u, av), m11 = sub(dot(v, av), ev);
  const double a00 = fabs(m00), a01 = fabs(m01), a11 = fabs(m11);
  double cu, cv;  // the result is cu*U - cv*V
  if (a00 >= a11) {
    if (!((a00 < a01 ? a01 : a00) > 0.0)) return u;
    if (a00 >= a01) {
      m01 = quo(m01, m00);
      m00 = quo(1.0, __dsqrt_rn(add(1.0, mul(m01, m01))));
      m01 = mul(m01, m00);
    } else {
      m00 = quo(m00, m01);
      m01 = quo(1.0, __dsqrt_rn(add(1.0, mul(m00, m00))));
      m00 = mul(m00, m01);
    }
    cu = m01;
    cv = m00;
  } else {
    if (!((a11 < a01 ? a01 : a11) > 0.0)) return u;
    if (a11 >= a01) {
      m01 = quo(m01, m11);
      m11 = quo(1.0, __dsqrt_rn(add(1.0, mul(m01, m01))));
      m01 = mul(m01, m11);
    } else {
      m11 = quo(m11, m01);
      m01 = quo(1.0, __dsqrt_rn(add(1.0, mul(m11, m11))));
      m11 = mul(m11, m01);
    }
    cu = m11;
    cv = m01;
  }
  return {sub(mul(cu, u.x), mul(cv, v.x)), sub(mul(cu, u.y), mul(cv, v.y)), sub(mul(cu, u.z), mul(cv, v.z))};
}

__device__ __forceinline__ V3 fast_eigen3x3(const double* cov) {
  // Eigen's maxCoeff: column-major over the full matrix, replacing on value > res
  const double full[9] = {cov[0], cov[1], cov[2], cov[1], cov[3], cov[4], cov[2], cov[4], cov[5]};
  double mc = full[0];
#pragma unroll
  for (int i = 1; i < 9; ++i)
    if (full[i] > mc) mc = full[i];
  if (mc == 0.0) return {0.0, 0.0, 0.0};
  double a[6];
#pragma unroll
  for (int i = 0; i < 6; ++i) a[i] = quo(cov[i], mc);
  const double norm = add(add(mul(a[1], a[1]), mul(a[2], a[2])), mul(a[4], a[4]));
  if (!(norm > 0.0)) {
    // a diagonal matrix: the axis of the smallest entry of A / max * max, z when none is strictly smallest
    const double d0 = mul(a[0], mc), d1 = mul(a[3], mc), d2 = mul(a[5], mc);
    if (d0 < d1 && d0 < d2) return {1.0, 0.0, 0.0};
    if (d1 < d0 && d1 < d2) return {0.0, 1.0, 0.0};
    return {0.0, 0.0, 1.0};
  }
  const double q = quo(add(add(a[0], a[3]), a[5]), 3.0);
  const double b00 = sub(a[0], q), b11 = sub(a[3], q), b22 = sub(a[5], q);
  const double p = __dsqrt_rn(quo(add(add(add(mul(b00, b00), mul(b11, b11)), mul(b22, b22)), mul(norm, 2.0)), 6.0));
  const double c00 = sub(mul(b11, b22), mul(a[4], a[4]));
  const double c01 = sub(mul(a[1], b22), mul(a[4], a[2]));
  const double c02 = sub(mul(a[1], a[4]), mul(b11, a[2]));
  const double det = quo(add(sub(mul(b00, c00), mul(a[1], c01)), mul(a[2], c02)), mul(mul(p, p), p));
  double hd = mul(det, 0.5);
  hd = hd < -1.0 ? -1.0 : hd;  // std::min(std::max(hd, -1.0), 1.0), NaN kept
  hd = 1.0 < hd ? 1.0 : hd;
  const double angle = quo(fd_acos(hd), 3.0);
  const double beta2 = mul(fd_cos(angle), 2.0);
  const double beta0 = mul(fd_cos(add(angle, 2.09439510239319549)), 2.0);
  const double beta1 = -add(beta0, beta2);
  const double ev0 = add(q, mul(p, beta0)), ev1 = add(q, mul(p, beta1)), ev2 = add(q, mul(p, beta2));
  if (hd >= 0.0) {
    const V3 e2 = eigenvector0(a, ev2);
    if (ev2 < ev0 && ev2 < ev1) return e2;
    const V3 e1 = eigenvector1(a, e2, ev1);
    if (ev1 < ev0 && ev1 < ev2) return e1;
    return cross(e1, e2);
  }
  const V3 e0 = eigenvector0(a, ev0);
  if (ev0 < ev1 && ev0 < ev2) return e0;
  const V3 e1 = eigenvector1(a, e0, ev1);
  if (ev1 < ev0 && ev1 < ev2) return e1;
  return cross(e0, e1);
}

// One thread per point: its k nearest grid points (the point itself among them when it is a grid point), their
// covariance (ComputeCovariance: nine cumulants from 0.0 in neighbour order, divided by the count, then c_ij - m_i*m_j;
// the identity for fewer than 3 neighbours), FastEigen3x3, and (0, 0, 1) where that gives a vector of zero norm.
__global__ void __launch_bounds__(128, 4) normals_kernel(const GsbPointGrid g, const double* __restrict__ pts, long long n,
                                                      int k, double* __restrict__ out) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  double d2s[kMaxK];
  long long ids[kMaxK];
  const int m = ring_knn(g, pts[3 * t], pts[3 * t + 1], pts[3 * t + 2], k, d2s, ids);
  double cov[6] = {1.0, 0.0, 0.0, 1.0, 0.0, 1.0};
  if (m >= 3) {
    double c[9] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    for (int j = 0; j < m; ++j) {
      const double* p = g.points + 3 * ids[j];
      const double x = p[0], y = p[1], z = p[2];
      c[0] = add(c[0], x);
      c[1] = add(c[1], y);
      c[2] = add(c[2], z);
      c[3] = add(c[3], mul(x, x));
      c[4] = add(c[4], mul(x, y));
      c[5] = add(c[5], mul(x, z));
      c[6] = add(c[6], mul(y, y));
      c[7] = add(c[7], mul(y, z));
      c[8] = add(c[8], mul(z, z));
    }
#pragma unroll
    for (int i = 0; i < 9; ++i) c[i] = quo(c[i], (double)m);
    cov[0] = sub(c[3], mul(c[0], c[0]));
    cov[1] = sub(c[4], mul(c[0], c[1]));
    cov[2] = sub(c[5], mul(c[0], c[2]));
    cov[3] = sub(c[6], mul(c[1], c[1]));
    cov[4] = sub(c[7], mul(c[1], c[2]));
    cov[5] = sub(c[8], mul(c[2], c[2]));
  }
  V3 nrm = fast_eigen3x3(cov);
  if (dot(nrm, nrm) == 0.0) nrm = {0.0, 0.0, 1.0};
  out[3 * t] = nrm.x;
  out[3 * t + 1] = nrm.y;
  out[3 * t + 2] = nrm.z;
}

// ---------------------------------------------------------------------------------------------------------------------
// RemoveStatisticalOutliers: m_i = (((0.0 + sqrt(d2_0)) + sqrt(d2_1)) + ...) / double(c) over the c = min(k, n) nearest
// grid points of grid point i (itself included), then mean and standard deviation of the positive m_i by a fixed-order
// sum S (chunks of kStatChunk consecutive indices summed sequentially from 0.0, then the chunk sums sequentially from
// 0.0), so every run writes the same bytes.  A skipped term adds nothing: a sum from +0.0 of values >= 0 is never -0.0,
// so skipping equals adding +0.0.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int kStatChunk = 1024;

__global__ void __launch_bounds__(128, 4) stat_mean_kernel(const GsbPointGrid g, int k, double* __restrict__ mean_dist) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= g.n_points) return;
  double d2s[kMaxK];
  long long ids[kMaxK];
  const double* p = g.points + 3 * t;
  const int c = ring_knn(g, p[0], p[1], p[2], k, d2s, ids);
  double s = 0.0;
  for (int j = 0; j < c; ++j) s = add(s, __dsqrt_rn(d2s[j]));
  mean_dist[t] = quo(s, (double)c);
}

// pass 0: the chunk sums of m_i over m_i > 0; pass 1: of (m_i - mean) * (m_i - mean) over m_i > 0, mean = stats[0]
__global__ void __launch_bounds__(128) stat_chunk_kernel(const double* __restrict__ mean_dist, long long n, int pass,
                                                         const double* __restrict__ stats, double* __restrict__ partial) {
  const long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (c * kStatChunk >= n) return;
  const double mean = pass ? stats[0] : 0.0;
  const long long e = min(n, (c + 1) * kStatChunk);
  double s = 0.0;
  for (long long i = c * kStatChunk; i < e; ++i) {
    const double m = mean_dist[i];
    if (m > 0.0) s = add(s, pass ? mul(sub(m, mean), sub(m, mean)) : m);
  }
  partial[c] = s;
}

// One thread: the chunk sums in chunk order.  pass 0 writes stats[0] = S / double(n); pass 1 writes stats[1] =
// sqrt(S / double(n - 1)) and stats[2] = mean + std_ratio * std.
__global__ void stat_total_kernel(const double* __restrict__ partial, long long n, int pass, double std_ratio,
                                  double* __restrict__ stats) {
  const long long chunks = (n + kStatChunk - 1) / kStatChunk;
  double s = 0.0;
  for (long long c = 0; c < chunks; ++c) s = add(s, partial[c]);
  if (pass == 0) {
    stats[0] = quo(s, (double)n);
  } else {
    const double sd = __dsqrt_rn(quo(s, (double)(n - 1)));
    stats[1] = sd;
    stats[2] = add(stats[0], mul(std_ratio, sd));
  }
}

__global__ void __launch_bounds__(256) stat_keep_kernel(const double* __restrict__ mean_dist, long long n,
                                                        const double* __restrict__ stats, uint8_t* __restrict__ keep) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double m = mean_dist[i];
  keep[i] = m > 0.0 && m < stats[2];
}

// RemoveRadiusOutliers: keep[i] = 1 iff more than nb_points grid points j (i itself included) have
// ((dx*dx)+dy*dy)+dz*dz < r2, strictly (nanoflann's radius result set).  The 27-cell walk stops once the count passes
// nb_points; a point with a non-finite coordinate is not kept.
__global__ void __launch_bounds__(256) radius_outlier_kernel(const GsbPointGrid g, long long nb_points, double r2,
                                                             uint8_t* __restrict__ keep) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= g.n_points) return;
  const double x = g.points[3 * t], y = g.points[3 * t + 1], z = g.points[3 * t + 2];
  long long count = 0;
  if (isfinite(x) && isfinite(y) && isfinite(z))
    visit_27_cells(g, x, y, z, [&](long long q) {
      count += sq_dist(x, y, z, g.points + 3 * q) < r2;
      return count <= nb_points;
    });
  keep[t] = count > nb_points;
}

// ---------------------------------------------------------------------------------------------------------------------
// ClusterDBSCAN.  core[i] = count_i >= min_points is radius_outlier_kernel with nb_points = min_points - 1 (-1 for
// min_points = 0 marks every point core).  Core points joined by a pair at d2 < r2 form components; each component's
// union-find root is its smallest index, so an exclusive scan of the root flags numbers the components by their
// smallest core index, as Open3D's ascending loop does.  A non-core point takes the smallest root among the core points
// within eps, which is the smallest component number; none gives -1.
// ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ bool finite3(const double* p) { return isfinite(p[0]) && isfinite(p[1]) && isfinite(p[2]); }

// parent[i] = i; a point with a non-finite coordinate is never core (radius_outlier_kernel marks it core for
// min_points = 0, its count 0 being > -1), so the later passes need not test finiteness of core points.
__global__ void __launch_bounds__(256) dbscan_init_kernel(const GsbPointGrid g, uint8_t* __restrict__ core,
                                                          int* __restrict__ parent) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= g.n_points) return;
  parent[t] = (int)t;
  if (!finite3(g.points + 3 * t)) core[t] = 0;
}

// One thread per core point i: every core q < i within eps is united with i, so each core-core pair is handled once.
__global__ void __launch_bounds__(256) dbscan_link_kernel(const GsbPointGrid g, double r2, const uint8_t* __restrict__ core,
                                                          int* parent) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= g.n_points || !core[t]) return;
  const double x = g.points[3 * t], y = g.points[3 * t + 1], z = g.points[3 * t + 2];
  visit_27_cells(g, x, y, z, [&](long long q) {
    if (q < t && core[q] && sq_dist(x, y, z, g.points + 3 * q) < r2) uf_union(parent, (int)t, (int)q);
    return true;
  });
}

// parent[i] = the root of core point i; head[i] = 1 for the roots (core points only)
__global__ void __launch_bounds__(256) dbscan_compress_kernel(const uint8_t* __restrict__ core, long long n, int* parent,
                                                              int* __restrict__ head) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  int r = (int)t;
  if (core[t]) {
    for (int p = uf_load(parent, r); p != r; p = uf_load(parent, r)) r = p;
    ParentRef(parent[t]).store(r, cuda::memory_order_relaxed);
  }
  head[t] = core[t] && r == (int)t;
}

// labels[i] = ordinal of i's root (core), of the smallest root among the core points within eps (non-core), or -1; the
// last thread writes the number of clusters.
__global__ void __launch_bounds__(256) dbscan_label_kernel(const GsbPointGrid g, double r2, const uint8_t* __restrict__ core,
                                                           const int* __restrict__ parent, const int* __restrict__ head,
                                                           const int* __restrict__ ordinal, int32_t* __restrict__ labels,
                                                           int32_t* __restrict__ n_clusters) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= g.n_points) return;
  const double* p = g.points + 3 * t;
  int root = -1;
  if (core[t]) {
    root = parent[t];
  } else if (finite3(p)) {
    const double x = p[0], y = p[1], z = p[2];
    visit_27_cells(g, x, y, z, [&](long long q) {
      if (core[q] && (root < 0 || parent[q] < root) && sq_dist(x, y, z, g.points + 3 * q) < r2) root = parent[q];
      return true;
    });
  }
  labels[t] = root < 0 ? -1 : ordinal[root];
  if (t == g.n_points - 1) *n_clusters = ordinal[t] + head[t];
}

// Workspace of gsb_pcd_dbscan; with a NULL base only `total` is meaningful.
struct DbscanWork {
  uint8_t* core;  // [n]
  int* parent;    // [n]
  int* head;      // [n]
  int* ordinal;   // [n]
  void* tmp;
  size_t tmp_bytes, total;
};

DbscanWork carve_dbscan(void* base, long long n) {
  Carver c(base);
  DbscanWork w;
  w.core = c.take<uint8_t>((size_t)n);
  w.parent = c.take<int>((size_t)n);
  w.head = c.take<int>((size_t)n);
  w.ordinal = c.take<int>((size_t)n);
  w.tmp_bytes = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, w.tmp_bytes, (int*)nullptr, (int*)nullptr, n);
  w.tmp = c.take<char>(w.tmp_bytes);
  w.total = c.total();
  return w;
}

}  // namespace
}  // namespace gsb

using namespace gsb;

extern "C" {

int gsb_eval_knn(const GsbPointGrid* grid, const double* queries, int64_t n_queries, int32_t k, double* dist2,
                 int64_t* index, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (!grid_ok(grid) || n_queries < 0 || k < 1 || k > kMaxK || (n_queries && (!queries || !dist2 || !index)))
    return fail(GSB_ERR_INVALID, "eval_knn: bad arguments (k must be in 1..%d)", kMaxK);
  if (n_queries == 0) return GSB_OK;
  knn_kernel<<<blocks_for(n_queries, 128), 128, 0, stream>>>(*grid, queries, n_queries, k, dist2,
                                                             reinterpret_cast<long long*>(index));
  count_launch();
  return check_launch("knn_kernel", stream, false);
}

int gsb_eval_estimate_normals(const GsbPointGrid* grid, const double* points, int64_t n_points, int32_t k, double* normals,
                              void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (!grid_ok(grid) || n_points < 0 || k < 1 || k > kMaxK || (n_points && (!points || !normals)))
    return fail(GSB_ERR_INVALID, "eval_estimate_normals: bad arguments (k must be in 1..%d)", kMaxK);
  if (n_points == 0) return GSB_OK;
  normals_kernel<<<blocks_for(n_points, 128), 128, 0, stream>>>(*grid, points, n_points, k, normals);
  count_launch();
  return check_launch("normals_kernel", stream, false);
}

size_t gsb_pcd_statistical_workspace_bytes(int64_t n_points) {
  if (n_points < 0 || n_points > 2147483647) return 0;
  return align_up(sizeof(double) * (size_t)((n_points + kStatChunk - 1) / kStatChunk), 256);
}

int gsb_pcd_statistical_outliers(const GsbPointGrid* grid, int32_t k, double std_ratio, void* workspace,
                                 size_t workspace_bytes, double* mean_dist, uint8_t* keep, double* stats, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (!grid_ok(grid) || grid->n_points > 2147483647 || k < 1 || k > kMaxK || !(std_ratio > 0.0) ||
      (grid->n_points && (!workspace || !mean_dist || !keep || !stats)))
    return fail(GSB_ERR_INVALID, "pcd_statistical_outliers: bad arguments (k must be in 1..%d, std_ratio > 0)", kMaxK);
  const long long n = grid->n_points;
  if (n == 0) return GSB_OK;
  if (workspace_bytes < gsb_pcd_statistical_workspace_bytes(n))
    return fail(GSB_ERR_WORKSPACE, "pcd_statistical_outliers: workspace %zu < %zu bytes", workspace_bytes,
                gsb_pcd_statistical_workspace_bytes(n));
  double* partial = static_cast<double*>(workspace);
  const long long chunks = (n + kStatChunk - 1) / kStatChunk;
  stat_mean_kernel<<<blocks_for(n, 128), 128, 0, stream>>>(*grid, k, mean_dist);
  for (int pass = 0; pass < 2; ++pass) {
    stat_chunk_kernel<<<blocks_for(chunks, 128), 128, 0, stream>>>(mean_dist, n, pass, stats, partial);
    stat_total_kernel<<<1, 1, 0, stream>>>(partial, n, pass, std_ratio, stats);
  }
  stat_keep_kernel<<<blocks_for(n), 256, 0, stream>>>(mean_dist, n, stats, keep);
  count_launch(6);
  return check_launch("statistical outliers", stream, false);
}

int gsb_pcd_radius_outliers(const GsbPointGrid* grid, int64_t nb_points, double radius, uint8_t* keep, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (!grid_ok(grid) || nb_points < 1 || !(radius > 0.0) || !(radius < INFINITY) || (grid->n_points && !keep) ||
      !(grid->cell >= radius * 1.0000001))
    return fail(GSB_ERR_INVALID,
                "pcd_radius_outliers: bad arguments (nb_points >= 1, a finite radius > 0, the grid cell above the radius)");
  if (grid->n_points == 0) return GSB_OK;
  radius_outlier_kernel<<<blocks_for(grid->n_points), 256, 0, stream>>>(*grid, nb_points, radius * radius, keep);
  count_launch();
  return check_launch("radius_outlier_kernel", stream, false);
}

size_t gsb_pcd_dbscan_workspace_bytes(int64_t n_points) {
  if (n_points <= 0 || n_points > 2147483647) return 0;
  return carve_dbscan(nullptr, n_points).total;
}

int gsb_pcd_dbscan(const GsbPointGrid* grid, double eps, int64_t min_points, void* workspace, size_t workspace_bytes,
                   int32_t* labels, int32_t* n_clusters, void* stream_v) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (!grid_ok(grid) || grid->n_points > 2147483647 || !(eps >= 0.0) || !(eps < INFINITY) || min_points < 0 ||
      !(grid->cell >= eps * 1.0000001) || (grid->n_points && (!workspace || !labels || !n_clusters)))
    return fail(GSB_ERR_INVALID,
                "pcd_dbscan: bad arguments (a finite eps >= 0, min_points >= 0, the grid cell above eps, at most 2^31 - 1 "
                "points)");
  const long long n = grid->n_points;
  if (n == 0) return GSB_OK;
  const size_t need = gsb_pcd_dbscan_workspace_bytes(n);
  if (workspace_bytes < need) return fail(GSB_ERR_WORKSPACE, "pcd_dbscan: workspace %zu < %zu bytes", workspace_bytes, need);
  const DbscanWork w = carve_dbscan(workspace, n);
  const double r2 = eps * eps;
  radius_outlier_kernel<<<blocks_for(n), 256, 0, stream>>>(*grid, min_points - 1, r2, w.core);
  dbscan_init_kernel<<<blocks_for(n), 256, 0, stream>>>(*grid, w.core, w.parent);
  dbscan_link_kernel<<<blocks_for(n), 256, 0, stream>>>(*grid, r2, w.core, w.parent);
  dbscan_compress_kernel<<<blocks_for(n), 256, 0, stream>>>(w.core, n, w.parent, w.head);
  count_launch(4);
  size_t tmp_bytes = w.tmp_bytes;
  GSB_CUDA_OK(cub::DeviceScan::ExclusiveSum(w.tmp, tmp_bytes, w.head, w.ordinal, n, stream));
  dbscan_label_kernel<<<blocks_for(n), 256, 0, stream>>>(*grid, r2, w.core, w.parent, w.head, w.ordinal, labels, n_clusters);
  count_launch();
  return check_launch("pcd_dbscan", stream, false);
}

}  // extern "C"
