"""numpy restatement of gsb_eval_knn and gsb_eval_estimate_normals (test infrastructure only; float64 throughout, every
operation a single correctly rounded numpy ufunc, so nothing is contracted into an FMA).  DESIGN.md section 7d gives the
operation orders:
  knn / knn_brute    the k nearest reference points in ascending (d2, index) order, d2 = ((dx*dx)+dy*dy)+dz*dz, padded
                     with (+inf, -1); a query with a non-finite coordinate gets only padding
  covariances        Open3D 0.17 ComputeCovariance: nine cumulants summed in neighbour order, divided by the count, then
                     c_ij - m_i*m_j; fewer than 3 neighbours give the identity
  fast_eigen3x3      Open3D 0.17 FastEigen3x3 (Eberly's robust 3x3 eigensolver): the eigenvector of the smallest eigenvalue
  acos / cos         the fdlibm algorithms the kernel uses instead of the device's libm, so both sides round alike
  estimate_normals   PointCloud::EstimateNormals(KDTreeSearchParamKNN(k)) on a cloud without normals
"""
from __future__ import annotations

import numpy as np

MAX_K = 32


def _f64(bits):
    return float(np.array(bits, dtype=np.uint64).view(np.float64))


def _hi(x):
    """The high 32 bits of |x| (fdlibm's __HI(x) & 0x7fffffff)."""
    return (np.asarray(x, np.float64).view(np.uint64) >> np.uint64(32)).astype(np.int64) & 0x7FFFFFFF


# ------------------------------------------------------------------------------------------------------------ k-NN
def sq_dist(q, p):
    d = q - p
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def _check_k(k):
    if not 1 <= int(k) <= MAX_K:
        raise ValueError(f"k must be in 1..{MAX_K}")
    return int(k)


def knn_brute(queries, reference, k, chunk=1 << 22):
    """(d2 [N,k], idx [N,k]) by comparing every query with every reference point."""
    k = _check_k(k)
    q = np.asarray(queries, np.float64).reshape(-1, 3)
    r = np.asarray(reference, np.float64).reshape(-1, 3)
    d2 = np.full((len(q), k), np.inf)
    idx = np.full((len(q), k), -1, np.int64)
    m = min(k, len(r))
    fin = np.isfinite(q).all(axis=1)
    if m == 0:
        return d2, idx
    step = max(1, chunk // len(r))
    ids = np.arange(len(r), dtype=np.int64)
    for a in range(0, len(q), step):
        dd = sq_dist(q[a:a + step, None, :], r[None, :, :])
        # lexsort by (d2, index): argsort by d2 is stable, and ids ascend along each row
        order = np.argsort(dd, axis=1, kind="stable")[:, :m]
        d2[a:a + step, :m] = np.take_along_axis(dd, order, axis=1)
        idx[a:a + step, :m] = ids[order]
    d2[~fin] = np.inf
    idx[~fin] = -1
    return d2, idx


def knn(queries, reference, k):
    """knn_brute's result through scipy's cKDTree: k + 4 candidates per query, re-sorted by the exact (d2, index); a row
    whose k-th d2 is not below its last candidate's d2 could have a tie outside the candidates and is redone by brute
    force against every reference point."""
    from scipy.spatial import cKDTree

    k = _check_k(k)
    q = np.asarray(queries, np.float64).reshape(-1, 3)
    r = np.asarray(reference, np.float64).reshape(-1, 3)
    n = len(r)
    if n <= k + 4 or len(q) == 0:
        return knn_brute(q, r, k)
    d2 = np.full((len(q), k), np.inf)
    idx = np.full((len(q), k), -1, np.int64)
    fin = np.where(np.isfinite(q).all(axis=1))[0]
    qf = q[fin]
    c = k + 4
    _, cand = cKDTree(r).query(qf, c)
    cd = sq_dist(qf[:, None, :], r[cand])
    order = np.lexsort((cand, cd), axis=-1)
    cd = np.take_along_axis(cd, order, axis=1)
    cand = np.take_along_axis(cand, order, axis=1)
    d2[fin], idx[fin] = cd[:, :k], cand[:, :k]
    redo = fin[~(cd[:, k - 1] < cd[:, c - 1])]
    if len(redo):
        d2[redo], idx[redo] = knn_brute(q[redo], r, k)
    return d2, idx


# ------------------------------------------------------------------------------------------------------ covariance
def covariances(points, idx):
    """[N,3,3] from the neighbour lists idx [N,k] (-1 = padding, always at the end of a row)."""
    p = np.asarray(points, np.float64).reshape(-1, 3)
    idx = np.asarray(idx, np.int64)
    n, k = idx.shape
    count = (idx >= 0).sum(axis=1)
    cum = np.zeros((n, 9))
    for j in range(k):
        live = idx[:, j] >= 0
        x = p[idx[live, j]]
        cum[live] += np.stack([x[:, 0], x[:, 1], x[:, 2], x[:, 0] * x[:, 0], x[:, 0] * x[:, 1], x[:, 0] * x[:, 2],
                               x[:, 1] * x[:, 1], x[:, 1] * x[:, 2], x[:, 2] * x[:, 2]], axis=1)
    with np.errstate(divide="ignore", invalid="ignore"):
        cum = cum / count[:, None].astype(np.float64)
    m0, m1, m2 = cum[:, 0], cum[:, 1], cum[:, 2]
    cov = np.empty((n, 3, 3))
    cov[:, 0, 0] = cum[:, 3] - m0 * m0
    cov[:, 1, 1] = cum[:, 6] - m1 * m1
    cov[:, 2, 2] = cum[:, 8] - m2 * m2
    cov[:, 0, 1] = cov[:, 1, 0] = cum[:, 4] - m0 * m1
    cov[:, 0, 2] = cov[:, 2, 0] = cum[:, 5] - m0 * m2
    cov[:, 1, 2] = cov[:, 2, 1] = cum[:, 7] - m1 * m2
    cov[count < 3] = np.eye(3)
    return cov


# ------------------------------------------------------------------------------------------------- fdlibm acos, cos
PI = _f64(0x400921FB54442D18)
PIO2_HI = _f64(0x3FF921FB54442D18)
PIO2_LO = _f64(0x3C91A62633145C07)
PS = [_f64(b) for b in (0x3FC5555555555555, 0xBFD4D61203EB6F7D, 0x3FC9C1550E884455, 0xBFA48228B5688F3B,
                        0x3F49EFE07501B288, 0x3F023DE10DFDF709)]
QS = [_f64(b) for b in (0xC0033A271C8A2D4B, 0x40002AE59C598AC8, 0xBFE6066C1B8D0159, 0x3FB3B8C5B12E9282)]
INVPIO2 = _f64(0x3FE45F306DC9C883)
PIO2_1 = _f64(0x3FF921FB54400000)
PIO2_2 = _f64(0x3DD0B4611A600000)
PIO2_2T = _f64(0x3BA3198A2E037073)
C = [_f64(b) for b in (0x3FA555555555554C, 0xBF56C16C16C15177, 0x3EFA01A019CB1590, 0xBE927E4F809C52AD,
                       0x3E21EE9EBDB4B1C4, 0xBDA8FAE9BE8838D4)]
S = [_f64(b) for b in (0xBFC5555555555549, 0x3F8111111110F8A6, 0xBF2A01A019C161D5, 0x3EC71DE357B1FE7D,
                       0xBE5AE5E68A2B9CEB, 0x3DE5D93A5ACFD57C)]
TWO_THIRDS_PI = 2.09439510239319549


def _rational(z):
    p = z * (PS[0] + z * (PS[1] + z * (PS[2] + z * (PS[3] + z * (PS[4] + z * PS[5])))))
    q = 1.0 + z * (QS[0] + z * (QS[1] + z * (QS[2] + z * QS[3])))
    return p / q


def acos(x):
    """fdlibm's __ieee754_acos for x in [-1, 1] (and NaN), without its tiny-argument shortcut."""
    x = np.asarray(x, np.float64)
    with np.errstate(all="ignore"):
        z = x * x  # |x| < 0.5
        small = PIO2_HI - (x - (PIO2_LO - x * _rational(z)))
        z = (1.0 + x) * 0.5  # x <= -0.5
        s = np.sqrt(z)
        neg = PI - 2.0 * (s + (_rational(z) * s - PIO2_LO))
        z = (1.0 - x) * 0.5  # x >= 0.5
        s = np.sqrt(z)
        df = (s.view(np.uint64) & np.uint64(0xFFFFFFFF00000000)).view(np.float64)
        c = (z - df * df) / (s + df)
        pos = 2.0 * (df + (_rational(z) * s + c))
    r = np.where(np.abs(x) < 0.5, small, np.where(x < 0.0, neg, pos))
    r = np.where(x == 1.0, 0.0, r)
    return np.where(x == -1.0, PI + 2.0 * PIO2_LO, r)


def _kernel_cos(x, y):
    z = x * x
    r = z * (C[0] + z * (C[1] + z * (C[2] + z * (C[3] + z * (C[4] + z * C[5])))))
    ix = _hi(x)
    qx = np.where(ix > 0x3FE90000, 0.28125, ((ix - 0x00200000).astype(np.uint64) << np.uint64(32)).view(np.float64))
    big = (1.0 - qx) - ((0.5 * z - qx) - (z * r - x * y))
    return np.where(ix < 0x3FD33333, 1.0 - (0.5 * z - (z * r - x * y)), big)


def _kernel_sin(x, y):
    z = x * x
    v = z * x
    r = S[1] + z * (S[2] + z * (S[3] + z * (S[4] + z * S[5])))
    return x - ((z * (0.5 * y - v * r) - y) - v * S[0])


def cos(x):
    """fdlibm's cos for x in [0, 4] (and NaN): n = floor(x * 2/pi + 0.5), x - n*pi/2 with the three-part pi/2 of
    __ieee754_rem_pio2's second step, then __kernel_cos or __kernel_sin."""
    x = np.asarray(x, np.float64)
    with np.errstate(all="ignore"):
        fn = np.floor(x * INVPIO2 + 0.5)
        t = x - fn * PIO2_1
        w = fn * PIO2_2
        r = t - w
        w = fn * PIO2_2T - ((t - r) - w)
        y0 = r - w
        y1 = (r - y0) - w
        kc, ks = _kernel_cos(y0, y1), _kernel_sin(y0, y1)
    return np.where(fn == 1.0, -ks, np.where(fn == 2.0, -kc, kc))


# ------------------------------------------------------------------------------------------------------ FastEigen3x3
def _cross(a, b):
    return np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                     a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], axis=-1)


def _dot(a, b):
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def _max(a, b):  # std::max
    return np.where(a < b, b, a)


def _eigenvector0(A, ev):
    r0 = np.stack([A[:, 0, 0] - ev, A[:, 0, 1], A[:, 0, 2]], axis=1)
    r1 = np.stack([A[:, 0, 1], A[:, 1, 1] - ev, A[:, 1, 2]], axis=1)
    r2 = np.stack([A[:, 0, 2], A[:, 1, 2], A[:, 2, 2] - ev], axis=1)
    c01, c02, c12 = _cross(r0, r1), _cross(r0, r2), _cross(r1, r2)
    d0, d1, d2 = _dot(c01, c01), _dot(c02, c02), _dot(c12, c12)
    imax = np.where(d1 > d0, 1, 0)
    imax = np.where(d2 > np.where(d1 > d0, d1, d0), 2, imax)
    return np.where((imax == 0)[:, None], c01 / np.sqrt(d0)[:, None],
                    np.where((imax == 1)[:, None], c02 / np.sqrt(d1)[:, None], c12 / np.sqrt(d2)[:, None]))


def _eigenvector1(A, e0, ev):
    x_first = np.abs(e0[:, 0]) > np.abs(e0[:, 1])
    inv_a = 1.0 / np.sqrt(e0[:, 0] * e0[:, 0] + e0[:, 2] * e0[:, 2])
    inv_b = 1.0 / np.sqrt(e0[:, 1] * e0[:, 1] + e0[:, 2] * e0[:, 2])
    zero = np.zeros(len(e0))
    U = np.where(x_first[:, None], np.stack([-e0[:, 2] * inv_a, zero, e0[:, 0] * inv_a], axis=1),
                 np.stack([zero, e0[:, 2] * inv_b, -e0[:, 1] * inv_b], axis=1))
    V = _cross(e0, U)
    rows = [np.stack([A[:, 0, 0], A[:, 0, 1], A[:, 0, 2]], 1), np.stack([A[:, 0, 1], A[:, 1, 1], A[:, 1, 2]], 1),
            np.stack([A[:, 0, 2], A[:, 1, 2], A[:, 2, 2]], 1)]
    AU = np.stack([_dot(row, U) for row in rows], axis=1)
    AV = np.stack([_dot(row, V) for row in rows], axis=1)
    m00 = _dot(U, AU) - ev
    m01 = _dot(U, AV)
    m11 = _dot(V, AV) - ev
    a00, a01, a11 = np.abs(m00), np.abs(m01), np.abs(m11)
    # branch 0: |m00| >= |m11|
    q = m01 / m00
    s = 1.0 / np.sqrt(1.0 + q * q)
    b0_a = (q * s, s)  # (m01, m00) when |m00| >= |m01|
    q = m00 / m01
    s = 1.0 / np.sqrt(1.0 + q * q)
    b0_b = (s, q * s)
    u0 = np.where(a00 >= a01, b0_a[0], b0_b[0])
    v0 = np.where(a00 >= a01, b0_a[1], b0_b[1])
    vec0 = u0[:, None] * U - v0[:, None] * V  # m01*U - m00*V
    ok0 = _max(a00, a01) > 0
    # branch 1: |m00| < |m11|
    q = m01 / m11
    s = 1.0 / np.sqrt(1.0 + q * q)
    b1_a = (s, q * s)  # (m11, m01) when |m11| >= |m01|
    q = m11 / m01
    s = 1.0 / np.sqrt(1.0 + q * q)
    b1_b = (q * s, s)
    u1 = np.where(a11 >= a01, b1_a[0], b1_b[0])
    v1 = np.where(a11 >= a01, b1_a[1], b1_b[1])
    vec1 = u1[:, None] * U - v1[:, None] * V  # m11*U - m01*V
    ok1 = _max(a11, a01) > 0
    first = a00 >= a11
    return np.where(first[:, None], np.where(ok0[:, None], vec0, U), np.where(ok1[:, None], vec1, U))


def fast_eigen3x3(cov):
    """The unit eigenvector of the smallest eigenvalue of each symmetric [3,3] (zero for a zero matrix)."""
    A = np.array(cov, dtype=np.float64).reshape(-1, 3, 3)
    n = len(A)
    out = np.zeros((n, 3))
    with np.errstate(all="ignore"):
        mc = A[:, 0, 0].copy()  # Eigen's maxCoeff: column-major, value > res
        for j in range(3):
            for i in range(3):
                if i or j:
                    mc = np.where(A[:, i, j] > mc, A[:, i, j], mc)
        nz = mc != 0
        A = A / np.where(nz, mc, 1.0)[:, None, None]
        norm = (A[:, 0, 1] * A[:, 0, 1] + A[:, 0, 2] * A[:, 0, 2]) + A[:, 1, 2] * A[:, 1, 2]
        # off-diagonal entries all zero: a coordinate axis, by the diagonal rescaled with (A / max) * max
        d = A[:, [0, 1, 2], [0, 1, 2]] * mc[:, None]
        axis = np.where((d[:, 0] < d[:, 1]) & (d[:, 0] < d[:, 2]), 0,
                        np.where((d[:, 1] < d[:, 0]) & (d[:, 1] < d[:, 2]), 1, 2))
        diag = np.eye(3)[axis]
        q = ((A[:, 0, 0] + A[:, 1, 1]) + A[:, 2, 2]) / 3.0
        b00, b11, b22 = A[:, 0, 0] - q, A[:, 1, 1] - q, A[:, 2, 2] - q
        p = np.sqrt((((b00 * b00 + b11 * b11) + b22 * b22) + norm * 2.0) / 6.0)
        c00 = b11 * b22 - A[:, 1, 2] * A[:, 1, 2]
        c01 = A[:, 0, 1] * b22 - A[:, 1, 2] * A[:, 0, 2]
        c02 = A[:, 0, 1] * A[:, 1, 2] - b11 * A[:, 0, 2]
        det = ((b00 * c00 - A[:, 0, 1] * c01) + A[:, 0, 2] * c02) / ((p * p) * p)
        hd = det * 0.5
        hd = np.where(hd < -1.0, -1.0, hd)  # std::min(std::max(hd, -1.0), 1.0)
        hd = np.where(1.0 < hd, 1.0, hd)
        angle = acos(hd) / 3.0
        beta2 = cos(angle) * 2.0
        beta0 = cos(angle + TWO_THIRDS_PI) * 2.0
        beta1 = -(beta0 + beta2)
        ev0, ev1, ev2 = q + p * beta0, q + p * beta1, q + p * beta2
        pos = hd >= 0
        v_first = _eigenvector0(A, np.where(pos, ev2, ev0))
        first_min = np.where(pos, (ev2 < ev0) & (ev2 < ev1), (ev0 < ev1) & (ev0 < ev2))
        v1 = _eigenvector1(A, v_first, ev1)
        one_min = (ev1 < ev0) & (ev1 < ev2)
        v_last = np.where(pos[:, None], _cross(v1, v_first), _cross(v_first, v1))
        full = np.where(first_min[:, None], v_first, np.where(one_min[:, None], v1, v_last))
        out = np.where((norm > 0)[:, None], full, diag)
        out[~nz] = 0.0
    return out


def estimate_normals(points, k=20, idx=None):
    """Open3D's EstimateNormals with fast_normal_computation: FastEigen3x3 of each point's k-NN covariance (the point
    itself included), (0, 0, 1) where that gives a zero vector; no orientation."""
    p = np.asarray(points, np.float64).reshape(-1, 3)
    if idx is None:
        idx = knn(p, p, k)[1]
    nrm = fast_eigen3x3(covariances(p, idx))
    zero = ((nrm[:, 0] * nrm[:, 0] + nrm[:, 1] * nrm[:, 1]) + nrm[:, 2] * nrm[:, 2]) == 0.0
    nrm[zero] = (0.0, 0.0, 1.0)
    return nrm
