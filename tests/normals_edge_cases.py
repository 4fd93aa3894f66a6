"""Edge cases for ring_knn and FastEigen3x3 (gs2mesh_b200/csrc/gsb_normals.cu), and a second restatement of the normal
computation that records the branches it takes (test infrastructure only).

trace_fast_eigen3x3 transliterates fast_eigen3x3, eigenvector0, eigenvector1, fd_acos, fd_cos, kernel_cos and kernel_sin
statement by statement in Python floats: one IEEE round-to-nearest per operation, no FMA, math.sqrt and math.floor.  It
shares no code with tests/normals_oracle.py, which evaluates every branch in numpy and selects with np.where; the two
must agree bit for bit.  It returns the vector and the set of branch labels it took; LABELS lists them all and
UNREACHABLE gives, for each label no case reaches, the reason: a proof, except for the one entry that says otherwise.

EIGEN_CASES are point clouds of m <= 32 points, run with k = m, so every point's neighbourhood is the whole cloud.  Most
have small dyadic coordinates, whose cumulant sums are exact in any order, so every point gets the same covariance bits;
the large-offset clouds get per-point bits from their neighbour order.  The k-NN builders place reference points and
queries on explicit grid layouts (origin, cell, dims) at the bounds of ring_knn's stop test `n == k && d2s[k-1] <
lb*lb`, lb = (K-1)*h*(1 - 1e-9) before ring K, and at ties past the k-th place.
"""
from __future__ import annotations

import functools
import math
import struct

import numpy as np

# ------------------------------------------------------------------------------------------------ Python-float IEEE ops


def _bits(x):
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def _f(b):
    return struct.unpack("<d", struct.pack("<Q", b & 0xFFFFFFFFFFFFFFFF))[0]


def _quo(a, b):
    """a / b in IEEE arithmetic (Python raises on a zero divisor)."""
    if b != 0.0 or math.isnan(b):
        return a / b
    if a == 0.0 or math.isnan(a):
        return math.nan
    return math.copysign(math.inf, a) * math.copysign(1.0, b)


def _sqrt(x):
    return math.nan if math.isnan(x) or x < 0.0 else math.sqrt(x)


def _floor(x):
    return x if math.isnan(x) or math.isinf(x) else float(math.floor(x))


def _hi_abs(x):
    return (_bits(x) >> 32) & 0x7FFFFFFF


def _hi_only(x):  # __hiloint2double(__double2hiint(x), 0)
    return _f(_bits(x) & 0xFFFFFFFF00000000)


# ------------------------------------------------------------------------------------------------ fdlibm acos, cos
_PS = [_f(b) for b in (0x3FC5555555555555, 0xBFD4D61203EB6F7D, 0x3FC9C1550E884455, 0xBFA48228B5688F3B,
                       0x3F49EFE07501B288, 0x3F023DE10DFDF709)]
_QS = [_f(b) for b in (0xC0033A271C8A2D4B, 0x40002AE59C598AC8, 0xBFE6066C1B8D0159, 0x3FB3B8C5B12E9282)]
_C = [_f(b) for b in (0x3FA555555555554C, 0xBF56C16C16C15177, 0x3EFA01A019CB1590, 0xBE927E4F809C52AD,
                      0x3E21EE9EBDB4B1C4, 0xBDA8FAE9BE8838D4)]
_S1 = [_f(b) for b in (0x3F8111111110F8A6, 0xBF2A01A019C161D5, 0x3EC71DE357B1FE7D, 0xBE5AE5E68A2B9CEB,
                       0x3DE5D93A5ACFD57C)]
_S0 = _f(0xBFC5555555555549)
_PI, _PIO2_HI, _PIO2_LO = _f(0x400921FB54442D18), _f(0x3FF921FB54442D18), _f(0x3C91A62633145C07)


def _acos_rational(z):
    p = z * (_PS[0] + z * (_PS[1] + z * (_PS[2] + z * (_PS[3] + z * (_PS[4] + z * _PS[5])))))
    qq = 1.0 + z * (_QS[0] + z * (_QS[1] + z * (_QS[2] + z * _QS[3])))
    return _quo(p, qq)


def _fd_acos(x, L):
    if x == 1.0:
        L.add("acos_one")
        return 0.0
    if x == -1.0:
        L.add("acos_minus_one")
        return _PI + 2.0 * _PIO2_LO
    if abs(x) < 0.5:
        L.add("acos_small")
        return _PIO2_HI - (x - (_PIO2_LO - x * _acos_rational(x * x)))
    if x < 0.0:
        L.add("acos_negative")
        z = (1.0 + x) * 0.5
        s = _sqrt(z)
        return _PI - 2.0 * (s + (_acos_rational(z) * s - _PIO2_LO))
    L.add("acos_positive")  # x > 0.5, or NaN
    z = (1.0 - x) * 0.5
    s = _sqrt(z)
    df = _hi_only(s)
    c = _quo(z - df * df, s + df)
    return 2.0 * (df + (_acos_rational(z) * s + c))


def _kernel_cos(x, y, L):
    z = x * x
    r = z * (_C[0] + z * (_C[1] + z * (_C[2] + z * (_C[3] + z * (_C[4] + z * _C[5])))))
    ix = _hi_abs(x)
    zr_xy = z * r - x * y
    if ix < 0x3FD33333:
        L.add("kcos_small")
        return 1.0 - (0.5 * z - zr_xy)
    if ix > 0x3FE90000:
        L.add("kcos_big")
        qx = 0.28125
    else:
        L.add("kcos_mid")
        qx = _f((ix - 0x00200000) << 32)
    return (1.0 - qx) - ((0.5 * z - qx) - zr_xy)


def _kernel_sin(x, y):
    z = x * x
    v = z * x
    r = _S1[0] + z * (_S1[1] + z * (_S1[2] + z * (_S1[3] + z * _S1[4])))
    return x - ((z * (0.5 * y - v * r) - y) - v * _S0)


def _fd_cos(x, L, call):
    fn = _floor(x * _f(0x3FE45F306DC9C883) + 0.5)
    t = x - fn * _f(0x3FF921FB54400000)
    w = fn * _f(0x3DD0B4611A600000)
    r = t - w
    w = fn * _f(0x3BA3198A2E037073) - ((t - r) - w)
    y0 = r - w
    y1 = (r - y0) - w
    if fn == 1.0:
        L.add(f"cos{call}_fn1")
        return -_kernel_sin(y0, y1)
    if fn == 2.0:
        L.add(f"cos{call}_fn2")
        return -_kernel_cos(y0, y1, L)
    L.add(f"cos{call}_fn0")  # fn == 0, or NaN
    return _kernel_cos(y0, y1, L)


# ------------------------------------------------------------------------------------------------ FastEigen3x3
def _cross(a, b):
    return (a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0])


def _dot(a, b):
    return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]


def _scaled(a, d):
    return (_quo(a[0], d), _quo(a[1], d), _quo(a[2], d))


def _eigenvector0(a, ev, L):
    r0, r1, r2 = (a[0] - ev, a[1], a[2]), (a[1], a[3] - ev, a[4]), (a[2], a[4], a[5] - ev)
    c01, c02, c12 = _cross(r0, r1), _cross(r0, r2), _cross(r1, r2)
    d0, d1, d2 = _dot(c01, c01), _dot(c02, c02), _dot(c12, c12)
    dmax, imax = d0, 0
    if d1 > dmax:
        dmax, imax = d1, 1
    elif d1 == dmax:
        L.add("ev0_tie_d0_d1")
    if d2 > dmax:
        imax = 2
    elif d2 == dmax and imax == 1:
        L.add("ev0_tie_d1_d2")
    L.add(f"ev0_imax{imax}")
    return _scaled((c01, c02, c12)[imax], _sqrt((d0, d1, d2)[imax]))


def _eigenvector1(a, e0, ev, L):
    if abs(e0[0]) > abs(e0[1]):
        L.add("ev1_x_first")
        inv = _quo(1.0, _sqrt(e0[0] * e0[0] + e0[2] * e0[2]))
        u = (-e0[2] * inv, 0.0, e0[0] * inv)
    else:
        L.add("ev1_y_first_equal" if abs(e0[0]) == abs(e0[1]) else "ev1_y_first")
        inv = _quo(1.0, _sqrt(e0[1] * e0[1] + e0[2] * e0[2]))
        u = (0.0, e0[2] * inv, -e0[1] * inv)
    v = _cross(e0, u)
    row0, row1, row2 = (a[0], a[1], a[2]), (a[1], a[3], a[4]), (a[2], a[4], a[5])
    au, av = (_dot(row0, u), _dot(row1, u), _dot(row2, u)), (_dot(row0, v), _dot(row1, v), _dot(row2, v))
    m00, m01, m11 = _dot(u, au) - ev, _dot(u, av), _dot(v, av) - ev
    a00, a01, a11 = abs(m00), abs(m01), abs(m11)
    if a00 >= a11:
        L.add("ev1_a00_ge_a11")
        if not ((a01 if a00 < a01 else a00) > 0.0):
            L.add("ev1_return_u_a00")
            return u
        if a00 >= a01:
            L.add("ev1_a00_ge_a01_equal" if a00 == a01 else "ev1_a00_ge_a01")
            if a00 == a01 and (m00 < 0.0) != (m01 < 0.0):
                L.add("ev1_a00_eq_a01_signs_differ")  # the only tie where the other branch gives another vector
            m01 = _quo(m01, m00)
            m00 = _quo(1.0, _sqrt(1.0 + m01 * m01))
            m01 = m01 * m00
        else:
            L.add("ev1_a00_lt_a01")
            m00 = _quo(m00, m01)
            m01 = _quo(1.0, _sqrt(1.0 + m00 * m00))
            m00 = m00 * m01
        cu, cv = m01, m00
    else:
        L.add("ev1_a00_lt_a11")
        if not ((a01 if a11 < a01 else a11) > 0.0):
            L.add("ev1_return_u_a11")
            return u
        if a11 >= a01:
            L.add("ev1_a11_ge_a01_equal" if a11 == a01 else "ev1_a11_ge_a01")
            m01 = _quo(m01, m11)
            m11 = _quo(1.0, _sqrt(1.0 + m01 * m01))
            m01 = m01 * m11
        else:
            L.add("ev1_a11_lt_a01")
            m11 = _quo(m11, m01)
            m01 = _quo(1.0, _sqrt(1.0 + m11 * m11))
            m11 = m11 * m01
        cu, cv = m11, m01
    return (cu * u[0] - cv * v[0], cu * u[1] - cv * v[1], cu * u[2] - cv * v[2])


def _axis(d):
    """The diagonal branch: the axis of the strictly smallest entry, else z."""
    if d[0] < d[1] and d[0] < d[2]:
        return 0
    if d[1] < d[0] and d[1] < d[2]:
        return 1
    return 2


def _ties(d):
    return {(i, j) for i in range(3) for j in range(i + 1, 3) if d[i] == d[j]}


def trace_fast_eigen3x3(cov):
    """(vector, labels): fast_eigen3x3 of the symmetric [3,3] cov, and the set of branch labels it took."""
    c = np.asarray(cov, np.float64).reshape(3, 3)
    cv = [float(c[0, 0]), float(c[0, 1]), float(c[0, 2]), float(c[1, 1]), float(c[1, 2]), float(c[2, 2])]
    L = set()
    full = [cv[0], cv[1], cv[2], cv[1], cv[3], cv[4], cv[2], cv[4], cv[5]]
    mc = full[0]
    for x in full[1:]:
        if x > mc:
            mc = x
    if mc < 0.0:
        L.add("mc_negative")
    if mc == 0.0:
        L.add("mc_zero_nonzero_entries" if any(x != 0.0 for x in full) else "mc_zero")
        return (0.0, 0.0, 0.0), L
    a = [_quo(x, mc) for x in cv]
    norm = (a[1] * a[1] + a[2] * a[2]) + a[4] * a[4]
    if not (norm > 0.0):
        d = (a[0] * mc, a[3] * mc, a[5] * mc)
        axis = _axis(d)
        if axis == 2:
            L.add("diag_z_smallest" if d[2] < d[0] and d[2] < d[1] else "diag_z_tie")
        else:
            L.add(("diag_x", "diag_y")[axis])
        raw = (cv[0], cv[3], cv[5])
        if _axis(raw) != axis:  # the rescale decided the axis: a tie it made, or one it undid
            L.add("diag_rescale_tie_created" if _ties(d) - _ties(raw) else "diag_rescale_tie_broken")
        return tuple(float(i == axis) for i in range(3)), L
    q = ((a[0] + a[3]) + a[5]) / 3.0
    b00, b11, b22 = a[0] - q, a[3] - q, a[5] - q
    p = _sqrt(((((b00 * b00) + b11 * b11) + b22 * b22) + norm * 2.0) / 6.0)
    c00 = b11 * b22 - a[4] * a[4]
    c01 = a[1] * b22 - a[4] * a[2]
    c02 = a[1] * a[4] - b11 * a[2]
    det = _quo((b00 * c00 - a[1] * c01) + a[2] * c02, (p * p) * p)
    hd = det * 0.5
    if math.isnan(hd):
        L.add("hd_nan")
    elif hd > 1.0:
        L.add("hd_clamp_high")
    elif hd < -1.0:
        L.add("hd_clamp_low")
    elif hd == 1.0:
        L.add("hd_one")
    elif hd == -1.0:
        L.add("hd_minus_one")
    elif hd == 0.0:
        L.add("hd_zero")
    hd = -1.0 if hd < -1.0 else hd
    hd = 1.0 if 1.0 < hd else hd
    angle = _fd_acos(hd, L) / 3.0
    beta2 = _fd_cos(angle, L, 1) * 2.0
    beta0 = _fd_cos(angle + 2.09439510239319549, L, 2) * 2.0
    beta1 = -(beta0 + beta2)
    ev0, ev1, ev2 = q + p * beta0, q + p * beta1, q + p * beta2
    if hd >= 0.0:
        L.add("hd_nonnegative")
        e2 = _eigenvector0(a, ev2, L)
        if ev2 < ev0 and ev2 < ev1:
            L.add("pos_return_e2")
            return e2, L
        e1 = _eigenvector1(a, e2, ev1, L)
        if ev1 < ev0 and ev1 < ev2:
            L.add("pos_return_e1")
            return e1, L
        L.add("pos_return_cross")
        return _cross(e1, e2), L
    L.add("hd_negative")  # hd < 0, or NaN
    e0 = _eigenvector0(a, ev0, L)
    if ev0 < ev1 and ev0 < ev2:
        L.add("neg_return_e0")
        return e0, L
    e1 = _eigenvector1(a, e0, ev1, L)
    if ev1 < ev0 and ev1 < ev2:
        L.add("neg_return_e1")
        return e1, L
    L.add("neg_return_cross")
    return _cross(e0, e1), L


# ------------------------------------------------------------------------------------------------ eigen cases
EIGEN_CASES = {
    # 32 points 2^-k apart at a large offset: per-point sum orders, hd = -1, an |m11| == |m01| tie
    'offset_cancellation': [(25043211.0078125, 25017625.0, 32802881.4921875), (25043211.0078125, 25017624.9921875, 32802881.4921875), (25043210.9921875, 25017625.0078125, 32802881.4921875), (25043211.0, 25017625.0078125, 32802881.5078125), (25043210.9921875, 25017625.0, 32802881.5078125), (25043210.9921875, 25017625.0078125, 32802881.5), (25043211.0, 25017625.0078125, 32802881.5), (25043210.9921875, 25017625.0078125, 32802881.5), (25043211.0, 25017625.0078125, 32802881.5078125), (25043211.0, 25017624.9921875, 32802881.4921875), (25043211.0078125, 25017625.0, 32802881.4921875), (25043210.9921875, 25017625.0078125, 32802881.5), (25043211.0, 25017625.0078125, 32802881.5), (25043211.0078125, 25017625.0, 32802881.4921875), (25043210.9921875, 25017624.9921875, 32802881.5), (25043211.0, 25017625.0078125, 32802881.5078125), (25043210.9921875, 25017625.0, 32802881.4921875), (25043211.0, 25017624.9921875, 32802881.5078125), (25043210.9921875, 25017625.0078125, 32802881.4921875), (25043211.0, 25017625.0078125, 32802881.5078125), (25043210.9921875, 25017625.0078125, 32802881.5), (25043210.9921875, 25017625.0078125, 32802881.5078125), (25043210.9921875, 25017625.0, 32802881.5078125), (25043211.0, 25017625.0, 32802881.5), (25043210.9921875, 25017624.9921875, 32802881.5078125), (25043211.0078125, 25017625.0078125, 32802881.5078125), (25043211.0, 25017625.0, 32802881.4921875), (25043211.0, 25017624.9921875, 32802881.5078125), (25043211.0, 25017625.0, 32802881.4921875), (25043211.0, 25017625.0, 32802881.5078125), (25043211.0078125, 25017624.9921875, 32802881.5), (25043211.0078125, 25017625.0, 32802881.5078125)],
    # cancellation leaves every entry of some rows <= 0: mc < 0, and mc == 0 with non-zero entries
    'offset_negative_max': [(-1076640.21875, -1024218.2813110352, -229941.4375), (-1076640.21875, -1024218.28125, -229941.4375), (-1076640.2188110352, -1024218.2811889648, -229941.4375), (-1076640.2188110352, -1024218.2811889648, -229941.4375), (-1076640.21875, -1024218.2811889648, -229941.43743896484), (-1076640.2186889648, -1024218.2813110352, -229941.43743896484), (-1076640.21875, -1024218.2811889648, -229941.4375), (-1076640.2186889648, -1024218.28125, -229941.43743896484), (-1076640.21875, -1024218.2811889648, -229941.4375), (-1076640.21875, -1024218.2813110352, -229941.4375), (-1076640.2188110352, -1024218.28125, -229941.43756103516), (-1076640.2186889648, -1024218.2811889648, -229941.4375), (-1076640.2186889648, -1024218.2813110352, -229941.4375), (-1076640.2186889648, -1024218.28125, -229941.43743896484), (-1076640.2188110352, -1024218.28125, -229941.43756103516)],
    # +-e1, +-e2, +-e3 with one y moved by 2^-535: norm subnormal, p*p*p == 0, det = 0/0
    'octahedron_nan': [(1.0, 8.89103499794031e-162, 0.0), (0.0, 1.0, 0.0), (0.0, 0.0, 1.0), (-1.0, -0.0, -0.0), (-0.0, -1.0, -0.0), (-0.0, -0.0, -1.0)],
    # the same moved by 2^-60: p below an ulp of q, hd == 0, |e0.x| == |e0.y|
    'octahedron_2m60': [(1.0, 8.673617379884035e-19, 0.0), (0.0, 1.0, 0.0), (0.0, 0.0, 1.0), (-1.0, 0.0, 0.0), (0.0, -1.0, 0.0), (0.0, 0.0, -1.0)],
    # a line with 2^-k jitter: hd == 1, |m11| < |m01|
    'needle': [(-7.9999847412109375, -8.0, -1.52587890625e-05), (-27.999984741210938, -27.999984741210938, -1.52587890625e-05), (1.52587890625e-05, -1.52587890625e-05, 1.52587890625e-05), (10.000015258789062, 9.999984741210938, -1.52587890625e-05), (9.999984741210938, 9.999984741210938, 0.0), (25.999984741210938, 26.0, -1.52587890625e-05), (12.0, 12.0, 0.0)],
    # a 2x2 block and an axis: det/2 below -1, d1 == d2
    'block_clamp_low': [(0.75, 0.25, 0.0), (0.25, 0.75, 0.0), (-0.75, -0.25, -0.0), (-0.25, -0.75, -0.0), (0.0, 0.0, 1.0), (-0.0, -0.0, -1.0)],
    # det/2 above 1
    'block_clamp_high': [(-0.125, 0.0, -0.625), (-0.625, 0.0, -0.125), (0.125, -0.0, 0.625), (0.625, -0.0, 0.125), (0.0, 0.5, 0.0), (-0.0, -0.5, -0.0)],
    # |m00| >= |m11| but |m00| < |m01| by rounding
    'block_a00_lt_a01': [(0.0, 0.125, -0.25), (0.0, -0.25, 0.125), (-0.0, -0.125, 0.25), (-0.0, 0.25, -0.125), (1.75, 0.0, 0.0), (-1.75, -0.0, -0.0)],
    # |m00| == |m01| with opposite signs: the one tie where > instead of >= gives the opposite vector
    'block_a00_eq_a01_signs_differ': [(0.0, 0.375, -0.5), (0.0, -0.5, 0.375), (-0.0, -0.375, 0.5),
                                      (-0.0, 0.5, -0.375), (2.5, 0.0, 0.0), (-2.5, -0.0, -0.0)],
    # |m00| == |m01| with equal signs: both branches give the same vector
    'block_a00_eq_a01':[(0.0, 0.125, 0.5), (0.0, 0.5, 0.125), (-0.0, -0.125, -0.5), (-0.0, -0.5, -0.125), (1.0, 0.0, 0.0), (-1.0, -0.0, -0.0)],
    # all points at the origin: the zero matrix
    'block_zero': [(0.0, 0.0, 0.0), (0.0, 0.0, 0.0), (-0.0, -0.0, -0.0), (-0.0, -0.0, -0.0), (0.0, 0.0, 0.0), (-0.0, -0.0, -0.0)],
    # +-a e1, +-b e2, +-c e3: a diagonal matrix, x smallest
    'axes_x': [(1.0, 0.0, 0.0), (0.0, 1.25, 0.0), (0.0, 0.0, 1.75), (-1.0, -0.0, -0.0), (-0.0, -1.25, -0.0), (-0.0, -0.0, -1.75)],
    # y smallest
    'axes_y': [(2.0, 0.0, 0.0), (0.0, 0.25, 0.0), (0.0, 0.0, 0.5), (-2.0, -0.0, -0.0), (-0.0, -0.25, -0.0), (-0.0, -0.0, -0.5)],
    # z strictly smallest
    'axes_z': [(1.75, 0.0, 0.0), (0.0, 2.0, 0.0), (0.0, 0.0, 0.5), (-1.75, -0.0, -0.0), (-0.0, -2.0, -0.0), (-0.0, -0.0, -0.5)],
    # x < y one ulp apart, equal after (A/mc)*mc: no strictly smallest entry, z
    'axes_rescale_tie': [(1.6412954979564338, 0.0, 0.0), (0.0, 1.641295497956434, 0.0), (0.0, 0.0, 3.924820095028968), (-1.6412954979564338, -0.0, -0.0), (-0.0, -1.641295497956434, -0.0), (-0.0, -0.0, -3.924820095028968)],
    # +-e1, +-e2, +-e3, +-(1,1,1): (I + 11^T)/4, eigenvalues (1, 1/4, 1/4)
    'cube_diagonal': [(1.0, 0.0, 0.0), (0.0, 1.0, 0.0), (0.0, 0.0, 1.0), (-1.0, -0.0, -0.0), (-0.0, -1.0, -0.0), (-0.0, -0.0, -1.0), (1.0, 1.0, 1.0), (-1.0, -1.0, -1.0)],
    # hd just below sqrt(2)/2: the second cos reduces to |y| > 0.78125
    'kcos_big_nonnegative': [(0.0, 1.0, 2.0), (2.0, 2.0, -2.0), (3.0, -3.0, 0.0), (-1.0, 1.0, 1.0), (0.0, -3.0, -2.0), (0.0, 0.0, -2.0)],
    # hd just above -sqrt(2)/2: the first cos keeps fn = 0 at angle > 0.78125
    'kcos_big_negative': [(2.0, -2.0, -2.0), (-3.0, 2.0, 2.0), (-3.0, -3.0, 3.0), (3.0, 0.0, 3.0), (2.0, -1.0, 1.0), (0.0, 1.0, 0.0), (2.0, 3.0, -1.0), (-3.0, 3.0, -1.0)],
}


def trace_normal(cov, count):
    """normals_kernel after the neighbour search: the identity for fewer than 3 neighbours, FastEigen3x3, and (0, 0, 1)
    for a vector whose ((x*x)+y*y)+z*z is 0 (a NaN vector stays)."""
    if count < 3:
        cov = np.eye(3)
    v, L = trace_fast_eigen3x3(cov)
    if _dot(v, v) == 0.0:
        L.add("normal_zero_vector")
        v = (0.0, 0.0, 1.0)
    return v, L


LABELS = frozenset("""
    mc_zero mc_zero_nonzero_entries mc_negative
    diag_x diag_y diag_z_smallest diag_z_tie diag_rescale_tie_created diag_rescale_tie_broken
    hd_nonnegative hd_negative hd_one hd_minus_one hd_zero hd_clamp_high hd_clamp_low hd_nan
    pos_return_e2 pos_return_e1 pos_return_cross neg_return_e0 neg_return_e1 neg_return_cross
    ev0_imax0 ev0_imax1 ev0_imax2 ev0_tie_d0_d1 ev0_tie_d1_d2
    ev1_x_first ev1_y_first ev1_y_first_equal ev1_a00_ge_a11 ev1_a00_lt_a11
    ev1_a00_ge_a01 ev1_a00_ge_a01_equal ev1_a00_lt_a01 ev1_a11_ge_a01 ev1_a11_ge_a01_equal ev1_a11_lt_a01
    ev1_a00_eq_a01_signs_differ
    ev1_return_u_a00 ev1_return_u_a11
    acos_one acos_minus_one acos_small acos_negative acos_positive
    cos1_fn0 cos1_fn1 cos1_fn2 cos2_fn0 cos2_fn1 cos2_fn2
    kcos_small kcos_mid kcos_big
    normal_zero_vector
""".split())

UNREACHABLE = {
    "diag_rescale_tie_broken":
        "x -> (x/mc)*mc is a function of x alone and monotone (mc != 0, each rounding monotone), so equal diagonal entries "
        "stay equal and unequal ones can only merge",
    "pos_return_e2":
        "hd >= 0 gives angle in [0, pi/6]: beta2 >= 1.73 > 0 > -1 >= beta0, and p >= 0, so ev2 = q + p*beta2 >= ev0 "
        "under monotone rounding",
    "pos_return_e1":
        "hd >= 0: beta1 - beta0 = 2*sqrt(3)*sin(angle) >= 1.7e-8 once angle > 0 (the least positive fd_acos(hd) is 1.49e-8), "
        "and at angle 0 the rounded betas are beta0 = -1 - 2^-51 < beta1 = -1 + 2^-51; p >= 0, so ev1 >= ev0",
    "neg_return_e1":
        "hd < 0 gives angle in (pi/6, pi/3]: beta1 in (0, 1] and beta0 in [-2, -1.73), so ev1 >= ev0 with p >= 0; a NaN "
        "hd fails every comparison",
    "cos1_fn2":
        "the first cos takes angle = fd_acos(hd)/3 <= (pi + 2^-52)/3 < 1.05, so fn = floor(angle*2/pi + 0.5) <= 1",
    "ev1_return_u_a00":
        "needs |m00| >= |m11| with m00 = m11 = 0 and m01 zero or NaN: a NaN m00 or m11 fails the >= and takes the other "
        "branch, and a finite exact zero needs the rounded ev1 to equal both u.Au and v.Av with u.Av == 0; no case reaches it",
}


# ------------------------------------------------------------------------------------------------ k-NN cases
KNN_CELLS = (1.0, 0.1, 2.0 ** -20)
KNN_ORIGINS = {1.0: (3.0, -5.0, 7.0), 0.1: (0.3, -7.7, 1e3), 2.0 ** -20: (1e3, 1e3, -1e3)}
KNN_KS = (2, 5, 20, 32)
RINGS = (2, 3, 6)


def sq_dist(q, p):
    d = (q[0] - p[0], q[1] - p[1], q[2] - p[2])
    return (d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]


def cell_of(x, o, h):
    """floor((x - o)/h), as the grid build and query_cell round it (before clamping)."""
    return math.floor((x - o) / h)


def ring_of(q, p, origin, h):
    """The Chebyshev ring of p's cell around q's cell."""
    return max(abs(cell_of(p[a], origin[a], h) - cell_of(q[a], origin[a], h)) for a in range(3))


def _steps(x, n):
    out, up, dn = [x], x, x
    for _ in range(n):
        up, dn = math.nextafter(up, math.inf), math.nextafter(dn, -math.inf)
        out += [up, dn]
    return out


@functools.lru_cache(maxsize=None)
def _ring_geometry(K, h, relation):
    """(origin, c, qx, px): a query and a point P along +x with P in ring K and d2 against lb0 = fl(fl((K-1)*h)^2) as
    relation says.  Queries sit within 3 ulp of a cell's upper face and P within 3 ulp of (K-1)*h beyond; the x origin
    steps by 0.37 until the cell arithmetic gives the relation, or None after 200 origins."""
    lb = ((K - 1) * h) * ((K - 1) * h)
    for j in range(200):
        o = (KNN_ORIGINS[h][0] + 0.37 * j,) + KNN_ORIGINS[h][1:]
        for c in range(4, 40):
            for qx in _steps(o[0] + (c + 1) * h, 3):
                for px in _steps(qx + (K - 1) * h, 3):
                    if cell_of(px, o[0], h) - cell_of(qx, o[0], h) != K:
                        continue
                    d2 = (px - qx) * (px - qx)
                    if {"<": d2 < lb, "==": d2 == lb, ">": d2 > lb}[relation]:
                        return o, c, qx, px
    return None


def ring_bound_case(K, k, h, relation):
    """The k-th neighbour R at squared distance D2 against lb0 = fl(fl((K-1)*h)^2), relation '<', '==' or '>', with a
    point P of lower index in ring K at the same D2: a search that stops before ring K returns R instead of P.  P lies
    along +x from the query, R along +y in ring K-1 or closer, and k-1 fillers along +z within a quarter cell.  Returns
    (ref, query, origin, dims), or None where the cell's arithmetic cannot give the relation: an exact h puts every
    ring-K point strictly beyond (K-1)*h, and for h = 0.1 only rounding in the cell index can bring one within it."""
    g = _ring_geometry(K, h, relation)
    if g is None:
        return None
    o, c, qx, px = g
    yq, zq = o[1] + 8.5 * h, o[2] + 8.5 * h
    q, p = (qx, yq, zq), (px, yq, zq)
    d2 = sq_dist(q, p)
    for ry in _steps(yq + (px - qx), 64):
        r = (qx, ry, zq)
        if sq_dist(q, r) == d2 and ring_of(q, r, o, h) < K:
            break
    else:
        return None
    fill = [(qx, yq, zq + h * j / (4 * k)) for j in range(k - 1)]
    ref = np.array([p, r] + fill + [o, (o[0] + (c + K + 4) * h, o[1] + 16 * h, o[2] + 16 * h)])
    return ref, np.array([q]), np.array(o), [c + K + 5, 17, 17]


def shell_case(k, seed=0):
    """The 84 integer points with x*x + y*y + z*z = 50 around an integer query, in shuffled index order, plus a farther
    shell: all 84 tie, so the k lowest indices win."""
    g = np.arange(-8, 9)
    pts = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)
    r2 = (pts * pts).sum(1)
    shell = pts[r2 == 50]
    far = pts[r2 == 51][:30]
    rng = np.random.default_rng(seed)
    q = np.array([[20.0, 20.0, 20.0]])
    ref = np.concatenate([shell, far])[rng.permutation(len(shell) + len(far))] + q
    return ref.astype(np.float64), q


def duplicates_case(k):
    """k + 8 exact copies of the query (d2 = 0) among other points: the k lowest indices of the copies win."""
    rng = np.random.default_rng(k)
    q = np.array([[1.25, -3.5, 2.0]])
    other = q + rng.integers(-6, 7, size=(60, 3)) * 0.25
    ref = np.concatenate([other[:30], np.repeat(q, k + 8, axis=0), other[30:]])
    return ref, q
