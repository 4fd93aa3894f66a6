"""The edge cases of tests/normals_edge_cases.py on the CPU: the branch-recording transliteration of FastEigen3x3 equals
the vectorised oracle (tests/normals_oracle.py) bit for bit, the eigen cases reach every label not proven unreachable,
and each k-NN case is where its docstring puts it."""
import math

import numpy as np
import pytest

from tests import normals_edge_cases as ec
from tests import normals_oracle as no


def _same(a, b):
    """Equal bits, with NaN equal to NaN by position (the device and x86 encode NaN differently)."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    nan = np.isnan(a)
    return a.shape == b.shape and np.array_equal(nan, np.isnan(b)) and np.array_equal(a[~nan].view(np.uint64),
                                                                                      b[~nan].view(np.uint64))


def _case_covariances(pts):
    pts = np.asarray(pts, np.float64)
    return no.covariances(pts, no.knn(pts, pts, len(pts))[1])


def test_trace_equals_vectorised_oracle_on_random_matrices():
    rng = np.random.default_rng(20)
    n = 100_000
    M = rng.normal(size=(n, 3, 3)) * rng.uniform(1e-3, 1e3, size=(n, 1, 1))
    A = M + M.transpose(0, 2, 1)  # indefinite
    A[: n // 2] = M[: n // 2] @ M[: n // 2].transpose(0, 2, 1)  # positive semi-definite
    A[:1000] = np.round(A[:1000] * 4) / 4  # small dyadic entries: exact ties
    want = no.fast_eigen3x3(A)
    got = np.array([ec.trace_fast_eigen3x3(a)[0] for a in A])
    assert _same(got, want)


@pytest.mark.parametrize("name", sorted(ec.EIGEN_CASES))
def test_eigen_case_trace_equals_oracle(name):
    pts = np.asarray(ec.EIGEN_CASES[name], np.float64)
    assert 3 <= len(pts) <= no.MAX_K
    cov = _case_covariances(pts)
    got = np.array([ec.trace_normal(c, len(pts))[0] for c in cov])
    assert _same(got, no.estimate_normals(pts, len(pts)))


def test_labels_cover_everything_reachable():
    assert set(ec.UNREACHABLE) <= ec.LABELS and all(ec.UNREACHABLE.values())
    seen = set()
    for pts in ec.EIGEN_CASES.values():
        for c in _case_covariances(pts):
            seen |= ec.trace_normal(c, len(pts))[1]
    assert seen <= ec.LABELS
    assert seen == ec.LABELS - set(ec.UNREACHABLE)


def test_trace_labels_of_named_cases():
    def labels(name):
        pts = ec.EIGEN_CASES[name]
        return set().union(*[ec.trace_normal(c, len(pts))[1] for c in _case_covariances(pts)])

    assert {"hd_nan", "cos2_fn0", "ev1_return_u_a11", "neg_return_cross"} <= labels("octahedron_nan")
    assert {"hd_one", "ev0_tie_d0_d1", "ev1_y_first_equal"} <= labels("cube_diagonal")
    assert {"diag_rescale_tie_created", "diag_z_tie"} == labels("axes_rescale_tie")
    assert "ev1_a00_ge_a01_equal" in labels("block_a00_eq_a01")
    assert labels("block_zero") == {"mc_zero", "normal_zero_vector"}
    # the NaN normal: every point of the octahedron gets it on both sides
    pts = np.asarray(ec.EIGEN_CASES["octahedron_nan"])
    assert np.isnan(no.estimate_normals(pts, len(pts))).all()
    # fewer than 3 neighbours: the identity, whose normal is z
    assert ec.trace_normal(np.full((3, 3), np.nan), 2)[0] == (0.0, 0.0, 1.0)


def test_unreachable_bounds_hold_numerically():
    """The numbers the UNREACHABLE proofs use: the betas at angle 0 and at the least positive angle, the largest angle."""
    L = set()
    b2, b0 = ec._fd_cos(0.0, L, 1) * 2.0, ec._fd_cos(0.0 + 2.09439510239319549, L, 2) * 2.0
    assert (b2, b0, -(b0 + b2)) == (2.0, -1.0 - 2.0 ** -51, -1.0 + 2.0 ** -51)
    angle = ec._fd_acos(math.nextafter(1.0, 0.0), L) / 3.0
    assert angle > 4.9e-9
    for a in (angle, math.pi / 12, math.pi / 6):
        b2, b0 = ec._fd_cos(a, L, 1) * 2.0, ec._fd_cos(a + 2.09439510239319549, L, 2) * 2.0
        assert -(b0 + b2) - b0 >= 1.7e-8 and b2 > 1.7 and b0 <= -1.0
    top = ec._fd_acos(-1.0, L) / 3.0
    assert math.floor(top * 0.6366197723675814 + 0.5) == 1 and top < 1.05


# ------------------------------------------------------------------------------------------------ k-NN cases
RING_CASES_PRESENT = {
    (1.0, 2): {"==", ">"}, (1.0, 3): {"==", ">"}, (1.0, 6): {"=="},
    (0.1, 2): set(), (0.1, 3): set(), (0.1, 6): {"=="},
    (2.0 ** -20, 2): {">"}, (2.0 ** -20, 3): {">"}, (2.0 ** -20, 6): {">"},
}


@pytest.mark.parametrize("k", ec.KNN_KS)
def test_ring_bound_cases_are_where_they_say(k):
    for (h, K), present in RING_CASES_PRESENT.items():
        for rel in ("<", "==", ">"):
            case = ec.ring_bound_case(K, k, h, rel)
            assert (case is not None) == (rel in present), (h, K, rel)
            if case is None:
                continue
            ref, q, o, dims = case
            lb = ((K - 1) * h) * ((K - 1) * h)
            d2, idx = no.knn_brute(q, ref, k)
            # P (index 0) in ring K and R (index 1) closer in ring, tied at the k-th place
            assert ec.ring_of(q[0], ref[0], o, h) == K and ec.ring_of(q[0], ref[1], o, h) < K
            assert d2[0, k - 1] == ec.sq_dist(q[0], ref[0]) == ec.sq_dist(q[0], ref[1])
            assert {"<": d2[0, k - 1] < lb, "==": d2[0, k - 1] == lb, ">": d2[0, k - 1] > lb}[rel]
            assert idx[0, k - 1] == 0 and 1 not in idx[0]
            # the grid holds every point
            for a in range(3):
                cells = [ec.cell_of(p[a], o[a], h) for p in ref]
                assert min(cells) >= 0 and max(cells) < dims[a]


@pytest.mark.parametrize("k", ec.KNN_KS)
def test_shell_and_duplicate_cases(k):
    ref, q = ec.shell_case(k)
    d2, idx = no.knn_brute(q, ref, k)
    shell = np.nonzero(ec_d2(q, ref) == 50.0)[0]
    assert len(shell) == 84 and (d2 == 50.0).all() and idx[0].tolist() == sorted(shell)[:k]
    ref, q = ec.duplicates_case(k)
    d2, idx = no.knn_brute(q, ref, k)
    assert (d2 == 0.0).all() and idx[0].tolist() == list(range(30, 30 + k))


def ec_d2(q, ref):
    return no.sq_dist(q[0][None, :], ref)
