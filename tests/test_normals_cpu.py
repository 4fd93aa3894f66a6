"""k nearest neighbours and normal estimation without a GPU: the numpy oracle (tests/normals_oracle.py) against scipy's
cKDTree and numpy's eigh, its fdlibm acos / cos against the host libm, the PLY layout with normals, and the C entry
points' refusals."""
import ctypes as C
import math

import numpy as np
import pytest

from gs2mesh_b200 import _lib
from tests import normals_oracle as no


def _tie_free(dist, k):
    """Rows whose k-th distance differs from the (k+1)-th: their k nearest form a unique set."""
    return dist[:, k - 1] < dist[:, k]


@pytest.mark.parametrize("k", [1, 2, 20, 32])
def test_knn_brute_equals_kd_tree(k):
    from scipy.spatial import cKDTree

    rng = np.random.default_rng(k)
    ref = np.concatenate([rng.uniform(-1, 1, size=(1500, 3)), rng.integers(-3, 4, size=(500, 3)) * 0.25])
    q = np.concatenate([rng.uniform(-1.2, 1.2, size=(700, 3)), ref[:100], rng.integers(-3, 4, size=(200, 3)) * 0.25])
    d2, idx = no.knn_brute(q, ref, k)
    kd, ki = cKDTree(ref).query(q, k)
    kd, ki = kd.reshape(len(q), k), ki.reshape(len(q), k)
    assert np.array_equal(np.sqrt(d2), kd)
    assert np.array_equal(d2, no.sq_dist(q[:, None, :], ref[idx]))
    free = _tie_free(cKDTree(ref).query(q, k + 1)[0], k)
    assert free.sum() > 0.5 * len(q) and (~free).sum() > 0  # the lattice points make ties at the k-th place
    assert all(set(a) == set(b) for a, b in zip(idx[free], ki[free]))
    # (d2, index) order: ties go to the lower index
    same = d2[:, 1:] == d2[:, :-1]
    assert (idx[:, 1:][same] > idx[:, :-1][same]).all()


def test_knn_through_kd_tree_equals_brute_force():
    rng = np.random.default_rng(7)
    for ref in (rng.normal(size=(4000, 3)), rng.integers(0, 6, size=(3000, 3)).astype(np.float64),
                np.repeat(rng.normal(size=(300, 3)), 7, axis=0)):
        q = np.concatenate([ref[::3], rng.normal(size=(300, 3)) * 2, [[np.nan, 0, 0], [0, np.inf, 0]]])
        for k in (1, 20, 32):
            a, b = no.knn(q, ref, k), no.knn_brute(q, ref, k)
            assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    d2, idx = no.knn(q, ref[:5], 20)  # fewer reference points than k, and non-finite queries: padding
    assert (idx[:, 5:] == -1).all() and np.isinf(d2[:, 5:]).all() and (idx[:-2, :5] >= 0).all()
    assert (idx[-2:] == -1).all() and np.isinf(d2[-2:]).all()
    with pytest.raises(ValueError):
        no.knn(q, ref, 33)


def test_fdlibm_acos_cos_within_an_ulp():
    rng = np.random.default_rng(0)
    x = np.concatenate([rng.uniform(-1, 1, 100000), [-1.0, 1.0, 0.5, -0.5, 0.0, -0.0, 1e-300, np.nextafter(1.0, 0)]])
    a = no.acos(x)
    ref = np.array([math.acos(v) for v in x])
    assert (np.abs(a - ref) <= np.spacing(ref)).all()
    y = np.concatenate([rng.uniform(0, math.pi, 100000), [0.0, math.pi / 4, math.pi / 2, 2.0943951023931955, math.pi]])
    c = no.cos(y)
    ref = np.array([math.cos(v) for v in y])
    assert (np.abs(c - ref) <= np.spacing(np.abs(ref))).all()
    assert np.isnan(no.acos(np.nan)) and np.isnan(no.cos(np.nan))


def test_fast_eigen3x3_smallest_eigenvector_of_random_psd():
    rng = np.random.default_rng(1)
    M = rng.normal(size=(20000, 3, 3)) * rng.uniform(1e-3, 1e3, size=(20000, 1, 1))
    A = M @ M.transpose(0, 2, 1)
    v = no.fast_eigen3x3(A)
    w, V = np.linalg.eigh(A)
    gap = w[:, 1] - w[:, 0] > 1e-6 * w[:, 2]  # a well-separated smallest eigenvalue pins the vector
    assert gap.mean() > 0.99
    assert (np.abs((v * V[:, :, 0]).sum(1))[gap] >= 1 - 1e-12).all()
    assert np.abs(np.linalg.norm(v, axis=1) - 1).max() < 1e-14


SPECIAL = {
    "diagonal": (np.diag([3.0, 1.0, 2.0]), [0.0, 1.0, 0.0]),
    "diagonal_tie": (np.diag([1.0, 1.0, 2.0]), [0.0, 0.0, 1.0]),  # no strictly smallest entry: z
    "isotropic": (np.eye(3) * 2.0, [0.0, 0.0, 1.0]),
    "rank2": (np.outer([1, 0, 1], [1, 0, 1]) + np.outer([0, 1, 1], [0, 1, 1]) * 1.0, None),
    "rank1": (np.outer([1, 2, 3], [1, 2, 3]) * 1.0, None),
    "zero": (np.zeros((3, 3)), [0.0, 0.0, 0.0]),
}


@pytest.mark.parametrize("scale", [1.0, 1e-300, 1e150])
@pytest.mark.parametrize("case", sorted(SPECIAL))
def test_fast_eigen3x3_special_matrices(case, scale):
    """Diagonal matrices give the axis of the strictly smallest entry (else z), a zero matrix the zero vector, a rank-2
    matrix its null vector and a rank-1 matrix a unit vector orthogonal to its range; scaling by 1e-300 or 1e150 keeps
    every result (FastEigen3x3 divides by the largest entry first)."""
    A, want = SPECIAL[case]
    v = no.fast_eigen3x3((A * scale)[None])[0]
    if want is not None:
        assert v.tolist() == want
    elif case == "rank2":
        null = np.cross([1, 0, 1], [0, 1, 1]) / math.sqrt(3)
        assert abs(v @ null) >= 1 - 1e-12
    else:
        assert abs(v @ np.array([1, 2, 3]) / math.sqrt(14)) <= 1e-12 and abs(np.linalg.norm(v) - 1) < 1e-14
    if case == "zero":
        assert no.estimate_normals(np.zeros((5, 3)), 4).tolist() == [[0.0, 0.0, 1.0]] * 5


def test_covariance_cumulants_and_small_neighbourhoods():
    pts = np.array([[0.0, 0, 0], [1, 0, 0], [0, 2, 0], [0, 0, 3], [1, 1, 1]])
    cov = no.covariances(pts, np.array([[0, 1, 2, 3], [4, 1, -1, -1], [0, -1, -1, -1]]))
    x = pts[[0, 1, 2, 3]]
    m = x.sum(0) / 4
    c = np.zeros((3, 3))
    for a in range(3):
        for b in range(3):
            c[a, b] = (x[:, a] * x[:, b]).sum() / 4 - m[a] * m[b]
    assert np.array_equal(cov[0], c)
    assert np.array_equal(cov[1], np.eye(3)) and np.array_equal(cov[2], np.eye(3))  # fewer than 3 neighbours
    plane = np.random.default_rng(2).uniform(-1, 1, size=(400, 3)) * [1, 1, 0]
    n = no.estimate_normals(plane, 20)
    assert (np.abs(n[:, 2]) > 1 - 1e-12).all()


def test_point_cloud_ply_with_normals_layout(tmp_path):
    from gs2mesh_b200.io import write_point_cloud_ply

    rng = np.random.default_rng(3)
    p, c, nrm = rng.normal(size=(50, 3)), rng.uniform(size=(50, 3)), rng.normal(size=(50, 3))
    with_n = open(write_point_cloud_ply(str(tmp_path / "n.ply"), p, c, nrm), "rb").read()
    plain = open(write_point_cloud_ply(str(tmp_path / "p.ply"), p, c), "rb").read()
    head, body = with_n.split(b"end_header\n")
    assert head.decode().splitlines()[3:] == ["property double x", "property double y", "property double z",
                                              "property double nx", "property double ny", "property double nz",
                                              "property uchar red", "property uchar green", "property uchar blue"]
    rows = np.frombuffer(body, dtype=[("xyz", "<f8", 3), ("n", "<f8", 3), ("rgb", "u1", 3)])
    assert np.array_equal(rows["n"], nrm) and np.array_equal(rows["xyz"], p)
    stripped = head.replace(b"property double nx\nproperty double ny\nproperty double nz\n", b"") + b"end_header\n"
    stripped += np.ascontiguousarray(rows[["xyz", "rgb"]]).astype([("xyz", "<f8", 3), ("rgb", "u1", 3)]).tobytes()
    assert stripped == plain  # everything but the normals is what the writer gives without them


def test_c_entry_points_refuse_bad_arguments(gsb_lib):
    L = gsb_lib
    fake = C.c_void_p(256)  # never dereferenced: every refusal happens before any device work
    g = _lib.GsbPointGrid((C.c_double * 3)(0, 0, 0), 1.0, (C.c_int32 * 3)(1, 1, 1), 256, 1, 256, 256)
    for k in (0, -1, 33, 1 << 30):
        assert L.gsb_eval_knn(C.byref(g), fake, 10, k, fake, fake, None) == _lib.GSB_ERR_INVALID
        assert b"1..32" in L.gsb_last_error()
        assert L.gsb_eval_estimate_normals(C.byref(g), fake, 10, k, fake, None) == _lib.GSB_ERR_INVALID
    assert L.gsb_eval_knn(C.byref(g), fake, -1, 20, fake, fake, None) == _lib.GSB_ERR_INVALID
    assert L.gsb_eval_estimate_normals(C.byref(g), fake, -1, 20, fake, None) == _lib.GSB_ERR_INVALID
    for args in ((None, fake, fake), (fake, None, fake), (fake, fake, None)):
        assert L.gsb_eval_knn(C.byref(g), args[0], 10, 20, args[1], args[2], None) == _lib.GSB_ERR_INVALID
    assert L.gsb_eval_estimate_normals(C.byref(g), None, 10, 20, fake, None) == _lib.GSB_ERR_INVALID
    assert L.gsb_eval_estimate_normals(C.byref(g), fake, 10, 20, None, None) == _lib.GSB_ERR_INVALID
    assert L.gsb_eval_knn(None, fake, 10, 20, fake, fake, None) == _lib.GSB_ERR_INVALID
    assert L.gsb_eval_estimate_normals(None, fake, 10, 20, fake, None) == _lib.GSB_ERR_INVALID
    big = _lib.GsbPointGrid((C.c_double * 3)(0, 0, 0), 1.0, (C.c_int32 * 3)((1 << 21) + 1, 1, 1), 256, 1, 256, 256)
    assert L.gsb_eval_knn(C.byref(big), fake, 10, 20, fake, fake, None) == _lib.GSB_ERR_INVALID
    assert L.gsb_eval_estimate_normals(C.byref(big), fake, 10, 20, fake, None) == _lib.GSB_ERR_INVALID
    # nothing to do: accepted without touching the device
    assert L.gsb_eval_knn(C.byref(g), None, 0, 32, None, None, None) == _lib.GSB_OK
    assert L.gsb_eval_estimate_normals(C.byref(g), None, 0, 1, None, None) == _lib.GSB_OK
    assert _lib.KNN_MAX_K == 32
