"""Tanks and Temples evaluation without a GPU: the oracle (oracle/tnt_oracle.py) against scalar restatements, the host
steps of gs2mesh_b200.tnt (readers, RANSAC alignment, F-score, CLI) and the C entry points' refusals."""
import bisect
import ctypes as C
import math
import os
from fractions import Fraction

import numpy as np
import pytest

from gs2mesh_b200 import _lib
from gs2mesh_b200 import tnt
from oracle import tnt_oracle as to

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tnt")


# ------------------------------------------------------------------------------------------------------------ crop
def _crop_scalar(points, axis, amin, amax, poly):
    """CropInPolygon's loop, one point at a time: crossings in Python floats, std::sort, std::lower_bound."""
    u, v, w = {"x": (1, 2, 0), "y": (0, 2, 1), "z": (0, 1, 2)}[axis.lower()]
    keep = []
    for p in points:
        p = [float(c) for c in p]
        if p[w] < amin or p[w] > amax:
            keep.append(False)
            continue
        nodes = []
        for i in range(len(poly)):
            j = (i + 1) % len(poly)
            Pi, Pj = [float(c) for c in poly[i]], [float(c) for c in poly[j]]
            if (Pi[v] < p[v] and Pj[v] >= p[v]) or (Pj[v] < p[v] and Pi[v] >= p[v]):
                nodes.append(Pi[u] + (p[v] - Pi[v]) / (Pj[v] - Pi[v]) * (Pj[u] - Pi[u]))
        nodes.sort()
        keep.append(bisect.bisect_left(nodes, p[u]) % 2 == 1)
    return np.array(keep)


POLYGONS = {
    "square": [[0, 0, 0], [2, 0, 0], [2, 2, 0], [0, 2, 0]],
    "concave": [[0, 0, 0], [4, 0, 0], [4, 4, 0], [2, 1, 0], [0, 4, 0]],
    "bowtie": [[0, 0, 0], [2, 2, 0], [2, 0, 0], [0, 2, 0]],  # self-intersecting
    "star": [[np.cos(k * 4 * np.pi / 5), np.sin(k * 4 * np.pi / 5), 0.3] for k in range(5)],
    "thirds": [[0.1, 0.2, 0], [0.7, 0.3, 0], [0.3, 0.9, 0]],
}


def crop_cases(rng, poly, axis):
    """Points on vertices, on horizontal edges, on the slab faces, and random ones, placed in the (u, v, w) frame."""
    u, v, w = {"x": (1, 2, 0), "y": (0, 2, 1), "z": (0, 1, 2)}[axis.lower()]
    P = np.asarray(poly, dtype=np.float64)
    uv = [P[:, [0, 1]]]
    for i in range(len(P)):  # edge midpoints and vertices
        j = (i + 1) % len(P)
        uv.append(((P[i, :2] + P[j, :2]) / 2)[None])
        uv.append((P[i, :2] * 0.25 + P[j, :2] * 0.75)[None])
    lo, hi = P[:, :2].min(0) - 0.5, P[:, :2].max(0) + 0.5
    uv.append(rng.uniform(lo, hi, size=(400, 2)))
    uv.append(np.round(rng.uniform(lo, hi, size=(200, 2)) * 4) / 4)  # on a lattice through the vertices
    uv = np.concatenate(uv)
    ws = np.array([-1.0, -0.5, 0.0, 0.25, 1.0, 1.5, np.nextafter(-0.5, -1), np.nextafter(1.0, 2)])
    out = np.zeros((len(uv) * len(ws), 3))
    out[:, u] = np.repeat(uv[:, 0], len(ws))
    out[:, v] = np.repeat(uv[:, 1], len(ws))
    out[:, w] = np.tile(ws, len(uv))
    # the polygon in the same frame: its (x, y) become (u, v)
    Q = np.zeros_like(P)
    Q[:, u], Q[:, v], Q[:, w] = P[:, 0], P[:, 1], P[:, 2]
    return out, Q


@pytest.mark.parametrize("axis", ["x", "y", "z", "X", "Y", "Z"])
@pytest.mark.parametrize("name", sorted(POLYGONS))
def test_crop_oracle_matches_scalar_loop(axis, name):
    rng = np.random.default_rng(len(name) * 7 + ord(axis))
    pts, poly = crop_cases(rng, POLYGONS[name], axis)
    got = to.crop_mask(pts, axis, -0.5, 1.0, poly)
    ref = _crop_scalar(pts, axis, -0.5, 1.0, poly)
    assert np.array_equal(got, ref)
    assert 0 < got.sum() < len(got)


def test_crop_edge_rules():
    poly = [[0, 0, 0], [2, 0, 0], [2, 2, 0], [0, 2, 0]]
    pts = np.array([[0, 0, 0], [1, 0, 0], [1, 2, 0], [0, 1, 0], [2, 1, 0], [1, 1, -0.5], [1, 1, 1.0], [1, 1, 1.0000001]])
    # the lower horizontal edge has no crossings (dropped), the upper one two (kept); the left edge's crossing is not
    # strictly below p_u (dropped), the right edge's is (kept); the slab faces are inclusive
    assert to.crop_mask(pts, "z", -0.5, 1.0, poly).tolist() == [False, False, True, False, True, True, True, False]
    assert np.array_equal(to.crop_mask(pts, "z", -0.5, 1.0, poly), _crop_scalar(pts, "z", -0.5, 1.0, poly))


# ----------------------------------------------------------------------------------------------------------- voxel
def _voxel_brute(points, vs):
    p = [tuple(float(c) for c in q) for q in points]
    lo = [min(q[a] for q in p) - vs * 0.5 for a in range(3)]
    acc = {}
    for q in p:
        key = tuple(int(math.floor((q[a] - lo[a]) / vs)) for a in range(3))
        s, n = acc.get(key, ([0.0, 0.0, 0.0], 0))
        acc[key] = ([s[a] + q[a] for a in range(3)], n + 1)
    keys = sorted(acc)
    return np.array([[s / acc[k][1] for s in acc[k][0]] for k in keys]).reshape(-1, 3), np.array(keys).reshape(-1, 3)


@pytest.mark.parametrize("case", ["random", "boundaries", "one", "duplicates", "far"])
def test_voxel_oracle_matches_brute_force(case):
    rng = np.random.default_rng(5)
    vs = 0.25
    if case == "random":
        pts = rng.normal(size=(3000, 3))
    elif case == "boundaries":  # exactly on voxel faces relative to lo = min - vs/2
        pts = np.concatenate([np.zeros((1, 3)), rng.integers(-8, 8, size=(2000, 3)) * (vs / 2)])
    elif case == "one":
        pts = np.array([[1.5, -2.0, 3.25]])
    elif case == "duplicates":
        pts = np.repeat(rng.normal(size=(50, 3)), 7, axis=0)[rng.permutation(350)]
    else:
        pts = rng.normal(size=(1000, 3)) * 0.3 + np.array([1e5, -3e4, 7.0])
    got, keys = to.voxel_down_sample(pts, vs)
    ref, rkeys = _voxel_brute(pts, vs)
    assert np.array_equal(keys, rkeys)
    assert np.array_equal(got.view(np.uint64), ref.view(np.uint64))


def test_voxel_too_small_raises():
    with pytest.raises(ValueError, match="too small"):
        to.voxel_down_sample(np.array([[0.0, 0, 0], [1e3, 0, 0]]), 1e-7)


# --------------------------------------------------------------------------------------------------------- umeyama
def _rot():
    # exact rational rotation: (3/5, 4/5) about z, then (5/13, 12/13) about x
    a = [[Fraction(3, 5), Fraction(-4, 5), 0], [Fraction(4, 5), Fraction(3, 5), 0], [0, 0, 1]]
    b = [[1, 0, 0], [0, Fraction(5, 13), Fraction(-12, 13)], [0, Fraction(12, 13), Fraction(5, 13)]]
    return [[sum(Fraction(b[i][k]) * a[k][j] for k in range(3)) for j in range(3)] for i in range(3)]


def _moments_exact(src, dst):
    n = len(src)
    mu_s = [sum(p[k] for p in src) / n for k in range(3)]
    mu_d = [sum(p[k] for p in dst) / n for k in range(3)]
    second = [sum((q[j] - mu_d[j]) * (p[k] - mu_s[k]) for p, q in zip(src, dst)) for j in range(3) for k in range(3)]
    second += [sum((p[k] - mu_s[k]) ** 2 for p in src) for k in range(3)]
    return mu_s, mu_d, second


@pytest.mark.parametrize("umeyama", [to.umeyama, tnt.umeyama])
def test_umeyama_recovers_exact_similarity(umeyama):
    rng = np.random.default_rng(9)
    src = [[Fraction(int(x), 8) for x in row] for row in rng.integers(-40, 40, size=(30, 3))]
    R, c, t = _rot(), Fraction(7, 4), [Fraction(1, 2), Fraction(-3), Fraction(5, 8)]
    dst = [[c * sum(R[j][k] * p[k] for k in range(3)) + t[j] for j in range(3)] for p in src]
    mu_s, mu_d, second = _moments_exact(src, dst)
    sums = np.array([0.0] + [float(sum(p[k] for p in src)) for k in range(3)] + [float(sum(p[k] for p in dst)) for k in range(3)])
    T = umeyama(sums, len(src), np.array([float(x) for x in second]), True)
    want = np.eye(4)
    want[:3, :3] = [[float(c * R[j][k]) for k in range(3)] for j in range(3)]
    want[:3, 3] = [float(x) for x in t]
    assert np.abs(T - want).max() < 1e-12
    # the two-pass moments of the oracle give the same answer
    s, d = np.array(src, dtype=np.float64), np.array(dst, dtype=np.float64)
    idx = np.arange(len(s))
    m0, n = to.moments(s, d, idx, np.zeros(len(s)))
    m1, _ = to.moments(s, d, idx, None, np.concatenate([m0[1:4], m0[4:7]]) * (1.0 / n))
    assert np.abs(umeyama(m0, n, m1, True) - want).max() < 1e-12


@pytest.mark.parametrize("umeyama", [to.umeyama, tnt.umeyama])
def test_umeyama_reflection_gives_rotation(umeyama):
    """dst = diag(1, 1, -1) src with a diagonal covariance d1 > d2 > d3: det U det V < 0, so S = diag(1, 1, -1), R = I,
    c = (d1 + d2 - d3) / (d1 + d2 + d3)."""
    base = [Fraction(v) for v in (3, -3, 2, -2, 1, -1)]
    src = [[base[0], 0, 0], [base[1], 0, 0], [0, base[2], 0], [0, base[3], 0], [0, 0, base[4]], [0, 0, base[5]]]
    dst = [[p[0], p[1], -p[2]] for p in src]
    mu_s, mu_d, second = _moments_exact(src, dst)
    d1, d2, d3 = Fraction(18, 6), Fraction(8, 6), Fraction(2, 6)
    c = (d1 + d2 - d3) / (d1 + d2 + d3)
    sums = np.zeros(7)
    T = umeyama(sums, len(src), np.array([float(x) for x in second]), True)
    assert np.abs(T[:3, :3] - float(c) * np.eye(3)).max() < 1e-14
    assert np.abs(T[:3, 3]).max() < 1e-14


# ------------------------------------------------------------------------------------------------------ ICP loop
def _arc(n_t, rot):
    a = np.linspace(0, np.pi, n_t)
    tgt = np.stack([np.cos(a), np.sin(a), 0 * a], 1)
    b = a[::4] + rot
    return np.stack([np.cos(b), np.sin(b), 0.01 * np.sin(7 * b)], 1), tgt


def test_icp_stops_on_fitness_while_rmse_changes():
    src, tgt = _arc(2000, 0.5)
    T, fit, rmse, it, hist = to.registration_icp(src, tgt, 0.3, np.eye(4), True, 1e-6, 20, 30)
    assert it < 30 and fit == 1.0
    # the RMSE was still moving: with relative_rmse = 1e-6 the same loop keeps going
    assert to.registration_icp(src, tgt, 0.3, np.eye(4), True, 1e-6, 1e-6, 30)[3] > it


def test_icp_positional_criteria_run_thirty_iterations():
    """ICPConvergenceCriteria(1e-6, 20): relative_rmse = 20, max_iteration stays 30; fitness changes every iteration here."""
    src, tgt = _arc(2000, 0.8)
    T, fit, rmse, it, hist = to.registration_icp(src, tgt, 0.2, np.eye(4), True, 1e-6, 20, 30)
    assert it == 30 and len(hist) == 30


def test_registration_stages_pass_criteria_positionally(monkeypatch):
    import inspect

    assert inspect.signature(tnt.registration_icp).parameters["max_iteration"].default == 30
    calls = []
    monkeypatch.setattr(tnt, "crop_and_downsample", lambda *a, **k: None)
    monkeypatch.setattr(tnt, "registration_icp",
                        lambda *a, **k: calls.append((a, k)) or tnt.ICPResult(np.eye(4), 1.0, 0.0, 1))
    tnt.registration_vol_ds(None, None, np.eye(4), None, 0.01, 0.8, 20, verbose=False)
    tnt.registration_unif(None, None, np.eye(4), None, 0.02, 20, verbose=False)
    assert len(calls) == 2
    for a, k in calls:
        assert a[4:] == (True, 1e-6, 20) and not k  # relative_rmse = max_itr; max_iteration keeps its default


# ------------------------------------------------------------------------------------------------ rough alignment
@pytest.mark.parametrize("seed", [0, 1, 7])
def test_ransac_self_registration_returns_gt_trans(seed):
    rng = np.random.default_rng(seed + 100)
    n = 300
    centres = np.cumsum(rng.normal(size=(n, 3)) * 0.05, axis=0)
    traj = [tnt.CameraPose([i, i, n], np.block([[np.eye(3), c[:, None]], [np.zeros((1, 3)), np.ones((1, 1))]]))
            for i, c in enumerate(centres)]
    c, s = math.cos(0.7), math.sin(0.7)
    gt_trans = np.array([[1.3 * c, -1.3 * s, 0, 0.4], [1.3 * s, 1.3 * c, 0, -2.0], [0, 0, 1.3, 0.25], [0, 0, 0, 1]])
    T = tnt.trajectory_alignment(None, traj, traj, gt_trans, "Scene", seed=seed)
    assert np.abs(T - gt_trans).max() <= 1e-9 * np.abs(gt_trans).max()


# ------------------------------------------------------------------------------------------------------- F-score
@pytest.mark.parametrize("seed", [0, 1])
def test_f1_histo_matches_reference_formulas(seed):
    rng = np.random.default_rng(seed)
    tau = 0.005
    d1 = np.abs(rng.normal(scale=tau, size=5000))
    d2 = np.concatenate([np.abs(rng.normal(scale=2 * tau, size=3000)), [tau, 0.0, 5 * tau, np.nextafter(tau, 0)]])
    got = tnt.get_f1_score_histo2(tau, ".", 5, d1, d2)
    ref = to.f1_score_histo2(tau, 5, d1, d2)
    assert type(got[0]) is float and got[:3] == list(ref[:3])
    for a, b in zip(got[3:], ref[3:]):
        assert np.array_equal(a, b)


def test_f1_histo_empty_and_zero():
    for d1, d2 in (([], [0.1]), ([0.1], []), ([], [])):
        r = tnt.get_f1_score_histo2(0.01, ".", 5, d1, d2)
        assert r[:3] == [0, 0, 0] and all(np.array_equal(x, [0]) for x in r[3:])
    with pytest.raises(ZeroDivisionError):
        tnt.get_f1_score_histo2(0.01, ".", 5, [1.0, 2.0], [0.5])
    with pytest.raises(ZeroDivisionError):
        to.f1_score_histo2(0.01, 5, [1.0, 2.0], [0.5])


# -------------------------------------------------------------------------------------------------------- readers
def test_read_trajectory_fixture():
    traj = tnt.read_trajectory(os.path.join(GOLDEN, "Tiny_COLMAP_SfM.log"))
    assert [t.metadata for t in traj] == [[0, 0, 3], [1, 1, 3], [2, 2, 3]]
    assert traj[0].pose[:3, 3].tolist() == [0.5, -1.25, 2.0]
    assert traj[1].pose[0].tolist() == [0.0, -1.0, 0.0, 3.5] and traj[1].pose[2, 3] == -7e-3
    assert traj[2].pose[:3, 3].tolist() == [100.0, -0.25, 0.0]
    assert tnt.convert_trajectory_to_points(traj).shape == (3, 3)


def test_read_mapping_fixture():
    n, total, mapping = tnt.read_mapping(os.path.join(GOLDEN, "Tiny_mapping_reference.txt"))
    assert (n, total) == (2, 3) and mapping.tolist() == [[1.0, 3.0], [2.0, 1.0]] and mapping.dtype == np.float64
    traj = tnt.read_trajectory(os.path.join(GOLDEN, "Tiny_COLMAP_SfM.log"))
    assert [t.metadata[0] for t in tnt.gen_sparse_trajectory(mapping, traj)] == [2, 0]


def test_read_selection_polygon_volume_fixture():
    vol = tnt.read_selection_polygon_volume(os.path.join(GOLDEN, "Tiny.json"))
    assert vol.orthogonal_axis == "Z" and (vol.axis_min, vol.axis_max) == (-1.25, 4.5)
    assert vol.bounding_polygon.shape == (4, 3) and vol.bounding_polygon[2].tolist() == [2.0, 3.0, 0.0]


# ------------------------------------------------------------------------------------------------------------ CLI
def test_cli_flags():
    p = tnt.build_parser()
    a = p.parse_args(["--dataset-dir", "d/Barn", "--traj-path", "t.log", "--ply-path", "m.ply"])
    assert (a.dataset_dir, a.traj_path, a.ply_path, a.out_dir, a.seed, a.tau) == ("d/Barn", "t.log", "m.ply", "", 0, None)
    a = p.parse_args(["--dataset-dir", "d", "--traj-path", "t", "--ply-path", "m", "--out-dir", "o", "--seed", "3",
                      "--tau", "0.02"])
    assert (a.out_dir, a.seed, a.tau) == ("o", 3, 0.02)
    with pytest.raises(SystemExit):
        p.parse_args(["--traj-path", "t", "--ply-path", "m"])


def test_scene_thresholds():
    assert tnt.SCENES_TAU == {"Barn": 0.01, "Caterpillar": 0.005, "Ignatius": 0.003, "Truck": 0.005}
    assert tnt.scene_tau("Truck") == 0.005 and tnt.scene_tau("Elsewhere", 0.02) == 0.02
    with pytest.raises(ValueError, match="not in the scene thresholds"):
        tnt.scene_tau("Elsewhere")
    with pytest.raises(ValueError):
        tnt.run_evaluation("/nonexistent/Elsewhere", "t.log", "m.ply", "out")


def test_uniform_rate_rounds_half_to_even():
    assert [int(round(n / float(tnt.MAX_POINT_NUMBER))) for n in (6e6, 1e7, 1.4e7, 1.8e7)] == [2, 2, 4, 4]


# ---------------------------------------------------------------------------------------------------- C refusals
def test_c_entry_points_refuse_bad_arguments(gsb_lib):
    L = gsb_lib
    fake = C.c_void_p(256)  # never dereferenced: every refusal happens before any device work
    T = (C.c_double * 16)(*np.eye(4).ravel())
    assert L.gsb_eval_transform_points(fake, 10, None, fake, None) == _lib.GSB_ERR_INVALID
    assert L.gsb_eval_transform_points(fake, -1, T, fake, None) == _lib.GSB_ERR_INVALID
    assert L.gsb_eval_transform_points(None, 0, T, None, None) == _lib.GSB_OK
    for nv, axis in ((2, 2), (0, 0), (3, 3), (3, -1), (4096, 2)):
        assert L.gsb_eval_crop_polygon(fake, 10, fake, nv, axis, 0.0, 1.0, fake, fake, fake, None) == _lib.GSB_ERR_INVALID
    assert b"3 .. 2048" in L.gsb_last_error() or b"bad arguments" in L.gsb_last_error()
    assert L.gsb_eval_crop_polygon(None, 0, fake, 3, 2, 0.0, 1.0, None, None, None, None) == _lib.GSB_OK
    ws = L.gsb_eval_voxel_workspace_bytes(10)
    assert ws > 10 * 41 and L.gsb_eval_voxel_workspace_bytes(-1) == 0
    g = _lib.GsbPointGrid((C.c_double * 3)(0, 0, 0), 1.0, (C.c_int32 * 3)(1, 1, 1), 256, 1, 256, 256)
    for r in (0.0, -1.0, float("inf"), float("nan")):
        assert L.gsb_eval_icp_correspond(C.byref(g), fake, 10, r, fake, fake, None) == _lib.GSB_ERR_INVALID
    assert L.gsb_eval_icp_correspond(None, fake, 10, 1.0, fake, fake, None) == _lib.GSB_ERR_INVALID
    means = (C.c_double * 6)()
    assert L.gsb_eval_icp_moments(fake, fake, fake, 10, fake, 2, means, fake, fake, None) == _lib.GSB_ERR_INVALID
    assert L.gsb_eval_icp_moments(fake, fake, fake, 10, fake, 1, None, fake, fake, None) == _lib.GSB_ERR_INVALID
    assert L.gsb_eval_icp_moments(fake, fake, None, 10, fake, 0, None, fake, fake, None) == _lib.GSB_ERR_INVALID
