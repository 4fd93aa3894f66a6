"""GPU Tanks and Temples evaluation (gs2mesh_b200.tnt) against the CPU oracle (oracle/tnt_oracle.py), bit for bit: the
transform, polygon crop, voxel downsampling, ICP correspondences and moments, every ICP iteration, and run_evaluation's
results and text files on a synthetic scene."""
import ctypes as C
import filecmp
import math
import os

import numpy as np
import pytest

from oracle import eval_oracle as eo
from oracle import tnt_oracle as to

pytestmark = pytest.mark.gpu


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def _dev(x, device):
    import torch

    return torch.as_tensor(np.ascontiguousarray(x, dtype=np.float64), device=device)


def _similarity(angle, axis, scale, t):
    axis = np.asarray(axis, dtype=np.float64) / np.linalg.norm(axis)
    K = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    R = np.eye(3) + math.sin(angle) * K + (1 - math.cos(angle)) * K @ K
    T = np.eye(4)
    T[:3, :3] = scale * R
    T[:3, 3] = t
    return T


def test_transform_matches_oracle(gsb_lib, cuda_device):
    from gs2mesh_b200.tnt import transform_points

    rng = np.random.default_rng(1)
    pts = np.concatenate([rng.normal(size=(100000, 3)) * 50, [[0.0, -0.0, 1e-300], [-0.0, -0.0, -0.0]]])
    for T in (_similarity(0.3, [1, 2, 3], 1.7, [0.1, -4, 2e3]), np.eye(4),
              np.array([[1, 0.2, 0, 1], [0, 1, 0.3, 0], [0.1, 0, 1, 0], [1e-3, 2e-3, -1e-3, 1.0]])):
        got = transform_points(_dev(pts, cuda_device), T).cpu().numpy()
        assert np.array_equal(_bits(got), _bits(to.transform(pts, T)))


POLY = np.array([[0, 0, 0], [4, 0, 0], [4, 4, 0], [2, 1, 0], [0.5, 3.7, 0], [0.5, 2, 0], [-1, 2, 0], [1, 1, 0], [-1, 0.5, 0],
                 [0.25, 0.25, 0]], dtype=np.float64)


def _crop_points(n, rng):
    if n <= 1:
        return np.array([[1.0, 1.0, 0.5]])[:n]
    pts = rng.uniform(-1.5, 4.5, size=(n, 3))
    k = min(n // 4, 100000)
    lattice = np.round(rng.uniform(-1.5, 4.5, size=(k, 3)) * 4) / 4  # on vertices, edges and the slab faces
    lattice[: k // 2, 2] = rng.choice([-1.0, -0.5, 0.0, 2.0, 2.5], size=k // 2)
    pts[:k] = lattice
    pts[k:k + len(POLY)] = POLY
    return pts


@pytest.mark.parametrize("n", [0, 1, 5000, 20_000_000])
@pytest.mark.parametrize("axis", ["z", "X", "y"])
def test_crop_matches_oracle(gsb_lib, cuda_device, n, axis):
    from gs2mesh_b200.tnt import SelectionPolygonVolume, crop_point_cloud

    if n == 20_000_000 and axis != "z":
        pytest.skip("the largest size runs once")
    rng = np.random.default_rng(n + ord(axis))
    pts = _crop_points(n, rng)
    u, v, w = to.AXES[axis.lower()]
    poly = np.zeros_like(POLY)
    poly[:, u], poly[:, v], poly[:, w] = POLY[:, 0], POLY[:, 1], POLY[:, 2]
    vol = SelectionPolygonVolume(axis, -0.5, 2.0, poly)
    got = crop_point_cloud(_dev(pts, cuda_device), vol).cpu().numpy()
    mask = to.crop_mask(pts, axis, -0.5, 2.0, poly)
    assert np.array_equal(_bits(got), _bits(pts[mask]))
    if n >= 5000:
        assert 0 < mask.sum() < n


def test_crop_refusals(gsb_lib, cuda_device):
    from gs2mesh_b200.tnt import SelectionPolygonVolume, crop_point_cloud

    pts = np.zeros((10, 3))
    pts[7, 1] = np.nan
    with pytest.raises(ValueError, match="not finite"):
        crop_point_cloud(_dev(pts, cuda_device), SelectionPolygonVolume("z", -1, 1, POLY))
    pts[7, 1] = np.inf
    with pytest.raises(ValueError, match="not finite"):
        crop_point_cloud(_dev(pts, cuda_device), SelectionPolygonVolume("z", -1, 1, POLY))
    with pytest.raises(ValueError, match="3 vertices"):
        crop_point_cloud(_dev(np.zeros((4, 3)), cuda_device), SelectionPolygonVolume("z", -1, 1, POLY[:2]))
    with pytest.raises(ValueError, match="orthogonal_axis"):
        crop_point_cloud(_dev(np.zeros((4, 3)), cuda_device), SelectionPolygonVolume("w", -1, 1, POLY))


@pytest.mark.parametrize("case", ["empty", "one", "boundaries", "random", "far", "large"])
def test_voxel_down_sample_matches_oracle(gsb_lib, cuda_device, case):
    from gs2mesh_b200.tnt import voxel_down_sample

    rng = np.random.default_rng(3)
    vs = 0.25
    pts = {"empty": np.zeros((0, 3)), "one": np.array([[1.5, -2.0, 3.25]]),
           "boundaries": np.concatenate([np.zeros((1, 3)), rng.integers(-40, 40, size=(200000, 3)) * (vs / 2)]),
           "random": rng.normal(size=(300000, 3)) * 3,
           "far": rng.normal(size=(100000, 3)) * 0.3 + np.array([1e5, -3e4, 7.0]),
           "large": rng.uniform(-20, 20, size=(5_000_000, 3))}[case]
    got = voxel_down_sample(_dev(pts, cuda_device), vs).cpu().numpy()
    ref = to.voxel_down_sample(pts, vs)[0]
    assert got.shape == ref.shape
    assert np.array_equal(_bits(got), _bits(ref))


def test_voxel_down_sample_refusals(gsb_lib, cuda_device):
    from gs2mesh_b200.tnt import voxel_down_sample

    with pytest.raises(ValueError, match="too small"):
        voxel_down_sample(_dev([[0.0, 0, 0], [1e3, 0, 0]], cuda_device), 1e-7)
    with pytest.raises(ValueError, match="not finite"):
        voxel_down_sample(_dev([[0.0, 0, 0], [np.nan, 0, 0]], cuda_device), 0.1)
    with pytest.raises(ValueError, match="63 bits"):
        voxel_down_sample(_dev([[0.0, 0, 0], [2e9, 2e9, 2e9]], cuda_device), 1.0)


def _correspond(source, target, radius, device):
    import torch

    from gs2mesh_b200 import _lib
    from gs2mesh_b200.evaluate import PointGrid, _stream

    grid = PointGrid(_dev(target, device))
    s = _dev(source, device)
    idx = torch.empty(len(source), dtype=torch.int64, device=device)
    d2 = torch.empty(len(source), dtype=torch.float64, device=device)
    _lib.check(_lib.lib().gsb_eval_icp_correspond(C.byref(grid.desc), _lib.ptr(s), len(source), float(radius),
                                                   _lib.ptr(idx), _lib.ptr(d2), _stream(device)))
    return idx.cpu().numpy(), d2.cpu().numpy()


def test_correspondences_match_oracle(gsb_lib, cuda_device):
    rng = np.random.default_rng(4)
    target = np.concatenate([rng.integers(-20, 20, size=(3000, 3)) * 0.5, rng.normal(size=(2000, 3)) * 5])
    at_r = target[:1000] + np.array([0.5, 0, 0]) * rng.choice([-1, 1], size=(1000, 1))  # exactly r from a lattice point
    source = np.concatenate([at_r, target[:500], rng.normal(size=(4000, 3)) * 6])
    for r in (0.5, 0.75, 3.0):
        idx, d2 = _correspond(source, target, r, cuda_device)
        oi, od = to.correspond(source, target, r)
        assert np.array_equal(idx, oi) and np.array_equal(_bits(d2), _bits(od))
    idx, _ = _correspond(source, target, 0.5, cuda_device)
    assert (idx[:1000] == -1).any() and (idx[1000:1500] >= 0).all()  # at exactly r: no correspondence


def test_moments_match_oracle(gsb_lib, cuda_device):
    import torch

    from gs2mesh_b200.tnt import _Moments

    rng = np.random.default_rng(5)
    for n in (0, 1, 1000, 1_000_003):
        src = rng.normal(size=(n, 3)) * 10 + 3
        tgt = rng.normal(size=(max(n, 1), 3)) * 10 - 1
        idx = np.where(rng.random(n) < 0.8, rng.integers(0, len(tgt), n), -1)
        d2 = rng.random(n)
        m = _Moments(cuda_device)
        args = (_dev(src, cuda_device), torch.as_tensor(idx, device=cuda_device), _dev(d2, cuda_device),
                _dev(tgt, cuda_device))
        s0, c0 = m(*args, 0)
        o0, oc0 = to.moments(src, tgt, idx, d2)
        assert c0 == oc0 and np.array_equal(_bits(s0[:7]), _bits(o0))
        mu = np.concatenate([o0[1:4], o0[4:7]]) * (1.0 / max(oc0, 1))
        s1, c1 = m(*args, 1, mu)
        o1, _ = to.moments(src, tgt, idx, d2, mu)
        assert c1 == oc0 and np.array_equal(_bits(s1), _bits(o1))
        assert np.array_equal(_bits(m(*args, 1, mu)[0]), _bits(s1))  # the same bits on every run


def _arc(n_t, rot):
    a = np.linspace(0, np.pi, n_t)
    tgt = np.stack([np.cos(a), np.sin(a), 0 * a], 1)
    b = a[::4] + rot
    return np.stack([np.cos(b), np.sin(b), 0.01 * np.sin(7 * b)], 1), tgt


def _surface(n, rng):
    xy = rng.uniform(-1.5, 1.5, size=(n, 2))
    return np.concatenate([xy, (0.3 * np.sin(3 * xy[:, 0]) * np.cos(2 * xy[:, 1]) + 0.1 * xy[:, 0] ** 2)[:, None]], 1)


@pytest.mark.parametrize("case", ["arc_fitness_stop", "arc_thirty", "surface", "no_overlap"])
def test_icp_matches_oracle(gsb_lib, cuda_device, case):
    from gs2mesh_b200.tnt import registration_icp

    rng = np.random.default_rng(6)
    init = np.eye(4)
    if case == "arc_fitness_stop":
        (src, tgt), r, crit = _arc(2000, 0.5), 0.3, (1e-6, 20)
    elif case == "arc_thirty":
        (src, tgt), r, crit = _arc(2000, 0.8), 0.2, (1e-6, 20)
    elif case == "surface":
        tgt = _surface(4000, rng)
        src = to.transform(_surface(3000, rng) + rng.normal(scale=0.003, size=(3000, 3)), _similarity(0.05, [1, 1, 0], 1.03,
                                                                                                      [0.02, -0.01, 0.03]))
        r, crit = 0.2, (1e-6, 1e-6)
        init = _similarity(0.01, [0, 0, 1], 0.99, [0.0, 0.01, 0.0])
    else:
        tgt, src, r, crit = _surface(500, rng), _surface(400, rng) + 10.0, 0.1, (1e-6, 1e-6)
    runs = [registration_icp(_dev(src, cuda_device), _dev(tgt, cuda_device), r, init, True, *crit, 30) for _ in range(2)]
    T, fit, rmse, it, hist = to.registration_icp(src, tgt, r, init, True, *crit, 30)
    for g in runs:
        assert (g.iterations, g.fitness, g.inlier_rmse) == (it, fit, rmse)
        assert len(g.transformations) == len(hist)
        for a, b in zip(g.transformations, hist):
            assert np.array_equal(_bits(a), _bits(b))
        assert np.array_equal(_bits(g.transformation), _bits(T))
    if case == "arc_thirty":
        assert it == 30
    if case == "arc_fitness_stop":
        assert it < 30 and fit == 1.0
    if case == "no_overlap":
        assert fit == 0.0 and rmse == 0.0 and it == 1 and np.array_equal(T, np.eye(4))


def test_icp_recovers_known_similarity(gsb_lib, cuda_device):
    from gs2mesh_b200.tnt import registration_icp

    rng = np.random.default_rng(8)
    g = np.linspace(-1.5, 1.5, 151)
    x, y = np.meshgrid(g, g)
    gt = np.stack([x.ravel(), y.ravel(), (0.3 * np.sin(3 * x) * np.cos(2 * y) + 0.1 * x ** 2).ravel()], 1)
    S = _similarity(0.01, [1, 2, 3], 1.004, [0.004, -0.003, 0.002])
    scan = gt[rng.permutation(len(gt))[:15000]] + rng.normal(scale=1e-6, size=(15000, 3))
    src = to.transform(scan, np.linalg.inv(S))
    res = registration_icp(_dev(src, cuda_device), _dev(gt, cuda_device), 0.05, np.eye(4), True, 1e-12, 1e-12, 100)
    assert res.fitness == 1.0
    assert np.abs(res.transformation - S).max() < 1e-6


def test_uniform_branch_above_four_million(gsb_lib, cuda_device):
    from gs2mesh_b200.tnt import SelectionPolygonVolume, crop_and_downsample

    vol = SelectionPolygonVolume("z", -10, 10, np.array([[-10, -10, 0], [10, -10, 0], [10, 10, 0], [-10, 10, 0]], float))
    rng = np.random.default_rng(9)
    for n, k in ((4_000_000, 1), (4_000_001, 1), (10_000_000, 2), (14_000_000, 4)):  # round(2.5) = 2, round(3.5) = 4
        pts = rng.uniform(-1, 1, size=(n, 3))
        got = crop_and_downsample(_dev(pts, cuda_device), vol, down_sample_method="uniform").cpu().numpy()
        assert np.array_equal(_bits(got), _bits(pts[::k]))


# ------------------------------------------------------------------------------------------------ end to end
SCENE, TAU = "Synth", 0.05


def _write_scene(root, rng):
    from gs2mesh_b200.io import write_point_cloud_ply

    d = os.path.join(root, SCENE)
    os.makedirs(d)
    gt_trans = _similarity(0.4, [0.2, 0.3, 1.0], 1.6, [0.5, -0.25, 0.1])
    gt = _surface(8000, rng)
    write_point_cloud_ply(os.path.join(d, SCENE + ".ply"), gt)
    np.savetxt(os.path.join(d, SCENE + "_trans.txt"), gt_trans)
    # the reconstruction lives in the SfM frame: the GT frame mapped back, with noise and a small residual misalignment
    recon = to.transform(_surface(6000, rng) + rng.normal(scale=0.01, size=(6000, 3)),
                         np.linalg.inv(gt_trans) @ _similarity(0.02, [1, 0, 0], 1.01, [0.02, 0.0, -0.01]))
    ply = os.path.join(root, "recon.ply")
    write_point_cloud_ply(ply, recon)
    with open(os.path.join(d, SCENE + ".json"), "w") as f:
        f.write('{"axis_max": 0.35, "axis_min": -0.3, "bounding_polygon": [[-1.2, -1.3, 0], [1.3, -1.1, 0], [1.0, 0.2, 0], '
                '[1.4, 1.3, 0], [-1.3, 1.2, 0]], "class_name": "SelectionPolygonVolume", "orthogonal_axis": "Z", '
                '"version_major": 1, "version_minor": 0}')
    log = os.path.join(d, SCENE + "_COLMAP_SfM.log")
    with open(log, "w") as f:
        for i in range(60):
            a = 2 * np.pi * i / 60
            pose = _similarity(a, [0, 0, 1], 1.0, [3 * np.cos(a), 3 * np.sin(a), 1.5 + 0.1 * np.sin(3 * a)])
            f.write(f"{i} {i} 60\n" + "\n".join(" ".join("%.12f" % x for x in row) for row in pose) + "\n")
    with open(os.path.join(d, SCENE + "_mapping_reference.txt"), "w") as f:
        f.write("60\n60\n" + "".join(f"{i} {i + 1}\n" for i in range(60)))
    return d, log, ply, gt, recon, gt_trans


def _oracle_pipeline(d, log, gt, recon, out, seed):
    from gs2mesh_b200 import tnt

    traj = tnt.read_trajectory(log)
    T0 = tnt.trajectory_alignment(os.path.join(d, SCENE + "_mapping_reference.txt"), traj, traj,
                                  np.loadtxt(os.path.join(d, SCENE + "_trans.txt")), SCENE, seed=seed)
    vol = tnt.read_selection_polygon_volume(os.path.join(d, SCENE + ".json"))

    def crop(p, T):
        p = to.transform(p, T)
        return p[to.crop_mask(p, vol.orthogonal_axis, vol.axis_min, vol.axis_max, vol.bounding_polygon)]

    T = T0
    for vs, thr in ((TAU, TAU * 80), (TAU / 2, TAU * 20)):
        s, t = to.voxel_down_sample(crop(recon, T), vs)[0], to.voxel_down_sample(crop(gt, np.eye(4)), vs)[0]
        T = to.registration_icp(s, t, thr, np.eye(4), True, 1e-6, 20, 30)[0] @ T
    T = to.registration_icp(crop(recon, T), crop(gt, np.eye(4)), 2 * TAU, np.eye(4), True, 1e-6, 20, 30)[0] @ T
    s = to.voxel_down_sample(crop(recon, T), TAU / 2)[0]
    t = to.voxel_down_sample(crop(gt, np.eye(4)), TAU / 2)[0]
    d1, d2 = eo.nearest(s, t)[0], eo.nearest(t, s)[0]
    p, r, f, _, cum_s, _, cum_t = to.f1_score_histo2(TAU, 5, d1, d2)
    os.makedirs(out)
    np.savetxt(os.path.join(out, SCENE + ".recall.txt"), cum_t)
    np.savetxt(os.path.join(out, SCENE + ".precision.txt"), cum_s)
    np.savetxt(os.path.join(out, SCENE + ".prf_tau_plotstr.txt"), np.array([p, r, f, TAU, 5]))
    return [p, r, f], T0


def test_run_evaluation_matches_oracle_pipeline(gsb_lib, cuda_device, tmp_path):
    from gs2mesh_b200 import tnt

    rng = np.random.default_rng(10)
    d, log, ply, gt, recon, gt_trans = _write_scene(str(tmp_path), rng)
    want, T0 = _oracle_pipeline(d, log, gt, recon, str(tmp_path / "oracle"), seed=3)
    assert np.abs(T0 - gt_trans).max() < 1e-9 * np.abs(gt_trans).max()
    outs = [str(tmp_path / f"gpu{k}") for k in range(2)]
    got = [tnt.run_evaluation(d, log, ply, o, seed=3, tau=TAU) for o in outs]
    assert got[0] == want and got[1] == want
    assert 0.5 < want[2] < 1.0
    for o in outs:
        for suffix in (".recall.txt", ".precision.txt", ".prf_tau_plotstr.txt"):
            assert filecmp.cmp(os.path.join(o, SCENE + suffix), str(tmp_path / "oracle" / (SCENE + suffix)), shallow=False)
    # the CLI runs the same evaluation
    assert tnt.main(["--dataset-dir", d, "--traj-path", log, "--ply-path", ply, "--out-dir", str(tmp_path / "cli"),
                     "--seed", "3", "--tau", str(TAU)]) == want
