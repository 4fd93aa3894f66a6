"""GPU mesh-quality evaluation (gs2mesh_b200.evaluate) against the CPU oracle (oracle/eval_oracle.py): sampled points,
nearest-neighbour distances and precision/recall/F1 must be bit-identical."""
import json
import math
import os

import numpy as np
import pytest

from oracle import eval_oracle as eo
from tests.test_gpu_tsdf import CX, CY, FX, FY, H, W, _gpu_volume, _views

pytestmark = pytest.mark.gpu


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def _adversarial_mesh():
    rng = np.random.default_rng(11)
    v = [[0, 0, 0], [1, 0, 0], [0, 1, 0], [0.1, 0, 0], [0, 10, 0], [10, 0, 0], [10, 0.01, 0], [2, 0, 0],
         [0, 0, 0], [40, 0.5, 0], [0.3, 25, 7]]  # a large triangle: rows far beyond one warp
    v = np.concatenate([np.array(v, np.float64), rng.normal(size=(300, 3)) * rng.uniform(0.01, 5, size=(300, 1))])
    t = [[0, 1, 2], [0, 3, 4], [0, 5, 6], [0, 1, 7], [8, 9, 10], [0, 0, 1]]
    t = np.concatenate([np.array(t), rng.integers(11, len(v), size=(2000, 3))])
    return v, t


def _tsdf_mesh(device):
    import torch

    from gs2mesh_b200.mesh import extract_triangle_mesh

    gvol = _gpu_volume(device, with_color=True)
    for depth, rgb, w2c in _views(5):
        gvol.integrate(gvol.prepare_depth(depth, W, H, depth_trunc=4.0), rgb, W, H, FX, FY, CX, CY, w2c)
    torch.cuda.synchronize()
    mesh = extract_triangle_mesh(gvol)
    assert len(mesh.triangles) > 2000
    return mesh.vertices * 1000.0, mesh.triangles  # metres -> millimetres, eval.py's unit


@pytest.mark.parametrize("density", [0.2, 1.0])
def test_sampling_matches_oracle(gsb_lib, cuda_device, density):
    import torch

    from gs2mesh_b200.evaluate import sample_mesh_points

    for v, t in (_adversarial_mesh(), _tsdf_mesh(cuda_device)):
        got = sample_mesh_points(torch.as_tensor(v, device=cuda_device), torch.as_tensor(t, device=cuda_device),
                                 density).cpu().numpy()
        ref = eo.sample_mesh(v, t, density)
        assert got.shape == ref.shape and len(ref) > len(v)
        assert np.array_equal(_bits(got), _bits(ref))


def _clouds(n):
    rng = np.random.default_rng(21)
    centres = rng.uniform(-50, 50, size=(4096, 3))
    clustered = centres[rng.integers(0, 4096, n)] + rng.normal(scale=0.5, size=(n, 3))
    uniform = rng.uniform(-50, 50, size=(n, 3))
    return rng, clustered, uniform


def _check_nearest(q, ref, dist, idx, max_dist=math.inf):
    od, oi = eo.nearest(q, ref)
    expect = np.where(od < max_dist, od, np.inf)
    same = _bits(dist) == _bits(expect)
    if not same.all():
        # the kd-tree candidate is not always the exact minimum under rounding: the GPU's must then be no larger
        bad = ~same
        mine = eo.distance(q[bad], ref[idx[bad]])
        assert (idx[bad] >= 0).all() and np.array_equal(_bits(mine), _bits(dist[bad])) and (mine <= od[bad]).all()
        assert bad.mean() < 1e-4
    hit = np.isfinite(dist)
    assert np.array_equal(_bits(eo.distance(q[hit], ref[idx[hit]])), _bits(dist[hit]))  # idx points at that distance
    assert (idx[~hit] == -1).all()


def test_nearest_matches_oracle(gsb_lib, cuda_device):
    import torch

    from gs2mesh_b200.evaluate import PointGrid

    rng, clustered, uniform = _clouds(1_000_000)
    outliers = rng.uniform(-1, 1, size=(2000, 3)) * 1e4
    dup = clustered[:1000].copy()  # exact hits and duplicated reference points (ties)
    ref = np.concatenate([clustered, dup])
    q = np.concatenate([uniform, outliers, dup, clustered[::7] + 1e-3])
    grid = PointGrid(torch.as_tensor(ref, device=cuda_device))
    d, i = grid.nearest(torch.as_tensor(q, device=cuda_device))
    d, i = d.cpu().numpy(), i.cpu().numpy()
    _check_nearest(q, ref, d, i)
    assert (d[len(uniform) + len(outliers):len(uniform) + len(outliers) + len(dup)] == 0).all()
    # ties go to the lowest index: every duplicate query resolves to the first copy
    assert (i[len(uniform) + len(outliers):len(uniform) + len(outliers) + len(dup)] == np.arange(1000)).all()

    # uniform reference, clustered queries; and the max_dist cut-off
    grid = PointGrid(torch.as_tensor(uniform, device=cuda_device))
    qc = np.concatenate([clustered, outliers])
    for max_dist in (math.inf, 0.75):
        d, i = grid.nearest(torch.as_tensor(qc, device=cuda_device), max_dist=max_dist)
        d, i = d.cpu().numpy(), i.cpu().numpy()
        _check_nearest(qc, uniform, d, i, max_dist)
    assert np.isinf(d[len(clustered):]).all() and np.isfinite(d).mean() > 0.5


def test_precision_recall_f1_matches_oracle(gsb_lib, cuda_device):
    import torch

    from gs2mesh_b200.evaluate import precision_recall_f1

    rng = np.random.default_rng(4)
    gt = rng.uniform(0, 1, size=(200_000, 3))
    pred = np.concatenate([gt[::2] + rng.normal(scale=0.003, size=(100_000, 3)), rng.uniform(0, 1, size=(5000, 3))])
    got = precision_recall_f1(torch.as_tensor(pred, device=cuda_device), torch.as_tensor(gt, device=cuda_device), 0.005)
    ref = eo.precision_recall_f1(pred, gt, 0.005)
    assert set(got) == set(ref)
    for k in ref:
        assert got[k] == ref[k], (k, got[k], ref[k])


def test_nearest_with_a_far_floater_in_the_reference(gsb_lib, cuda_device):
    """One floater 10 units from a 0.3-unit object stretches the bounding box 33-fold per axis: cells are sized from the
    point spacing of the bulk (then limited by the cell budget of the dense grid), and the search stays exact."""
    import torch

    from gs2mesh_b200.evaluate import PointGrid

    rng = np.random.default_rng(8)
    ref = np.concatenate([rng.uniform(0, 0.3, size=(1_000_000, 3)), [[10.0, 10.0, 10.0]]])
    q = np.concatenate([rng.uniform(-0.05, 0.35, size=(200_000, 3)), [[9.9, 10.1, 10.0]]])
    grid = PointGrid(torch.as_tensor(ref, device=cuda_device))
    assert grid.cell < 0.03  # sized over the bounding box it would be 0.063
    d, i = grid.nearest(torch.as_tensor(q, device=cuda_device))
    _check_nearest(q, ref, d.cpu().numpy(), i.cpu().numpy())
    assert i[-1].item() == len(ref) - 1


def test_radius_downsample_matches_sequential_loop(gsb_lib, cuda_device):
    import torch

    from gs2mesh_b200.evaluate import radius_downsample

    rng = np.random.default_rng(9)
    thresh = 0.2
    p = rng.uniform(0, 20, size=(1_000_000, 3))
    axis = np.zeros((20000, 3))
    axis[np.arange(20000), rng.integers(0, 3, 20000)] = thresh * rng.choice([-1.0, 1.0], 20000)
    p = np.concatenate([p, p[:20000], p[20000:40000] + axis])  # duplicates and pairs at exactly thresh along an axis
    order = np.random.default_rng(3).permutation(len(p))
    shuffled, keep = radius_downsample(torch.as_tensor(p, device=cuda_device), thresh, seed=3)
    assert np.array_equal(_bits(shuffled.cpu().numpy()), _bits(p[order]))
    ref = eo.radius_downsample(p[order], thresh)
    got = keep.cpu().numpy()
    assert 0 < ref.sum() < len(p)
    assert np.array_equal(got, ref), int((got != ref).sum())


def _dtu_layout(root, device):
    """A DTU-layout dataset around a mesh from the pipeline: ObsMask with a hole, a ground plane cutting off the bottom,
    an stl scan sampled densely from the mesh surface, jittered, plus stray points."""
    from scipy.io import savemat

    from gs2mesh_b200.io import write_point_cloud_ply
    from gs2mesh_b200.mesh import TriangleMesh

    v, t = _tsdf_mesh(device)
    lo, hi = v.min(0), v.max(0)
    D = float(np.linalg.norm(hi - lo))
    density = D / 300
    rng = np.random.default_rng(2)
    stl = eo.sample_mesh(v, t, density / 2)
    stl = stl + rng.normal(scale=D / 2000, size=stl.shape)
    stl = np.concatenate([stl, rng.uniform(lo, hi, size=(2000, 3))])
    res = D / 40
    BB = np.stack([lo - D / 40, hi + D / 40])
    shape = tuple(int(x) for x in np.ceil((BB[1] - BB[0]) / res) + 1)
    obs = np.ones(shape, np.uint8)
    c = [s // 2 for s in shape]
    obs[c[0] - 3:c[0] + 3, c[1] - 3:c[1] + 3, :] = 0  # a hole through the middle
    z_cut = lo[2] + 0.2 * (hi[2] - lo[2])
    P = np.array([[0.0], [0.0], [1.0], [-z_cut]])
    os.makedirs(os.path.join(root, "ObsMask"))
    os.makedirs(os.path.join(root, "Points", "stl"))
    savemat(os.path.join(root, "ObsMask", "ObsMask1_10.mat"), {"ObsMask": obs, "BB": BB, "Res": np.array([[res]])})
    savemat(os.path.join(root, "ObsMask", "Plane1.mat"), {"P": P})
    write_point_cloud_ply(os.path.join(root, "Points", "stl", "stl001_total.ply"), stl)
    TriangleMesh(v, t).write_ply(os.path.join(root, "mesh.ply"))
    params = dict(downsample_density=density, patch_size=D / 20, max_dist=D / 50)
    return v, t, stl, obs, BB, res, P, params


def test_dtu_chamfer_and_cli_match_oracle(gsb_lib, cuda_device, tmp_path):
    import subprocess
    import sys

    from gs2mesh_b200.evaluate import dtu_chamfer

    root = str(tmp_path)
    v, t, stl, obs, BB, res, P, prm = _dtu_layout(root, cuda_device)
    seed = 5
    data_pcd = eo.sample_mesh(v, t, prm["downsample_density"])
    ref = eo.dtu_chamfer(data_pcd, stl, obs, BB, np.array([[res]]), P, np.random.default_rng(seed).permutation(len(data_pcd)),
                         **prm)
    assert len(ref["dist_d2s"]) > 1000 and np.isfinite(ref["overall"])
    assert (ref["dist_d2s"] >= prm["max_dist"]).any() or (ref["dist_s2d"] >= prm["max_dist"]).any()
    got = dtu_chamfer((v, t), stl, obs, BB, np.array([[res]]), P, seed=seed, device=cuda_device, **prm)
    assert np.array_equal(_bits(got["data_down"]), _bits(ref["data_down"]))
    for k in ("mean_d2s", "mean_s2d", "overall"):
        assert got[k] == ref[k], (k, got[k], ref[k])

    root_dir = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable, "-m", "gs2mesh_b200.evaluate", "--data", os.path.join(root, "mesh.ply"), "--scan", "1", "--mode",
           "mesh", "--dataset_dir", root, "--vis_out_dir", root, "--downsample_density", repr(prm["downsample_density"]),
           "--patch_size", repr(prm["patch_size"]), "--max_dist", repr(prm["max_dist"]), "--seed", str(seed)]
    output = subprocess.check_output(cmd, cwd=root_dir).decode("utf-8")
    output = output.replace(" ", ",").split(",")  # run_and_evaluate_dtu.py:58-59
    output[-1] = output[-1].strip()
    assert [float(x) for x in output] == [ref["mean_d2s"], ref["mean_s2d"], ref["overall"]]
    with open(os.path.join(root, "results.json")) as f:
        assert json.load(f)["overall"] == ref["overall"]
    for name in ("vis_001_d2s.ply", "vis_001_s2d.ply"):
        assert os.path.getsize(os.path.join(root, name)) > 0
