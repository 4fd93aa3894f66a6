"""The MobileBrick evaluation on the GPU (gsb_mobilebrick.cu, gs2mesh_b200/mobilebrick.py) against its CPU restatement
(oracle/mobilebrick_oracle.py), bit for bit: uniform samples, the kept Poisson-disk set at full size and on the tie and
round-heavy clouds, the visibility mask (also against the reference's literal F.grid_sample expression), the compacted
mesh and its normals, the ICP branch around fitness 0.99, the written cropped PLY, the seven numbers, repeatability and
the no-triangle fallback."""
import os

import numpy as np
import pytest

from oracle import mobilebrick_oracle as mo
from tests import mobilebrick_cases as mc

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _peak_memory():
    yield
    import torch

    if torch.cuda.is_available():
        print(f"\ntest_gpu_mobilebrick: peak torch memory {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def test_uniform_samples(gsb_lib, cuda_device):
    from gs2mesh_b200 import mobilebrick as mb

    for v, t, M in [(*mc.grid_mesh(40, 30, seed=1), 20000), (*mc.half_round_mesh(), 10), (*mc.half_round_mesh(), 7)]:
        got = mb.sample_points_uniformly(v, t, M, stream=mb.Mt19937Stream(11), device=cuda_device).cpu().numpy()
        want = mo.sample_uniform(v, t, M, mo.Stream(11).uniform(2 * M))[0]
        assert np.array_equal(_bits(got), _bits(want))
    with pytest.raises(ValueError, match="Input mesh has no triangles."):
        mb.sample_points_uniformly(np.zeros((3, 3)), np.zeros((0, 3), np.int64), 5, device=cuda_device)
    with pytest.raises(ValueError, match="Invalid surface area"):
        mb.sample_points_uniformly(np.zeros((3, 3)), np.array([[0, 1, 2]]), 5, device=cuda_device)


CLOUDS = mc.elimination_clouds(40)
EDGE = ["at_r_max", "r_min_clamp", "isolated", "gradient_chain", "n_is_m_minus_1", "n_is_m"]


@pytest.mark.parametrize("name", EDGE + sorted(k for k in CLOUDS if k.startswith("random_")))
def test_elimination_clouds(gsb_lib, cuda_device, name):
    import torch

    from gs2mesh_b200 import mobilebrick as mb

    p, N, r_max, r_min = CLOUDS[name]
    kept, info = mb.eliminate(torch.as_tensor(p, device=cuda_device), N, r_max, r_min, return_info=True)
    want = mc.oracle_elimination(p, N, r_max, r_min, heap=True)
    assert np.array_equal(kept.cpu().numpy(), want)
    if N < len(p):
        _, key, rnd, rounds = mc.oracle_elimination(p, N, r_max, r_min, heap=False)
        assert info["rounds"] == rounds
        assert np.array_equal(_bits(info["keys"].cpu().numpy()), _bits(key))
        assert np.array_equal(info["round_of"].cpu().numpy(), rnd)


def test_poisson_full_size(gsb_lib, cuda_device):
    """100 000 points from 500 000 samples: the kept indices and points equal the round-based oracle's."""
    import torch

    from gs2mesh_b200 import mobilebrick as mb

    v, t = mc.grid_mesh(300, 300, seed=5)
    N = 100000
    torch.cuda.reset_peak_memory_stats()
    got, info = mb.sample_points_poisson_disk(v, t, N, stream=mb.Mt19937Stream(0), device=cuda_device, return_info=True)
    peak = torch.cuda.max_memory_allocated() / 2 ** 20
    pts, kept, samples, rounds = mo.poisson_disk(v, t, N, mo.Stream(0))
    assert np.array_equal(_bits(info["samples"].cpu().numpy()), _bits(samples))
    assert np.array_equal(info["kept"].cpu().numpy(), kept)
    assert np.array_equal(_bits(got.cpu().numpy()), _bits(pts))
    assert info["rounds"] == rounds
    print(f"\npoisson 100000 of 500000: {info['rounds']} rounds, {info['neighbours'] / 500000:.1f} neighbours per point, "
          f"peak torch memory {peak:.0f} MiB")


def _vis_cases():
    rng = np.random.default_rng(3)
    res = np.array([7, 5, 9])
    min_pts = np.array([0.1, -0.2, 0.3])
    vs = 0.05
    vol = rng.random(tuple(res)) > 0.4
    ijk = np.stack(np.meshgrid(*[np.arange(-1, r + 1) for r in res], indexing="ij"), -1).reshape(-1, 3)
    pts = [min_pts + ijk * vs,  # voxel centres, g = +-1 at the volume's corners, one voxel outside
           min_pts + (ijk + 0.5) * vs,  # half-integer voxel coordinates
           min_pts + rng.uniform(-0.2, 1.2, (20000, 3)) * (res - 1) * vs]  # inside and outside
    return np.concatenate(pts), vol, min_pts, res, vs


def test_visibility(gsb_lib, cuda_device):
    import torch
    import torch.nn.functional as F

    from gs2mesh_b200 import mobilebrick as mb

    points, vol, min_pts, res, vs = _vis_cases()
    got = mb.visibility_test(torch.as_tensor(points, device=cuda_device), vol.reshape(-1), min_pts, res, vs).cpu().numpy()
    assert np.array_equal(got, mo.visibility(points, vol, min_pts, res, vs))
    # evaluate.py:36-41 literally, on the device
    volume = torch.from_numpy(vol.astype(np.float64)).float().to(cuda_device)
    voxels = (points - min_pts) / vs
    voxels = voxels / (res - 1) * 2 - 1
    voxels = torch.from_numpy(voxels)[..., [2, 1, 0]].float().to(cuda_device)
    mask = F.grid_sample(volume.unsqueeze(0).unsqueeze(0), voxels.unsqueeze(0).unsqueeze(0).unsqueeze(0), mode="nearest",
                         padding_mode="zeros", align_corners=True)
    ref = mask[0, 0, 0, 0].cpu().numpy() > 0
    assert np.array_equal(got, ref)
    assert got.any() and not got.all()


def test_remove_vertices_and_normals(gsb_lib, cuda_device):
    from gs2mesh_b200 import mobilebrick as mb
    from gs2mesh_b200.mesh import TriangleMesh

    v, t = mc.grid_mesh(30, 20, seed=2)
    v = np.concatenate([v, [[9.0, 9.0, 9.0]]])  # unreferenced
    rng = np.random.default_rng(4)
    remove = rng.random(len(v)) < 0.2
    remove[-1] = False
    col = rng.random((len(v), 3))
    nrm = rng.random((len(v), 3))
    gv, gt_, gc, gn = mb.remove_vertices_by_mask(v, t, remove, col, nrm)
    wv, wt, wc, wn = mo.remove_vertices_by_mask(v, t, remove, col, nrm)
    for a, b in [(gv, wv), (gc, wc), (gn, wn)]:
        assert np.array_equal(_bits(a.cpu().numpy()), _bits(b))
    assert np.array_equal(gt_.cpu().numpy(), wt)
    m = TriangleMesh(gv.cpu().numpy(), gt_.cpu().numpy()).compute_vertex_normals(cuda_device)
    assert np.array_equal(_bits(m.vertex_normals), _bits(mo.vertex_normals(wv, wt)))


@pytest.mark.parametrize("hits,total,branch", [(991, 1000, True), (99, 100, False), (98, 100, False)])
def test_icp_branch(gsb_lib, cuda_device, hits, total, branch):
    """fitness just above 0.99, exactly 0.99 (99 of 100 correspondences: not taken, the comparison is strict) and below."""
    from gs2mesh_b200 import mobilebrick as mb
    from oracle import tnt_oracle as to

    rng = np.random.default_rng(hits)
    gt = rng.uniform(0, 0.3, (total, 3))
    gt[hits:] += 5.0  # no prediction vertex within 0.02
    pred = to.transform(gt[:hits], mc.rigid(0.3, [1, 2, 3], [0.002, 0.001, -0.001]))
    got, reg = mb.align_prediction(gt, mb._points(pred, cuda_device))
    T, fitness, rmse, it, _ = to.registration_icp(gt, pred, 0.02, np.eye(4), False, 1e-6, 1e-6, 10)
    assert reg.fitness == fitness and (fitness > 0.99) == branch
    assert np.array_equal(_bits(reg.transformation), _bits(T))
    want = to.transform(pred, np.linalg.inv(T)) if branch else pred
    assert np.array_equal(_bits(got.cpu().numpy()), _bits(want))


def _expected_ply(v, t, c, n):
    props = [("x", "<f8"), ("y", "<f8"), ("z", "<f8"), ("nx", "<f8"), ("ny", "<f8"), ("nz", "<f8")]
    head = ["ply", "format binary_little_endian 1.0", "comment Created by gs2mesh_b200", f"element vertex {len(v)}",
            "property double x", "property double y", "property double z", "property double nx", "property double ny",
            "property double nz"]
    if c is not None:
        props += [("red", "u1"), ("green", "u1"), ("blue", "u1")]
        head += ["property uchar red", "property uchar green", "property uchar blue"]
    head += [f"element face {len(t)}", "property list uchar uint vertex_indices", "end_header"]
    tab = np.zeros(len(v), props)
    for k, name in enumerate("xyz"):
        tab[name] = v[:, k]
        tab["n" + name] = n[:, k]
    if c is not None:
        rgb = np.rint(c * 255).astype(np.uint8)  # the file's own bytes: colours read as u8 / 255 round back exactly
        tab["red"], tab["green"], tab["blue"] = rgb.T
    face = np.zeros(len(t), [("n", "u1"), ("v", "<u4", (3,))])
    face["n"] = 3
    face["v"] = t
    return ("\n".join(head) + "\n").encode() + tab.tobytes() + face.tobytes()


def test_evaluate_single(gsb_lib, cuda_device, tmp_path):
    from gs2mesh_b200 import mobilebrick as mb

    gt_dir, pred, exp, _ = mc.write_scan(str(tmp_path))
    gv, gt, pv, pt, pc, m = mc.load_scan(gt_dir, pred)
    N = 3000
    got = mb.evaluate_single(gt_dir, pred, exp, "scan", device=cuda_device, seed=7, number_of_points=N)
    want, (v, t, c, n), fitness = mo.evaluate_single(gv, gt, pv, pt, m, seed=7, number_of_points=N, pred_colors=pc)
    assert fitness > 0.99
    assert np.array_equal(_bits(got), _bits(want)), (got, want)
    path = os.path.join(exp, "scan_cropped.ply")
    with open(path, "rb") as f:
        assert f.read() == _expected_ply(v, t, c, n)
    again = mb.evaluate_single(gt_dir, pred, exp, "scan", device=cuda_device, seed=7, number_of_points=N)
    assert np.array_equal(_bits(again), _bits(got))  # one seed, the same bits


def test_evaluate_single_fallback(gsb_lib, cuda_device, tmp_path):
    from gs2mesh_b200 import mobilebrick as mb

    gt_dir, pred, exp, _ = mc.write_scan(str(tmp_path), nx=6, ny=6, no_triangles=True)
    gv, gt, pv, pt, pc, m = mc.load_scan(gt_dir, pred)
    got = mb.evaluate_single(gt_dir, pred, exp, "fb", device=cuda_device, seed=3, number_of_points=50)
    want, (v, t, c, n), _ = mo.evaluate_single(gv, gt, pv, pt, m, seed=3, number_of_points=50, pred_colors=pc)
    assert len(t) == 0 and len(v) > 0
    assert np.array_equal(_bits(got), _bits(want))
    with open(os.path.join(exp, "fb_cropped.ply"), "rb") as f:
        assert f.read() == _expected_ply(v, t, c, n)


def test_cli(gsb_lib, cuda_device, tmp_path, capsys):
    from gs2mesh_b200 import mobilebrick as mb

    gt_dir, pred, exp, _ = mc.write_scan(str(tmp_path), nx=30, ny=30)
    out = mb.main(["--gt_dir", gt_dir, "--pred_path", pred, "--exp_path", exp, "--scan_name", "cli", "--seed", "1"])
    text = capsys.readouterr().out
    assert len(out) == 7 and all(h in text for h in mb.CSV_HEADER)
    assert os.path.exists(os.path.join(exp, "cli_cropped.ply"))
