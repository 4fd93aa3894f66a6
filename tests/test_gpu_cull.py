"""GPU mask cull (gs2mesh_b200.cull) against the CPU oracle (oracle/cull_oracle.py) and against the reference's own torch
expressions (evaluate_single_scene.py:57-99) on the device: dilated masks, keep masks and culled meshes bit for bit."""
import os

import numpy as np
import pytest

from oracle import cull_oracle as co
from oracle import eval_oracle as eo
from tests.test_cull_oracle import adversarial_masks, adversarial_vertices
from tests.test_gpu_eval import _bits, _tsdf_mesh

pytestmark = pytest.mark.gpu

IW, IH = 1600, 1200


def _dilate_gpu(masks, radius, device):
    from gs2mesh_b200.cull import dilate_masks

    return dilate_masks(masks, radius, device=device).cpu().numpy()


def test_dilation_matches_oracle_64_views(gsb_lib, cuda_device):
    masks = adversarial_masks(64, IH, IW, seed=3)
    got = _dilate_gpu(masks, 24, cuda_device)
    assert got.shape == masks.shape and got.dtype == np.bool_
    ref = co.dilate_masks(masks, 24)
    assert np.array_equal(got, ref), int((got != ref).sum())
    assert 0.2 < ref.mean() < 0.99


@pytest.mark.parametrize("radius", [0, 1])
@pytest.mark.parametrize("shape", [(3, 37, 45), (2, 5, 33), (2, 9, 1), (1, 1, 70)])
def test_dilation_matches_oracle_odd_sizes(gsb_lib, cuda_device, radius, shape):
    rng = np.random.default_rng(sum(shape) + radius)
    masks = (rng.uniform(size=shape) < 0.1).astype(np.uint8) * 200
    masks[..., 0, -1] = 1
    got = _dilate_gpu(masks, radius, cuda_device)
    assert np.array_equal(got, co.dilate_masks(masks, radius))


def _look_at(eye):
    f = -eye / np.linalg.norm(eye)
    r = np.cross(f, [0.0, 0.0, 1.0])
    r /= np.linalg.norm(r)
    d = np.cross(f, r)
    R = np.stack([r, d, f])  # camera x right, y down, z forward
    return R, -R @ eye


def _ring(n=49, radius=3.0, seed=0):
    """n cameras on a ring around the unit sphere looking at the origin: K [R | t] in the normalised frame."""
    rng = np.random.default_rng(seed)
    K = np.array([[1400.0, 0.0, 800.0], [0.0, 1400.0, 600.0], [0.0, 0.0, 1.0]])
    out = []
    for k in range(n):
        a = 2 * np.pi * k / n
        eye = np.array([radius * np.cos(a), radius * np.sin(a), rng.uniform(0.5, 1.5)])
        R, t = _look_at(eye)
        out.append(K @ np.concatenate([R, t[:, None]], 1))
    return out


def _cut_masks(Ps, H=IH, W=IW):
    """Per view the silhouette of a sphere of radius 1.2 around the origin (a disc about the principal point, since the
    cameras look at the origin) with its upper part removed, at a height that varies with the view: together the views
    cut off the top of the unit-sphere mesh."""
    yy, xx = np.mgrid[:H, :W]
    masks = []
    for k, P in enumerate(Ps):
        d = np.linalg.norm(np.linalg.lstsq(P[:, :3], -P[:, 3], rcond=None)[0])  # distance of the camera centre
        r = 1400.0 * np.tan(np.arcsin(1.2 / d))
        inside = ((xx - 800.0) ** 2 + (yy - 600.0) ** 2 < r * r) & (yy > 600.0 - (0.3 + 0.1 * np.sin(k)) * r)
        masks.append(np.where(inside, 255, 0).astype(np.uint8))
    return np.stack(masks)


def _normalised_mesh(device):
    v, t = _tsdf_mesh(device)
    c = 0.5 * (v.min(0) + v.max(0))
    return (v - c) / np.linalg.norm(v - c, axis=1).max(), t


SCALE = np.array([[20.0, 0, 0, 5.0], [0, 20.0, 0, -3.0], [0, 0, 20.0, 400.0], [0, 0, 0, 1]], np.float32)


def _scan_dir(root, Ps, masks):
    """DTU's scan<k>/{images,mask,cameras.npz}: world_mat = P @ inverse(scale_mat), so that world_mat @ scale_mat = P."""
    import cv2

    os.makedirs(os.path.join(root, "images"))
    os.makedirs(os.path.join(root, "mask"))
    d = {}
    inv = np.linalg.inv(SCALE.astype(np.float64))
    for i, (P, m) in enumerate(zip(Ps, masks)):
        world = np.eye(4)
        world[:3] = P @ inv[:, :]
        d[f"world_mat_{i}"], d[f"scale_mat_{i}"] = world, SCALE.astype(np.float64)
        cv2.imwrite(os.path.join(root, "images", f"{i:06d}.png"), np.zeros((8, 8, 3), np.uint8))
        cv2.imwrite(os.path.join(root, "mask", f"{i:03d}.png"), np.repeat(m[:, :, None], 3, 2))
    np.savez(os.path.join(root, "cameras.npz"), **d)


def _check_against_oracle(vn, t, M, masks, device, image_size=(IW, IH)):
    import torch

    from gs2mesh_b200.cull import cull_mesh, cull_vertices

    keep = cull_vertices(torch.as_tensor(vn, device=device), M, masks, image_size=image_size).cpu().numpy()
    okeep, ov, ot = co.cull_scan_mesh(vn, t, M.cpu().numpy(), masks, SCALE, image_size=image_size)
    assert np.array_equal(keep, okeep), int((keep != okeep).sum())
    mesh = cull_mesh(vn, t, M, masks, SCALE, image_size=image_size)
    assert np.array_equal(_bits(mesh.vertices), _bits(ov)) and np.array_equal(mesh.triangles, ot)
    return okeep, ov, ot


def test_pipeline_mesh_ring_of_49_cameras_matches_oracle(gsb_lib, cuda_device, tmp_path):
    from gs2mesh_b200.cull import dtu_cameras

    vn, t = _normalised_mesh(cuda_device)
    Ps = _ring(49)
    masks = _cut_masks(Ps)
    _scan_dir(str(tmp_path / "scan1"), Ps, masks)
    M, scale_mats = dtu_cameras(str(tmp_path / "scan1"), device=cuda_device)
    assert M.shape == (49, 4, 4) and np.array_equal(scale_mats[0], SCALE)
    keep, ov, ot = _check_against_oracle(vn, t, M, masks, cuda_device)
    assert 0.05 < keep.mean() < 0.98 and 0 < len(ot) < len(t)


def test_adversarial_vertices_match_oracle(gsb_lib, cuda_device):
    import torch

    v, mats = adversarial_vertices()
    rng = np.random.default_rng(4)
    t = rng.integers(0, len(v), size=(4000, 3))
    M = torch.as_tensor(mats, device=cuda_device)
    for H, W in ((IH, IW), (450, 600)):
        keep, _, _ = _check_against_oracle(v, t, M, adversarial_masks(len(mats), H, W), cuda_device)
        assert 0.05 < keep.mean() < 0.95


def _torch_cull_scan_keep(vertices_np, M, dilated, W=IW, H=IH):
    """evaluate_single_scene.py:57-99 verbatim on the device, with M = intrinsic @ w2c given per view."""
    import torch
    import torch.nn.functional as F

    vertices = torch.from_numpy(vertices_np).cuda()
    vertices = torch.cat((vertices, torch.ones_like(vertices[:, :1])), dim=-1)
    vertices = vertices.permute(1, 0)
    vertices = vertices.float()
    sampled_masks, pix = [], []
    for i in range(len(M)):
        with torch.no_grad():
            cam_points = M[i] @ vertices
            pix_coords = cam_points[:2, :] / (cam_points[2, :].unsqueeze(0) + 1e-6)
            pix_coords = pix_coords.permute(1, 0)
            pix_coords[..., 0] /= W - 1
            pix_coords[..., 1] /= H - 1
            pix_coords = (pix_coords - 0.5) * 2
            valid = ((pix_coords > -1.) & (pix_coords < 1.)).all(dim=-1).float()
            maski = torch.from_numpy(dilated[i]).float()[None, None].cuda()
            sampled_mask = F.grid_sample(maski, pix_coords[None, None], mode='nearest', padding_mode='zeros',
                                         align_corners=True)[0, -1, 0]
            sampled_mask = sampled_mask + (1. - valid)
            sampled_masks.append(sampled_mask)
            pix.append(pix_coords.cpu().numpy())
    sampled_masks = torch.stack(sampled_masks, -1)
    return (sampled_masks > 0.).all(dim=-1).cpu().numpy(), np.stack(pix)


def _near_boundary(v, M, dilated, W=IW, H=IH, tol=1e-3):
    """Whether fp64 places vertex v within tol pixels of a decision boundary in some view: a half-integer pixel, the
    image border (g = +-1), or the edge of the dilated mask."""
    h, w = dilated.shape[1:]
    for k in range(len(M)):
        c = M[k].astype(np.float64) @ np.append(v, 1.0)
        p = c[:2] / (c[2] + 1e-6)
        g = (p / [W - 1, H - 1] - 0.5) * 2
        f = (g + 1) / 2 * [w - 1, h - 1]
        if not np.isfinite(f).all():
            continue
        if (np.abs(np.abs(g) - 1) * [W - 1, H - 1] < tol).any() or (np.abs(f - np.floor(f) - 0.5) < tol).any():
            return True
        if (np.abs(g) < 1).all():
            vals = {bool(dilated[k][int(np.clip(np.rint(f[1] + dy), 0, h - 1)), int(np.clip(np.rint(f[0] + dx), 0, w - 1))])
                    for dx in (-tol, tol) for dy in (-tol, tol)}
            if len(vals) > 1:
                return True
    return False


def test_keep_agrees_with_torch_cull_scan_on_device(gsb_lib, cuda_device):
    import torch

    from gs2mesh_b200.cull import cull_vertices

    vn, _ = _normalised_mesh(cuda_device)
    rng = np.random.default_rng(12)
    n = 300_000  # cuBLAS sums M @ v without FMA at this size (DESIGN.md section 7a): the boundary rule is exercised
    base = vn[rng.integers(0, len(vn), n)]
    v = base + rng.normal(scale=0.02, size=base.shape)
    Ps = _ring(49)
    masks = _cut_masks(Ps)
    M = torch.as_tensor(np.stack([np.concatenate([P, [[0, 0, 0, 1]]]) for P in Ps]).astype(np.float32), device=cuda_device)
    dil = co.dilate_masks(masks, 24)
    ref, pix = _torch_cull_scan_keep(v, M, dil)
    got = cull_vertices(torch.as_tensor(v, device=cuda_device), M, masks).cpu().numpy()
    g = co.project(v, M.cpu().numpy())
    same_g = int(((g == pix) | (np.isnan(g) & np.isnan(pix))).all(-1).all(0).sum())
    bad = np.nonzero(got != ref)[0]
    print(f"\ncull vs torch on the device: {len(bad)} of {n} keep decisions differ; grid coordinates bit-identical "
          f"for {same_g} of {n} vertices in all 49 views")
    assert 0.05 < ref.mean() < 0.98
    assert len(bad) <= 1e-5 * n
    Mn = M.cpu().numpy()
    for i in bad:
        assert _near_boundary(v[i], Mn, dil), i


def test_cli_end_to_end_matches_oracle(gsb_lib, cuda_device, tmp_path):
    import subprocess
    import sys

    from scipy.io import savemat

    from gs2mesh_b200.io import read_triangle_mesh_ply, write_point_cloud_ply
    from gs2mesh_b200.mesh import TriangleMesh
    from gs2mesh_b200.cull import dtu_cameras

    vn, t = _normalised_mesh(cuda_device)
    Ps = _ring(49)
    masks = _cut_masks(Ps)
    _scan_dir(str(tmp_path / "scan1"), Ps, masks)
    dtu = str(tmp_path / "data" / "Offical_DTU_Dataset")
    TriangleMesh(vn, t).write_ply(str(tmp_path / "mesh.ply"))

    # the ground truth in DTU world coordinates (eval.py's defaults: 0.2 density, patch 60, max_dist 20)
    vw = vn * SCALE[0, 0] + SCALE[:3, 3][None]
    rng = np.random.default_rng(2)
    lo, hi = vw.min(0), vw.max(0)
    stl = eo.sample_mesh(vw, t, 0.4)
    stl = np.concatenate([stl + rng.normal(scale=0.05, size=stl.shape), rng.uniform(lo, hi, size=(2000, 3))])
    res = 1.0
    BB = np.stack([lo - 1, hi + 1])
    shape = tuple(int(x) for x in np.ceil((BB[1] - BB[0]) / res) + 1)
    obs = np.ones(shape, np.uint8)
    obs[: shape[0] // 3] = 0
    P = np.array([[0.0], [0.0], [1.0], [-(lo[2] + 0.2 * (hi[2] - lo[2]))]])
    os.makedirs(os.path.join(dtu, "ObsMask"))
    os.makedirs(os.path.join(dtu, "Points", "stl"))
    savemat(os.path.join(dtu, "ObsMask", "ObsMask1_10.mat"), {"ObsMask": obs, "BB": BB, "Res": np.array([[res]])})
    savemat(os.path.join(dtu, "ObsMask", "Plane1.mat"), {"P": P})
    write_point_cloud_ply(os.path.join(dtu, "Points", "stl", "stl001_total.ply"), stl)

    M, _ = dtu_cameras(str(tmp_path / "scan1"), device=cuda_device)
    keep, ov, ot = co.cull_scan_mesh(vn, t, M.cpu().numpy(), masks, SCALE)
    assert 0.05 < keep.mean() < 0.98
    seed = 3
    data_pcd = eo.sample_mesh(ov, ot, 0.2)
    ref = eo.dtu_chamfer(data_pcd, stl, obs, BB, np.array([[res]]), P, np.random.default_rng(seed).permutation(len(data_pcd)))
    assert np.isfinite(ref["overall"])

    out = str(tmp_path / "out")
    root_dir = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable, "-m", "gs2mesh_b200.cull", "--input_mesh", str(tmp_path / "mesh.ply"), "--scan_id", "1",
           "--output_dir", out, "--DTU", dtu, "--seed", str(seed)]
    output = subprocess.check_output(cmd, cwd=root_dir).decode("utf-8")
    cv, ct = read_triangle_mesh_ply(os.path.join(out, "culled_mesh.ply"))
    assert np.array_equal(_bits(cv), _bits(ov)) and np.array_equal(ct, ot)
    output = output.strip().splitlines()[-1].replace(" ", ",").split(",")  # run_and_evaluate_dtu.py:58-59
    assert [float(x) for x in output] == [ref["mean_d2s"], ref["mean_s2d"], ref["overall"]]
