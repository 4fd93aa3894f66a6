"""CPU oracle of the DTU mask cull (oracle/cull_oracle.py, evaluate_single_scene.py:21-142): the disk dilation against a
brute-force definition, the fp32 fma against exact arithmetic, sampling and decision against the reference's torch
expressions, the camera setup against the reference's expression sequence, and the command line's flags."""
import os
from fractions import Fraction

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from gs2mesh_b200 import cull
from oracle import cull_oracle as co

FX, FY, CX, CY = 1000.0, 1000.0, 800.0, 600.0


def _k4():
    K = np.eye(4, dtype=np.float32)
    K[0, 0], K[1, 1], K[0, 2], K[1, 2] = FX, FY, CX, CY
    return K


def adversarial_vertices(seed=0):
    """Vertices and three cameras (float32 [3,4,4]) that hit every decision boundary of the cull: projections near
    half-integer pixels of a 1600x1200 and of a smaller mask (walked in fp32 ulp steps so that some land exactly on a
    tie), grid coordinates at and next to +-1, depth -1e-6 (cam_2 + 1e-6 == 0, non-finite projections), points behind
    the camera, plus a random cloud."""
    rng = np.random.default_rng(seed)
    K = _k4()
    R = np.eye(4, dtype=np.float32)  # second camera: rotated about y and shifted
    a = 0.3
    R[:3, :3] = [[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]]
    R[:3, 3] = [0.1, -0.05, 0.4]
    mats = np.stack([K, K @ R, np.eye(4)]).astype(np.float32)  # third: pixel = camera x / (z + 1e-6)
    ulps = np.arange(-12, 13)
    pts = []
    z = np.float32(1.5)
    for target in np.concatenate([rng.integers(0, 1600, 40) + 0.5, rng.integers(0, 600, 20) * (1599 / 599) + 0.5 * 1599 / 599,
                                  [0.0, 1599.0]]):
        x0 = np.float32((target - CX) / FX * z)
        xs = x0 + ulps * np.spacing(x0)
        y = np.float32((rng.uniform(100, 1100) - CY) / FY * z)
        pts.append(np.stack([xs, np.full_like(xs, y), np.full_like(xs, z)], 1))
    for target in np.concatenate([rng.integers(0, 1200, 40) + 0.5, [0.0, 1199.0]]):
        y0 = np.float32((target - CY) / FY * z)
        ys = y0 + ulps * np.spacing(y0)
        x = np.float32((rng.uniform(100, 1500) - CX) / FX * z)
        pts.append(np.stack([np.full_like(ys, x), ys, np.full_like(ys, z)], 1))
    pts.append(np.array([[0.0, 0.0, -1e-6], [0.1, 0.0, -1e-6], [0.0, -0.2, -1e-6], [0.0, 0.0, 0.0]]))
    # the identity camera at a depth where z + 1e-6f == 1 exactly: the pixel is x itself, so g reaches exactly -1 at 0 and
    # exactly +1 at the x next to 1599 with x * fp32(1/1599) == 1
    zs = (np.float32(1) - np.float32(1e-6) + np.arange(-8, 9) * np.spacing(np.float32(0.9))).astype(np.float32)
    z1 = zs[zs + np.float32(1e-6) == np.float32(1)][0]
    for size in (1600, 1200):
        e = np.float32(size - 1) + np.arange(-16, 17) * np.spacing(np.float32(size - 1))
        for edge in (np.float32(0), *e):
            pts.append(np.array([[edge, 600.0, z1]] if size == 1600 else [[800.0, edge, z1]], np.float64))
    behind = rng.uniform(-1, 1, size=(400, 3)) * [1.0, 1.0, 0.0] + [0.0, 0.0, -2.0]
    pts.append(behind)
    pts.append(rng.uniform(-1.5, 1.5, size=(3000, 3)) + [0, 0, 2.0])
    return np.concatenate(pts).astype(np.float64), mats


def adversarial_masks(V, H, W, seed=1):
    """Blobs with holes and set pixels on the border (uint8, values 0 or 1..255)."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[:H, :W]
    m = np.zeros((V, H, W), np.uint8)
    for v in range(V):
        for _ in range(6):
            cy, cx, r = rng.uniform(0, H), rng.uniform(0, W), rng.uniform(0.05, 0.3) * min(H, W)
            m[v][(yy - cy) ** 2 + (xx - cx) ** 2 < r * r] = rng.integers(1, 256)
        m[v][rng.uniform(size=(H, W)) < 0.002] = 7
        m[v][0, rng.integers(0, W)] = m[v][H - 1, rng.integers(0, W)] = m[v][rng.integers(0, H), W - 1] = 255
        m[v][(yy - H / 2) ** 2 + (xx - W / 3) ** 2 < (0.1 * min(H, W)) ** 2] = 0
    return m


def torch_decision(g, dilated):
    """evaluate_single_scene.py:76-99, literally, with torch on the CPU on the given pix_coords (g [V,N,2])."""
    sampled_masks = []
    for i in range(len(g)):
        pix_coords = torch.from_numpy(np.ascontiguousarray(g[i]))
        valid = ((pix_coords > -1.) & (pix_coords < 1.)).all(dim=-1).float()
        maski = torch.from_numpy(dilated[i]).float()[None, None]
        sampled_mask = F.grid_sample(maski, pix_coords[None, None], mode='nearest', padding_mode='zeros',
                                     align_corners=True)[0, -1, 0]
        sampled_mask = sampled_mask + (1. - valid)
        sampled_masks.append(sampled_mask)
    sampled_masks = torch.stack(sampled_masks, -1)
    return (sampled_masks > 0.).all(dim=-1).numpy()


def test_disk_footprint_is_skimage_disk():
    assert co.disk(24).shape == (49, 49) and int(co.disk(24).sum()) == 1793
    assert co.disk(0).tolist() == [[True]]
    assert co.disk(1).astype(int).tolist() == [[0, 1, 0], [1, 1, 1], [0, 1, 0]]
    assert int(co.disk(5).sum()) == 81


@pytest.mark.parametrize("radius", [0, 1, 5, 24])
def test_oracle_dilation_equals_brute_force(radius):
    rng = np.random.default_rng(radius)
    H, W = 61, 83
    m = (rng.uniform(size=(2, H, W)) < 0.01).astype(np.uint8) * rng.integers(1, 256, size=(2, H, W)).astype(np.uint8)
    m[0, 0, 0] = m[0, H - 1, W - 1] = m[1, 0, W - 1] = m[1, H // 2, 0] = 3
    want = np.zeros((2, H, W), bool)
    for v, y, x in zip(*np.nonzero(m)):
        for dy in range(-radius, radius + 1):
            for dx in range(-radius, radius + 1):
                if dx * dx + dy * dy <= radius * radius and 0 <= y + dy < H and 0 <= x + dx < W:
                    want[v, y + dy, x + dx] = True
    assert np.array_equal(co.dilate_masks(m, radius), want)


def test_fma32_is_correctly_rounded():
    rng = np.random.default_rng(3)
    a = rng.normal(size=3000).astype(np.float32)
    b = rng.normal(size=3000).astype(np.float32)
    c = (-(a.astype(np.float64) * b) * (1 + rng.normal(size=3000) * 1e-7)).astype(np.float32)  # heavy cancellation
    c[::3] = (rng.normal(size=1000) * 1e-9).astype(np.float32)
    # exact ties of a*b at float32 precision, nudged either way by a tiny c
    t = np.float32(1 + 2 ** -12)
    a = np.concatenate([a, [t, t, t]]).astype(np.float32)
    b = np.concatenate([b, [t, t, t]]).astype(np.float32)
    c = np.concatenate([c, [2 ** -60, -2 ** -60, 0.0]]).astype(np.float32)
    got = co.fma32(a, b, c)
    for i in range(len(a)):
        exact = Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i]))
        f = np.float32(float(exact))
        cands = [np.nextafter(f, np.float32(-np.inf)), f, np.nextafter(f, np.float32(np.inf))]
        best = min(cands, key=lambda q: (abs(Fraction(float(q)) - exact), int(np.float32(q).view(np.uint32)) & 1))
        assert got[i] == best, i
    one = np.float32(1).view(np.uint32)
    assert (got[-3:].view(np.uint32) - one).tolist() == [4097, 4096, 4096]


def test_oracle_grid_coords_follow_the_torch_expressions():
    """evaluate_single_scene.py:71-75 with torch on the CPU on the same cam_points; lines 73-74 multiply by the fp32
    reciprocal, which is how torch divides a CUDA tensor by a Python scalar (on the CPU torch divides)."""
    v, mats = adversarial_vertices()
    cam = co.camera_points(v, mats)
    g = co.grid_coords(cam)
    W, H = 1600, 1200
    for i in range(len(mats)):
        cam_points = torch.from_numpy(cam[i])
        pix_coords = cam_points[:2, :] / (cam_points[2, :].unsqueeze(0) + 1e-6)
        pix_coords = pix_coords.permute(1, 0)
        pix_coords[..., 0] *= torch.tensor(1.0, dtype=torch.float32) / (W - 1)
        pix_coords[..., 1] *= torch.tensor(1.0, dtype=torch.float32) / (H - 1)
        pix_coords = (pix_coords - 0.5) * 2
        assert np.array_equal(pix_coords.numpy().view(np.uint32), g[i].view(np.uint32))
    assert (np.abs(g) == 1).any() and not np.isfinite(g).all()


@pytest.mark.parametrize("mask_size", [(1200, 1600), (450, 600)])
def test_oracle_sampling_and_decision_equal_torch(mask_size):
    v, mats = adversarial_vertices()
    g = co.project(v, mats)
    dil = co.dilate_masks(adversarial_masks(len(mats), *mask_size), 3)
    keep = co.keep_vertices(g, dil)
    assert np.array_equal(keep, torch_decision(g, dil))
    assert 0.05 < keep.mean() < 0.95
    # the inputs reach the boundaries: exact half-pixel ties, g == +-1, non-finite and behind-the-camera projections
    h, w = mask_size
    fx = ((g[..., 0] + np.float32(1)) / np.float32(2)) * np.float32(w - 1)
    fx = fx[np.isfinite(fx)]
    assert (np.abs(fx - np.floor(fx)) == 0.5).any()
    assert (g == 1).any() and (g == -1).any() and np.isnan(g).any()
    behind = (co.camera_points(v, mats)[:, 2] < 0) & ((g > -1) & (g < 1)).all(-1)
    assert behind.any() and not keep[behind.any(0)].all()


def test_oracle_cull_scan_mesh_compacts_in_order():
    rng = np.random.default_rng(5)
    v, mats = adversarial_vertices()
    t = rng.integers(0, len(v), size=(5000, 3))
    masks = adversarial_masks(len(mats), 1200, 1600)
    s = np.array([[2.5, 0, 0, 10.0], [0, 2.5, 0, -3.0], [0, 0, 2.5, 7.0], [0, 0, 0, 1]], np.float32)
    keep, vw, tw = co.cull_scan_mesh(v, t, mats, masks, s, radius=24)
    assert np.array_equal(keep, co.keep_vertices(co.project(v, mats), co.dilate_masks(masks, 24)))
    kept = np.nonzero(keep)[0]
    assert np.array_equal(vw, v[kept] * np.float64(np.float32(2.5)) + np.array([10.0, -3.0, 7.0]))
    ft = t[keep[t].all(1)]
    assert np.array_equal(kept[tw], ft) and 0 < len(tw) < len(t)


def _write_cameras(root, K, Rs, ts, scale):
    import cv2

    inst = os.path.join(root, "scan7")
    os.makedirs(os.path.join(inst, "images"))
    d = {}
    for i, (R, t) in enumerate(zip(Rs, ts)):
        world = np.eye(4)
        world[:3, :4] = K @ np.concatenate([R, t[:, None]], 1)
        d[f"world_mat_{i}"] = world
        d[f"scale_mat_{i}"] = scale
        cv2.imwrite(os.path.join(inst, "images", f"{i:06d}.png"), np.zeros((4, 4, 3), np.uint8))
    np.savez(os.path.join(inst, "cameras.npz"), **d)
    return inst


def _rotation(rng):
    q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
    return q * np.sign(np.linalg.det(q))


def test_dtu_cameras_equal_reference_expressions_and_recover_K_R_t(tmp_path):
    import cv2

    rng = np.random.default_rng(6)
    K = np.array([[2892.33, 0.0, 823.2], [0.0, 2883.18, 619.07], [0.0, 0.0, 1.0]])
    Rs = [_rotation(rng) for _ in range(3)]
    ts = [rng.normal(size=3) * 50 + [0, 0, 600] for _ in range(3)]
    scale = np.array([[200.0, 0, 0, -10.0], [0, 200.0, 0, 5.0], [0, 0, 200.0, 640.0], [0, 0, 0, 1]])
    inst = _write_cameras(str(tmp_path), K, Rs, ts, scale)
    M, scale_mats = cull.dtu_cameras(inst, device="cpu")
    assert M.dtype == torch.float32 and M.shape == (3, 4, 4) and len(scale_mats) == 3

    camera_dict = np.load(os.path.join(inst, "cameras.npz"))  # evaluate_single_scene.py:28-38, 64-66
    for i in range(3):
        scale_mat = camera_dict['scale_mat_%d' % i].astype(np.float32)
        world_mat = camera_dict['world_mat_%d' % i].astype(np.float32)
        P = (world_mat @ scale_mat)[:3, :4]
        out = cv2.decomposeProjectionMatrix(P)
        Ki, Ri, ti = out[0], out[1], out[2]
        Ki = Ki / Ki[2, 2]
        intrinsics = np.eye(4)
        intrinsics[:3, :3] = Ki
        pose = np.eye(4, dtype=np.float32)
        pose[:3, :3] = Ri.transpose()
        pose[:3, 3] = (ti[:3] / ti[3])[:, 0]
        w2c = torch.inverse(torch.from_numpy(pose).float())
        ref = torch.from_numpy(intrinsics).float() @ w2c
        assert np.array_equal(M[i].numpy().view(np.uint32), ref.numpy().view(np.uint32))
        assert np.array_equal(scale_mats[i], scale_mat)
        # recovered: K, R and the camera centre in the normalised frame
        assert np.allclose(intrinsics[:3, :3], K, rtol=1e-4, atol=1e-3)
        assert np.allclose(pose[:3, :3], Rs[i].T, atol=1e-4)
        c_world = -Rs[i].T @ ts[i]
        assert np.allclose(pose[:3, 3], (c_world - scale[:3, 3]) / scale[0, 0], atol=1e-3)
        # the matrix projects a world point to its pixel
        X = rng.normal(size=3) * 30 + scale[:3, 3]
        p = K @ (Rs[i] @ X + ts[i])
        c = M[i].double().numpy() @ np.append((X - scale[:3, 3]) / scale[0, 0], 1.0)
        assert np.allclose(c[:2] / c[2], p[:2] / p[2], atol=0.05)


def test_cli_flags_and_defaults_match_evaluate_single_scene():
    a = cull.build_parser().parse_args([])
    assert vars(a) == {"input_mesh": None, "scan_id": None, "output_dir": "evaluation_results_single",
                       "DTU": "Offical_DTU_Dataset", "seed": 0}
    a = cull.build_parser().parse_args(["--input_mesh", "m.ply", "--scan_id", "24", "--output_dir", "o", "--DTU", "d",
                                        "--seed", "3"])
    assert (a.input_mesh, a.scan_id, a.output_dir, a.DTU, a.seed) == ("m.ply", "24", "o", "d", 3)


@pytest.mark.parametrize("n_masks", [None, 0, 2])
def test_missing_or_short_mask_directory_raises(tmp_path, n_masks):
    import cv2

    from gs2mesh_b200.mesh import TriangleMesh

    rng = np.random.default_rng(7)
    dtu = os.path.join(str(tmp_path), "data", "Offical_DTU_Dataset")
    os.makedirs(dtu)
    inst = _write_cameras(str(tmp_path), np.diag([1000.0, 1000.0, 1.0]), [np.eye(3)] * 3, [np.array([0, 0, 5.0])] * 3,
                          np.eye(4))
    if n_masks is not None:
        os.makedirs(os.path.join(inst, "mask"))
        for i in range(n_masks):
            cv2.imwrite(os.path.join(inst, "mask", f"{i:03d}.png"), np.full((12, 16, 3), 255, np.uint8))
    TriangleMesh(rng.normal(size=(10, 3)), rng.integers(0, 10, (5, 3))).write_ply(str(tmp_path / "m.ply"))
    with pytest.raises(ValueError, match="masks for 3 images"):
        cull.cull_scan(7, str(tmp_path / "m.ply"), str(tmp_path / "out.ply"), dtu)


def test_unequal_masks_and_non_finite_vertices_rejected():
    v, mats = adversarial_vertices()
    with pytest.raises(ValueError, match="same size"):
        cull.cull_vertices(v, mats, [np.ones((12, 16), np.uint8), np.ones((12, 15), np.uint8)] * 2)
    with pytest.raises(ValueError, match="masks for 3 views"):
        cull.cull_vertices(v, mats, [np.ones((12, 16), np.uint8)])
    bad = v.copy()
    bad[5, 1] = np.nan
    with pytest.raises(ValueError, match="finite"):
        cull.cull_vertices(bad, mats, np.ones((3, 12, 16), np.uint8))
    bad[5, 1] = np.inf
    with pytest.raises(ValueError, match="finite"):
        cull.cull_vertices(bad, mats, np.ones((3, 12, 16), np.uint8))
