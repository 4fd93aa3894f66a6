"""GPU k nearest neighbours (gsb_eval_knn) and normal estimation (gsb_eval_estimate_normals) against the numpy oracle
(tests/normals_oracle.py), bit for bit, on random and adversarial clouds; and run_evaluation's PLYs with normals."""
import math
import os

import numpy as np
import pytest

from oracle import eval_oracle as eo
from oracle import tnt_oracle as to
from tests import normals_oracle as no

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tnt")


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def _dev(x, device):
    import torch

    return torch.as_tensor(np.ascontiguousarray(x, dtype=np.float64), device=device)


def _check_knn(ref, q, k, device):
    from gs2mesh_b200.evaluate import PointGrid

    d2, idx = PointGrid(_dev(ref, device)).knn(_dev(q, device), k)
    od2, oidx = no.knn(q, ref, k)
    assert np.array_equal(idx.cpu().numpy(), oidx)
    assert np.array_equal(_bits(d2.cpu().numpy()), _bits(od2))
    return oidx


def _check_normals(pts, k, device):
    from gs2mesh_b200.tnt import estimate_normals

    got = estimate_normals(_dev(pts, device), k).cpu().numpy()
    want = no.estimate_normals(pts, k)
    assert np.array_equal(_bits(got), _bits(want))
    return want


def _sphere(n, rng):
    v = rng.normal(size=(n, 3))
    return v / np.linalg.norm(v, axis=1, keepdims=True)


def _surface(n, rng, noise=0.0):
    xy = rng.uniform(-1.5, 1.5, size=(n, 2))
    z = 0.3 * np.sin(3 * xy[:, 0]) * np.cos(2 * xy[:, 1]) + 0.1 * xy[:, 0] ** 2
    return np.concatenate([xy, z[:, None]], 1) + rng.normal(scale=noise, size=(n, 3))


@pytest.mark.parametrize("n", [1, 2, 3, 19, 20, 21, 1000, 100_000, 1_000_000])
def test_random_clouds_match_oracle(gsb_lib, cuda_device, n):
    rng = np.random.default_rng(n)
    pts = rng.uniform(-1, 1, size=(n, 3)) * [3.0, 1.0, 0.2]
    for k in ((20,) if n >= 100_000 else (1, 2, 20, 32)):
        q = np.concatenate([pts, rng.uniform(-4, 4, size=(min(n, 1000), 3))])
        _check_knn(pts, q, k, cuda_device)
        nrm = _check_normals(pts, k, cuda_device)
    if n >= 3:
        assert np.abs(np.linalg.norm(nrm, axis=1) - 1).max() < 1e-12


def _lattice(rng):
    return np.stack(np.meshgrid(*[np.arange(12.0)] * 3, indexing="ij"), -1).reshape(-1, 3)[rng.permutation(1728)]


CASES = {
    # integer coordinates: exact ties in d2 at the k-th place for almost every point
    "lattice": lambda rng: _lattice(rng),
    "lattice_plane": lambda rng: _lattice(rng) * [1, 1, 0],
    "duplicates": lambda rng: np.repeat(rng.normal(size=(400, 3)), 7, axis=0)[rng.permutation(2800)],
    "plane": lambda rng: np.concatenate([rng.uniform(-1, 1, size=(5000, 2)), np.zeros((5000, 1))], 1),
    "tilted_plane": lambda rng: rng.uniform(-1, 1, size=(5000, 2)) @ np.array([[1.0, 0.3, -0.2], [0.1, 1.0, 0.7]]),
    "line": lambda rng: np.outer(rng.uniform(-5, 5, 3000), [0.3, -0.5, 0.8]),
    "axis_line": lambda rng: np.stack([rng.uniform(-5, 5, 3000), np.zeros(3000), np.zeros(3000)], 1),
    "sphere": lambda rng: _sphere(20000, rng),
    "noisy_surface": lambda rng: _surface(30000, rng, 0.01),
    "smaller_than_k": lambda rng: rng.normal(size=(7, 3)),
    "two_points": lambda rng: rng.normal(size=(2, 3)),
    "one_point": lambda rng: np.array([[1.5, -2.0, 0.25]]),
    "coincident": lambda rng: np.tile([[0.1, 0.2, 0.3]], (50, 1)),
    "far_floaters": lambda rng: np.concatenate([_surface(20000, rng, 0.002), rng.normal(size=(5, 3)) * 1e4]),
    "offset": lambda rng: _surface(10000, rng, 0.001) + [1e5, -3e4, 7e3],
    "tiny_scale": lambda rng: _surface(5000, rng, 0.01) * 1e-150,
    "huge_scale": lambda rng: _surface(5000, rng, 0.01) * 1e100,
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_adversarial_clouds_match_oracle(gsb_lib, cuda_device, case):
    rng = np.random.default_rng(sorted(CASES).index(case))
    pts = CASES[case](rng)
    for k in (1, 3, 20, 32):
        _check_knn(pts, pts, k, cuda_device)
        nrm = _check_normals(pts, k, cuda_device)
        if k < 3 or len(pts) < 3:
            assert (nrm == [0.0, 0.0, 1.0]).all()  # fewer than 3 neighbours: the identity, whose normal is z
    if case == "plane":
        assert (np.abs(nrm[:, 2]) > 1 - 1e-12).all()
    if case == "lattice":
        # ties at the 20th place decide the set: the GPU keeps the lower indices, like the oracle
        d2 = no.knn_brute(pts, pts, 21)[0]
        assert (d2[:, 19] == d2[:, 20]).mean() > 0.3


def test_non_finite_and_far_queries(gsb_lib, cuda_device):
    rng = np.random.default_rng(11)
    ref = _surface(5000, rng)
    q = np.array([[np.nan, 0, 0], [0, np.inf, 0], [0, 0, -np.inf], [1e6, -1e6, 3.0], [-1e12, 0, 0], [0.1, 0.2, 0.3]])
    idx = _check_knn(ref, q, 20, cuda_device)
    assert (idx[:3] == -1).all() and (idx[3:] >= 0).all()
    _check_knn(ref[:5], q, 20, cuda_device)  # fewer points than k: rows end in (+inf, -1)


def test_knn_api(gsb_lib, cuda_device):
    from gs2mesh_b200 import evaluate
    from gs2mesh_b200.tnt import estimate_normals

    rng = np.random.default_rng(12)
    ref, q = rng.normal(size=(3000, 3)), rng.normal(size=(500, 3))
    d2, idx = evaluate.knn(_dev(q, cuda_device), _dev(ref, cuda_device), 20)
    assert d2.shape == (500, 20) and idx.shape == (500, 20)
    d, i = evaluate.nearest(_dev(q, cuda_device), _dev(ref, cuda_device))
    assert np.array_equal(idx[:, 0].cpu().numpy(), i.cpu().numpy())
    assert np.array_equal(_bits(np.sqrt(d2[:, 0].cpu().numpy())), _bits(d.cpu().numpy()))
    for k in (0, 33):
        with pytest.raises(ValueError, match="1..32"):
            evaluate.knn(_dev(q, cuda_device), _dev(ref, cuda_device), k)
        with pytest.raises(ValueError, match="1..32"):
            estimate_normals(_dev(ref, cuda_device), k)
    assert estimate_normals(_dev(np.zeros((0, 3)), cuda_device)).shape == (0, 3)
    assert np.array_equal(d2.cpu().numpy(), evaluate.knn(_dev(q, cuda_device), _dev(ref, cuda_device), 20)[0].cpu().numpy())


# ------------------------------------------------------------------------------------------------ run_evaluation
class _Colormap:
    """A stand-in for matplotlib's hot_r: RGBA from a fixed formula, so the PLYs are written without matplotlib."""

    def get_cmap(self, name):
        assert name == "hot_r"
        return lambda x: np.stack([1 - x, (1 - x) ** 2, x * 0.5, np.ones_like(x)], axis=-1)


def _read_ply(path):
    raw = open(path, "rb").read()
    head, body = raw.split(b"end_header\n")
    return head.decode().splitlines(), body


def test_run_evaluation_writes_oracle_normals(gsb_lib, cuda_device, tmp_path, monkeypatch):
    from gs2mesh_b200 import tnt
    from gs2mesh_b200.io import write_point_cloud_ply

    tau, scene = 0.05, "Tiny"
    d = tmp_path / scene
    d.mkdir()
    for f in ("Tiny.json", "Tiny_COLMAP_SfM.log", "Tiny_mapping_reference.txt"):
        (d / f).write_bytes(open(os.path.join(GOLDEN, f), "rb").read())
    np.savetxt(str(d / "Tiny_trans.txt"), np.eye(4))
    rng = np.random.default_rng(13)

    def surface(n):
        xy = rng.uniform(0, 1, size=(n, 2)) * [2.0, 3.0]
        return np.concatenate([xy, (0.2 * np.sin(3 * xy[:, 0]) * np.cos(2 * xy[:, 1]))[:, None]], 1)

    gt = surface(12000)
    recon = surface(9000) + rng.normal(scale=0.01, size=(9000, 3)) + [0.01, -0.005, 0.0]
    write_point_cloud_ply(str(d / "Tiny.ply"), gt)
    write_point_cloud_ply(str(tmp_path / "recon.ply"), recon)
    monkeypatch.setattr(tnt, "_matplotlib", lambda: _Colormap())
    monkeypatch.setattr(tnt, "plot_graph", lambda *a, **k: None)
    out = tmp_path / "out"
    got = tnt.run_evaluation(str(d), str(d / "Tiny_COLMAP_SfM.log"), str(tmp_path / "recon.ply"), str(out), tau=tau)

    # the oracle pipeline: three camera centres are fewer than RANSAC's 6, so the alignment is the identity
    vol = tnt.read_selection_polygon_volume(str(d / "Tiny.json"))

    def crop(p, T):
        p = to.transform(p, T)
        return p[to.crop_mask(p, vol.orthogonal_axis, vol.axis_min, vol.axis_max, vol.bounding_polygon)]

    T = np.eye(4)
    for vs, thr in ((tau, tau * 80), (tau / 2, tau * 20)):
        s, t = to.voxel_down_sample(crop(recon, T), vs)[0], to.voxel_down_sample(crop(gt, np.eye(4)), vs)[0]
        T = to.registration_icp(s, t, thr, np.eye(4), True, 1e-6, 20, 30)[0] @ T
    T = to.registration_icp(crop(recon, T), crop(gt, np.eye(4)), 2 * tau, np.eye(4), True, 1e-6, 20, 30)[0] @ T
    s = to.voxel_down_sample(crop(recon, T), tau / 2)[0]
    t = to.voxel_down_sample(crop(gt, np.eye(4)), tau / 2)[0]
    d1, d2 = eo.nearest(s, t)[0], eo.nearest(t, s)[0]
    p, r, f, _, cum_s, _, cum_t = to.f1_score_histo2(tau, 5, d1, d2)
    assert got == [p, r, f] and 0.5 < f <= 1.0
    for name, arr in ((".recall.txt", cum_t), (".precision.txt", cum_s), (".prf_tau_plotstr.txt", [p, r, f, tau, 5])):
        np.savetxt(str(tmp_path / ("want" + name)), np.asarray(arr))
        assert open(str(out / (scene + name)), "rb").read() == open(str(tmp_path / ("want" + name)), "rb").read()

    for suffix, pts, dist in ((".precision.ply", s, d1), (".recall.ply", t, d2)):
        head, body = _read_ply(str(out / (scene + suffix)))
        assert head[3:12] == ["property double x", "property double y", "property double z", "property double nx",
                              "property double ny", "property double nz", "property uchar red", "property uchar green",
                              "property uchar blue"]
        rows = np.frombuffer(body, dtype=[("xyz", "<f8", 3), ("n", "<f8", 3), ("rgb", "u1", 3)])
        assert len(rows) == len(pts) > 100
        assert np.array_equal(_bits(rows["n"]), _bits(no.estimate_normals(pts, 20)))
        # without the normals, the file is what the writer made before normals were added
        plain = tnt.write_color_distances(str(tmp_path / ("plain" + suffix)), pts, dist, 3 * tau)
        want_head, want_body = _read_ply(plain)
        assert [h for h in head if not h.startswith("property double n")] == want_head
        stripped = np.ascontiguousarray(rows[["xyz", "rgb"]]).astype([("xyz", "<f8", 3), ("rgb", "u1", 3)]).tobytes()
        assert stripped == want_body
    assert not math.isnan(f)
