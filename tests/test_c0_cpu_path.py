"""BASELINE.json configs[0]: "synthetic 10k-Gaussian scene, 4 stereo pairs @640x480, 128^3 TSDF on CPU reference path
(plumbing, no GPU)".  The whole hot path end to end on the CPU ORACLE (raster restatement -> expected depth ->
Open3D-restatement TSDF -> marching-cubes restatement), with the host logic of the product (scene generator, camera
maths, stage-class depth rules, view sharding and merge).  It pins the plumbing the GPU tests rely on: the same scene
generator, the same conventions, the same filters."""
import numpy as np
import pytest


@pytest.fixture(scope="module")
def c0(oracle):
    from gs2mesh_b200 import camera as cam
    from gs2mesh_b200 import scene

    cfg = scene.CONFIGS["C0"]
    W, H = cfg["width"], cfg["height"]
    cloud = scene.make_gaussians(cfg["num_points"], seed=0)
    rigs, baseline = scene.make_stereo_cameras(cfg["pairs"], W, H, layout=cfg["layout"])
    frames = []
    for pair in rigs:
        views = {}
        for side in ("left", "right"):
            vt = cam.view_transforms_from_camera(pair[side])
            views[side] = oracle.forward(cloud.xyz, cloud.opacity, vt.world_view, vt.full_proj, vt.cam_center, W, H, vt.tan_fovx,
                                         vt.tan_fovy, shs=cloud.features, scales=cloud.scaling, rotations=cloud.rotation)
        frames.append(views)
    return dict(cfg=cfg, W=W, H=H, cloud=cloud, rigs=rigs, baseline=baseline, frames=frames)


def _depth_and_rgb(c0, i):
    """What the stage classes hand to the fusion (SURVEY 8(d)): expected depth D/alpha where alpha > 0.5, the reference's
    min-depth rule (tsdf_utils.py:83), uint8 colour with cv2's rounding (renderer_utils.py:389-390)."""
    cfg, left = c0["cfg"], c0["frames"][i]["left"]
    alpha = 1.0 - left["final_T"]
    d = np.where(alpha > 0.5, left["depth"] / np.maximum(alpha, 1e-30), 0).astype(np.float32)
    d = np.where(d < np.float32(cfg["min_db"] * c0["baseline"]), 0, d).astype(np.float32)
    rgb = np.clip(np.rint(left["color"].transpose(1, 2, 0) * 255.0), 0, 255).astype(np.uint8)
    return d, rgb


def _integrate(c0, ovol, i):
    cfg, cam_l = c0["cfg"], c0["rigs"][i]["left"]
    d, rgb = _depth_and_rgb(c0, i)
    ovol.integrate(d, rgb, c0["W"], c0["H"], cam_l["fx"], cam_l["fy"], cam_l["cx"], cam_l["cy"], np.linalg.inv(cam_l["extrinsic"]),
                   depth_scale=1.0, depth_trunc=cfg["max_db"] * c0["baseline"])


def test_stereo_pairs_render_the_object_with_disparity(c0):
    W, H = c0["W"], c0["H"]
    for i, views in enumerate(c0["frames"]):
        left, right = views["left"], views["right"]
        cover = (1.0 - left["final_T"]) > 0.5
        assert 0.4 < cover.mean() < 0.8, cover.mean()  # the object fills the middle of the frame
        assert left["num_rendered"] > 100_000 and (left["radii"] > 0).sum() > 0.9 * c0["cfg"]["num_points"]
        assert np.isfinite(left["color"]).all() and left["color"].min() >= 0
        # the right eye sees the same object shifted: horizontal centroid of the coverage moves left by fx*B/z pixels
        cover_r = (1.0 - right["final_T"]) > 0.5
        xs = np.arange(W)[None, :]
        shift = (cover * xs).sum() / cover.sum() - (cover_r * xs).sum() / cover_r.sum()
        z = np.median(left["depth"][cover] / (1.0 - left["final_T"][cover]))
        expect = c0["rigs"][i]["left"]["fx"] * c0["baseline"] / z
        assert abs(shift - expect) < 0.2 * expect, (shift, expect)


def test_fused_volume_and_mesh_recover_the_surface(c0, oracle):
    cfg = c0["cfg"]
    vl = 2.0 / cfg["tsdf_res"]
    trunc = max(0.04, 3 * vl)
    ovol = oracle.OracleTSDFVolume(vl, trunc, with_color=True)
    for i in range(cfg["pairs"]):
        _integrate(c0, ovol, i)
    nb = cfg["tsdf_res"] // 16
    origin, count = (-(nb // 2),) * 3, (nb,) * 3  # gs2mesh_b200.tsdf.default_window without importing torch-side code
    tw, alloc, outside = ovol.export_bricks(origin, count)
    assert outside < 50  # the scene fits the reference's default lattice over [-1,1]^3
    w = tw[..., 1]
    assert w.max() >= 2 and (w > 0).sum() > 300_000  # overlapping views fuse into the same voxels
    assert np.abs(tw[..., 0]).max() <= 1.0
    mesh = oracle.extract_mesh_from_bricks(tw, origin, count, vl)
    v, t = mesh["vertices"], mesh["triangles"]
    assert len(t) > 50_000
    r = np.linalg.norm(v, axis=1)
    # the generator's surface: radius 0.8 sphere with low-frequency bumps (scene.make_gaussians)
    assert 0.55 < np.percentile(r, 1) and np.percentile(r, 99) < 1.05 and abs(np.median(r) - 0.8) < 0.03, np.percentile(r, [1, 50, 99])


def test_shard_views_round_robin():
    from gs2mesh_b200.tsdf import shard_views

    assert shard_views(7, 0, 2) == [0, 2, 4, 6] and shard_views(7, 1, 2) == [1, 3, 5]
    got = sorted(v for r in range(8) for v in shard_views(500, r, 8))
    assert got == list(range(500))
    assert max(len(shard_views(500, r, 8)) for r in range(8)) - min(len(shard_views(500, r, 8)) for r in range(8)) <= 1
    assert shard_views(3, 5, 8) == []


def test_view_shards_merged_by_merge_oracle_equal_sequential_fusion(c0, oracle):
    """SURVEY 8(e) on the C0 case: ranks take views round-robin, and the multi-GPU merge's host restatement
    (tests/merge_oracle.py) of the two ranks' volumes opens the sequential fusion's units with the same weights and tsdf."""
    from gs2mesh_b200.tsdf import shard_views
    from tests.merge_oracle import merge_oracle

    cfg = c0["cfg"]
    vl = 2.0 / cfg["tsdf_res"]
    trunc = max(0.04, 3 * vl)

    def fuse(views):
        """{(bx,by,bz): (tsdf, weight) [4096,2]} of every unit the views open."""
        vol = oracle.OracleTSDFVolume(vl, trunc, with_color=False)
        for i in views:
            _integrate(c0, vol, i)
        return {tuple(int(v) for v in k): np.stack(vol.unit_data(i)[:2], -1) for i, k in enumerate(vol.unit_indices())}

    ref = fuse(range(cfg["pairs"]))
    ranks = [{k: (tw, None) for k, tw in fuse(shard_views(cfg["pairs"], rank, 2)).items()} for rank in range(2)]
    merged = merge_oracle(ranks, None, len(set(ranks[0]) | set(ranks[1])))[0].merged
    assert set(merged) == set(ref)
    for k, (tw, _) in merged.items():  # two ranks: one candidate per voxel
        np.testing.assert_array_equal(tw[0][:, 1], ref[k][:, 1])
        assert np.abs(tw[0][:, 0] - ref[k][:, 0]).max() < 1e-6
