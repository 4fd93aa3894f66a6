"""Times surface and voxel point-cloud extraction (ScalableTSDFVolume::ExtractPointCloud / ExtractVoxelPointCloud) on
the TSDF volume of the synthetic C1 scene (voxel 2/512), on the GPU and with the numpy restatement the tests compare
against (tests/pointcloud_oracle.py), checks that both give the same arrays, and prints one JSON line with the card's
name and power limit, read in the same run.  Everything it writes goes to a temporary directory.

The GPU path is timed with CUDA events around the whole call after a warm-up, so the count, scan, emit, sort, attribute
kernels and the download of the arrays to the host are all inside the window; the numpy path with a host clock, on the
dense window of the same bricks (the read-back itself is not timed).

    python scripts/pointcloud_time.py [--views 20] [--reps 5]
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from scripts.mesh_clean_time import _card  # noqa: E402  (the card's name and power limit)


def _c1_volume(dev, views, tmp):
    """The TSDF volume the stage fuses from the C1 scene, with the reference's defaults at voxel 2/512 (as in
    scripts/mesh_clean_time.py)."""
    from gs2mesh_b200 import scene
    from gs2mesh_b200.renderer import Renderer
    from gs2mesh_b200.tsdf import TSDF

    cfg = scene.CONFIGS["C1"]

    class Args:
        GS_white_background = False
        TSDF_scale = 1.0
        TSDF_voxel = 2.0
        TSDF_sdf_trunc = 0.04
        TSDF_dilate = 1
        TSDF_valid = None
        TSDF_skip = None
        TSDF_use_mask = False
        TSDF_use_occlusion_mask = False
        TSDF_min_depth_baselines = cfg["min_db"]
        TSDF_max_depth_baselines = cfg["max_db"]

    cloud = scene.make_gaussians(cfg["num_points"], seed=1)
    rigs, baseline = scene.make_stereo_cameras(views, cfg["width"], cfg["height"], layout=cfg["layout"])
    r = Renderer.from_scene(rigs, baseline, cloud, output_dir_root=tmp, args=Args(), device=str(dev))
    r.prepare_renderer()
    r.keep_frames = True
    for i in range(len(r)):
        r.render_image_pair(i)
    stage = TSDF(r, None, Args(), "c1", window_resolution=cfg["tsdf_res"], device=str(dev))
    stage.run()
    return stage.volume


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--max-window-bricks", type=int, default=150000)
    args = ap.parse_args()

    import torch

    from gs2mesh_b200.mesh import extract_point_cloud, extract_voxel_point_cloud
    from tests.pointcloud_oracle import extract_point_cloud_from_bricks, extract_voxel_point_cloud_from_bricks

    dev = torch.device("cuda", 0)
    with tempfile.TemporaryDirectory() as tmp:
        vol = _c1_volume(dev, args.views, tmp)
    name, power = _card()

    def gpu_ms(fn):
        fn()
        torch.cuda.synchronize()
        out = []
        for _ in range(args.reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            r = fn()
            b.record()
            torch.cuda.synchronize()
            out.append(a.elapsed_time(b))
        return float(np.median(out)), r

    surf_ms, surf = gpu_ms(lambda: extract_point_cloud(vol))
    vox_ms, vox = gpu_ms(lambda: extract_voxel_point_cloud(vol))

    b0, nb = surf.key_window
    units = vol.export_units()
    total = int(np.prod(nb))
    if total > args.max_window_bricks:  # the numpy path works on the dense window: 8 bytes per voxel and temporaries
        raise SystemExit(f"key window of {total} bricks is larger than --max-window-bricks {args.max_window_bricks}")
    tw = np.zeros((total, 4096, 2), np.float32)
    col = np.zeros((total, 4096, 3), np.float32)
    alloc = np.zeros(total, bool)
    for (bx, by, bz), (t, c) in units.items():
        i = ((bx - b0[0]) * nb[1] + (by - b0[1])) * nb[2] + (bz - b0[2])
        tw[i], col[i], alloc[i] = t, c[:, :3], True
    t0 = time.perf_counter()
    ref = extract_point_cloud_from_bricks(tw, b0, nb, vol.voxel_length, color=col, allocated=alloc)
    host_surf_ms = (time.perf_counter() - t0) * 1e3
    t0 = time.perf_counter()
    vref = extract_voxel_point_cloud_from_bricks(tw, b0, nb, vol.voxel_length)
    host_vox_ms = (time.perf_counter() - t0) * 1e3
    same = (np.array_equal(surf.keys, ref["keys"]) and surf.points.tobytes() == ref["points"].tobytes()
            and surf.colors.tobytes() == ref["colors"].tobytes() and surf.normals.tobytes() == ref["normals"].tobytes()
            and np.array_equal(vox.keys, vref["keys"]) and vox.points.tobytes() == vref["points"].tobytes()
            and vox.colors.tobytes() == vref["colors"].tobytes())
    print(json.dumps(dict(card=name, power_limit=power, scene="C1", views=args.views, bricks=vol.num_bricks(),
                          key_window=[list(b0), list(nb)], surface_points=len(surf.points), voxel_points=len(vox.points),
                          gpu_surface_ms=round(surf_ms, 3), gpu_voxel_ms=round(vox_ms, 3),
                          numpy_surface_ms=round(host_surf_ms, 1), numpy_voxel_ms=round(host_vox_ms, 1),
                          reps=args.reps, identical=bool(same))))


if __name__ == "__main__":
    main()
