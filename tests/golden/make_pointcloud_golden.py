#!/usr/bin/env python
"""Generates tests/golden/pointcloud_o3d_<case>.npz from the wheel the reference's TSDF half is, open3d==0.17.0.  On the
frames and cases of make_tsdf_golden.py it runs the literal call sequence

    volume = o3d.pipelines.integration.ScalableTSDFVolume(voxel_length, sdf_trunc, color_type=RGB8)
    volume.integrate(rgbd, PinholeCameraIntrinsic(w, h, fx, fy, cx, cy), inv(extrinsic))     # per frame
    pcd = volume.extract_point_cloud()            # points, colors, normals (fp64)
    vox = volume.extract_voxel_point_cloud()      # points, colors (fp64)

and stores the inputs next to the outputs, so the consuming test (tests/test_pointcloud_golden.py) needs neither open3d
nor this script.  Open3D's point order follows its hash map; the test compares sorted sets.

STATUS: open3d 0.17.0 publishes no cp312 wheel, so the fixtures do not exist yet and the consuming test skips.

    python tests/golden/make_pointcloud_golden.py                 # needs `import open3d` == 0.17.0
    python tests/golden/make_pointcloud_golden.py --backend oracle --out /tmp/x   # plumbing check of the consuming test
                                                                                  # ONLY; never commit those files
"""
from __future__ import annotations

import argparse
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tests.golden.make_tsdf_golden import CASES, make_frames, oracle_volume, reference_filters  # noqa: E402


def run_open3d(case):
    import open3d as o3d

    if not o3d.__version__.startswith("0.17.0"):
        raise SystemExit(f"open3d {o3d.__version__} is not the reference's 0.17.0")
    c = CASES[case]
    frames = make_frames(case)
    volume = o3d.pipelines.integration.ScalableTSDFVolume(voxel_length=c["voxel"] / 512, sdf_trunc=c["trunc"],
                                                          color_type=o3d.pipelines.integration.TSDFVolumeColorType.RGB8)
    for f in frames:
        d, e, trunc = reference_filters(f["depth"], f["extrinsic"], c["scale"])
        rgbd = o3d.geometry.RGBDImage.create_from_color_and_depth(o3d.geometry.Image(f["rgb"]), o3d.geometry.Image(d),
                                                                   depth_scale=c["scale"], depth_trunc=trunc,
                                                                   convert_rgb_to_intensity=False)
        intr = o3d.camera.PinholeCameraIntrinsic(c["W"], c["H"], c["fx"], c["fy"], c["cx"], c["cy"])
        volume.integrate(rgbd, intr, np.linalg.inv(e))
    pcd = volume.extract_point_cloud()
    vox = volume.extract_voxel_point_cloud()
    out = dict(points=np.asarray(pcd.points), colors=np.asarray(pcd.colors), normals=np.asarray(pcd.normals),
               voxel_points=np.asarray(vox.points), voxel_colors=np.asarray(vox.colors), backend=f"open3d {o3d.__version__}")
    return frames, out


def oracle_clouds(case, vol):
    """The same read-outs from the CPU restatement of the volume and tests/pointcloud_oracle.py."""
    from tests.pointcloud_oracle import extract_point_cloud_from_bricks, extract_voxel_point_cloud_from_bricks

    vl = CASES[case]["voxel"] / 512
    units = vol.unit_indices()
    b0 = units.min(axis=0)
    nb = units.max(axis=0) - b0 + 2
    tw, alloc, outside = vol.export_bricks(b0, nb)
    assert outside == 0
    col = np.zeros((tw.shape[0], 4096, 3), np.float32)
    for i, idx in enumerate(units):
        b = idx - b0
        col[(b[0] * nb[1] + b[1]) * nb[2] + b[2]] = vol.unit_data(i)[2]
    s = extract_point_cloud_from_bricks(tw, b0, nb, vl, color=col, allocated=alloc.astype(bool))
    v = extract_voxel_point_cloud_from_bricks(tw, b0, nb, vl)
    return dict(points=s["points"], colors=s["colors"], normals=s["normals"], voxel_points=v["points"],
                voxel_colors=v["colors"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--backend", default="open3d", choices=["open3d", "oracle"])
    ap.add_argument("--out", default=HERE)
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    for case in CASES:
        if args.backend == "open3d":
            frames, out = run_open3d(case)
        else:
            frames = make_frames(case)
            out = dict(oracle_clouds(case, oracle_volume(case, frames)), backend="oracle (plumbing check, NOT golden)")
        path = os.path.join(args.out, f"pointcloud_o3d_{case}.npz")
        np.savez_compressed(path, case=case, depth=np.stack([f["depth"] for f in frames]), rgb=np.stack([f["rgb"] for f in frames]),
                            extrinsic=np.stack([f["extrinsic"] for f in frames]), **out)
        print("wrote", path, out["backend"], "points", len(out["points"]), "voxels", len(out["voxel_points"]))


if __name__ == "__main__":
    main()
