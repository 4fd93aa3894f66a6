"""Times point-cloud cleaning and downsampling (gs2mesh_b200.pointcloud: remove_statistical_outlier,
remove_radius_outlier, voxel_down_sample with colours and normals, select_by_index, uniform_down_sample,
compute_nearest_neighbor_distance, compute_point_cloud_distance) on the surface cloud of the synthetic C1 scene's TSDF
volume (voxel 2/512, the cloud of scripts/pointcloud_time.py), checks every output against the numpy restatement
(tests/pcd_oracle.py) in the same run, and prints one JSON line with the card's name and power limit, read in the same
run.  Everything it writes goes to a temporary directory.

Each GPU call is the whole method (upload, grid build, kernels, compaction, download), the median of --reps calls after
a warm-up, timed with CUDA events and a final synchronise.  The numpy restatement runs once per operation, timed with a
host clock.

    python scripts/pointcloud_filter_time.py [--views 20] [--reps 5]
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
from scripts.pointcloud_time import _c1_volume  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()

    import torch

    from gs2mesh_b200.mesh import extract_point_cloud
    from tests import pcd_oracle as po

    dev = torch.device("cuda", 0)
    if not torch.cuda.is_available():
        raise SystemExit("pointcloud_filter_time.py needs a CUDA device")
    with tempfile.TemporaryDirectory() as tmp:
        vol = _c1_volume(dev, args.views, tmp)
    pcd = extract_point_cloud(vol)
    vl = vol.voxel_length
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

    def host_ms(fn):
        t0 = time.perf_counter()
        r = fn()
        return (time.perf_counter() - t0) * 1e3, r

    same = lambda a, b: a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()
    rng = np.random.default_rng(0)
    half = rng.permutation(len(pcd.points))[: len(pcd.points) // 2]
    rows = []

    def row(op, fn, ref_fn, check):
        g_ms, got = gpu_ms(fn)
        h_ms, ref = host_ms(ref_fn)
        rows.append(dict(op=op, gpu_ms=round(g_ms, 3), numpy_ms=round(h_ms, 1), identical=bool(check(got, ref))))
        return got

    def cloud_check(got, ref):
        p, c, n = ref
        return same(got.points, p) and same(got.colors, c) and same(got.normals, n)

    def selected(keep):
        return pcd.points[keep], pcd.colors[keep], pcd.normals[keep]

    def stat_ref():
        keep = po.statistical(pcd.points, 20, 2.0)[1]
        return selected(keep), np.nonzero(keep)[0]

    clean, _ = row("remove_statistical_outlier(20, 2.0)", lambda: pcd.remove_statistical_outlier(20, 2.0), stat_ref,
                   lambda g, r: cloud_check(g[0], r[0]) and same(g[1], r[1].astype(np.int64)))

    def radius_ref():
        keep = po.radius(pcd.points, 8, 2 * vl)
        return selected(keep), np.nonzero(keep)[0]

    row("remove_radius_outlier(8, 2 voxels)", lambda: pcd.remove_radius_outlier(8, 2 * vl), radius_ref,
        lambda g, r: cloud_check(g[0], r[0]) and same(g[1], r[1].astype(np.int64)))
    thin = row("voxel_down_sample(2 voxels)", lambda: pcd.voxel_down_sample(2 * vl),
               lambda: po.voxel_down_sample(pcd.points, 2 * vl, pcd.colors, pcd.normals), cloud_check)
    row("select_by_index(half, shuffled)", lambda: pcd.select_by_index(half),
        lambda: selected(po.select(len(pcd.points), half)), cloud_check)
    row("uniform_down_sample(5)", lambda: pcd.uniform_down_sample(5),
        lambda: (pcd.points[::5], pcd.colors[::5], pcd.normals[::5]), cloud_check)
    row("compute_nearest_neighbor_distance()", pcd.compute_nearest_neighbor_distance,
        lambda: po.nearest_neighbor_distance(pcd.points), same)
    from tests.normals_oracle import knn

    row("compute_point_cloud_distance(voxel_down_sample)", lambda: pcd.compute_point_cloud_distance(thin),
        lambda: np.sqrt(knn(pcd.points, thin.points, 1)[0][:, 0]), same)
    print(json.dumps(dict(card=name, power_limit=power, scene="C1", views=args.views, points=len(pcd.points),
                          kept_statistical=len(clean.points), voxel_points=len(thin.points), voxel_length=vl,
                          reps=args.reps, rows=rows)))


if __name__ == "__main__":
    main()
