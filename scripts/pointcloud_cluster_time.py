"""Times density clustering (gs2mesh_b200.pointcloud.cluster_dbscan) on the surface cloud of the synthetic C1 scene's
TSDF volume (voxel 2/512, the cloud of scripts/pointcloud_time.py) at eps = 2, 4 and 8 voxels with min_points = 10, and
on 50,000 points inside a ball of diameter below eps (every pair within eps: the link pass's worst case).  Checks every
label against the numpy restatement (tests/dbscan_oracle.py) in the same run; the ball is checked against its known
answer instead (every label 0), because the restatement would hold its 1.25e9 pairs.  Prints one JSON line with the
card's name and power limit, read in the same run.  Everything it writes goes to a temporary directory.

Each GPU time is the whole call (upload, grid build, kernels, download), the median of --reps calls after a warm-up,
timed with CUDA events and a final synchronise.  The restatement runs once per row, timed with a host clock.

    python scripts/pointcloud_cluster_time.py [--views 20] [--reps 5]
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

    from gs2mesh_b200.mesh import PointCloud, extract_point_cloud
    from tests import dbscan_oracle as do

    dev = torch.device("cuda", 0)
    if not torch.cuda.is_available():
        raise SystemExit("pointcloud_cluster_time.py needs a CUDA device")
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

    same = lambda a, b: a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()
    rows = []
    for voxels in (2, 4, 8):
        eps = voxels * vl
        g_ms, got = gpu_ms(lambda: pcd.cluster_dbscan(eps, 10))
        t0 = time.perf_counter()
        ref, n_clusters = do.dbscan(pcd.points, eps, 10)
        h_ms = (time.perf_counter() - t0) * 1e3
        rows.append(dict(op=f"cluster_dbscan({voxels} voxels, 10)", points=len(pcd.points), gpu_ms=round(g_ms, 3),
                         numpy_ms=round(h_ms, 1), clusters=n_clusters, noise=int((ref == -1).sum()),
                         identical=bool(same(got, ref))))

    rng = np.random.default_rng(0)
    v = rng.normal(size=(50000, 3))
    ball = PointCloud(v / np.linalg.norm(v, axis=1, keepdims=True) * 0.45 * rng.uniform(size=(50000, 1)) ** (1 / 3),
                      device=dev)
    g_ms, got = gpu_ms(lambda: ball.cluster_dbscan(1.0, 10))
    rows.append(dict(op="cluster_dbscan(1.0, 10), 50,000 points in a ball of diameter 0.9", points=50000,
                     gpu_ms=round(g_ms, 3), numpy_ms=None, clusters=int(got.max()) + 1,
                     identical=bool(same(got, np.zeros(50000, np.int32)))))
    print(json.dumps(dict(card=name, power_limit=power, scene="C1", views=args.views, voxel_length=vl, reps=args.reps,
                          rows=rows)))


if __name__ == "__main__":
    main()
