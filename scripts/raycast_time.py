"""Times the TSDF ray cast (gsb_tsdf_raycast) per view on the volume the stage fuses from the synthetic C1 scene (1M
Gaussians, 1600x1200, voxel 2/512), fused over each given number of views, and prints one JSON line per view count with
the card's name and power limit, read in the same run.  Everything it writes goes to a temporary directory.

Each left camera is cast with TSDF.raycast (depth, normals and colours, the integration's own depth range) after one
warm-up cast per camera; CUDA events around each call give its time, reported as the median and the spread over all
left cameras.

    python scripts/raycast_time.py [--views 20 200] [--reps 3]
"""
import argparse
import json
import os
import sys
import tempfile

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from scripts.mesh_clean_time import _card  # noqa: E402  (the card's name and power limit)
from scripts.pointcloud_time import _c1_volume  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, nargs="+", default=[20, 200])
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()

    import torch

    from gs2mesh_b200 import scene
    from gs2mesh_b200.tsdf import TSDF

    dev = torch.device("cuda", 0)
    name, power = _card()
    cfg = scene.CONFIGS["C1"]
    for views in args.views:
        with tempfile.TemporaryDirectory() as tmp:
            vol = _c1_volume(dev, views, tmp)
        rigs, baseline = scene.make_stereo_cameras(views, cfg["width"], cfg["height"], layout=cfg["layout"])

        class Args:
            TSDF_scale = 1.0
            TSDF_min_depth_baselines = cfg["min_db"]
            TSDF_max_depth_baselines = cfg["max_db"]

        class Rig:
            pass

        rig = Rig()
        rig.baseline = baseline
        stage = TSDF(rig, None, Args(), "c1", device=str(dev))
        stage.volume = vol
        cams = [r["left"] for r in rigs]
        for cam in cams:
            stage.raycast(cam)
        torch.cuda.synchronize()
        ms, hits = [], []
        for cam in cams:
            per = []
            for _ in range(args.reps):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                out = stage.raycast(cam)
                b.record()
                torch.cuda.synchronize()
                per.append(a.elapsed_time(b))
            ms.append(float(np.median(per)))
            hits.append(int((out.depth > 0).sum().item()))
        ms = np.array(ms)
        print(json.dumps(dict(card=name, power_limit=power, scene="C1", views=views, bricks=vol.num_bricks(),
                              width=cfg["width"], height=cfg["height"], cameras=len(cams),
                              median_ms=round(float(np.median(ms)), 3), min_ms=round(float(ms.min()), 3),
                              p90_ms=round(float(np.percentile(ms, 90)), 3), max_ms=round(float(ms.max()), 3),
                              median_hit_fraction=round(float(np.median(hits)) / (cfg["width"] * cfg["height"]), 4),
                              reps=args.reps)), flush=True)
        del vol, stage


if __name__ == "__main__":
    main()
