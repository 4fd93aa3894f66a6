"""Times gs2mesh_b200.mobilebrick.evaluate_single phase by phase on a synthetic MobileBrick scan (default: a GT mesh and a
prediction of about 1M triangles each, 100 000 Poisson-disk points per mesh) and prints one JSON line with the card's
name and power limit, read in the same run.  Each phase is timed with CUDA events around it (the host work inside a
phase included), the median of --repeats runs after one warm-up run.  Everything it writes goes to a temporary
directory.

    python scripts/mobilebrick_eval_time.py [--grid 708] [--points 100000] [--repeats 5]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in q.split(",")]
        return name, power
    except Exception as e:  # the timing is still reported; the card stays unknown
        return f"unknown ({e})", "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--grid", type=int, default=708, help="vertices per side of the heightfield (2 (g-1)^2 triangles)")
    ap.add_argument("--points", type=int, default=100000)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()

    import torch

    from __graft_entry__ import build
    from gs2mesh_b200 import mobilebrick as mb
    from gs2mesh_b200.evaluate import precision_recall_f1
    from gs2mesh_b200.io import read_triangle_mesh_ply
    from gs2mesh_b200.mesh import TriangleMesh
    from tests import mobilebrick_cases as mc

    assert torch.cuda.is_available(), "mobilebrick_eval_time needs a CUDA device"
    build()
    dev = torch.device("cuda", 0)
    N = args.points

    with tempfile.TemporaryDirectory() as tmp:
        gt_dir, pred_path, exp, _ = mc.write_scan(tmp, nx=args.grid, ny=args.grid, seed=args.seed)
        d = np.load(os.path.join(gt_dir, "visibility_mask.npy"), allow_pickle=True).item()

        def run():
            ev = []

            def mark():
                e = torch.cuda.Event(enable_timing=True)
                e.record()
                ev.append(e)

            mark()
            gv, gt = read_triangle_mesh_ply(os.path.join(gt_dir, "mesh", "gt_mesh.ply"))
            pv, pt, pc = read_triangle_mesh_ply(pred_path, with_colors=True)
            gvd, gtd = mb._mesh(gv, gt, dev)
            pvd = mb._points(pv, dev)
            mark()
            stream = mb.Mt19937Stream(args.seed)
            gt_points, info = mb.sample_points_poisson_disk(gvd, gtd, N, stream=stream, return_info=True)
            mark()
            pvd, reg = mb.align_prediction(gvd, pvd)
            mark()
            keep = mb.visibility_test(pvd, d["mask"], d["min_pts"], d["resolutions"], d["voxel_size"])
            v, t, c, _ = mb.remove_vertices_by_mask(pvd, pt, ~keep, pc)
            mesh = TriangleMesh(v.cpu().numpy(), t.cpu().numpy(), c.cpu().numpy())
            mesh.compute_vertex_normals(dev)
            mark()
            pred_points = mb.sample_points_poisson_disk(v, t, N, stream=stream)
            mark()
            mesh.write_ply(os.path.join(exp, "timing_cropped.ply"))
            mark()
            a = precision_recall_f1(pred_points, gt_points, 0.0025)
            b = precision_recall_f1(pred_points, gt_points, 0.005)
            mark()
            torch.cuda.synchronize()
            names = ["read_ms", "gt_poisson_ms", "icp_ms", "crop_normals_ms", "pred_poisson_ms", "write_ply_ms", "metrics_ms"]
            ms = {k: ev[i].elapsed_time(ev[i + 1]) for i, k in enumerate(names)}
            ms["total_ms"] = ev[0].elapsed_time(ev[-1])
            out = [a["chamfer"], a["accuracy"], a["recall"], a["F1"], b["accuracy"], b["recall"], b["F1"]]
            return ms, out, info["rounds"], reg.iterations, len(gt), len(t)

        run()  # warm-up: module load, allocations, every kernel
        runs = [run() for _ in range(args.repeats)]
    name, power = _card()
    keys = runs[0][0].keys()
    med = {k: round(statistics.median(r[0][k] for r in runs), 2) for k in keys}
    same = all(r[1] == runs[0][1] for r in runs)
    print(json.dumps({"card": name, "power_limit": power, "gt_triangles": runs[0][4], "cropped_pred_triangles": runs[0][5],
                      "points": N, "gt_elimination_rounds": runs[0][2], "icp_iterations": runs[0][3],
                      "repeats": args.repeats, "identical_results": same, "result": runs[0][1], **med}))


if __name__ == "__main__":
    main()
