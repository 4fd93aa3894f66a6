"""Times gs2mesh_b200.tnt.run_evaluation stage by stage on a synthetic Tanks and Temples scene (default: a 5M-point
reconstruction against a 20M-point GT) and prints one JSON line with the card's name and power limit, read in the same
run.  Everything it writes goes to a temporary directory.

    python scripts/tnt_eval_time.py [--recon 5000000] [--gt 20000000] [--tau 0.005]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

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


def _surface(n, rng):
    xy = rng.uniform(-5, 5, size=(n, 2))
    z = 0.5 * np.sin(1.3 * xy[:, 0]) * np.cos(0.7 * xy[:, 1]) + 0.02 * xy[:, 0] ** 2
    return np.concatenate([xy, z[:, None]], 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--recon", type=int, default=5_000_000)
    ap.add_argument("--gt", type=int, default=20_000_000)
    ap.add_argument("--tau", type=float, default=0.005)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()

    import torch

    from __graft_entry__ import build
    from gs2mesh_b200 import tnt
    from gs2mesh_b200.io import write_point_cloud_ply

    assert torch.cuda.is_available(), "tnt_eval_time needs a CUDA device"
    build()
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(args.seed)
    tau = args.tau
    gt_trans = np.eye(4)
    gt_trans[:3, :3] *= 1.5
    gt_trans[:3, 3] = [0.3, -0.2, 0.1]
    gt = _surface(args.gt, rng)
    delta = np.eye(4)
    delta[:3, 3] = [0.4 * tau, -0.3 * tau, 0.2 * tau]
    recon = tnt._host_transform(_surface(args.recon, rng) + rng.normal(scale=tau / 4, size=(args.recon, 3)),
                                np.linalg.inv(gt_trans) @ delta)
    poly = [[-4.5, -4.5, 0], [4.5, -4.2, 0], [3.0, 0.5, 0], [4.5, 4.5, 0], [-4.5, 4.4, 0]]
    vol = tnt.SelectionPolygonVolume("z", -1.0, 1.0, np.array(poly, dtype=np.float64))
    traj = [tnt.CameraPose([i, i, 200], np.block([[np.eye(3), np.array([[6 * np.cos(a)], [6 * np.sin(a)], [2.0]])],
                                                  [np.zeros((1, 3)), np.ones((1, 1))]]))
            for i, a in enumerate(np.linspace(0, 2 * np.pi, 200, endpoint=False))]

    def timed(fn):
        torch.cuda.synchronize()
        t = time.perf_counter()
        r = fn()
        torch.cuda.synchronize()
        return r, (time.perf_counter() - t) * 1e3

    with tempfile.TemporaryDirectory() as tmp:
        pcd = torch.as_tensor(recon, device=dev)
        gt_pcd = torch.as_tensor(gt, device=dev)
        # warm-up of every kernel and allocation shape at a small size
        tnt.registration_vol_ds(pcd[:100000], gt_pcd[:400000], gt_trans, vol, tau, 80 * tau, 20, verbose=False)
        tnt.estimate_normals(pcd[:100000], 20)
        stages = {}
        T0, stages["alignment_ms"] = timed(lambda: tnt.trajectory_alignment(None, traj, traj, gt_trans, seed=args.seed))
        r2, stages["vol_ds_1_ms"] = timed(lambda: tnt.registration_vol_ds(pcd, gt_pcd, T0, vol, tau, tau * 80, 20,
                                                                          verbose=False))
        r3, stages["vol_ds_2_ms"] = timed(lambda: tnt.registration_vol_ds(pcd, gt_pcd, r2.transformation, vol, tau / 2,
                                                                          tau * 20, 20, verbose=False))
        r, stages["unif_ms"] = timed(lambda: tnt.registration_unif(pcd, gt_pcd, r3.transformation, vol, 2 * tau, 20,
                                                                   verbose=False))
        res, stages["histo_ms"] = timed(lambda: tnt.evaluate_histo(pcd, gt_pcd, r.transformation, vol, tau / 2, tau, tmp, 5,
                                                                   "Synth"))
        # the normals evaluate_histo estimates, alone: the downsampled GT (the larger of its two clouds), grid included
        t_ds = tnt.voxel_down_sample(tnt.crop_point_cloud(gt_pcd, vol), tau / 2)
        _, stages["normals_gt_ms"] = timed(lambda: tnt.estimate_normals(t_ds, 20))
        # the whole run_evaluation from files, PLY reads included
        d = os.path.join(tmp, "Synth")
        os.makedirs(d)
        write_point_cloud_ply(os.path.join(d, "Synth.ply"), gt)
        write_point_cloud_ply(os.path.join(tmp, "recon.ply"), recon)
        np.savetxt(os.path.join(d, "Synth_trans.txt"), gt_trans)
        with open(os.path.join(d, "Synth.json"), "w") as f:
            json.dump({"orthogonal_axis": "Z", "axis_min": -1.0, "axis_max": 1.0, "bounding_polygon": poly}, f)
        with open(os.path.join(d, "Synth_COLMAP_SfM.log"), "w") as f:
            for t in traj:
                f.write(" ".join(map(str, t.metadata)) + "\n" + "\n".join(" ".join("%.12f" % x for x in row) for row in t.pose)
                        + "\n")
        log = os.path.join(d, "Synth_COLMAP_SfM.log")
        eva, stages["run_evaluation_ms"] = timed(lambda: tnt.run_evaluation(d, log, os.path.join(tmp, "recon.ply"),
                                                                            os.path.join(tmp, "out"), seed=args.seed,
                                                                            tau=tau))
    name, power = _card()
    print(json.dumps({"card": name, "power_limit": power, "recon_points": args.recon, "gt_points": args.gt, "tau": tau,
                      "icp_iterations": [r2.iterations, r3.iterations, r.iterations], "precision_recall_fscore": eva,
                      "normals_gt_points": int(t_ds.shape[0]),
                      **{k: round(v, 2) for k, v in stages.items()}}))


if __name__ == "__main__":
    main()
