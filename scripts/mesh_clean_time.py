"""Times TriangleMesh cluster cleaning (tsdf_utils.py:122-142) on the host path (numpy / scipy) and on the GPU path, on
shuffled grid meshes of about 1M and 4M triangles and on the TSDF mesh of the synthetic C1 scene (voxel 2/512), checks
that both paths give the same output, and prints one JSON line with the card's name and power limit, read in the same
run.  Everything it writes goes to a temporary directory.

The host path is timed with a host clock; the GPU path with CUDA events and a final synchronise around the whole call
after a warm-up, so the triangle upload, the kernels, the index download and the host gather of the vertex arrays are
all inside the window.

    python scripts/mesh_clean_time.py [--grids 1000000,4000000] [--views 20] [--threshold 100000] [--reps 5]
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


def _shuffled_grid(n_triangles, rng):
    """One edge-connected sheet of ~n_triangles triangles with shuffled vertex ids and triangle order, colours and
    normals; plus 1000 lone triangles so that the cleaning removes something."""
    n = int(round(np.sqrt(n_triangles / 2)))
    g = np.arange((n + 1) * (n + 1)).reshape(n + 1, n + 1)
    a, b, c, d = g[:-1, :-1].ravel(), g[:-1, 1:].ravel(), g[1:, :-1].ravel(), g[1:, 1:].ravel()
    t = np.concatenate([np.stack([a, b, d], 1), np.stack([a, d, c], 1), g.size + np.arange(3000).reshape(1000, 3)])
    nv = g.size + 3000
    perm = rng.permutation(nv)
    t = perm[t][rng.permutation(len(t))]
    v = np.empty((nv, 3))
    v[perm] = rng.normal(size=(nv, 3))
    return v, t, rng.random((nv, 3)), rng.normal(size=(nv, 3))


def _c1_mesh(dev, views, tmp):
    from gs2mesh_b200 import scene
    from gs2mesh_b200.renderer import Renderer
    from gs2mesh_b200.tsdf import TSDF

    cfg = scene.CONFIGS["C1"]

    class Args:  # the reference's defaults (argument_utils.py:29-42,74-90) at voxel 2/512
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
    return stage.extract_mesh()


def _same(a, b):
    if a is None or b is None:
        return a is None and b is None
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


def _time(mesh, threshold, reps):
    import torch

    from gs2mesh_b200.mesh import TriangleMesh

    host = TriangleMesh(mesh.vertices, mesh.triangles, mesh.vertex_colors, mesh.vertex_normals)
    gpu = TriangleMesh(mesh.vertices, mesh.triangles, mesh.vertex_colors, mesh.vertex_normals, device=mesh.device)
    out = {"triangles": int(len(mesh.triangles)), "vertices": int(len(mesh.vertices))}

    def host_clock(fn):
        t = time.perf_counter()
        r = fn()
        return r, (time.perf_counter() - t) * 1e3

    def gpu_clock(fn):
        fn()  # warm-up
        ev, wall, r = [], [], None
        for _ in range(reps):
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t = time.perf_counter()
            a.record()
            r = fn()
            b.record()
            torch.cuda.synchronize()
            wall.append((time.perf_counter() - t) * 1e3)
            ev.append(a.elapsed_time(b))
        return r, float(np.median(ev)), float(np.median(wall))

    want, out["host_remove_small_clusters_ms"] = host_clock(lambda: host.remove_small_clusters(threshold))
    hc, out["host_cluster_connected_triangles_ms"] = host_clock(host.cluster_connected_triangles)
    got, out["gpu_remove_small_clusters_ms"], out["gpu_remove_small_clusters_wall_ms"] = gpu_clock(
        lambda: gpu.remove_small_clusters(threshold))
    gc, out["gpu_cluster_connected_triangles_ms"], out["gpu_cluster_connected_triangles_wall_ms"] = gpu_clock(
        gpu.cluster_connected_triangles)
    out["speedup_remove_small_clusters"] = round(out["host_remove_small_clusters_ms"] / out["gpu_remove_small_clusters_ms"], 1)
    out["kept_triangles"] = int(len(got.triangles))
    out["same_cleaned_mesh"] = all(_same(getattr(got, k), getattr(want, k))
                                   for k in ("vertices", "triangles", "vertex_colors", "vertex_normals"))
    out["same_labels_counts"] = _same(gc[0], hc[0]) and _same(gc[1], hc[1])
    out["area_max_rel_diff"] = float(np.max(np.abs(gc[2] - hc[2]) / np.maximum(np.abs(hc[2]), 1e-300))) if len(hc[2]) else 0.0
    return {k: round(v, 2) if isinstance(v, float) and k != "area_max_rel_diff" else v for k, v in out.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--grids", default="1000000,4000000")
    ap.add_argument("--views", type=int, default=20)
    ap.add_argument("--threshold", type=float, default=100000.0)  # TSDF_cleaning_threshold / TSDF_scale, the defaults
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()

    import torch

    from __graft_entry__ import build
    from gs2mesh_b200.mesh import TriangleMesh

    assert torch.cuda.is_available(), "mesh_clean_time needs a CUDA device"
    build()
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(args.seed)
    results = {}
    with torch.cuda.device(dev):
        for n in (int(x) for x in args.grids.split(",") if x):
            v, t, col, nrm = _shuffled_grid(n, rng)
            results[f"grid_{n}"] = _time(TriangleMesh(v, t, col, nrm, device=dev), args.threshold, args.reps)
        with tempfile.TemporaryDirectory() as tmp:
            results[f"c1_tsdf_{args.views}_views"] = _time(_c1_mesh(dev, args.views, tmp), args.threshold, args.reps)
    name, power = _card()
    print(json.dumps({"card": name, "power_limit": power, "threshold": args.threshold, "reps": args.reps,
                      "host_cpus": os.cpu_count(), **results}))


if __name__ == "__main__":
    main()
