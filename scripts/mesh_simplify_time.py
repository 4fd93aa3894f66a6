"""Times TriangleMesh.simplify_vertex_clustering on the GPU and the numpy restatement (tests/simplify_oracle.py) on the
host, on shuffled grid meshes of about 1M and 4M triangles and on the TSDF mesh of the synthetic C1 scene (voxel 2/512),
at voxel sizes of 2x and 4x the mesh's spacing with both contractions; checks that both give the same arrays, and prints
one JSON line with the card's name and power limit, read in the same run.  Everything it writes goes to a temporary
directory.

The GPU call is timed with CUDA events and a final synchronise around the whole call after a warm-up, so the uploads,
the kernels and the downloads are all inside the window; the restatement once with a host clock.

    python scripts/mesh_simplify_time.py [--grids 1000000,4000000] [--views 20] [--reps 5]
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from mesh_clean_time import _c1_mesh, _card, _same  # noqa: E402


def _shuffled_grid(n_triangles, rng):
    """One sheet of ~n_triangles triangles at spacing 0.01 on a wavy surface, with shuffled vertex ids and triangle
    order, colours and normals."""
    n = int(round(np.sqrt(n_triangles / 2)))
    g = np.arange((n + 1) * (n + 1)).reshape(n + 1, n + 1)
    a, b, c, d = g[:-1, :-1].ravel(), g[:-1, 1:].ravel(), g[1:, :-1].ravel(), g[1:, 1:].ravel()
    t = np.concatenate([np.stack([a, b, d], 1), np.stack([a, d, c], 1)])
    perm = rng.permutation(g.size)
    t = perm[t][rng.permutation(len(t))]
    xy = np.stack(np.meshgrid(np.arange(n + 1.0), np.arange(n + 1.0), indexing="ij"), -1).reshape(-1, 2) * 0.01
    v = np.empty((g.size, 3))
    v[perm] = np.concatenate([xy, np.sin(xy[:, :1] * 3) * 0.1], 1)
    return v, t, rng.random(v.shape), rng.normal(size=v.shape), 0.01


def _time(mesh, spacing, reps):
    import torch

    from gs2mesh_b200.mesh import SimplificationContraction, TriangleMesh
    from tests import simplify_oracle as so

    gpu = TriangleMesh(mesh.vertices, mesh.triangles, mesh.vertex_colors, mesh.vertex_normals, device=mesh.device)
    out = {"triangles": int(len(mesh.triangles)), "vertices": int(len(mesh.vertices)), "spacing": spacing}
    for mult in (2, 4):
        s = mult * spacing
        for mode in (SimplificationContraction.Average, SimplificationContraction.Quadric):
            key = f"{mult}x_{mode.name.lower()}"
            t0 = time.perf_counter()
            wv, wt, wc, wn, wq = so.simplify(mesh.vertices, mesh.triangles, s, int(mode), mesh.vertex_colors,
                                             mesh.vertex_normals)
            host_ms = (time.perf_counter() - t0) * 1e3
            gpu.simplify_vertex_clustering(s, mode)  # warm-up
            ev, got = [], None
            for _ in range(reps):
                torch.cuda.synchronize()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                got = gpu.simplify_vertex_clustering(s, mode)
                b.record()
                torch.cuda.synchronize()
                ev.append(a.elapsed_time(b))
            same = all(_same(x, y) for x, y in ((got.vertices, wv), (got.triangles, wt), (got.vertex_colors, wc),
                                               (got.vertex_normals, wn)))
            out[key] = {"gpu_ms": round(float(np.median(ev)), 2), "host_ms": round(host_ms, 1),
                        "out_vertices": int(len(wv)), "out_triangles": int(len(wt)),
                        "quadric_cells": gpu.last_simplify_stats["quadric_cells"], "same_output": bool(same and
                                                                                                         gpu.last_simplify_stats["quadric_cells"] == wq)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--grids", default="1000000,4000000")
    ap.add_argument("--views", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()

    import torch

    from __graft_entry__ import build
    from gs2mesh_b200.mesh import TriangleMesh

    assert torch.cuda.is_available(), "mesh_simplify_time needs a CUDA device"
    build()
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(args.seed)
    results = {}
    with torch.cuda.device(dev):
        for n in (int(x) for x in args.grids.split(",") if x):
            v, t, col, nrm, spacing = _shuffled_grid(n, rng)
            results[f"grid_{n}"] = _time(TriangleMesh(v, t, col, nrm, device=dev), spacing, args.reps)
        with tempfile.TemporaryDirectory() as tmp:
            mesh = _c1_mesh(dev, args.views, tmp)
            results[f"c1_tsdf_{args.views}_views"] = _time(mesh, 2.0 / 512, args.reps)  # the TSDF voxel
    name, power = _card()
    print(json.dumps({"card": name, "power_limit": power, "reps": args.reps, "host_cpus": os.cpu_count(), **results}))


if __name__ == "__main__":
    main()
