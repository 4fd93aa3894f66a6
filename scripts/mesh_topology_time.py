"""Times the topology queries (TriangleMesh.get_non_manifold_edges, get_non_manifold_vertices,
get_self_intersecting_triangles, is_orientable, get_surface_area, is_watertight) on the GPU, on the shuffled grid meshes
and the TSDF mesh of the synthetic C1 scene that scripts/mesh_filter_time.py uses; checks them against the numpy
restatement (tests/topology_oracle.py) and prints one JSON line with the card's name and power limit, read in the same
run.  Everything it writes goes to a temporary directory.

Per mesh and query:
- `call_ms`: the whole method call (upload, kernels, download), timed with CUDA events and a final synchronise after a
  warm-up, median of --reps;
- `device_ms`: the self-intersection count pass alone through the C ABI with the mesh and workspace already on the
  device, between two CUDA events (median of --reps);
- `candidates`, `registrations`, `level`: the grid's candidate pairs, (triangle, cell) registrations and level;
- `fan_<n>`: the worst case of the grid, a fan of n triangles around one vertex: every box holds the centre, so one cell
  holds every triangle and the count pass visits n(n-1)/2 candidate pairs; only `self_intersections_device` is timed
  there (every pair shares the centre, so none is found);
- `host_ms` / `same_output`: the restatement once and whether the GPU gave the same answer.  The restatement's
  self-intersection sweep along x visits about n^1.5 pairs on a surface mesh, so it runs on the first
  --host-isect-triangles triangles only (`host_isect_triangles`), and the GPU is compared with it there.

    python scripts/mesh_topology_time.py [--grids 1000000] [--views 20] [--reps 5] [--host-isect-triangles 50000]
                                        [--fan 120000]
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

from mesh_clean_time import _c1_mesh, _card  # noqa: E402
from mesh_simplify_time import _shuffled_grid  # noqa: E402

QUERIES = ("get_non_manifold_edges", "get_non_manifold_vertices", "is_orientable", "get_surface_area",
           "get_self_intersecting_triangles", "is_watertight")


def _events(fn, reps):
    import torch

    fn()  # warm-up
    ms = []
    for _ in range(reps):
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    return round(float(np.median(ms)), 3)


def _device_isect(mesh, reps):
    """Device time of the counting self-intersection pass, inputs and workspace resident, and its stats."""
    import ctypes as C

    import torch

    from gs2mesh_b200 import _lib
    from gs2mesh_b200._lib import ptr

    L = _lib.lib()
    dev = mesh.device
    nv, nt = len(mesh.vertices), len(mesh.triangles)
    xyz = torch.as_tensor(mesh.vertices).to(dev).contiguous()
    tri = torch.as_tensor(mesh.triangles).to(dev).contiguous()
    dbl3 = C.c_double * 3
    lo, hi = dbl3(*mesh.vertices.min(axis=0).tolist()), dbl3(*mesh.vertices.max(axis=0).tolist())
    work = torch.empty(L.gsb_mesh_self_intersections_workspace_bytes(nt, nv, 0), dtype=torch.uint8, device=dev)
    stats = torch.empty(4, dtype=torch.int64, device=dev)

    def call():
        _lib.check(L.gsb_mesh_self_intersections(ptr(xyz), nv, ptr(tri), nt, lo, hi, ptr(work), work.numel(), None, 0,
                                                 ptr(stats), _lib.stream(dev)))

    ms = _events(call, reps)
    pairs, candidates, registrations, level = (int(x) for x in stats.cpu().tolist())
    return {"device_ms": ms, "pairs": pairs, "candidates": candidates, "registrations": registrations, "level": level,
            "workspace_mb": round(work.numel() / 2**20, 1)}


def _host(name, v, t):
    from tests import topology_oracle as to

    nv = len(v)
    if name == "get_non_manifold_edges":
        return to.edges(t, nv, True)[0]
    if name == "get_non_manifold_vertices":
        return to.non_manifold_vertices(t, nv)
    if name == "is_orientable":
        return to.is_orientable(t, nv)
    if name == "get_surface_area":
        return to.surface_area(v, t)
    if name == "get_self_intersecting_triangles":
        return to.self_intersecting_triangles(v, t)
    return (len(to.edges(t, nv, False)[0]) == 0 and len(to.non_manifold_vertices(t, nv)) == 0
            and len(to.self_intersecting_triangles(v, t)) == 0)


def _equal(a, b):
    return bool(np.asarray(a).tobytes() == np.asarray(b).tobytes()) if isinstance(a, np.ndarray) else a == b


def _time(mesh, args):
    from gs2mesh_b200.mesh import TriangleMesh

    gpu = TriangleMesh(mesh.vertices, mesh.triangles, device=mesh.device)
    v, t = gpu.vertices, gpu.triangles
    out = {"triangles": int(len(t)), "vertices": int(len(v))}
    for name in QUERIES:
        res = {"call_ms": _events(getattr(gpu, name), args.reps)}
        if name in ("get_self_intersecting_triangles", "is_watertight"):
            k = min(len(t), args.host_isect_triangles)
            sub = TriangleMesh(v, t[:k], device=mesh.device)
            res["host_isect_triangles"] = k
            got, (hv, ht) = getattr(sub, name)(), (v, t[:k])
        else:
            got, (hv, ht) = getattr(gpu, name)(), (v, t)
        t0 = time.perf_counter()
        want = _host(name, hv, ht)
        res["host_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
        res["same_output"] = _equal(got, want)
        out[name] = res
    out["self_intersections_device"] = _device_isect(gpu, args.reps)
    return out


def _fan(n):
    ang = np.linspace(0, 2 * np.pi, n + 1)[:-1]
    v = np.concatenate([[[0, 0, 0]], np.stack([np.cos(ang), np.sin(ang), 0.1 * np.sin(7 * ang)], 1)])
    return v, np.stack([np.zeros(n - 1, np.int64), np.arange(1, n), np.arange(2, n + 1)], 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--grids", default="1000000")
    ap.add_argument("--views", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--host-isect-triangles", type=int, default=50000)
    ap.add_argument("--fan", type=int, default=120000)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()

    import torch

    from __graft_entry__ import build
    from gs2mesh_b200.mesh import TriangleMesh

    assert torch.cuda.is_available(), "mesh_topology_time needs a CUDA device"
    build()
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(args.seed)
    results = {}
    with torch.cuda.device(dev):
        for n in (int(x) for x in args.grids.split(",") if x):
            v, t, _, _, _ = _shuffled_grid(n, rng)
            results[f"grid_{n}"] = _time(TriangleMesh(v, t, device=dev), args)
        if args.fan:
            v, t = _fan(args.fan)
            results[f"fan_{args.fan}"] = {"triangles": int(len(t)),
                                          "self_intersections_device": _device_isect(TriangleMesh(v, t, device=dev), args.reps)}
        with tempfile.TemporaryDirectory() as tmp:
            results[f"c1_tsdf_{args.views}_views"] = _time(_c1_mesh(dev, args.views, tmp), args)
    name, power = _card()
    print(json.dumps({"card": name, "power_limit": power, "reps": args.reps, "host_cpus": os.cpu_count(), **results}))


if __name__ == "__main__":
    main()
