"""Times the smoothing and sharpening filters (TriangleMesh.filter_smooth_simple / _laplacian / _taubin, filter_sharpen)
on the GPU, on shuffled grid meshes of about 1M and 4M triangles and on the TSDF mesh of the synthetic C1 scene (voxel
2/512), at 1, 10 and 100 iterations with every attribute filtered (FilterScope.All); checks them against the numpy
restatement (tests/filter_oracle.py) and prints one JSON line with the card's name and power limit, read in the same run.
Everything it writes goes to a temporary directory.

Per mesh and filter:
- `call_ms`: the whole method call, timed with CUDA events and a final synchronise after a warm-up (median of --reps), so
  the uploads, the CSR build, the kernels and the downloads are all inside the window;
- `pass_us`: the device time of one pass, with the inputs and the CSR already on the device, through the C ABI: one
  gsb_mesh_filter call of --device-iterations iterations between two CUDA events, divided by its number of passes;
- `floor_us`: the pass's algorithmic HBM floor at 3.35 TB/s, each array read once (offsets 8 B (nv + 1), neighbours
  8 B nnz, and 24 B nv read plus 24 B nv written per filtered attribute, the positions being among them); the neighbour
  gathers are L2 traffic and not counted.  It is a floor, not a measurement: `floor_over_pass` is how close a pass gets;
- `host_ms` / `same_output`: the restatement once, at --check-iterations iterations, and whether the GPU call at that
  count gave the same bytes.

    python scripts/mesh_filter_time.py [--grids 1000000,4000000] [--views 20] [--reps 5] [--check-iterations 1]
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
from mesh_simplify_time import _shuffled_grid  # noqa: E402

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet
ITERATIONS = (1, 10, 100)
NAMES = ("filter_smooth_simple", "filter_smooth_laplacian", "filter_smooth_taubin", "filter_sharpen")
DEFAULTS = ((0.0, 0.0), (0.5, 0.0), (0.5, -0.53), (1.0, 0.0))  # the methods' (lambda_filter, mu) or (strength, -)


def _device_pass_us(mesh, kind, iterations):
    """Device time of one pass through gsb_mesh_filter with device-resident inputs and CSR."""
    import torch

    from gs2mesh_b200 import _lib
    from gs2mesh_b200._lib import ptr
    from gs2mesh_b200.mesh import _adjacency

    dev = mesh.device
    L = _lib.lib()
    up = lambda a: None if a is None else torch.as_tensor(a).to(dev).contiguous()
    xyz, rgb, nrm = up(mesh.vertices), up(mesh.vertex_colors), up(mesh.vertex_normals)
    nv = len(mesh.vertices)
    offsets, neighbours = _adjacency(up(mesh.triangles), nv)
    like = lambda a: None if a is None else torch.empty_like(a)
    out_v, out_c, out_n = like(xyz), like(rgb), like(nrm)
    work = torch.empty(L.gsb_mesh_filter_workspace_bytes(nv, rgb is not None, nrm is not None), dtype=torch.uint8, device=dev)

    def call(n):
        _lib.check(L.gsb_mesh_filter(kind, ptr(xyz), ptr(rgb), ptr(nrm), nv, ptr(offsets), ptr(neighbours), n,
                                     *DEFAULTS[kind], 0, ptr(work), work.numel(), ptr(out_v), ptr(out_c), ptr(out_n),
                                     _lib.stream(dev)))

    call(2)  # warm-up
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    call(iterations)
    b.record()
    torch.cuda.synchronize()
    passes = iterations * (2 if kind == _lib.GSB_FILTER_TAUBIN else 1)
    return a.elapsed_time(b) * 1e3 / passes, int(neighbours.numel())


def _time(mesh, args):
    import torch

    from gs2mesh_b200.mesh import TriangleMesh
    from tests import filter_oracle as fo

    gpu = TriangleMesh(mesh.vertices, mesh.triangles, mesh.vertex_colors, mesh.vertex_normals, device=mesh.device)
    nv = len(mesh.vertices)
    attrs = 1 + (mesh.vertex_colors is not None) + (mesh.vertex_normals is not None)
    out = {"triangles": int(len(mesh.triangles)), "vertices": nv, "attributes": attrs}
    for kind, name in enumerate(NAMES):
        method = getattr(gpu, name)
        res = {}
        for it in ITERATIONS:
            method(it)  # warm-up
            ev = []
            for _ in range(args.reps):
                torch.cuda.synchronize()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                method(it)
                b.record()
                torch.cuda.synchronize()
                ev.append(a.elapsed_time(b))
            res[f"call_ms_{it}"] = round(float(np.median(ev)), 2)
        pass_us, nnz = _device_pass_us(gpu, kind, args.device_iterations)
        floor_us = (8 * (nv + 1) + 8 * nnz + 48 * nv * attrs) / HBM_BYTES_PER_S * 1e6
        res.update(pass_us=round(pass_us, 1), floor_us=round(floor_us, 1), floor_over_pass=round(floor_us / pass_us, 3),
                   neighbours=nnz)
        got = method(args.check_iterations)
        t0 = time.perf_counter()
        want = fo.filter_mesh(kind, mesh.vertices, mesh.triangles, args.check_iterations, *DEFAULTS[kind], fo.ALL,
                              mesh.vertex_colors, mesh.vertex_normals)
        res["host_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
        res["same_output"] = bool(all(_same(g, w) for g, w in zip((got.vertices, got.vertex_colors, got.vertex_normals), want)))
        out[name] = res
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--grids", default="1000000,4000000")
    ap.add_argument("--views", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--device-iterations", type=int, default=100)
    ap.add_argument("--check-iterations", type=int, default=1)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()

    import torch

    from __graft_entry__ import build
    from gs2mesh_b200.mesh import TriangleMesh

    assert torch.cuda.is_available(), "mesh_filter_time needs a CUDA device"
    build()
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(args.seed)
    results = {}
    with torch.cuda.device(dev):
        for n in (int(x) for x in args.grids.split(",") if x):
            v, t, col, nrm, _ = _shuffled_grid(n, rng)
            results[f"grid_{n}"] = _time(TriangleMesh(v, t, col, nrm, device=dev), args)
        with tempfile.TemporaryDirectory() as tmp:
            results[f"c1_tsdf_{args.views}_views"] = _time(_c1_mesh(dev, args.views, tmp), args)
    name, power = _card()
    print(json.dumps({"card": name, "power_limit": power, "reps": args.reps, "device_iterations": args.device_iterations,
                      "check_iterations": args.check_iterations, "host_cpus": os.cpu_count(), **results}))


if __name__ == "__main__":
    main()
