"""Times mesh extraction (`extract_triangle_mesh`, ScalableTSDFVolume::ExtractTriangleMesh) on the TSDF volume of the
synthetic C1 scene (voxel 2/512), as in scripts/pointcloud_time.py, and prints one JSON line with the card's name and
power limit, read in the same run, and a digest of the mesh so that two builds can be checked for the same output.

Two windows, both timed with CUDA events after a warm-up: the whole call (count, scan, emit, unique, vertex kernel and the
download of the arrays to the host; median of --reps calls), and the marching-cubes kernels alone (gsb_mesh_count and
gsb_mesh_emit on the brick list the extraction passes, mean over --launches back-to-back launches each).

    python scripts/mesh_extract_time.py [--views 20] [--reps 5] [--launches 50]
"""
import argparse
import ctypes as C
import hashlib
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
    ap.add_argument("--views", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--launches", type=int, default=50)
    args = ap.parse_args()

    import torch

    from gs2mesh_b200 import _lib
    from gs2mesh_b200.mesh import extract_triangle_mesh

    dev = torch.device("cuda", 0)
    with tempfile.TemporaryDirectory() as tmp:
        vol = _c1_volume(dev, args.views, tmp)
    name, power = _card()

    def events(fn, n):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(n):
            r = fn()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / n, r

    mesh = extract_triangle_mesh(vol)
    torch.cuda.synchronize()
    whole = [events(lambda: extract_triangle_mesh(vol), 1)[0] for _ in range(args.reps)]

    # the kernels alone, on the extraction's brick list (ascending lattice index) and key window
    L = _lib.lib()
    stream = _lib.stream(dev)
    nb = vol.num_bricks()
    idx = vol._index[:nb, :3].long()
    lo, hi = idx.min(0).values, idx.max(0).values
    n = hi - lo + 2
    lin = ((idx[:, 0] - lo[0]) * n[1] + (idx[:, 1] - lo[1])) * n[2] + (idx[:, 2] - lo[2])
    bricks = torch.sort(lin).indices.to(torch.int32)
    window = (C.c_int32 * 6)(*[int(v) for v in lo.tolist()], *[int(v) for v in n.tolist()])
    counts = torch.zeros(nb, dtype=torch.int32, device=dev)
    count = lambda: _lib.check(L.gsb_mesh_count(vol._h, window, _lib.ptr(bricks), nb, _lib.ptr(counts), stream))
    count()
    offsets = (torch.cumsum(counts.to(torch.int64), 0) - counts.to(torch.int64)).contiguous()
    keys = torch.empty(3 * int(counts.sum().item()), dtype=torch.int64, device=dev)
    emit = lambda: _lib.check(L.gsb_mesh_emit(vol._h, window, _lib.ptr(bricks), nb, _lib.ptr(offsets), _lib.ptr(keys), stream))
    emit()
    torch.cuda.synchronize()
    count_ms, _ = events(count, args.launches)
    emit_ms, _ = events(emit, args.launches)

    digest = hashlib.sha256(mesh.vertices.tobytes() + mesh.triangles.tobytes() + mesh.vertex_colors.tobytes()).hexdigest()[:16]
    print(json.dumps(dict(card=name, power_limit=power, scene="C1", views=args.views, bricks=nb, triangles=len(mesh.triangles),
                          vertices=len(mesh.vertices), extract_ms=round(float(np.median(whole)), 3),
                          count_kernel_ms=round(count_ms, 4), emit_kernel_ms=round(emit_ms, 4), reps=args.reps,
                          launches=args.launches, mesh_sha256=digest)))


if __name__ == "__main__":
    main()
