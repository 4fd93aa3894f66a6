"""Dump what gsb_tsdf_reduce computes, so that two builds of the library can be compared byte for byte.

    torchrun --nproc-per-node N scripts/merge_dump.py OUT_DIR [--package-root TREE]
    python scripts/merge_dump.py --compare DIR_A DIR_B

Every rank fuses its round-robin share of six seeded synthetic views (a sphere of depth, random colours) and merges:
  allreduce  ncclAllReduce, every rank's volume after the merge;
  reduce     ncclReduce to the last rank, every rank's volume after the merge;
  overflow   an all-reduce into pools that hold each rank's own bricks but not the union: only the counters are dumped,
             because which bricks find room depends on the order of the insertions.
Each dump is OUT_DIR/<case>_rank<r>.npz: the open bricks sorted by lattice index, their (tsdf, weight) and colour, and the
volume's eight counter words.  --package-root imports gs2mesh_b200 from another tree (the build to compare against).
--compare checks that the bricks are bitwise equal and prints the counters that differ."""
import argparse
import glob
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
W, H, F, NV = 800, 600, 700.0, 6


def look_at(pos):
    pos = np.asarray(pos, float)
    f = -pos / np.linalg.norm(pos)
    r = np.cross(f, [0, 0, 1.0])
    r /= np.linalg.norm(r)
    c2w = np.eye(4)
    c2w[:3, :3] = np.stack([r, np.cross(f, r), f], 1)
    c2w[:3, 3] = pos
    return np.linalg.inv(c2w)


def sphere_depth(w2c, dev, radius=0.6):
    import torch

    c2w = torch.tensor(np.linalg.inv(w2c), dtype=torch.float64, device=dev)
    ys, xs = torch.meshgrid(torch.arange(H, device=dev, dtype=torch.float64), torch.arange(W, device=dev, dtype=torch.float64),
                            indexing="ij")
    dw = torch.stack([(xs - W / 2) / F, (ys - H / 2) / F, torch.ones_like(xs)], -1) @ c2w[:3, :3].T
    o = c2w[:3, 3]
    a, b, c = (dw * dw).sum(-1), 2 * (dw @ o), o @ o - radius ** 2
    disc = b * b - 4 * a * c
    return torch.where(disc > 0, (-b - torch.sqrt(disc.clamp_min(0))) / (2 * a), torch.zeros_like(a)).float().contiguous()


def fuse(views, dev, pool_bricks=None):
    import torch

    from gs2mesh_b200.tsdf import TSDFVolume

    vol = TSDFVolume(2.0 / 512, 4 * 2.0 / 512, with_color=True, device=dev, pool_bricks=pool_bricks)
    for k in views:
        az = 2 * np.pi * k / NV
        w2c = look_at(1.6 * np.array([np.cos(az), np.sin(az), 0.4 * np.sin(2 * az)]))
        rgb = torch.randint(0, 256, (H, W, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(k)).to(dev)
        vol.integrate(sphere_depth(w2c, dev), rgb, W, H, F, F, W / 2, H / 2, w2c)
    return vol


def dump(path, vol, units=True):
    arrays = {"counters": vol._counters.cpu().numpy()}
    if units:
        u = vol.export_units()
        keys = sorted(u)
        arrays["keys"] = np.array(keys, dtype=np.int32).reshape(-1, 3)
        arrays["tsdf_weight"] = np.stack([u[k][0] for k in keys])
        arrays["color"] = np.stack([u[k][1] for k in keys])
    np.savez(path, **arrays)


def run(out_dir):
    import torch
    import torch.distributed as dist

    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    dev = torch.device("cuda", local)
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl", device_id=dev)
    from gs2mesh_b200.tsdf import shard_views

    os.makedirs(out_dir, exist_ok=True)
    mine = shard_views(NV, rank, world)
    for case, dst in (("allreduce", None), ("reduce", world - 1)):
        vol = fuse(mine, dev)
        vol.reduce_across_ranks(dst=dst)
        torch.cuda.synchronize()
        dump(os.path.join(out_dir, f"{case}_rank{rank}.npz"), vol)
    most = torch.tensor([fuse(mine, dev).num_bricks()], dtype=torch.int64, device=dev)
    dist.all_reduce(most, op=dist.ReduceOp.MAX)
    vol = fuse(mine, dev, pool_bricks=int(most))
    vol.reduce_across_ranks(dst=None)
    torch.cuda.synchronize()
    dump(os.path.join(out_dir, f"overflow_rank{rank}.npz"), vol, units=False)
    dist.destroy_process_group()


def compare(a_dir, b_dir):
    names = sorted(os.path.basename(p) for p in glob.glob(os.path.join(a_dir, "*.npz")))
    if not names or names != sorted(os.path.basename(p) for p in glob.glob(os.path.join(b_dir, "*.npz"))):
        print(f"different dumps: {names}")
        return 1
    bad = 0
    for n in names:
        a, b = np.load(os.path.join(a_dir, n)), np.load(os.path.join(b_dir, n))
        for k in sorted(set(a.files) - {"counters"}):
            same = a[k].shape == b[k].shape and a[k].tobytes() == b[k].tobytes()
            bad += not same
            print(f"{n} {k}: {'identical' if same else 'DIFFERENT'} {a[k].shape}")
        if not np.array_equal(a["counters"], b["counters"]):
            print(f"{n} counters: {a['counters'].tolist()} vs {b['counters'].tolist()}")
    return 1 if bad else 0


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("dirs", nargs="+")
    ap.add_argument("--compare", action="store_true")
    ap.add_argument("--package-root", default=ROOT)
    args = ap.parse_args()
    if args.compare:
        sys.exit(compare(*args.dirs))
    sys.path.insert(0, os.path.abspath(args.package_root))
    run(args.dirs[0])
