"""One rank of the multi-GPU merge tests (tests/test_gpu_merge.py): `python -m tests.merge_ranks --rank R --world N ...`.

Rank 0 makes an NCCL id with gsb_comm_unique_id and hands it to the other ranks through a file in --dir (written, then
renamed); every rank joins with gsb_comm_create.  Each rank then runs the whole case list of CASES in order -- the same
collectives in the same order on every rank -- building its volumes brick by brick from seeded descriptions, and writes per
case its bricks before and after the merge, its pool statistics, a digest of every array of the volume and the return codes
to --dir/<case>_r<rank>.npz.  The cases that go through TSDFVolume.reduce_across_ranks (unequal pools, colour mismatch,
integration end to end) run last, in a torch.distributed NCCL group on 127.0.0.1.

--mode one_gpu puts every rank on device 0 (the parent sets NCCL_HOSTID per rank so that NCCL accepts that), per_gpu puts
rank r on device r."""
from __future__ import annotations

import argparse
import ctypes as C
import gc
import hashlib
import os
import sys
import time
import traceback

import numpy as np

POOL = 24            # pool of the plain cases (hash of 64 slots)
SMALL_POOL = 16      # pool of the fill / overflow cases
BIAS = 1 << 20
ROOTS = ("all", "root0", "rootlast")


# ----------------------------------------------------------------------------------------------------------- case list

def _case_list():
    out = []
    for name in ("disjoint", "identical", "partial", "one_empty", "all_empty", "collide", "fill_exact", "overflow",
                 "pre_overflow", "alpha", "ws_below_fixed", "ws_fixed_then_retry"):
        for root in ROOTS:
            for color in ((True,) if name == "alpha" else (True, False)):
                out.append((name, root, color))
    for name in ("unequal_pools", "end_to_end"):
        for root in ROOTS:
            for color in (True, False):
                out.append((name, root, color))
    out.append(("color_mismatch", "all", True))
    return out


CASES = _case_list()
DIST_CASES = ("unequal_pools", "end_to_end", "color_mismatch")


def case_id(name, root, color):
    return f"{name}-{root}-{'color' if color else 'nocolor'}"


def root_of(root, world):
    return {"all": -1, "root0": 0, "rootlast": world - 1}[root]


def _collide_keys():
    """Lattice keys at the ends of the brick range and near the origin whose home slots in a 64-slot table are one slot H
    (8 keys) and H + 1 (4 keys): probe chains that run through each other's keys."""
    from tests.tsdf_host import brick_hash, brick_key

    xs = [-BIAS, -BIAS + 1, -1, 0, 1, BIAS - 2, BIAS - 1]
    cand = [(x, y, z) for x in xs for y in xs for z in xs]
    homes = {}
    for k in cand:
        homes.setdefault(brick_hash(brick_key(k), 63), []).append(k)
    h = max(homes, key=lambda s: min(len(homes[s]), 8) * 10 + min(len(homes.get((s + 1) & 63, [])), 4))
    return homes[h][:8] + homes.get((h + 1) & 63, [])[:4]


def case_spec(name, world, rank):
    """(pool, keys in the order this rank opens them, keys to leave dead in the hash after an overflow)."""
    base = [(i, 1, -2) for i in range(40)]
    if name == "disjoint":
        return POOL, [(10 * rank + i, 2, -3) for i in range(6)], []
    if name == "identical":
        return POOL, [(i, 0, 0) for i in range(6)], []
    if name in ("partial", "alpha", "ws_below_fixed", "ws_fixed_then_retry"):
        keys = base[3 * rank:3 * rank + 8]
        return POOL, keys[::-1] if rank == 1 else keys, []
    if name == "one_empty":
        return POOL, [] if rank == 0 else base[3 * rank:3 * rank + 7], []
    if name == "all_empty":
        return POOL, [], []
    if name == "collide":
        ks = _collide_keys()
        rng = np.random.default_rng(100 + rank)
        return POOL, [ks[i] for i in rng.permutation(len(ks))[:8]], []
    if name == "fill_exact":  # the union is exactly SMALL_POOL bricks
        u = base[:SMALL_POOL]
        parts = {2: [u[0:10], u[6:16]], 3: [u[0:8], u[5:12], u[10:16] + [u[0]]]}[world]
        return SMALL_POOL, parts[rank], []
    if name == "overflow":  # the union is SMALL_POOL + 3 bricks
        u = base[:SMALL_POOL + 3]
        parts = {2: [u[0:10], u[9:19]], 3: [u[0:8], u[6:14], u[12:19] + [u[1]]]}[world]
        return SMALL_POOL, parts[rank], []
    if name == "pre_overflow":  # rank 1's own pool overflowed on keys rank 0 holds
        if rank == 0:
            return SMALL_POOL, base[:12], []
        if rank == 1:
            return SMALL_POOL, base[20:20 + SMALL_POOL - 1], base[0:4]
        return SMALL_POOL, base[8:14], []
    if name == "unequal_pools":
        pools = (16, 32, 24)
        return pools[rank], base[5 * rank:5 * rank + (12, 20, 9)[rank]], []
    raise KeyError(name)


def voxels(rng, with_color, alpha=False):
    """(tw [4096,2], colour [4096,4] | None) drawn over the values where a merge can go wrong: weight 0 (tsdf and colour 0,
    the pool invariant), weights 1 ... 2^20, tsdf +-1, +-0, subnormals and values whose products round; the colour's fourth
    channel is 0 unless `alpha`."""
    f32 = np.float32
    n = 4096
    u = rng.random(n)
    w = np.where(u < 0.12, 0, np.where(u < 0.42, 1, np.where(u < 0.72, rng.integers(2, 65, n),
                 np.where(u < 0.9, rng.integers(65, (1 << 20) + 1, n), 1 << 20)))).astype(f32)
    special = np.array([1.0, -1.0, -0.0, 0.0, 1e-45, -1e-45, 1e-40, -1e-40, 3e-39, -3e-39, 1.1e-38, -1.1e-38], f32)
    v = rng.random(n)
    t = np.where(v < 0.35, special[rng.integers(0, len(special), n)], rng.uniform(-1, 1, n).astype(f32)).astype(f32)
    t[w == 0] = 0.0
    tw = np.stack([t, w], -1).astype(f32)
    col = None
    if with_color:
        col = np.zeros((n, 4), f32)
        col[:, :3] = rng.uniform(0, 255, (n, 3)).astype(f32)
        if alpha:
            col[:, 3] = rng.uniform(0, 1, n).astype(f32)
        col[w == 0] = 0.0
    return tw, col


# ----------------------------------------------------------------------------------------------------------- volumes

class Rank:
    def __init__(self, rank, world, dev, out_dir):
        import torch

        from gs2mesh_b200 import _lib

        self.torch, self._lib, self.L = torch, _lib, _lib.lib()
        self.rank, self.world, self.dev, self.dir = rank, world, dev, out_dir

    def volume(self, pool, with_color, voxel_length=2.0 / 512):
        from gs2mesh_b200.tsdf import TSDFVolume

        return TSDFVolume(voxel_length, 4 * voxel_length, (0, 0, 0), (1, 1, 1), with_color=with_color, device=self.dev,
                          pool_bricks=pool)

    def fill(self, vol, keys, seed, alpha=False):
        """Opens `keys` one launch at a time (pool order = list order) and writes seeded contents."""
        torch = self.torch
        for k in keys:
            slot = int(vol.find_bricks(np.array([k], np.int32), insert=True)[0].item())
            assert slot >= 0, (k, slot)
            rng = np.random.default_rng([seed, k[0] + BIAS, k[1] + BIAS, k[2] + BIAS])
            tw, col = voxels(rng, vol.with_color, alpha)
            vol.pool()[slot] = torch.from_numpy(tw).to(self.dev)
            if col is not None:
                vol.color.view(vol.pool_bricks, 4096, 4)[slot] = torch.from_numpy(col).to(self.dev)
        torch.cuda.synchronize(self.dev)

    def make_dead(self, vol, keys):
        """Opens `keys` in one launch into a pool with one free slot: threads that pass the pool check together leave dead
        keys (hash entry without a pool slot).  A key that found the pool full and left no entry is then given the state
        such a race leaves: key stored on its probe chain, slot 0xFFFFFFFF."""
        from tests.tsdf_host import brick_hash, brick_key

        vol.find_bricks(np.array(keys, np.int32), insert=True)
        self.torch.cuda.synchronize(self.dev)
        hk = vol._hash_keys.cpu().numpy()
        mask = vol.hash_slots - 1
        for k in keys:
            key = brick_key(k)
            if (hk == key).any():
                continue
            h = brick_hash(key, mask)
            while hk[h] != -1:
                h = (h + 1) & mask
            hk[h] = key
            vol._hash_keys[h] = key
            vol._hash_vals[h] = -1
        self.torch.cuda.synchronize(self.dev)

    def state(self, vol, prefix):
        """Bricks in pool order, dead keys, statistics and a digest of every array of the volume."""
        torch = self.torch
        torch.cuda.synchronize(self.dev)
        n = vol.num_bricks()
        out = {f"{prefix}_keys": vol._index[:n, :3].cpu().numpy().astype(np.int32),
               f"{prefix}_tw": vol.pool()[:n].cpu().numpy()}
        if vol.color is not None:
            out[f"{prefix}_col"] = vol.color.view(vol.pool_bricks, 4096, 4)[:n].cpu().numpy()
        keys = vol._hash_keys.cpu().numpy()
        vals = vol._hash_vals.cpu().numpy()
        k = keys[(keys != -1) & (vals == -1)].view(np.uint64)
        out[f"{prefix}_dead"] = np.stack([((k >> np.uint64(s)) & np.uint64(0x1FFFFF)).astype(np.int64) - BIAS
                                          for s in (42, 21, 0)], -1).reshape(-1, 3).astype(np.int32)
        s = vol.pool_stats()
        out[f"{prefix}_stats"] = np.array([s["bricks"], s["dropped_total"], vol.pool_bricks], np.int64)
        h = hashlib.sha256()
        for t in (vol.tsdf_weight, vol.color, vol._index, vol._hash_keys, vol._hash_vals, vol._hash_stamp, vol._list,
                  vol._counters):
            if t is not None:
                h.update(t.cpu().numpy().tobytes())
        out[f"{prefix}_digest"] = np.array(h.hexdigest())
        return out

    def reduce(self, vol, comm, root, scratch_bytes):
        torch = self.torch
        buf = torch.empty(max(int(scratch_bytes), 1), dtype=torch.uint8, device=self.dev)
        req = C.c_size_t(0)
        with torch.cuda.device(self.dev):
            rc = self.L.gsb_tsdf_reduce(vol._h, comm, self.world, self.rank, root, self._lib.ptr(buf), int(scratch_bytes),
                                        C.byref(req), vol._stream())
        torch.cuda.synchronize(self.dev)
        return int(rc), int(req.value)

    def save(self, cid, rec):
        np.savez(os.path.join(self.dir, f"{cid}_r{self.rank}.npz"), **rec)

    # ------------------------------------------------------------------------------------------------------- C-ABI cases
    def run_case(self, comm, name, root_mode, with_color):
        pool, keys, dead = case_spec(name, self.world, self.rank)
        content = "partial" if name.startswith("ws_") else name
        seed = sum(map(ord, content)) * 10 + self.rank
        vol = self.volume(pool, with_color)
        self.fill(vol, keys, seed, alpha=name == "alpha")
        if dead:
            self.make_dead(vol, dead)
        root = root_of(root_mode, self.world)
        rec = dict(pool=np.int64(pool))
        rec.update(self.state(vol, "pre"))
        L = self.L
        fixed = int(L.gsb_tsdf_reduce_scratch_bytes(vol._h, self.world, 0))
        ample = int(L.gsb_tsdf_reduce_scratch_bytes(vol._h, self.world, pool))
        if name == "ws_below_fixed":
            calls = [fixed - 1]
        elif name == "ws_fixed_then_retry":
            calls = [fixed, None]
        else:
            calls = [ample]
        req = 0
        for i, nbytes in enumerate(calls):
            nbytes = req if nbytes is None else nbytes
            rc, req = self.reduce(vol, comm, root, nbytes)
            rec[f"call{i}_bytes"] = np.int64(nbytes)
            rec[f"call{i}_rc"] = np.int64(rc)
            rec[f"call{i}_required"] = np.int64(req)
            rec[f"call{i}_need_own"] = np.int64(L.gsb_tsdf_reduce_scratch_bytes(vol._h, self.world, vol.num_bricks()))
            rec.update(self.state(vol, f"call{i}"))
        rec["fixed"] = np.int64(fixed)
        self.save(case_id(name, root_mode, with_color), rec)
        del vol
        gc.collect()

    # ------------------------------------------------------------------------------------------------ reduce_across_ranks
    def release(self, vol):
        for c in vol._comms.values():
            self.L.gsb_comm_destroy(c)
        vol._comms.clear()

    def run_dist_case(self, name, root_mode, with_color):
        torch = self.torch
        dst = None if root_mode == "all" else max(root_of(root_mode, self.world), 0)
        rec = {}
        if name == "end_to_end":
            vol = self.volume(1024, with_color, voxel_length=1.0 / 64)
            self.integrate_views(vol, with_color)
        elif name == "color_mismatch":
            vol = self.volume(POOL, self.rank == 0)
            self.fill(vol, case_spec("partial", self.world, self.rank)[1], 7 + self.rank)
        else:
            pool, keys, _ = case_spec(name, self.world, self.rank)
            vol = self.volume(pool, with_color)
            self.fill(vol, keys, 11 * self.rank + 3)
        rec["pool"] = np.int64(vol.pool_bricks)
        rec.update(self.state(vol, "pre"))
        rec["error"] = np.array("")
        try:
            vol.reduce_across_ranks(dst=dst)
        except ValueError as e:
            rec["error"] = np.array(f"ValueError: {e}")
        torch.cuda.synchronize(self.dev)
        rec.update(self.state(vol, "call0"))
        rec["call0_rc"] = np.int64(0)
        self.save(case_id(name, root_mode, with_color), rec)
        self.release(vol)
        del vol
        gc.collect()

    def integrate_views(self, vol, with_color):
        """Two seeded views per rank of a sphere of radius 0.6 at the origin, fused with TSDFVolume.integrate."""
        torch = self.torch
        W, H, f = 96, 72, 80.0
        rng = np.random.default_rng(500 + self.rank)
        for k in range(2):
            az = 2 * np.pi * (2 * self.rank + k) / (2 * self.world) + 0.3
            pos = 1.6 * np.array([np.cos(az), np.sin(az), 0.35])
            fwd = -pos / np.linalg.norm(pos)
            right = np.cross(fwd, [0, 0, 1.0])
            right /= np.linalg.norm(right)
            c2w = np.eye(4)
            c2w[:3, :3] = np.stack([right, np.cross(fwd, right), fwd], 1)
            c2w[:3, 3] = pos
            ys, xs = np.mgrid[0:H, 0:W].astype(np.float64)
            d = np.stack([(xs - W / 2) / f, (ys - H / 2) / f, np.ones_like(xs)], -1) @ c2w[:3, :3].T
            a, b, c = (d * d).sum(-1), 2 * (d @ pos), pos @ pos - 0.36
            disc = b * b - 4 * a * c
            depth = np.where(disc > 0, (-b - np.sqrt(np.maximum(disc, 0))) / (2 * a), 0).astype(np.float32)
            rgb = rng.integers(0, 256, (H, W, 3), dtype=np.uint8) if with_color else None
            vol.integrate(torch.from_numpy(depth).to(self.dev), None if rgb is None else torch.from_numpy(rgb).to(self.dev),
                          W, H, f, f, W / 2, H / 2, np.linalg.inv(c2w))
        torch.cuda.synchronize(self.dev)


# ----------------------------------------------------------------------------------------------------------- main

def _exchange_id(L, rank, out_dir, deadline):
    path = os.path.join(out_dir, "nccl_id.bin")
    if rank == 0:
        buf = (C.c_uint8 * 128)()
        if L.gsb_comm_unique_id(buf) != 0:
            raise RuntimeError(L.gsb_last_error().decode())
        tmp = path + ".tmp"
        with open(tmp, "wb") as fh:
            fh.write(bytes(buf))
        os.replace(tmp, path)
        return buf
    while not os.path.exists(path):
        if time.monotonic() > deadline:
            raise TimeoutError("rank 0 did not publish the NCCL id")
        time.sleep(0.05)
    with open(path, "rb") as fh:
        return (C.c_uint8 * 128)(*fh.read())


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--rank", type=int, required=True)
    ap.add_argument("--world", type=int, required=True)
    ap.add_argument("--mode", choices=("one_gpu", "per_gpu"), required=True)
    ap.add_argument("--dir", required=True)
    ap.add_argument("--port", type=int, required=True)
    a = ap.parse_args(argv)
    import torch

    dev = torch.device("cuda", 0 if a.mode == "one_gpu" else a.rank)
    torch.cuda.set_device(dev)
    r = Rank(a.rank, a.world, dev, a.dir)
    ident = _exchange_id(r.L, a.rank, a.dir, time.monotonic() + 60)
    with torch.cuda.device(dev):
        comm = r.L.gsb_comm_create(ident, a.world, a.rank)
    if not comm:
        with open(os.path.join(a.dir, f"refused_r{a.rank}.txt"), "w") as fh:
            fh.write(r.L.gsb_last_error().decode("utf-8", "replace"))
        return 3
    t0 = time.monotonic()
    for name, root, color in CASES:
        if name not in DIST_CASES:
            r.run_case(comm, name, root, color)
    r.L.gsb_comm_destroy(comm)
    import datetime

    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(a.port))
    dist.init_process_group("nccl", rank=a.rank, world_size=a.world, device_id=dev, timeout=datetime.timedelta(seconds=120))
    for name, root, color in CASES:
        if name in DIST_CASES:
            r.run_dist_case(name, root, color)
    dist.barrier()
    dist.destroy_process_group()
    with open(os.path.join(a.dir, f"done_r{a.rank}.txt"), "w") as fh:
        fh.write(f"{time.monotonic() - t0:.2f}")
    return 0


if __name__ == "__main__":
    try:
        sys.exit(main())
    except SystemExit:
        raise
    except BaseException:
        traceback.print_exc()
        sys.stderr.flush()
        os._exit(1)
