"""Multi-GPU check (run under torchrun on a box with >= 2 GPUs; not collected by pytest):
view-sharded integration + ONE NCCL sum-reduce of the brick volume == sequential single-GPU fusion.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29511 tests/dist_gpu_check.py
"""
import ctypes
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    from gs2mesh_b200 import scene
    from gs2mesh_b200.renderer import Renderer
    from gs2mesh_b200.tsdf import TSDF, shard_views

    class A:
        GS_white_background = False
        TSDF_voxel = 8
        TSDF_sdf_trunc = 0.06
        TSDF_scale = 1.0
        TSDF_min_depth_baselines = 4
        TSDF_max_depth_baselines = 20

    W, H, NV = 320, 240, 6
    cloud = scene.make_gaussians(8000, seed=3)
    rigs, baseline = scene.make_stereo_cameras(NV, W, H)
    r = Renderer.from_scene(rigs, baseline, cloud, args=A(), device=f"cuda:{local}")
    r.prepare_renderer()

    def fuse(views, pool_bricks=None):
        st = TSDF(r, None, A(), "d", window_resolution=128, device=f"cuda:{local}", pool_bricks=pool_bricks)
        st.volume = st._make_volume()
        for i in views:
            out = r.render_image_pair(i, to_host=False)
            st.integrate(out["depth"], out["left_u8"], rigs[i]["left"], final_T=out["final_T"])
        return st.volume

    def compare(merged, seq, what):
        a, b = merged.export_units(), seq.export_units()
        assert set(a) == set(b), f"{what}: merged volume holds {len(a)} bricks, sequential fusion {len(b)}"
        err = cerr = 0.0
        nvox = 0
        for k in a:
            assert np.array_equal(a[k][0][:, 1], b[k][0][:, 1]), f"{what}: merged weights differ from sequential fusion in brick {k}"
            err = max(err, float(np.abs(a[k][0][:, 0] - b[k][0][:, 0]).max()))
            cerr = max(cerr, float(np.abs(a[k][1] - b[k][1]).max()))
            nvox += int((b[k][0][:, 1] > 0).sum())
        assert err <= 2e-6, (what, err)
        assert cerr <= 1e-3, (what, cerr)
        return len(a), nvox, err, cerr

    mine = shard_views(NV, rank, world)
    seq = fuse(range(NV))
    # (1) all-reduce: every rank ends with the merged volume (C-ABI gsb_tsdf_reduce, root < 0)
    vol = fuse(mine)
    own = vol.num_bricks()
    vol.reduce_across_ranks(dst=None)
    torch.cuda.synchronize()
    n, nvox, err, cerr = compare(vol, seq, f"all-reduce on rank {rank}")
    assert vol.pool_stats()["dropped_total"] == 0, f"all-reduce on rank {rank} dropped bricks"
    # (2) reduce to the last rank: only its volume changes.  First with a scratch that holds the index exchange but no payload:
    #     every rank must get GSB_ERR_WORKSPACE together, with the same required size (the workspace protocol of the C ABI)
    from gs2mesh_b200 import _lib

    root = world - 1
    vol2 = fuse(mine)
    before = vol2.export_units()
    comm = vol2._comm(None)
    small = torch.empty(int(vol2._L.gsb_tsdf_reduce_scratch_bytes(vol2._h, world, 0)), dtype=torch.uint8, device=vol2.device)
    required = ctypes.c_size_t(0)
    rc = vol2._L.gsb_tsdf_reduce(vol2._h, comm, world, rank, root, _lib.ptr(small), small.numel(), ctypes.byref(required),
                                 vol2._stream())
    assert rc == _lib.GSB_ERR_WORKSPACE, rc
    need = torch.tensor([required.value], dtype=torch.int64, device=vol2.device)
    lo, hi = need.clone(), need.clone()
    dist.all_reduce(lo, op=dist.ReduceOp.MIN)
    dist.all_reduce(hi, op=dist.ReduceOp.MAX)
    assert int(lo) == int(hi) > small.numel(), "ranks disagree on the scratch the merge needs"
    vol2.reduce_across_ranks(dst=root)
    torch.cuda.synchronize()
    if rank == root:
        compare(vol2, seq, "reduce to root")
    else:
        after = vol2.export_units()
        assert set(after) == set(before) and all(np.array_equal(after[k][0], before[k][0]) for k in before), "a non-root volume changed"
    assert vol2.pool_stats()["dropped_total"] == 0, f"reduce to root: rank {rank} dropped bricks"
    # (3) every rank's pool holds its own bricks but not the union: the all-reduce drops the bricks that find no room, and
    #     counts them where the volume reports its drops
    most = torch.tensor([own], dtype=torch.int64, device=vol.device)
    dist.all_reduce(most, op=dist.ReduceOp.MAX)
    assert n > int(most), "the test needs a union larger than every rank's own bricks"
    vol3 = fuse(mine, pool_bricks=int(most))
    assert vol3.pool_stats()["dropped_total"] == 0
    vol3.reduce_across_ranks(dst=None)
    torch.cuda.synchronize()
    assert vol3.num_bricks() == int(most) and vol3.pool_stats()["dropped_total"] > 0, (rank, vol3.pool_stats())
    dist.barrier()
    if rank == 0:
        print(f"dist_gpu_check ok: world={world} views/rank={[len(shard_views(NV, q, world)) for q in range(world)]} "
              f"bricks own/union={own}/{n} touched voxels={nvox} max|dtsdf|={err:.2e} max|dcolor|={cerr:.2e}")
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
