"""TSDF fusion stage: H100-native replacement for the Open3D calls in
gs2mesh_utils/tsdf_utils.py (reference), behind the reference's own class surface.

Three layers, thinnest first:

* `TSDFVolume`          torch-owned device memory + the C-ABI volume handle
                        (`gsb_tsdf_*` in include/gs2mesh_b200.h).
* `ScalableTSDFVolume`  Open3D-shaped facade (`integrate(rgbd, intrinsic, extrinsic)`,
                        `extract_triangle_mesh()`), so the body of tsdf_utils.py:53-108 reads the
                        same with `o3d` replaced by `gs2mesh_b200.o3d_compat`.
* `TSDF`                the stage class run_single.py:154-174 drives:
                        `TSDF(renderer, stereo, args, out_name)`, `.run()`, `.save_mesh()`,
                        `.clean_mesh()`, plus the `integrate()` / `extract_mesh()` aliases
                        BASELINE.json's north_star names.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional, Sequence

import numpy as np
import torch

from . import _lib
from ._lib import BRICK, BRICK_VOXELS, GsbVolumeDesc, ptr


def default_window(resolution: int = 512):
    """Brick window of the dense `resolution`^3 lattice centred on the origin: the dense equivalent
    of `voxel_length = TSDF_voxel / 512` (tsdf_utils.py:51, SURVEY F3).  Only a VIEW for dense read-backs
    (`TSDFVolume.bricks()` / `.dense()`): the volume itself is unbounded."""
    nb = resolution // BRICK
    return (-(nb // 2),) * 3, (nb,) * 3


DEFAULT_POOL_BRICKS = 1 << 15  # 32768 bricks = 1 GiB of (tsdf, weight) + 2 GiB of colour; grown on demand
LATTICE_LIMIT = 1 << 20  # brick lattice indices lie in [-2^20, 2^20) per axis (21-bit hash keys)


class TSDFVolume:
    """Open3D's ScalableTSDFVolume in HBM: an unbounded set of 16^3-voxel bricks, opened on first touch, addressed by their
    integer lattice index through a device hash table and stored in a brick pool (GsbVolumeDesc in include/gs2mesh_b200.h).
    `brick_origin` / `brick_count` only define the window the dense read-backs `bricks()` / `dense()` look at."""

    def __init__(self, voxel_length: float, sdf_trunc: float, brick_origin: Optional[Sequence[int]] = None,
                 brick_count: Optional[Sequence[int]] = None, with_color: bool = True, device="cuda",
                 pool_bricks: Optional[int] = None):
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("TSDFVolume needs a CUDA device (gs2mesh_b200 has no CPU path)")
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        self.voxel_length = float(voxel_length)
        self.sdf_trunc = float(sdf_trunc)
        if brick_origin is None or brick_count is None:
            brick_origin, brick_count = default_window(512)
        self.brick_origin = tuple(int(v) for v in brick_origin)
        self.brick_count = tuple(int(v) for v in brick_count)
        self.with_color = bool(with_color)
        self._L = _lib.lib()
        self._h = None
        self._comms = {}
        self._reduce_scratch = None
        self._allocate(int(pool_bricks or DEFAULT_POOL_BRICKS))
        self.frames_integrated = 0

    # ------------------------------------------------------------------ storage
    def _allocate(self, pool_bricks: int):
        dev = self.device
        self.pool_bricks = int(pool_bricks)
        self.hash_slots = 1 << max(4, int(2 * self.pool_bricks - 1).bit_length())
        n_vox = self.pool_bricks * BRICK_VOXELS
        self.tsdf_weight = torch.zeros(n_vox * 2, dtype=torch.float32, device=dev)
        self.color = torch.zeros(n_vox * 4, dtype=torch.float32, device=dev) if self.with_color else None
        self._index = torch.zeros(self.pool_bricks, 4, dtype=torch.int32, device=dev)
        self._hash_keys = torch.full((self.hash_slots,), -1, dtype=torch.int64, device=dev)  # all-ones = empty
        self._hash_vals = torch.zeros(self.hash_slots, dtype=torch.int32, device=dev)
        self._hash_stamp = torch.zeros(self.hash_slots, dtype=torch.int32, device=dev)
        self._list = torch.zeros(self.hash_slots, dtype=torch.int32, device=dev)
        self._counters = torch.zeros(8, dtype=torch.int32, device=dev)
        desc = GsbVolumeDesc()
        desc.voxel_length = self.voxel_length
        desc.sdf_trunc = self.sdf_trunc
        desc.pool_bricks = self.pool_bricks
        desc.hash_slots = self.hash_slots
        desc.tsdf_weight = ptr(self.tsdf_weight)
        desc.color = ptr(self.color)
        desc.brick_index = ptr(self._index)
        desc.hash_keys = ptr(self._hash_keys)
        desc.hash_vals = ptr(self._hash_vals)
        desc.hash_stamp = ptr(self._hash_stamp)
        desc.brick_list = ptr(self._list)
        desc.counters = ptr(self._counters)
        if self._h:
            self._L.gsb_tsdf_destroy(self._h)
        self._h = self._L.gsb_tsdf_create(C.byref(desc))
        if not self._h:
            raise _lib.GsbError(_lib.GSB_ERR_INVALID, self._L.gsb_last_error().decode())

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            self._L.gsb_tsdf_destroy(h)
            self._h = None
        for comm in getattr(self, "_comms", {}).values():
            self._L.gsb_comm_destroy(comm)

    def grow(self, pool_bricks: Optional[int] = None):
        """Re-house the volume in a larger pool (synchronises): every open brick keeps its content and its pool slot."""
        n = self.num_bricks()
        old_tw, old_color, old_index = self.tsdf_weight, self.color, self._index
        self._allocate(int(pool_bricks or 2 * self.pool_bricks))
        if n:
            perm = self.find_bricks(old_index[:n], insert=True).long()  # where the parallel insert put each brick
            self.tsdf_weight.view(self.pool_bricks, -1)[perm] = old_tw.view(-1, BRICK_VOXELS * 2)[:n]
            if self.color is not None:
                self.color.view(self.pool_bricks, -1)[perm] = old_color.view(-1, BRICK_VOXELS * 4)[:n]

    # ------------------------------------------------------------------ helpers
    @property
    def resolution(self):
        return tuple(n * BRICK for n in self.brick_count)

    @property
    def origin(self):
        """World position of the view window's minimum corner."""
        return tuple(o * BRICK * self.voxel_length for o in self.brick_origin)

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def _f32(self, t, name):
        if not isinstance(t, torch.Tensor):
            t = torch.as_tensor(np.ascontiguousarray(t, dtype=np.float32))
        if not t.is_cuda:
            t = t.to(self.device, non_blocking=True)
        return t.contiguous().float()

    def _u8(self, t):
        if t is None:
            return None
        if not isinstance(t, torch.Tensor):
            t = torch.as_tensor(np.ascontiguousarray(t, dtype=np.uint8))
        if not t.is_cuda:
            t = t.to(self.device, non_blocking=True)
        if t.dtype == torch.bool:
            t = t.to(torch.uint8)
        return t.contiguous()

    # ------------------------------------------------------------------ hot path
    def prepare_depth(self, depth, width, height, *, final_T=None, mask=None, alpha_min=0.5, min_depth=0.0,
                      depth_scale=1.0, depth_trunc=float("inf"), out=None):
        """Fused per-view depth preparation (tsdf_utils.py:78-93 + Open3D's depth conversion)."""
        with torch.cuda.device(self.device):
            depth = self._f32(depth, "depth")
            final_T = None if final_T is None else self._f32(final_T, "final_T")
            mask = self._u8(mask)
            if out is None:
                out = torch.empty(height, width, dtype=torch.float32, device=self.device)
            trunc = float(depth_trunc) if np.isfinite(depth_trunc) else 3.0e38
            _lib.check(self._L.gsb_tsdf_prepare_depth(ptr(depth), ptr(final_T), ptr(mask), int(width), int(height),
                                                      float(alpha_min), float(min_depth), float(depth_scale), trunc,
                                                      ptr(out), self._stream()))
        return out

    def integrate(self, depth, rgb, width, height, fx, fy, cx, cy, extrinsic_w2c):
        """`volume.integrate(rgbd, intrinsic, extrinsic)` (tsdf_utils.py:107) on prepared inputs:
        depth = float32 [H,W] already converted (see prepare_depth), rgb = uint8 [H,W,3] or None,
        extrinsic_w2c = 4x4 world->camera (float64, host)."""
        with torch.cuda.device(self.device):
            depth = self._f32(depth, "depth")
            if depth.numel() != width * height:
                raise RuntimeError("[TSDFVolume::integrate] Unsupported image format.")  # Open3D's size check
            rgb = self._u8(rgb)
            if rgb is not None and rgb.numel() != width * height * 3:
                raise RuntimeError("[TSDFVolume::integrate] Unsupported image format.")
            e = np.ascontiguousarray(np.asarray(extrinsic_w2c, dtype=np.float64).reshape(16))
            _lib.check(self._L.gsb_tsdf_integrate(self._h, ptr(depth), ptr(rgb if self.color is not None else None), int(width),
                                                  int(height), float(fx), float(fy), float(cx), float(cy),
                                                  e.ctypes.data_as(C.POINTER(C.c_double)), self._stream()))
        self.frames_integrated += 1

    def integrate_exact(self, depth, rgb, width, height, fx, fy, cx, cy, extrinsic_w2c):
        """integrate() that can never lose a brick: the frame's bricks are opened first (`gsb_tsdf_touch`), the pool is grown
        if they did not fit, and only then are the voxels updated.  Two host synchronisations per frame -- for callers that
        want Open3D's unbounded behaviour frame by frame (the o3d_compat facade); the stage class checks once per run."""
        with torch.cuda.device(self.device):
            depth = self._f32(depth, "depth")
            e = np.ascontiguousarray(np.asarray(extrinsic_w2c, dtype=np.float64).reshape(16))
            for _ in range(16):
                _lib.check(self._L.gsb_tsdf_touch(self._h, ptr(depth), int(width), int(height), float(fx), float(fy), float(cx),
                                                  float(cy), e.ctypes.data_as(C.POINTER(C.c_double)), self._stream()))
                if self.ensure_capacity():
                    break
        self.integrate(depth, rgb, width, height, fx, fy, cx, cy, extrinsic_w2c)

    def pool_stats(self):
        """dict(touched, dropped, frame, bricks, dropped_total, out_of_range, out_of_range_total) -- synchronises.
        `dropped` counts bricks the last integrate could not store for want of pool slots; `dropped_total` since creation /
        reset.  `out_of_range` counts the brick-box cells of the last integrate whose lattice index lies outside
        [-2^20, 2^20) (one per sampled pixel and cell); no pool can hold those."""
        out = torch.zeros(8, dtype=torch.int32, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(self._L.gsb_tsdf_last_stats(self._h, ptr(out), self._stream()))
        v = out.cpu().numpy().astype(np.int64) & 0xFFFFFFFF
        return dict(touched=int(v[0]), dropped=int(v[1]), frame=int(v[2]), bricks=int(v[3]), dropped_total=int(v[4]),
                    out_of_range=int(v[5]), out_of_range_total=int(v[6]))

    def last_stats(self):
        """(bricks touched, bricks dropped, frame id) of the last integrate (syncs)."""
        s = self.pool_stats()
        return s["touched"], s["dropped"], s["frame"]

    def num_bricks(self) -> int:
        """Bricks opened so far (synchronises)."""
        return int(self._counters[4].item())

    def ensure_capacity(self):
        """After a batch of integrations: True if every brick found room.  Otherwise the pool is doubled (content kept, the
        dropped-bricks counter cleared) and False is returned -- the views since the last check must be integrated again.
        Raises RuntimeError, without growing, if some brick lay outside the lattice range: integrating again cannot help."""
        s = self.pool_stats()
        if s["out_of_range_total"]:
            lim = LATTICE_LIMIT * BRICK * self.voxel_length
            raise RuntimeError(f"TSDFVolume: {s['out_of_range_total']} brick-box cells lie outside the brick lattice range "
                               f"[-2^20, 2^20) per axis (|coordinate| >= {lim:.6g} at voxel_length {self.voxel_length:.6g}); "
                               "such bricks cannot be stored")
        if s["dropped_total"] == 0:
            return True
        self.grow()
        self._counters[5] = 0
        return False

    # ------------------------------------------------------------------ brick access
    def find_bricks(self, indices, insert: bool = False):
        """Lattice indices [n,3|4] -> pool slots int32[n] (-1 = not in the volume)."""
        idx = torch.as_tensor(indices).to(self.device, dtype=torch.int32)
        if idx.ndim != 2 or idx.shape[1] not in (3, 4):
            raise ValueError("indices must be [n,3]")
        n = int(idx.shape[0])
        idx4 = torch.zeros(n, 4, dtype=torch.int32, device=self.device)
        idx4[:, :3] = idx[:, :3]
        slots = torch.empty(n, dtype=torch.int32, device=self.device)
        scratch = torch.empty(n, dtype=torch.int32, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(self._L.gsb_tsdf_find_bricks(self._h, ptr(idx4), n, 1 if insert else 0, ptr(slots), ptr(scratch), self._stream()))
        return slots

    def brick_indices(self):
        """int32 [n,3] lattice indices of the open bricks, in pool order (synchronises)."""
        return self._index[: self.num_bricks(), :3]

    def pool(self):
        """View [pool_bricks, 4096, 2] of the brick pool (no copy); slots >= num_bricks() are unused (zero)."""
        return self.tsdf_weight.view(self.pool_bricks, BRICK_VOXELS, 2)

    def brick_at(self, index):
        """[4096, 2] (tsdf, weight) view of the brick with integer lattice index (bx, by, bz) (Open3D's volume-unit index)."""
        slot = int(self.find_bricks(np.asarray(index, dtype=np.int32).reshape(1, -1)[:, :3])[0].item())
        if slot < 0:
            raise KeyError(f"brick {tuple(int(v) for v in index)} was never opened")
        return self.pool()[slot]

    def export_units(self):
        """{(bx,by,bz): (tsdf_weight float32 [4096,2], colour float32 [4096,4] | None)} of every open brick, on the host
        (Open3D: the contents of volume_units_)."""
        n = self.num_bricks()
        idx = self._index[:n, :3].cpu().numpy()
        tw = self.pool()[:n].cpu().numpy()
        col = self.color.view(self.pool_bricks, BRICK_VOXELS, 4)[:n].cpu().numpy() if self.color is not None else None
        return {tuple(int(v) for v in idx[i]): (tw[i], None if col is None else col[i]) for i in range(n)}

    def bricks(self, brick_origin=None, brick_count=None):
        """Dense read-back [n_window_bricks, 4096, 2] of a window of the lattice (default: the view window), bricks row-major
        over (bx,by,bz), never-opened bricks zero: the layout oracle.OracleTSDFVolume.export_bricks produces.  A COPY."""
        b0 = self.brick_origin if brick_origin is None else tuple(int(v) for v in brick_origin)
        nb = self.brick_count if brick_count is None else tuple(int(v) for v in brick_count)
        g = torch.stack(torch.meshgrid(*[torch.arange(b0[k], b0[k] + nb[k], dtype=torch.int32) for k in range(3)], indexing="ij"),
                        -1).reshape(-1, 3)
        slots = self.find_bricks(g).long()
        out = torch.zeros(len(g), BRICK_VOXELS, 2, dtype=torch.float32, device=self.device)
        have = slots >= 0
        out[have] = self.pool()[slots[have]]
        return out

    def colors(self, brick_origin=None, brick_count=None):
        """Colour companion of bricks(): [n_window_bricks, 4096, 4] running-mean (r, g, b, unused), zeros where never opened."""
        b0 = self.brick_origin if brick_origin is None else tuple(int(v) for v in brick_origin)
        nb = self.brick_count if brick_count is None else tuple(int(v) for v in brick_count)
        g = torch.stack(torch.meshgrid(*[torch.arange(b0[k], b0[k] + nb[k], dtype=torch.int32) for k in range(3)], indexing="ij"),
                        -1).reshape(-1, 3)
        slots = self.find_bricks(g).long()
        out = torch.zeros(len(g), BRICK_VOXELS, 4, dtype=torch.float32, device=self.device)
        have = slots >= 0
        out[have] = self.color.view(self.pool_bricks, BRICK_VOXELS, 4)[slots[have]]
        return out

    def dense(self, brick_origin=None, brick_count=None):
        """(tsdf, weight) of a window of the lattice as dense [X,Y,Z] grids in Open3D UniformTSDFVolume index order."""
        b0 = self.brick_origin if brick_origin is None else tuple(int(v) for v in brick_origin)
        nb = self.brick_count if brick_count is None else tuple(int(v) for v in brick_count)
        rx, ry, rz = (n * BRICK for n in nb)
        tsdf = torch.empty(rx, ry, rz, dtype=torch.float32, device=self.device)
        weight = torch.empty_like(tsdf)
        with torch.cuda.device(self.device):
            _lib.check(self._L.gsb_tsdf_export_dense(self._h, (C.c_int32 * 3)(*b0), (C.c_int32 * 3)(*nb), ptr(tsdf), ptr(weight),
                                                     self._stream()))
        return tsdf, weight

    def reset(self):
        self.tsdf_weight.zero_()
        if self.color is not None:
            self.color.zero_()
        self._index.zero_()
        self._hash_keys.fill_(-1)
        self._hash_vals.zero_()
        self._hash_stamp.zero_()
        self._counters.zero_()
        self.frames_integrated = 0

    # ------------------------------------------------------------------ multi-GPU merge
    def to_sums(self):
        with torch.cuda.device(self.device):
            _lib.check(self._L.gsb_tsdf_to_sums(self._h, self._stream()))

    def from_sums(self):
        with torch.cuda.device(self.device):
            _lib.check(self._L.gsb_tsdf_from_sums(self._h, self._stream()))

    def _comm(self, group):
        """ncclComm_t of this volume's merge, created once per process group: rank 0 makes the id, torch.distributed carries
        its 128 bytes to the others (plumbing), every rank joins with gsb_comm_create."""
        import torch.distributed as dist

        key = id(group) if group is not None else 0
        if key not in self._comms:
            world, rank = dist.get_world_size(group), dist.get_rank(group)
            buf = (C.c_uint8 * 128)()
            if rank == 0:
                _lib.check(self._L.gsb_comm_unique_id(buf))
            t = torch.tensor(list(bytes(buf)), dtype=torch.uint8, device=self.device)
            dist.broadcast(t, src=dist.get_global_rank(group, 0) if group is not None else 0, group=group)
            ident = (C.c_uint8 * 128)(*t.cpu().tolist())
            with torch.cuda.device(self.device):
                comm = self._L.gsb_comm_create(ident, world, rank)
            if not comm:
                raise _lib.GsbError(_lib.GSB_ERR_CUDA, self._L.gsb_last_error().decode())
            self._comms[key] = comm
        return self._comms[key]

    def reduce_across_ranks(self, group=None, dst: Optional[int] = None):
        """Merge view-sharded volumes with ONE `gsb_tsdf_reduce` call per rank (include/gs2mesh_b200.h): the ranks exchange
        their brick lattice indices, agree on the union, and sum-reduce (sum tsdf*w, w, sum rgb*w) of exactly those bricks in
        one NCCL reduce (dst = rank) or all-reduce (dst=None); everything runs on the current stream, the only host
        synchronisation is the read of the union's size.  The root exchanges its pool in place.
        A rank whose pool is smaller than another's grows to the largest first; volumes that disagree on `with_color` raise
        ValueError on every rank."""
        import torch.distributed as dist

        if not dist.is_initialized() or dist.get_world_size(group) == 1:
            return
        world, rank = dist.get_world_size(group), dist.get_rank(group)
        # gsb_tsdf_reduce needs the same pool size, colour setting and scratch size on every rank, but each rank grows its
        # pool on its own while it integrates: agree on the largest pool (grow keeps every brick) and check the colour
        agree = torch.tensor([self.pool_bricks, int(self.with_color), 1 - int(self.with_color)], dtype=torch.int64,
                             device=self.device)
        dist.all_reduce(agree, op=dist.ReduceOp.MAX, group=group)
        pool, some_color, some_plain = (int(v) for v in agree.tolist())
        if some_color and some_plain:
            raise ValueError("reduce_across_ranks: the ranks' volumes disagree on with_color; all of them must keep colour, "
                             "or none")
        if pool > self.pool_bricks:
            self.grow(pool)
        comm = self._comm(group)
        with torch.cuda.device(self.device):
            # scratch for the worst case (the union fills the pool): the same size on every rank -- a rank must never take the
            # "too small, retry" exit of gsb_tsdf_reduce alone, so the size passed is `need`, not what an earlier merge left
            # allocated -- and allocated once, so no merge pays for an allocation or for a repeated index exchange (an
            # undersized first guess cost 1.75 ms instead of ~1 ms on 8 GPUs, 61 ms on C4)
            need = int(self._L.gsb_tsdf_reduce_scratch_bytes(self._h, world, self.pool_bricks))
            required = C.c_size_t(0)
            for _ in range(3):
                if self._reduce_scratch is None or self._reduce_scratch.numel() < need:
                    self._reduce_scratch = None
                    self._reduce_scratch = torch.empty(need, dtype=torch.uint8, device=self.device)
                rc = self._L.gsb_tsdf_reduce(self._h, comm, world, rank, -1 if dst is None else int(dst), ptr(self._reduce_scratch),
                                             need, C.byref(required), self._stream())
                if rc != _lib.GSB_ERR_WORKSPACE:
                    break
                need = required.value  # the same on every rank: all ranks retry together
            _lib.check(rc)


def filter_object_mask(mask, closing_kernel_size: int = 10, erosion_kernel_size: int = 10, invert: bool = False, device="cuda"):
    """tsdf_utils.py:69-77 on the GPU: optional inversion, cv2.morphologyEx(MORPH_CLOSE, ones(ck,ck)) (dilate, then
    erode) and cv2.erode(ones(ek,ek)); returns a uint8 0/1 device mask [H,W] that `prepare_depth(mask=...)` takes."""
    L = _lib.lib()
    if not isinstance(mask, torch.Tensor):
        mask = torch.as_tensor(np.ascontiguousarray(np.asarray(mask).astype(np.uint8)))
    dev = mask.device if mask.is_cuda else torch.device(device)
    m = (mask.to(dev) != 0)
    if invert:
        m = ~m
    a = m.to(torch.uint8).contiguous()
    h, w = a.shape
    b = torch.empty_like(a)
    with torch.cuda.device(dev):
        stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        for k, dilate in ((closing_kernel_size, 1), (closing_kernel_size, 0), (erosion_kernel_size, 0)):
            _lib.check(L.gsb_mask_morphology(ptr(a), w, h, int(k), dilate, ptr(b), stream))
            a, b = b, a
    return a


def merge_units_protocol(units, group=None, dst: Optional[int] = None, pool_bricks: int = 4096):
    """Host-side statement of `gsb_tsdf_reduce`'s protocol (csrc/gsb_reduce.cu), step for step, on numpy units
    {(bx,by,bz): tsdf_weight float32 [4096,2]} with torch.distributed collectives of ANY backend -- what the CPU (gloo,
    world_size 2) tests run, since the device path needs GPUs:
      1. all-gather of every rank's (count, fixed-size padded list of brick lattice indices);
      2. the receiving ranks open the bricks they lack (zero-filled);
      3. broadcast of the canonical rank's brick order;
      4. pack in canonical order, (mean,w) -> (sum,w), bricks a rank never saw travel as zeros;
      5. ONE sum reduce (dst) / all-reduce (dst=None) of the packed payload;
      6. (sum,w) -> (mean,w) where the result lives.
    Returns this rank's units after the merge."""
    import torch.distributed as dist

    world, rank = dist.get_world_size(group), dist.get_rank(group)
    canon_rank = 0 if dst is None else int(dst)
    receives = dst is None or rank == canon_rank
    units = {k: np.array(v, dtype=np.float32, copy=True) for k, v in units.items()}
    order = list(units)  # pool order of this rank
    # 1.
    mine = torch.zeros(1 + pool_bricks, 4, dtype=torch.int32)
    mine[0, 0] = len(order)
    if order:
        mine[1:1 + len(order), :3] = torch.tensor(order, dtype=torch.int32)
    gathered = [torch.zeros_like(mine) for _ in range(world)]
    dist.all_gather(gathered, mine, group=group)
    # 2.
    if receives:
        for r in range(world):
            if r == rank:
                continue
            for k in gathered[r][1:1 + int(gathered[r][0, 0])].tolist():
                key = tuple(k[:3])
                if key not in units:
                    units[key] = np.zeros((BRICK_VOXELS, 2), np.float32)
                    order.append(key)
    # 3.
    canon = torch.zeros(1 + pool_bricks, 4, dtype=torch.int32)
    if rank == canon_rank:
        canon[0, 0] = len(order)
        canon[1:1 + len(order), :3] = torch.tensor(order, dtype=torch.int32)
    dist.broadcast(canon, src=canon_rank if group is None else dist.get_global_rank(group, canon_rank), group=group)
    n = int(canon[0, 0])
    canon_keys = [tuple(k[:3]) for k in canon[1:1 + n].tolist()]
    # 4.
    packed = torch.zeros(n, BRICK_VOXELS, 2, dtype=torch.float32)
    for i, key in enumerate(canon_keys):
        if key in units:
            tw = units[key]
            packed[i, :, 0] = torch.from_numpy(tw[:, 0] * tw[:, 1])
            packed[i, :, 1] = torch.from_numpy(tw[:, 1])
    # 5.
    if dst is None:
        dist.all_reduce(packed, op=dist.ReduceOp.SUM, group=group)
    else:
        dist.reduce(packed, dst=canon_rank if group is None else dist.get_global_rank(group, canon_rank), op=dist.ReduceOp.SUM,
                    group=group)
    # 6.
    if receives:
        p = packed.numpy()
        for i, key in enumerate(canon_keys):
            w = p[i, :, 1]
            units[key] = np.stack([np.where(w > 0, p[i, :, 0] / np.maximum(w, 1e-30), 0).astype(np.float32), w], -1)
    return units


def merge_bricks_reference(volumes_tw):
    """Host-side statement of the cross-rank merge (used by the CPU gloo tests):
    given per-rank [n,4096,2] (mean, weight) arrays returns the merged (mean, weight)."""
    total_w = sum(tw[..., 1] for tw in volumes_tw)
    total_s = sum(tw[..., 0] * tw[..., 1] for tw in volumes_tw)
    mean = np.where(total_w > 0, total_s / np.maximum(total_w, 1e-30), 0.0).astype(np.float32)
    return np.stack([mean, total_w.astype(np.float32)], axis=-1)


def shard_views(num_views: int, rank: int, world_size: int):
    """View -> rank assignment of the multi-GPU path: round-robin (SURVEY 8(e))."""
    return list(range(rank, num_views, world_size))


class TSDF:
    """Stage class with the reference's surface (gs2mesh_utils/tsdf_utils.py:23-142)."""

    def __init__(self, renderer, stereo, args, out_name, *, window_resolution: int = 512, device=None,
                 pool_bricks: Optional[int] = None):
        self.model_name = getattr(stereo, "model_name", "rendered")  # tsdf_utils.py:34
        self.renderer = renderer
        self.out_name = out_name
        self.args = args
        self.window_resolution = window_resolution  # only the window dense read-backs look at; the volume is unbounded
        self.pool_bricks = pool_bricks
        self.device = device or getattr(renderer, "device", "cuda")
        self.volume: Optional[TSDFVolume] = None
        self.mesh = None

    # -- argument access with the reference's defaults (argument_utils.py:74-90)
    def _arg(self, name, default):
        return getattr(self.args, name, default)

    def _make_volume(self):
        voxel_length = float(self._arg("TSDF_voxel", 2)) / 512  # tsdf_utils.py:51
        origin, count = default_window(self.window_resolution)
        return TSDFVolume(voxel_length, float(self._arg("TSDF_sdf_trunc", 0.04)), origin, count, with_color=True,
                          device=self.device, pool_bricks=self.pool_bricks)

    @staticmethod
    def _view_list(value):
        """`--TSDF_valid` / `--TSDF_skip` are declared `type=str` in the reference (argument_utils.py:76-77) yet used with
        `camera_number in ...` (tsdf_utils.py:61-63), which only works for lists handed in programmatically.  Both are
        accepted here: a list / tuple / set of ints, or a string such as "0,5,10" or "[0, 5, 10]"."""
        if value is None:
            return None
        if isinstance(value, str):
            import re

            return {int(tok) for tok in re.findall(r"-?\d+", value)}
        return {int(v) for v in value}

    def _selected(self, camera_number):
        valid = self._view_list(self._arg("TSDF_valid", None))
        skip = self._view_list(self._arg("TSDF_skip", None))
        if camera_number % int(self._arg("TSDF_dilate", 1)) != 0:
            return False
        if valid is not None and camera_number not in valid:
            return False
        if skip is not None and camera_number in skip:
            return False
        return True

    def _load_view(self, camera_number):
        """(rgb uint8 [H,W,3], depth float32 [H,W], object_mask|None, occlusion_mask|None) for one view: from the
        renderer's in-memory frames when it kept them, else from the files the reference stages exchange
        (tsdf_utils.py:65-80)."""
        frame = None
        getter = getattr(self.renderer, "get_frame", None)
        if getter is not None:
            frame = getter(camera_number)
        out_dir = self.renderer.render_folder_name(camera_number)
        obj_mask = occ_mask = None
        have_mem = frame is not None and "left_u8" in frame and "depth" in frame
        if have_mem:
            rgb, depth = frame["left_u8"], frame["depth"]
            occ_mask = frame.get("occlusion_mask")  # handed over by the stereo stage (Renderer.put_stereo_outputs)
        else:
            from PIL import Image

            rgb = np.array(Image.open(os.path.join(out_dir, "left.png"))).astype(np.uint8)
            depth = np.load(os.path.join(out_dir, f"out_{self.model_name}", "depth.npy"))
        if self._arg("TSDF_use_mask", False):
            m = np.load(os.path.join(out_dir, "left_mask.npy")).astype(bool)
            invert = bool(self._arg("TSDF_invert_mask", False))
            if self._arg("TSDF_erode_mask", True):  # tsdf_utils.py:72-77, on the GPU
                obj_mask = filter_object_mask(m, int(self._arg("TSDF_closing_kernel_size", 10)),
                                              int(self._arg("TSDF_erosion_kernel_size", 10)), invert, device=self.device)
            else:
                obj_mask = ~m if invert else m
        if self._arg("TSDF_use_occlusion_mask", True) and not have_mem:
            occ_path = os.path.join(out_dir, f"out_{self.model_name}", "occlusion_mask.npy")
            if os.path.exists(occ_path):
                occ_mask = np.load(occ_path).astype(bool)
        return rgb, depth, obj_mask, occ_mask

    # -- north_star alias: one view
    def integrate(self, depth, rgb, left_camera, *, final_T=None, mask=None):
        """Fuse one view.  `depth`: float [H,W] metric depth (host or device); when `final_T` is
        given `depth` is the rasterizer's sum(z*alpha*T) and is normalised by alpha on the GPU."""
        if self.volume is None:
            self.volume = self._make_volume()
        scale = float(self._arg("TSDF_scale", 1.0))
        baseline = float(self.renderer.baseline)
        w, h = int(left_camera["width"]), int(left_camera["height"])
        extrinsic = np.array(left_camera["extrinsic"], dtype=np.float64).copy()
        extrinsic[:3, 3] /= scale  # tsdf_utils.py:85-86
        prepared = self.volume.prepare_depth(
            depth, w, h, final_T=final_T, mask=mask,
            min_depth=float(self._arg("TSDF_min_depth_baselines", 4)) * baseline,  # :83
            depth_scale=scale, depth_trunc=baseline * float(self._arg("TSDF_max_depth_baselines", 20)) / scale)  # :92
        self.volume.integrate(prepared, rgb, w, h, left_camera["fx"], left_camera["fy"], left_camera["cx"],
                              left_camera["cy"], np.linalg.inv(extrinsic))  # :106-107

    def run(self, visualize=False, views: Optional[Sequence[int]] = None):
        """tsdf_utils.py:39-110.  `views` restricts the loop (used for view sharding across ranks).  The volume is unbounded
        like Open3D's; if the brick pool turns out too small it is doubled and the loop repeated."""
        check = getattr(self.renderer, "check_status", None)
        if check is not None and getattr(self.renderer, "_ready", False):
            torch.cuda.synchronize()
            check()  # no frame of the renderer's cache came out of an overflowed binning scratch
        self.volume = self._make_volume()
        for _attempt in range(8):
            self._fuse_views(views)
            if self.volume.ensure_capacity():
                break
            self.volume.reset()
        else:
            raise RuntimeError("TSDF.run: the brick pool kept overflowing")
        self.mesh = None
        return self.volume

    def _fuse_views(self, views):
        for camera_number, left_camera in enumerate(self.renderer.left_cameras):
            if views is not None and camera_number not in views:
                continue
            if not self._selected(camera_number):
                continue
            rgb, depth, obj_mask, occ_mask = self._load_view(camera_number)
            mask = None
            for m in (obj_mask, occ_mask):  # depth * object_mask * occlusion_mask (tsdf_utils.py:78-81)
                if m is None:
                    continue
                m = self.volume._u8(m if isinstance(m, torch.Tensor) else np.asarray(m).astype(np.uint8))
                mask = m if mask is None else mask * m
            self.integrate(depth, rgb, left_camera, mask=mask)

    def extract_mesh(self):
        """`volume.extract_triangle_mesh()` + scale + vertex normals (tsdf_utils.py:108-110)."""
        from .mesh import extract_triangle_mesh

        if self.volume is None:
            raise RuntimeError("TSDF.extract_mesh() called before run()/integrate()")
        self.mesh = extract_triangle_mesh(self.volume)
        self.mesh.scale(float(self._arg("TSDF_scale", 1.0)), (0, 0, 0))
        self.mesh.compute_vertex_normals(self.volume.device)
        return self.mesh

    def save_mesh(self):
        """tsdf_utils.py:112-120"""
        if self.mesh is None:
            self.extract_mesh()
        path = os.path.join(self.renderer.output_dir_root, f"{self.out_name}_mesh.ply")
        self.mesh.write_ply(path)
        print("SAVED MESH")
        return path

    def clean_mesh(self):
        """tsdf_utils.py:122-142 (the reference overwrites this method with the cleaned mesh on first
        call; here the result is kept in `.cleaned_mesh` and returned)."""
        if self.mesh is None:
            self.extract_mesh()
        thres = float(self._arg("TSDF_cleaning_threshold", 100000)) / float(self._arg("TSDF_scale", 1.0))
        self.cleaned_mesh = self.mesh.remove_small_clusters(thres)
        path = os.path.join(self.renderer.output_dir_root, f"{self.out_name}_cleaned_mesh.ply")
        self.cleaned_mesh.write_ply(path)
        print("SAVED CLEANED MESH")
        return path
