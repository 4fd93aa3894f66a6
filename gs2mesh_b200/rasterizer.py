"""Torch-facing wrapper of the C-ABI rasterizer (`gsb_raster_forward`).

PyTorch is used for device memory and streams only; all compute happens in
libgs2mesh_b200.so.  Mirrors the marshalling the reference does in
DGR/rasterize_points.cu:35-115 (allocate outputs, hand raw pointers to the kernels),
with a grow-only `Scratch` block per frame in flight instead of three byte tensors that
are resized on every call (rasterize_points.cu:27-33, 71-75).
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import torch

from . import _lib
from ._lib import GsbRasterArgs, ptr

# ONE default for every caller (stage class, compat module, raw wrapper): exact tile culling + the ex2.approx blend (the
# table kernel).  EXACT_EXP_FLAGS selects the blend with the reference's own exponent expression and full-precision expf
# (transmittance bit-identical to the reference binary; ~8 % slower per frame).
DEFAULT_FLAGS = _lib.RASTER_EXACT_TILE_CULL | _lib.RASTER_FAST_EXP
EXACT_EXP_FLAGS = _lib.RASTER_EXACT_TILE_CULL
# first guess of the binning capacity of a block that has not seen a frame: instances per Gaussian / floor
GUESS_PER_GAUSSIAN = 4
MIN_GUESS = 1 << 20


def capacity_for(need: int) -> int:
    """Binning capacity for frames that need up to `need` instances (what `num_rendered[0]` reports, also for a frame
    that overflowed)."""
    return int(need * 1.1) + 4096


class Scratch:
    """Scratch block of one frame in flight: the binning workspace, its capacity for one (P, W, H), and the int64[4]
    counts buffer of synchronous calls that do not ask for counts.

    Two frames in flight at the same time need two blocks; the owner of the streams a block is used on orders its reuse.
    Its tensors are recorded on every stream they are enqueued on, so releasing them -- on growth, on a new frame shape or
    when the owner drops the block -- waits for the work those streams hold at that moment."""

    def __init__(self, device, max_instances=0):
        self.device = device
        self.max_instances = int(max_instances)  # 0: the first frame starts from the first guess
        self.key = None
        self.workspace: Optional[torch.Tensor] = None
        self.counts: Optional[torch.Tensor] = None
        self._recorded = set()  # handles of the streams the current tensors are recorded on

    def ensure(self, P, W, H, min_instances, streams):
        """Workspace for a P-Gaussian W x H frame with room for at least `min_instances` instances, enqueued on `streams`
        (its work starts on streams[0]); the capacity for one frame shape never shrinks."""
        key = (P, W, H)
        if self.key not in (None, key):
            self.max_instances = 0
        max_instances = max(self.max_instances or max(GUESS_PER_GAUSSIAN * P, MIN_GUESS), int(min_instances))
        if self.workspace is None or key != self.key or max_instances > self.max_instances:
            need = _lib.lib().gsb_raster_workspace_bytes(P, W, H, max_instances)
            if self.workspace is None or self.workspace.numel() < need:
                self.workspace = None  # release before re-allocating
                # on the stream the frame starts on: the memory may still be in use by work queued there, and the
                # frame's work on its other streams is ordered behind its start
                with torch.cuda.stream(streams[0]):
                    self.workspace = torch.empty(need, dtype=torch.uint8, device=self.device)
                    if self.counts is None:
                        self.counts = torch.zeros(4, dtype=torch.int64, device=self.device)
                self._recorded = set()
            self.max_instances = max_instances
            self.key = key
        for s in streams:
            if s.cuda_stream not in self._recorded:
                self._recorded.add(s.cuda_stream)
                self.workspace.record_stream(s)
                self.counts.record_stream(s)
        return self.workspace


_scratch = {}  # (device index, stream handle) -> the block of synchronous single-view calls that bring none


def _default_scratch(device, stream) -> Scratch:
    """The block of synchronous single-view calls that bring none, one per (device, stream): the stream orders its reuse."""
    key = (device.index, stream.cuda_stream)
    if key not in _scratch:
        _scratch[key] = Scratch(device)
    return _scratch[key]


def _dev_f32(t, name, device):
    if t is None:
        return None
    if not isinstance(t, torch.Tensor):
        raise TypeError(f"{name} must be a torch.Tensor")
    if t.numel() == 0:  # the reference's "absent" sentinel is an empty tensor (__init__.py:197-207)
        return None
    if not t.is_cuda:
        raise RuntimeError(f"{name} must live on a CUDA device (gs2mesh_b200 has no CPU path)")
    if t.device != device:
        raise RuntimeError(f"{name} is on {t.device}, expected {device}")
    if t.dtype != torch.float32:
        t = t.float()
    return t.contiguous()


def rasterize_forward(*, means3D, opacities, viewmatrix, projmatrix, campos, bg, width, height, tan_fovx, tan_fovy,
                      shs=None, colors_precomp=None, scales=None, rotations=None, cov3D_precomp=None, sh_degree=0,
                      scale_modifier=1.0, prefiltered=False, flags=DEFAULT_FLAGS, want_depth=True, want_final_T=True,
                      want_radii=True, want_counts=False, out_color=None, out_depth=None, out_final_T=None,
                      async_mode=False, counts_out=None, min_instances=0, scratch: Optional[Scratch] = None):
    """One forward rasterization on the current CUDA stream, in the scratch block `scratch`.

    Returns dict(color[3,H,W], depth[H,W]|None, final_T[H,W]|None, radii[P]|None,
    counts (int64[4]: binned instances, reference-equivalent instances, overflow flag, large tiles)|None).

    async_mode=False (default): the call waits for the stream once at the end of the frame so that an
    undersized scratch block can be grown and the frame redone transparently.
    async_mode=True: nothing waits; pass `counts_out` (int64[4], device or pinned host memory) and check
    counts_out[2] == 0 after your own synchronisation (see Renderer.check_status()).
    An asynchronous call (async_mode, or RASTER_ASYNC in `flags`) needs a `scratch` block of its own; a synchronous call
    without one uses the block of the current stream.
    """
    flags = int(flags) | (_lib.RASTER_ASYNC if async_mode else 0)
    asynchronous = bool(flags & _lib.RASTER_ASYNC)
    if asynchronous and scratch is None:
        raise ValueError("an asynchronous rasterize_forward needs its own scratch block (scratch=Scratch(device))")
    if means3D.ndim != 2 or means3D.shape[1] != 3:
        raise RuntimeError("means3D must have dimensions (num_points, 3)")  # rasterize_points.cu:57-59
    device = means3D.device
    if not means3D.is_cuda:
        raise RuntimeError("means3D must live on a CUDA device (gs2mesh_b200 has no CPU path)")
    if means3D.shape[0] == 0:
        # rasterize_points.cu:68-77: with no points the zero-filled outputs are returned untouched
        W, H = int(width), int(height)
        z = lambda *s, dt=torch.float32: torch.zeros(*s, dtype=dt, device=device)
        return dict(color=z(3, H, W), depth=z(H, W) if want_depth else None, final_T=z(H, W) if want_final_T else None,
                    radii=z(0, dt=torch.int32) if want_radii else None, counts=z(4, dt=torch.int64) if want_counts else None)
    means3D = _dev_f32(means3D, "means3D", device)
    opacities = _dev_f32(opacities, "opacities", device)
    shs = _dev_f32(shs, "shs", device)
    colors_precomp = _dev_f32(colors_precomp, "colors_precomp", device)
    scales = _dev_f32(scales, "scales", device)
    rotations = _dev_f32(rotations, "rotations", device)
    cov3D_precomp = _dev_f32(cov3D_precomp, "cov3D_precomp", device)
    viewmatrix = _dev_f32(viewmatrix, "viewmatrix", device)
    projmatrix = _dev_f32(projmatrix, "projmatrix", device)
    campos = _dev_f32(campos, "campos", device)
    bg = _dev_f32(bg, "bg", device)
    P = means3D.shape[0]
    W, H = int(width), int(height)
    M = 0 if shs is None else int(shs.shape[1])

    with torch.cuda.device(device):
        f32 = dict(dtype=torch.float32, device=device)
        color = out_color if out_color is not None else torch.empty(3, H, W, **f32)
        depth = (out_depth if out_depth is not None else torch.empty(H, W, **f32)) if want_depth else None
        final_T = (out_final_T if out_final_T is not None else torch.empty(H, W, **f32)) if want_final_T else None
        radii = torch.empty(P, dtype=torch.int32, device=device) if want_radii else None
        counts = counts_out if counts_out is not None else (torch.zeros(4, dtype=torch.int64, device=device) if want_counts else None)
        st = torch.cuda.current_stream(device)
        if scratch is None:
            scratch = _default_scratch(device, st)
        stream = C.c_void_p(st.cuda_stream)
        L = _lib.lib()
        for attempt in range(1 if asynchronous else 3):
            ws = scratch.ensure(P, W, H, min_instances, (st,))
            status = counts if counts is not None else scratch.counts  # [0] is the frame's instance need, also on overflow
            args = GsbRasterArgs(
                P=P, sh_degree=int(sh_degree), sh_coeffs=M, width=W, height=H, background=ptr(bg), means3D=ptr(means3D),
                shs=ptr(shs), colors_precomp=ptr(colors_precomp), opacities=ptr(opacities), scales=ptr(scales),
                rotations=ptr(rotations), cov3D_precomp=ptr(cov3D_precomp), scale_modifier=float(scale_modifier),
                viewmatrix=ptr(viewmatrix), projmatrix=ptr(projmatrix), cam_pos=ptr(campos), tan_fovx=float(tan_fovx),
                tan_fovy=float(tan_fovy), prefiltered=int(bool(prefiltered)), flags=flags, out_color=ptr(color),
                out_depth=ptr(depth), out_final_T=ptr(final_T), radii=ptr(radii), num_rendered=ptr(status),
                workspace=ptr(ws), workspace_bytes=ws.numel(), max_instances=scratch.max_instances)
            rc = L.gsb_raster_forward(C.byref(args), stream)
            if rc == _lib.GSB_ERR_WORKSPACE and attempt < 2 and not asynchronous:
                min_instances = capacity_for(int(status[0]))
                continue
            _lib.check(rc)
            break
    return dict(color=color, depth=depth, final_T=final_T, radii=radii, counts=counts)


def rasterize_forward_pair(*, means3D, opacities, shs, scales, rotations, sh_degree, bg, width, height, eyes, streams,
                           scratch=None, flags=DEFAULT_FLAGS, shared_depth=False, scale_modifier=1.0, min_instances=0):
    """Both eyes of a stereo pair through `gsb_raster_forward_pair` (one fused preprocess pass over the Gaussian
    parameters; with `shared_depth` also one depth sort).  Always asynchronous.

    eyes: two dicts with viewmatrix[16], projmatrix[16], campos[3] (device), tan_fovx, tan_fovy, out_color[3,H,W],
          out_depth / out_final_T ([H,W] or None), counts_out (int64[4], device or pinned host, or None).
    streams: (left, right) torch streams; the shared part runs on the left one.
    scratch: (left, right) `Scratch` blocks, one per eye.  The shared part writes both on the left stream, and each
    eye's binning and blend read them on its own stream, so both blocks are recorded on both streams.  The left stream
    first waits for the right one: a pair may reuse the blocks of the previous pair on the same streams.
    The caller checks counts_out[2] (scratch overflow) and counts_out[3] (shared_depth claimed but depths differ) after
    its own synchronisation."""
    if scratch is None:
        raise ValueError("rasterize_forward_pair needs one scratch block per eye (scratch=(left, right))")
    device = means3D.device
    P = means3D.shape[0]
    W, H = int(width), int(height)
    M = int(shs.shape[1])
    L = _lib.lib()
    if P == 0:  # rasterize_points.cu:68-77: with no points the zero-filled outputs are returned untouched
        for eye, st in zip(eyes, streams):
            with torch.cuda.stream(st):
                for k in ("out_color", "out_depth", "out_final_T", "counts_out"):
                    if eye.get(k) is not None:
                        eye[k].zero_()
        return
    with torch.cuda.device(device):
        if streams[1] != streams[0]:
            streams[0].wait_stream(streams[1])
        blocks = []
        for eye, block in zip(eyes, scratch):
            ws = block.ensure(P, W, H, min_instances, streams)
            fl = int(flags) | _lib.RASTER_ASYNC | (_lib.RASTER_PAIR_SHARED_DEPTH if shared_depth else 0)
            blocks.append(GsbRasterArgs(
                P=P, sh_degree=int(sh_degree), sh_coeffs=M, width=W, height=H, background=ptr(bg), means3D=ptr(means3D),
                shs=ptr(shs), colors_precomp=None, opacities=ptr(opacities), scales=ptr(scales), rotations=ptr(rotations),
                cov3D_precomp=None, scale_modifier=float(scale_modifier), viewmatrix=ptr(eye["viewmatrix"]),
                projmatrix=ptr(eye["projmatrix"]), cam_pos=ptr(eye["campos"]), tan_fovx=float(eye["tan_fovx"]),
                tan_fovy=float(eye["tan_fovy"]), prefiltered=0, flags=fl, out_color=ptr(eye["out_color"]),
                out_depth=ptr(eye.get("out_depth")), out_final_T=ptr(eye.get("out_final_T")), radii=None,
                num_rendered=ptr(eye.get("counts_out")), workspace=ptr(ws), workspace_bytes=ws.numel(),
                max_instances=block.max_instances))
        _lib.check(L.gsb_raster_forward_pair(C.byref(blocks[0]), C.byref(blocks[1]), C.c_void_p(streams[0].cuda_stream),
                                             C.c_void_p(streams[1].cuda_stream)))


def mark_visible(positions, viewmatrix, projmatrix):
    """`_C.mark_visible` (DGR/ext.cpp:18): bool[P], z_view > 0.2."""
    device = positions.device
    positions = _dev_f32(positions, "positions", device)
    viewmatrix = _dev_f32(viewmatrix, "viewmatrix", device)
    projmatrix = _dev_f32(projmatrix, "projmatrix", device)
    P = positions.shape[0]
    present = torch.zeros(P, dtype=torch.uint8, device=device)
    with torch.cuda.device(device):
        stream = C.c_void_p(torch.cuda.current_stream(device).cuda_stream)
        _lib.check(_lib.lib().gsb_raster_mark_visible(P, ptr(positions), ptr(viewmatrix), ptr(projmatrix), ptr(present), stream))
    return present.bool()


def image_to_u8(chw: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """[3,H,W] float in [0,1] -> [H,W,3] uint8, cv2.imwrite's float->u8 rule (renderer_utils.py:389-390)."""
    if not chw.is_cuda:
        raise RuntimeError("image_to_u8 needs a CUDA tensor")
    chw = chw.contiguous().float()
    _, H, W = chw.shape
    hwc = out if out is not None else torch.empty(H, W, 3, dtype=torch.uint8, device=chw.device)
    with torch.cuda.device(chw.device):
        stream = C.c_void_p(torch.cuda.current_stream(chw.device).cuda_stream)
        _lib.check(_lib.lib().gsb_image_to_u8(ptr(chw), W, H, ptr(hwc), stream))
    return hwc
