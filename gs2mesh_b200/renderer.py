"""Stereo-pair renderer stage: H100-native replacement for
gs2mesh_utils/renderer_utils.py `Renderer` (reference), same class surface:

    Renderer(base_dir, colmap_dir, output_dir_root, args, dataset=, splatting=, experiment_name=, device=)
    .prepare_renderer()  .render_image_pair(i, visualize=False)  .render_folder_name(i)  len()
    .cameras  .left_cameras  .baseline  .output_dir_root
plus `render(i)` (the name BASELINE.json's north_star uses) and `Renderer.from_scene(...)` for
in-memory scenes.

What changes relative to the reference loop (renderer_utils.py:363-395), by design:
* activations / SH concatenation are done once in prepare_renderer(), not per view
  (gaussian_renderer/__init__.py:53-80 recomputes them for every camera);
* all camera matrices are uploaded once as a device table; no per-view `Camera` object, no
  dummy `torch.rand(3,h,w)` image upload (renderer_utils.py:386, cameras.py:39);
* the float->uint8 conversion (x255, saturate, HWC) runs on the GPU, so the D2H copy is 3 bytes
  per pixel instead of 12 (renderer_utils.py:389);
* the left view's expected depth (sum z*alpha*T) and transmittance are produced in the same
  blend loop and stay on the device for the TSDF stage.
PNG files are still written when `write_images` is on, so downstream reference stages (Stereo,
Masker) keep working.
"""
from __future__ import annotations

import os
from typing import Optional

import numpy as np
import torch

from . import camera as cam
from . import rasterizer as rast


# two stream sets: the device-resident rate is the same from 2 up (the GPU is busy); three gained 3-4 % on the host-buffer path
# on one box and nothing on another, and two of five runs with three showed a slow device-resident loop (profiles/r03a_*, r03c_*)
DEFAULT_PAIRS_IN_FLIGHT = 2
# D2H copies of the uint8 frames on their own streams (one per eye and stream set) instead of the eye's render stream: the
# render stream is free for the next pair of its set as soon as the frame is converted, not once it has crossed PCIe.
# GSB_COPY_STREAMS=0|1 overrides (A/B switch)
DEFAULT_COPY_STREAMS = 0
# Buffer sets beyond pairs_in_flight + 2.  The tensors of call n stay valid until call n + pairs_in_flight + 1 is entered,
# so the renders of call c may overwrite their buffer set once everything the caller enqueued before call
# c - (spare sets) - 1 was entered has run.  With no spare set that is the PREVIOUS call's entry -- which, in a loop that
# fuses every pair right after rendering it, sits behind the TSDF kernels of the pair that has just left this call's stream
# set: the set idles for their duration.  One spare set moves the gate one call back (the other stream set's pair).
# GSB_SPARE_BUFFER_SETS=0|1|2 overrides (A/B switch)
DEFAULT_SPARE_BUFFER_SETS = 0


class _StreamSet(list):
    """The (left, right) streams a stereo pair is rendered on, and the scratch blocks of its two eyes (`scratch`): the
    blocks are only ever used by the pair in flight on these streams."""

    def __init__(self, streams, scratch):
        super().__init__(streams)
        self.scratch = scratch


class _PairReady:
    """Completion handle of an asynchronously rendered pair (render_image_pair(..., wait=False)).  synchronize() waits for
    both eyes and -- like the synchronous call -- transparently re-renders the pair if its binning scratch turned out too
    small (the reference resizes inside every frame, rasterizer_impl.cu:281-285)."""

    def __init__(self, events, redo=None):
        self._events = events
        self._redo = redo

    def synchronize(self):
        for e in self._events:
            e.synchronize()
        if self._redo is not None:
            redo, self._redo = self._redo, None
            redo()


class Renderer:
    def __init__(self, base_dir=None, colmap_dir=None, output_dir_root=None, args=None, dataset="custom", splatting="custom",
                 experiment_name=None, device="cuda", *, cameras=None, baseline=None, gaussians=None):
        self.args = args
        self.base_dir = base_dir
        self.colmap_dir = colmap_dir
        self.output_dir_root = output_dir_root
        self.device = device
        self.dataset = dataset
        self.render_name = getattr(args, "colmap_name", None)
        self.white_background = bool(getattr(args, "GS_white_background", False))
        self.splatting_iteration = getattr(args, "GS_iterations", 30000)
        self._cloud = gaussians
        if cameras is None:
            # reference path: COLMAP text model + trained point_cloud.ply on disk (renderer_utils.py:127-216)
            from .io import load_reference_scene

            cameras, baseline, self._cloud, self.poses, self.sorted_camera_indices = load_reference_scene(
                base_dir, colmap_dir, args, splatting)
        self.cameras = cameras
        self.baseline = baseline
        self.left_cameras = [c["left"] for c in self.cameras]
        print(f"num views: {len(self.cameras)}")
        print(f"baseline: {self.baseline}")
        if output_dir_root is not None and getattr(args, "renderer_save_json", True):  # argument_utils.py:63 default
            self.save_camera_data()
        self.write_images = output_dir_root is not None
        # the library default (rasterizer.DEFAULT_FLAGS): ex2.approx blend in the table kernel, parity-tested against the
        # reference rasterizer at C1..C4; False selects the full-precision expf kernel (rasterizer.EXACT_EXP_FLAGS)
        self.fast_exp = True
        # render the left and the right eye on two side streams (each with its own scratch) so that the
        # small latency-bound binning kernels of one eye overlap the other eye's blend kernel
        self.overlap_eyes = True
        # how many stereo pairs may be in flight at once (stream sets); GSB_PAIRS_IN_FLIGHT overrides (A/B switch)
        self.pairs_in_flight = int(os.environ.get("GSB_PAIRS_IN_FLIGHT", DEFAULT_PAIRS_IN_FLIGHT))
        self.copy_streams = bool(int(os.environ.get("GSB_COPY_STREAMS", DEFAULT_COPY_STREAMS)))
        self.spare_buffer_sets = max(0, int(os.environ.get("GSB_SPARE_BUFFER_SETS", DEFAULT_SPARE_BUFFER_SETS)))
        self.keep_frames = False
        self._frames = {}
        self._ready = False

    @classmethod
    def from_scene(cls, cameras, baseline, gaussians, output_dir_root=None, args=None, device="cuda"):
        return cls(None, None, output_dir_root, args, device=device, cameras=cameras, baseline=baseline, gaussians=gaussians)

    def __len__(self):
        return len(self.cameras)

    def render_folder_name(self, render_number):
        return os.path.join(self.output_dir_root or ".", f"{render_number:03}")

    def save_camera_data(self):
        """renderer_utils.py:298-314"""
        import copy
        import json

        os.makedirs(self.output_dir_root, exist_ok=True)
        out = copy.deepcopy(self.cameras)
        for pair in out:
            for side in ("left", "right"):
                pair[side]["intrinsic"] = np.asarray(pair[side]["intrinsic"]).tolist()
                pair[side]["extrinsic"] = np.asarray(pair[side]["extrinsic"]).tolist()
        with open(os.path.join(self.output_dir_root, "camera_data.json"), "w") as f:
            json.dump(out, f, indent=4)

    # ------------------------------------------------------------------------------------------
    def prepare_renderer(self):
        """Upload the Gaussian cloud and every camera once (reference: renderer_utils.py:316-361)."""
        dev = torch.device(self.device)
        if dev.type != "cuda":
            raise RuntimeError("Renderer needs a CUDA device (gs2mesh_b200 has no CPU path)")
        g = self._cloud
        if g is None:
            raise RuntimeError("Renderer has no Gaussian cloud")
        up = lambda a: torch.as_tensor(np.ascontiguousarray(a, dtype=np.float32)).to(dev)
        self.means3D = up(g.xyz)
        self.shs = up(g.features)  # [P,16,3] == cat(features_dc, features_rest) (gaussian_model.py:107-111)
        self.opacity = up(g.opacity).reshape(-1)
        self.scales = up(g.scaling)
        self.rotations = up(g.rotation)
        self.sh_degree = int(g.sh_degree)
        bg = [1, 1, 1] if self.white_background else [0, 0, 0]  # renderer_utils.py:359
        self.background = torch.tensor(bg, dtype=torch.float32, device=dev)
        # camera table: [n_views, 2 (left,right), 36] floats
        recs = np.zeros((len(self.cameras), 2, cam.CAMERA_RECORD_FLOATS), dtype=np.float32)
        self._views = []
        for i, pair in enumerate(self.cameras):
            vts = []
            for s, side in enumerate(("left", "right")):  # dict order of the reference: left then right (:378)
                vt = cam.view_transforms_from_camera(pair[side])
                recs[i, s] = vt.packed()
                vts.append(vt)
            self._views.append(vts)
        self._camera_table = torch.as_tensor(recs).to(dev)
        # One depth sort can serve both eyes of a rig when every Gaussian has the same view depth in both, i.e. when the z
        # rows of the two view matrices are bitwise equal (same rotation, translation along the camera x axis).  The right
        # camera's rotation goes through a float32 Euler round trip (renderer_utils.py:186-196), which moves an entry by
        # one ulp in about one rig of five: those pairs keep one depth sort per eye.
        zrow = recs[:, :, [2, 6, 10, 14]].view(np.uint32)
        self._shared_depth = [bool(np.array_equal(zrow[i, 0], zrow[i, 1])) for i in range(len(self.cameras))]
        self._bufs = {}
        # per-(view, side) rasterizer status words, written by the GPU straight into pinned host memory
        self._status = torch.zeros(len(self.cameras), 2, 4, dtype=torch.int64).pin_memory()
        self._min_instances = 0
        # the block of the synchronous single-view calls; the serial pair path (both eyes on the caller's stream) uses it
        # for its left eye, since both only ever run on the caller's stream
        self._view_block = rast.Scratch(dev)
        self._serial_blocks = (self._view_block, rast.Scratch(dev))
        self._ready = True
        self.calibrate_capacity()

    def calibrate_capacity(self, sample_views=None):
        """Size the binning scratch once so that the hot loop can run without ever waiting for the GPU (the reference
        re-sizes -- and blocks -- inside every frame, rasterizer_impl.cu:281-285).  By default EVERY view of the rig is
        rendered once (instance counts are deterministic per camera), so a frame of this camera set cannot outgrow the
        scratch; `sample_views=k` looks at k evenly spaced views only (then an overflowing frame is caught by its status
        word and re-rendered, see render_image_pair)."""
        n = len(self.cameras)
        if sample_views is None or sample_views >= n:
            views = range(n)
        else:
            views = sorted(set(int(round(k * (n - 1) / max(sample_views - 1, 1))) for k in range(sample_views)))
        counts = [self.render_view(i, s, want_counts=True)["counts"] for i in views for s in range(2)]  # grow-and-redo renders
        worst = int(torch.stack(counts)[:, 0].max().item()) if counts else 0
        self._min_instances = rast.capacity_for(worst)

    def check_status(self, views=None):
        """After a synchronisation: raise if any asynchronously rendered frame is invalid (binning scratch too small, or a
        shared depth order claimed for eyes whose depths differ).  render_image_pair repairs such frames itself on every
        path that synchronises; this check is for callers of the pure device path (to_host=False, wait=False)."""
        st = self._status if views is None else self._status[list(views)]
        bad = ((st[..., 2] != 0) | (st[..., 3] != 0)).nonzero()
        if len(bad):
            need = int(st[..., 0].max().item())
            self._min_instances = max(self._min_instances, rast.capacity_for(need))
            raise RuntimeError(f"{len(bad)} frame(s) are invalid (needed up to {need} instances of binning scratch); "
                               "capacity has been raised, render them again")

    def _frame_ok(self, camera_number):
        """Status words of one pair after a synchronisation; repairs the renderer's settings if the pair must be redone."""
        st = self._status[camera_number]
        ok = True
        if bool((st[:, 2] != 0).any()):
            self._min_instances = max(self._min_instances, rast.capacity_for(int(st[:, 0].max().item())))
            ok = False
        if bool((st[:, 3] != 0).any()):
            self._shared_depth[camera_number] = False
            ok = False
        return ok

    def _buffers(self, w, h, parity=0):
        key = (w, h, parity)
        if key not in self._bufs:
            dev = self._camera_table.device
            f32 = dict(dtype=torch.float32, device=dev)
            self._bufs[key] = dict(
                color=[torch.empty(3, h, w, **f32) for _ in range(2)],
                u8=[torch.empty(h, w, 3, dtype=torch.uint8, device=dev) for _ in range(2)],
                depth=torch.empty(h, w, **f32), final_T=torch.empty(h, w, **f32),
                host_u8=[torch.empty(h, w, 3, dtype=torch.uint8).pin_memory() for _ in range(2)],
                host_depth=torch.empty(h, w, dtype=torch.float32).pin_memory(),
            )
        return self._bufs[key]

    def render_view(self, camera_number, side, *, want_depth=False, out_color=None, out_depth=None, out_final_T=None,
                    flags=None, want_counts=False, async_mode=False, scratch=None):
        """One forward rasterization of view `camera_number`, side 0 (left) / 1 (right), on the current stream.  A
        synchronous call without `scratch` uses the renderer's single-view block; an asynchronous one needs its own."""
        if not self._ready:
            raise RuntimeError("call prepare_renderer() first")
        if flags is None:
            flags = rast.DEFAULT_FLAGS if self.fast_exp else rast.EXACT_EXP_FLAGS
        vt = self._views[camera_number][side]
        rec = self._camera_table[camera_number, side]
        return rast.rasterize_forward(
            means3D=self.means3D, opacities=self.opacity, viewmatrix=rec[0:16], projmatrix=rec[16:32], campos=rec[32:35],
            bg=self.background, width=vt.width, height=vt.height, tan_fovx=vt.tan_fovx, tan_fovy=vt.tan_fovy, shs=self.shs,
            scales=self.scales, rotations=self.rotations, sh_degree=self.sh_degree, scale_modifier=1.0, flags=flags,
            want_depth=want_depth, want_final_T=want_depth, want_radii=False, want_counts=want_counts,
            out_color=out_color, out_depth=out_depth, out_final_T=out_final_T, async_mode=async_mode,
            counts_out=self._status[camera_number, side] if async_mode else None, min_instances=self._min_instances,
            scratch=scratch if scratch is not None or async_mode else self._view_block)

    def _enqueue_pair(self, camera_number, b, streams):
        """Both eyes of one view into buffer set `b`: rasterize (+ u8 conversion) on the _StreamSet `streams`."""
        mode = os.environ.get("GSB_PAIR_MODE", "fused")  # A/B switch: fused | noshare (fused preprocess, two depth sorts) | separate
        flags = rast.DEFAULT_FLAGS if self.fast_exp else rast.EXACT_EXP_FLAGS
        self._status[camera_number].zero_()
        if mode == "separate":
            for s in range(2):
                with torch.cuda.stream(streams[s]):
                    self.render_view(camera_number, s, want_depth=(s == 0), out_color=b["color"][s],
                                     out_depth=b["depth"] if s == 0 else None, out_final_T=b["final_T"] if s == 0 else None,
                                     async_mode=True, scratch=streams.scratch[s])
        else:
            eyes = []
            for s in range(2):
                vt = self._views[camera_number][s]
                rec = self._camera_table[camera_number, s]
                eyes.append(dict(viewmatrix=rec[0:16], projmatrix=rec[16:32], campos=rec[32:35], tan_fovx=vt.tan_fovx,
                                 tan_fovy=vt.tan_fovy, out_color=b["color"][s], out_depth=b["depth"] if s == 0 else None,
                                 out_final_T=b["final_T"] if s == 0 else None, counts_out=self._status[camera_number, s]))
            vt = self._views[camera_number][0]
            rast.rasterize_forward_pair(means3D=self.means3D, opacities=self.opacity, shs=self.shs, scales=self.scales,
                                        rotations=self.rotations, sh_degree=self.sh_degree, bg=self.background, width=vt.width,
                                        height=vt.height, eyes=eyes, streams=streams, scratch=streams.scratch, flags=flags,
                                        shared_depth=self._shared_depth[camera_number] and mode != "noshare",
                                        min_instances=self._min_instances)
        for s in range(2):
            with torch.cuda.stream(streams[s]):
                rast.image_to_u8(b["color"][s], out=b["u8"][s])

    def render_image_pair(self, camera_number, visualize=False, *, to_host: Optional[bool] = None, wait: bool = True):
        """Render the stereo-aligned left/right pair of view `camera_number`
        (reference: renderer_utils.py:363-395).  Returns a dict of DEVICE tensors
        (left/right float CHW, left_u8/right_u8 HWC, depth = left sum(z*alpha*T), final_T) and, when
        `to_host` (default: whenever PNGs are written), pinned host copies `host_left_u8`,
        `host_right_u8`.  With `wait=False` the call only enqueues: `result["ready"].synchronize()` waits for the pair
        (lets the caller overlap the next pair's rendering with the host-side consumption of this one).

        Both eyes go through ONE `gsb_raster_forward_pair` call: the Gaussian parameters are read once, and -- for rigs whose
        eyes see every Gaussian at the same view depth -- depth-sorted once.

        A frame whose binning scratch turns out too small is re-rendered transparently wherever the call (or the handle's
        synchronize()) waits for the GPU anyway; prepare_renderer() sizes the scratch from every view of the rig, so the
        pure device path (to_host=False) cannot overflow for this camera set.

        Buffer rotation: the returned tensors belong to one of pairs_in_flight + 2 buffer sets.  The tensors of call n
        stay valid for work enqueued on the CALLER'S CURRENT STREAM until call n + pairs_in_flight + 1 is entered (the
        renders that overwrite them wait for an event recorded on that stream at that moment); consumers on other
        streams must order themselves (e.g. wait on an event recorded after the call)."""
        with torch.no_grad():
            vt = self._views[camera_number][0]
            dev = self._camera_table.device
            main = torch.cuda.current_stream(dev)
            to_host = self.write_images if to_host is None else to_host
            if self.write_images:
                to_host = True  # PNGs are written from the pinned host copies
            cstreams = None  # streams of the D2H copies, when they do not ride on the render streams
            if self.overlap_eyes:
                self._call_index = getattr(self, "_call_index", -1) + 1
                depth = max(1, int(self.pairs_in_flight))
                spare = int(self.spare_buffer_sets)
                nslots = depth + 2 + spare
                slot = self._call_index % nslots
                if not hasattr(self, "_stream_sets") or len(self._stream_sets) != depth:
                    # `pairs_in_flight` sets of (left, right) streams, used round-robin: consecutive pairs run on
                    # different stream sets (each with its own scratch blocks), so pair n+1's latency-bound binning
                    # kernels fill the gaps of pair n's blend kernels
                    self._stream_sets = [_StreamSet([torch.cuda.Stream(dev), torch.cuda.Stream(dev)],
                                                    (rast.Scratch(dev), rast.Scratch(dev))) for _ in range(depth)]
                if not hasattr(self, "_entry_events") or len(self._entry_events) != nslots:
                    main.synchronize()  # (re)configuration only: nothing may still use the old rotation
                    self._call_index = 0
                    slot = 0
                    self._entry_events = [None] * nslots
                    self._slot_done = [[] for _ in range(nslots)]
                b = self._buffers(vt.width, vt.height, slot)
                entry = torch.cuda.Event()
                entry.record(main)
                # everything that read this buffer set (handed out nslots calls ago, valid until call
                # c - nslots + depth + 1 = c - 1 - spare was entered) was enqueued on the caller's stream before that entry
                gate = self._entry_events[(self._call_index - 1 - spare) % nslots] if self._call_index > spare else None
                self._entry_events[slot] = entry
                streams = self._stream_sets[self._call_index % depth]
                if self.copy_streams and to_host:
                    if not hasattr(self, "_copy_streams") or len(self._copy_streams) != depth:
                        self._copy_streams = [[torch.cuda.Stream(dev), torch.cuda.Stream(dev)] for _ in range(depth)]
                    cstreams = self._copy_streams[self._call_index % depth]
                for st in streams:
                    if gate is not None:
                        st.wait_event(gate)
                    else:
                        st.wait_stream(main)
                    for done in self._slot_done[slot]:  # the renders that last wrote this buffer set (another stream set)
                        st.wait_event(done)
            else:
                b = self._buffers(vt.width, vt.height)
                streams = _StreamSet([main, main], self._serial_blocks)

            # the streams whose completion means "this pair is done": the copy streams when the frames travel on their own
            # streams (each copy is ordered behind everything its eye's render stream holds at that point), else the render streams
            tails = streams if cstreams is None else cstreams

            def enqueue():
                self._enqueue_pair(camera_number, b, streams)
                if to_host:
                    for s in range(2):
                        if cstreams is not None:
                            cstreams[s].wait_stream(streams[s])
                        with torch.cuda.stream(tails[s]):
                            b["host_u8"][s].copy_(b["u8"][s], non_blocking=True)

            def redo_if_invalid():
                """Called after the pair's streams have been waited for: grow the scratch / drop the shared depth order and
                render the pair again, synchronously, until its status words are clean."""
                for _ in range(4):
                    if self._frame_ok(camera_number):
                        return
                    enqueue()
                    for st in tails:
                        st.synchronize()
                self.check_status([camera_number])

            enqueue()
            result = dict(left=b["color"][0], right=b["color"][1], left_u8=b["u8"][0], right_u8=b["u8"][1],
                          depth=b["depth"], final_T=b["final_T"])
            if self.overlap_eyes:
                self._slot_done[slot] = [st.record_event() for st in tails]
            asynchronous = to_host and not wait and not self.write_images and not self.keep_frames and self.overlap_eyes
            if self.overlap_eyes and not asynchronous:
                for st in tails:
                    main.wait_stream(st)  # device-side dependency only: later work on the caller's stream sees both eyes
            if to_host:
                result["host_left_u8"], result["host_right_u8"] = b["host_u8"]
                if asynchronous:
                    result["ready"] = _PairReady([st.record_event() for st in tails], redo_if_invalid)
                else:
                    main.synchronize()
                    redo_if_invalid()
                    result["ready"] = _PairReady([])
            elif self.keep_frames:
                main.synchronize()
                redo_if_invalid()
            if self.write_images:
                import cv2

                out_dir = self.render_folder_name(camera_number)
                os.makedirs(out_dir, exist_ok=True)
                for s, name in enumerate(("left", "right")):
                    cv2.imwrite(os.path.join(out_dir, f"{name}.png"), cv2.cvtColor(b["host_u8"][s].numpy(), cv2.COLOR_RGB2BGR))
            if self.keep_frames:  # in-memory hand-off to the TSDF stage (the caller's stream already waits for both eyes)
                self._frames[camera_number] = dict(left_u8=b["u8"][0].clone(), right_u8=b["u8"][1].clone(),
                                                   depth=self.expected_depth(b["depth"], b["final_T"]))
            return result

    # north_star alias
    def render(self, camera_number, **kw):
        return self.render_image_pair(camera_number, **kw)

    @staticmethod
    def expected_depth(depth_sum, final_T, alpha_min=0.5):
        """Expected depth D/alpha where alpha = 1 - T > alpha_min, else 0 (SURVEY 8(d))."""
        alpha = 1.0 - final_T
        return torch.where(alpha > alpha_min, depth_sum / alpha.clamp_min(1e-12), torch.zeros_like(depth_sum))

    def get_frame(self, camera_number):
        return self._frames.get(camera_number)

    # ---- in-memory hand-off to / from the stereo stage (SURVEY 8(f) rank 2) ---------------------------------------------
    def stereo_inputs(self, camera_number, device=None):
        """What `Stereo.run` builds by re-reading left.png / right.png right after render_image_pair
        (stereo_utils.py:68-80,100-103): two float tensors [1,3,H,W] holding the uint8-quantised RGB frames -- bit for bit
        the values `load_image` returns, without the PNG encode / file / decode round trip.  Renders the pair if it is not
        in the frame cache (`keep_frames`)."""
        f = self._frames.get(camera_number)
        if f is None:
            keep, self.keep_frames = self.keep_frames, True
            try:
                self.render_image_pair(camera_number)
            finally:
                self.keep_frames = keep
            f = self._frames[camera_number]
            if not keep:
                self._frames.pop(camera_number, None)
        to = lambda u8: u8.permute(2, 0, 1).float()[None].to(device or u8.device)
        return to(f["left_u8"]), to(f["right_u8"])

    def put_stereo_outputs(self, camera_number, depth, occlusion_mask=None):
        """The other direction: the stereo stage's depth (= fx * baseline / disparity_LR, stereo_utils.py:133) and
        left-right occlusion mask (:132) for one view, as tensors / arrays, instead of depth.npy / occlusion_mask.npy on disk
        (stereo_utils.py:135-137 -> tsdf_utils.py:67,79-80).  TSDF.run() picks them up from the frame cache."""
        f = self._frames.setdefault(camera_number, {})
        f["depth"] = depth
        if occlusion_mask is not None:
            f["occlusion_mask"] = occlusion_mask
