"""Stereo stage: GPU replacement for gs2mesh_utils/stereo_utils.py `Stereo` (reference), same class surface:

    Stereo(base_dir, renderer, args, device='cuda')
    .run(start=0)  .get_occlusion_mask(L2R, R2L, threshold)  .load_image(imfile)
    .base_dir  .renderer  .args  .model_name  .device  .disparity_signs  .model  .model_args

The disparity model (DLNR) stays the caller's torch module, built exactly as stereo_utils.py:43-63 builds it.  Around it,
the reference reads the rendered pair back from PNG files, pads it, and computes the occlusion mask and the depth in numpy
on the host (stereo_utils.py:100-140).  Here the pair comes from the renderer's frame cache, and three kernels of
include/gs2mesh_b200.h (gs2mesh_b200/csrc/gsb_stereo.cu) do the rest on the device:
  gsb_stereo_pack_inputs      the model's four padded (and flipped) inputs, from the uint8 frames
  gsb_stereo_disparities      sign * the model's outputs, LR cropped, RL flipped back and NOT cropped (SURVEY Appendix A)
  gsb_stereo_occlusion_depth  get_occlusion_mask and depth = fx*B / disparity_LR in numpy's dtypes (DESIGN.md section 7c)
Depth and occlusion mask go to the TSDF stage through `Renderer.put_stereo_outputs`; the reference's files are still
written when the renderer writes images.  There is no CPU fallback.
"""
from __future__ import annotations

import os
import sys
from argparse import Namespace

import numpy as np
import torch

from . import _lib
from ._lib import ptr

DISPARITY_SIGNS = {"DLNR_Middlebury": -1, "DLNR_SceneFlow": -1}  # stereo_utils.py:41
DIVIS_BY = 32  # InputPadder(image1.shape, divis_by=32), stereo_utils.py:107
MAX_WIDTH, MAX_HEIGHT = 65536, 32768  # GSB_TSDF_MAX_WIDTH / _HEIGHT


def padding(height, width):
    """DLNR's InputPadder(dims, divis_by=32) in its default 'sintel' mode: [left, right, top, bottom]."""
    ph = ((height // DIVIS_BY + 1) * DIVIS_BY - height) % DIVIS_BY
    pw = ((width // DIVIS_BY + 1) * DIVIS_BY - width) % DIVIS_BY
    return [pw // 2, pw - pw // 2, ph // 2, ph - ph // 2]


def padded_shape(height, width):
    l, r, t, b = padding(height, width)
    return height + t + b, width + l + r


def _check_frame(height, width):
    if not (1 <= width <= MAX_WIDTH and 1 <= height <= MAX_HEIGHT):
        raise ValueError(f"stereo frames must be 1..{MAX_WIDTH} wide and 1..{MAX_HEIGHT} high, not {width}x{height}")


def _cuda(t, dtype, name):
    if not isinstance(t, torch.Tensor):
        t = torch.as_tensor(np.ascontiguousarray(t))
    if t.dtype != dtype:
        raise TypeError(f"{name} must be {dtype}, not {t.dtype}")
    if not t.is_cuda:
        t = t.to("cuda")
    return t.contiguous()


def pack_inputs(left_u8, right_u8):
    """The model inputs of stereo_utils.py:106-116 from two uint8 [H,W,3] frames: float [4,3,Hp,Wp] holding pad(left),
    pad(right), flip_x(pad(right)), flip_x(pad(left)) (replicate padding, float(u8)).  Rows [0:1],[1:2] are the LR pair,
    [2:3],[3:4] the RL pair."""
    left, right = _cuda(left_u8, torch.uint8, "left"), _cuda(right_u8, torch.uint8, "right")
    if left.dim() != 3 or left.shape[2] != 3 or left.shape != right.shape or left.device != right.device:
        raise ValueError(f"frames must be equal uint8 [H,W,3] tensors on one device, not {tuple(left.shape)} and {tuple(right.shape)}")
    H, W = int(left.shape[0]), int(left.shape[1])
    _check_frame(H, W)
    Hp, Wp = padded_shape(H, W)
    out = torch.empty(4, 3, Hp, Wp, dtype=torch.float32, device=left.device)
    with torch.cuda.device(left.device):
        _lib.check(_lib.lib().gsb_stereo_pack_inputs(ptr(left), ptr(right), W, H, ptr(out), _lib.stream(left.device)))
    return out


def disparities(flow_lr, flow_rl, height, width, sign):
    """sign * the model's full-resolution outputs (each [1,1,Hp,Wp] float32): (disparity_LR float [H,W], cropped to the
    frame; disparity_RL float [Hp,Wp], flipped back and not cropped, as the reference's RL padder has no pad)."""
    _check_frame(height, width)
    Hp, Wp = padded_shape(height, width)
    fl, fr = _cuda(flow_lr, torch.float32, "flow_lr"), _cuda(flow_rl, torch.float32, "flow_rl")
    for name, f in (("flow_lr", fl), ("flow_rl", fr)):
        if f.numel() != Hp * Wp or f.shape[-2:] != (Hp, Wp):
            raise ValueError(f"{name} must be [1,1,{Hp},{Wp}] for a {width}x{height} frame, not {tuple(f.shape)}")
    if fl.device != fr.device:
        raise ValueError("flow_lr and flow_rl must be on one device")
    d_lr = torch.empty(height, width, dtype=torch.float32, device=fl.device)
    d_rl = torch.empty(Hp, Wp, dtype=torch.float32, device=fl.device)
    with torch.cuda.device(fl.device):
        _lib.check(_lib.lib().gsb_stereo_disparities(ptr(fl), ptr(fr), width, height, float(sign), ptr(d_lr), ptr(d_rl),
                                                     _lib.stream(fl.device)))
    return d_lr, d_rl


def depth_numerator(fx, baseline):
    """`fx * baseline` as stereo_utils.py:133 forms it (double), rounded once to float32: NumPy 1.x divides a float32 array
    by a float64 scalar in float32 (value-based casting).  A product outside the float32 range would make NumPy 1.x divide
    in float64 instead, so it is refused."""
    with np.errstate(over="ignore"):
        num = np.float32(fx * baseline)
    if not np.isfinite(num):
        raise ValueError(f"fx * baseline = {fx * baseline!r} does not fit a float32")
    return num


def occlusion_depth(disp_lr, disp_rl, threshold, numerator=None, *, want_mask=True):
    """get_occlusion_mask(disp_lr, disp_rl, threshold) (stereo_utils.py:149-179) and, when `numerator` (depth_numerator) is
    given, depth = numerator / disp_lr (:133), on the device.  disp_lr: float32 [H,W]; disp_rl: float32 with at least H rows
    and W columns, read at row y, column xc.  Returns (visible bool [H,W] or None, depth float32 [H,W] or None)."""
    dl = _cuda(disp_lr, torch.float32, "disparity_LR")
    if dl.dim() != 2:
        raise ValueError(f"disparity_LR must be [H,W], not {tuple(dl.shape)}")
    H, W = int(dl.shape[0]), int(dl.shape[1])
    _check_frame(H, W)
    dr = None
    if want_mask:
        dr = _cuda(disp_rl, torch.float32, "disparity_RL").to(dl.device)
        if dr.dim() != 2:
            raise ValueError(f"disparity_RL must be 2-D, not {tuple(dr.shape)}")
        if dr.shape[0] < H or dr.shape[1] < W:  # numpy's R2L[y, xc] would index past its end
            raise IndexError(f"disparity_RL {tuple(dr.shape)} is smaller than disparity_LR {(H, W)}")
    visible = torch.empty(H, W, dtype=torch.bool, device=dl.device) if want_mask else None
    depth = torch.empty(H, W, dtype=torch.float32, device=dl.device) if numerator is not None else None
    if visible is None and depth is None:
        return None, None
    with torch.cuda.device(dl.device):
        _lib.check(_lib.lib().gsb_stereo_occlusion_depth(
            ptr(dl), ptr(dr), W, H, int(dr.shape[1]) if dr is not None else 0, float(threshold),
            float(numerator) if numerator is not None else 0.0, ptr(visible), ptr(depth), _lib.stream(dl.device)))
    return visible, depth


def get_shading(img, shading_eps):
    """transformation_utils.py:226-240: 1 / sqrt(gX^2 + gY^2 + eps) of cv2's 3x3 Sobel derivatives, in float64."""
    import cv2

    gX = cv2.Sobel(img, cv2.CV_64F, 1, 0)
    gY = cv2.Sobel(img, cv2.CV_64F, 0, 1)
    return 1 / (np.sqrt((gX ** 2) + (gY ** 2) + shading_eps))


class Stereo:
    """Stage class with the reference's surface (gs2mesh_utils/stereo_utils.py:25-179)."""

    def __init__(self, base_dir, renderer, args, device="cuda"):
        self.base_dir = base_dir
        self.renderer = renderer
        self.args = args
        self.model_name = self.args.stereo_model
        self.device = device
        self.disparity_signs = dict(DISPARITY_SIGNS)
        if self.model_name not in self.disparity_signs:
            raise ValueError(f"stereo model {self.model_name!r} is not supported (supported: {sorted(self.disparity_signs)})")
        dlnr_dir = os.path.abspath(os.path.join(self.base_dir, "third_party", "DLNR"))
        if dlnr_dir not in sys.path:
            sys.path.append(dlnr_dir)
        from core.dlnr import DLNR

        self.model_args = Namespace(corr_implementation="reg", corr_levels=4, corr_radius=4, dataset="things",
                                    hidden_dims=[128, 128, 128], mixed_precision=True, n_downsample=2, n_gru_layers=3,
                                    restore_ckpt=os.path.join(self.base_dir, "third_party", "DLNR", "pretrained",
                                                              f"{self.model_name}.pth"),
                                    shared_backbone=False, slow_fast_gru=False, valid_iters=10)
        model = torch.nn.DataParallel(DLNR(self.model_args), device_ids=[0])
        model.load_state_dict(torch.load(self.model_args.restore_ckpt, map_location="cpu"))
        model = model.module
        model.to(self.device)
        model.eval()
        self.model = model

    def load_image(self, imfile):
        """stereo_utils.py:68-80: an RGB image file as a float [1,3,H,W] tensor on the stage's device."""
        from PIL import Image

        img = np.array(Image.open(imfile)).astype(np.uint8)
        img = torch.from_numpy(img).permute(2, 0, 1).float()
        return img[None].to(self.device)

    def get_occlusion_mask(self, L2R_disparity, R2L_disparity, occlusion_threshold):
        """stereo_utils.py:149-179 on the GPU: numpy bool [H,W], True where the pixel is visible in both directions.
        Disparities are float32 (float16 is widened exactly); an R2L smaller than L2R raises IndexError."""
        L2R, R2L = (torch.as_tensor(np.asarray(d)) if not isinstance(d, torch.Tensor) else d for d in (L2R_disparity, R2L_disparity))
        L2R, R2L = (d.float() if d.dtype == torch.float16 else d for d in (L2R, R2L))
        visible, _ = occlusion_depth(L2R, R2L, occlusion_threshold)
        return visible.cpu().numpy()

    def run(self, start=0, visualize=False):
        """stereo_utils.py:82-147 for every view from `start`: render the pair into the frame cache, run the model LR and
        RL (warm-started like the reference when args.stereo_warm), then hand depth and occlusion mask to the TSDF stage
        with renderer.put_stereo_outputs.  When the renderer writes images, out_<model>/ gets the reference's files."""
        if visualize:
            raise NotImplementedError("Stereo.run(visualize=True): the visualisation helpers are not provided")
        r = self.renderer
        sign = self.disparity_signs[self.model_name]
        iters = self.model_args.valid_iters
        warm = bool(self.args.stereo_warm)
        threshold = float(self.args.stereo_occlusion_threshold)
        keep = r.keep_frames
        r.keep_frames = True  # TSDF.run then reads frames, depth and occlusion mask from memory
        try:
            with torch.no_grad():
                prev_flows = {"LR": None, "RL": None}
                for camera_number, left_camera in enumerate(r.left_cameras):
                    if camera_number < start:
                        continue
                    r.render_image_pair(camera_number, visualize=False)
                    frame = r.get_frame(camera_number)
                    H, W = int(frame["left_u8"].shape[0]), int(frame["left_u8"].shape[1])
                    block = pack_inputs(frame["left_u8"], frame["right_u8"])
                    flows = {}
                    for direction, (a, b) in (("LR", (0, 1)), ("RL", (2, 3))):
                        prev_flow, flows[direction] = self.model(block[a:a + 1], block[b:b + 1], iters=iters, test_mode=True,
                                                                 flow_init=prev_flows[direction] if warm else None)
                        # the reference keeps the RL flow flipped back, and feeds it so to the next flipped pair
                        prev_flows[direction] = torch.flip(prev_flow, dims=[3]) if direction == "RL" else prev_flow
                    d_lr, d_rl = disparities(flows["LR"], flows["RL"], H, W, sign)
                    visible, depth = occlusion_depth(d_lr, d_rl, threshold, depth_numerator(left_camera["fx"], r.baseline))
                    r.put_stereo_outputs(camera_number, depth, visible)
                    if r.write_images:
                        self._write_outputs(camera_number, d_lr, d_rl, visible, depth)
        finally:
            r.keep_frames = keep

    def _write_outputs(self, camera_number, d_lr, d_rl, visible, depth):
        """The files of stereo_utils.py:126-140, same names, shapes and dtypes; the matplotlib images only when
        matplotlib is installed."""
        import cv2

        out = os.path.join(self.renderer.render_folder_name(camera_number), f"out_{self.model_name}")
        os.makedirs(out, exist_ok=True)
        arrays = {"disparity_LR": d_lr.cpu().numpy(), "disparity_RL": d_rl.cpu().numpy(),
                  "occlusion_mask": visible.cpu().numpy(), "depth": depth.cpu().numpy()}
        for name, a in arrays.items():
            np.save(os.path.join(out, f"{name}.npy"), a)
        try:
            import matplotlib.pyplot as plt
        except ImportError:
            plt = None
        if plt is not None:
            for direction in ("LR", "RL"):
                plt.imsave(os.path.join(out, f"disparity_{direction}.png"), arrays[f"disparity_{direction}"], cmap="jet")
            plt.imsave(os.path.join(out, "occlusion_mask.png"), arrays["occlusion_mask"])
        cv2.imwrite(os.path.join(out, "depth.png"), arrays["depth"])
        cv2.imwrite(os.path.join(out, "shading.png"), get_shading(arrays["depth"], self.args.stereo_shading_eps))
