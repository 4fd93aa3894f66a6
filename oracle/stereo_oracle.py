"""CPU restatement of the stereo stage's arithmetic (test infrastructure only; numpy).

Written from the reference's behaviour (file:line in the gs2mesh sources), with every dtype made explicit so that the
result does not depend on the installed NumPy version:
  third_party/DLNR/core/utils/utils.py InputPadder   divis_by=32, 'sintel' split, replicate padding
  gs2mesh_utils/stereo_utils.py:106-124             model inputs, RL flip, crop (LR) / no crop (RL), sign
  gs2mesh_utils/stereo_utils.py:149-179             occlusion mask
  gs2mesh_utils/stereo_utils.py:133                 depth under NumPy 1.x value-based casting (float32 result)
"""
from __future__ import annotations

import numpy as np

INT32_MIN = -(2 ** 31)


def padding(height, width, divis_by=32):
    """[left, right, top, bottom] of InputPadder(dims, divis_by) in 'sintel' mode."""
    ph = ((height // divis_by + 1) * divis_by - height) % divis_by
    pw = ((width // divis_by + 1) * divis_by - width) % divis_by
    return [pw // 2, pw - pw // 2, ph // 2, ph - ph // 2]


def pack(left_u8, right_u8):
    """float32 [4,3,Hp,Wp]: pad(left), pad(right), flip_x(pad(right)), flip_x(pad(left)), replicate padding."""
    H, W = left_u8.shape[:2]
    l, r, t, b = padding(H, W)

    def pad(img):
        chw = np.asarray(img, np.uint8).transpose(2, 0, 1).astype(np.float32)
        return np.pad(chw, ((0, 0), (t, b), (l, r)), mode="edge")

    L, R = pad(left_u8), pad(right_u8)
    return np.stack([L, R, R[..., ::-1], L[..., ::-1]]).astype(np.float32)


def disparities(flow_lr, flow_rl, height, width, sign):
    """(float32 [H,W], float32 [Hp,Wp]): sign * flow_lr cropped to the frame, sign * flow_rl flipped in x, not cropped."""
    l, r, t, b = padding(height, width)
    s = np.float32(sign)
    fl = np.asarray(flow_lr, np.float32).reshape(height + t + b, width + l + r)
    fr = np.asarray(flow_rl, np.float32).reshape(fl.shape)
    return (s * fl[t:t + height, l:l + width]).astype(np.float32), (s * fr[:, ::-1]).astype(np.float32)


def trunc_int32(x):
    """x86 cvttsd2si of float64 values: truncation toward zero; NaN and results outside int32 give INT32_MIN."""
    x = np.asarray(x, np.float64)
    ok = (x > -2147483649.0) & (x < 2147483648.0)
    return np.where(ok, np.trunc(np.where(ok, x, 0.0)), INT32_MIN).astype(np.int64)


def occlusion_terms(L2R, R2L):
    """The mask's intermediates, each [H,W]: xp (int64 holding int32 values), the float64 reprojection xr and |x - clip(xr)|.
    R2L is read at row y, column clip(xp) of its own plane."""
    L2R = np.asarray(L2R, np.float32)
    R2L = np.asarray(R2L, np.float32)
    H, W = L2R.shape
    x = np.broadcast_to(np.arange(W, dtype=np.float64)[None, :], (H, W))
    y = np.broadcast_to(np.arange(H)[:, None], (H, W))
    xp = trunc_int32(x - L2R.astype(np.float64))
    xc = np.clip(xp, 0, W - 1)
    xr = xc.astype(np.float64) + R2L[y, xc].astype(np.float64)
    xrc = np.where(np.isnan(xr), xr, np.minimum(np.maximum(xr, 0.0), float(W - 1)))  # np.clip keeps NaN
    return xp, xr, np.abs(x - xrc)


def occlusion_mask(L2R, R2L, threshold):
    """bool [H,W], True = visible: not |x - clip(xr)| > threshold, and 0 <= xp < W."""
    xp, _, diff = occlusion_terms(L2R, R2L)
    with np.errstate(invalid="ignore"):
        occluded = diff > np.float64(threshold)
    return ~occluded & (xp >= 0) & (xp < diff.shape[1])


def depth(fx, baseline, L2R):
    """fx * baseline / L2R as NumPy 1.x evaluates it: the float64 scalar is rounded to float32, the division is float32."""
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        return np.float32(fx * baseline) / np.asarray(L2R, np.float32)


def depth_float64_route(fx, baseline, L2R):
    """What NumPy >= 2 gives for a float64 scalar (a float64 quotient), after tsdf_utils.py:88's astype(float32)."""
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        return (np.float64(fx * baseline) / np.asarray(L2R, np.float32).astype(np.float64)).astype(np.float32)
