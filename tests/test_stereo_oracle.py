"""CPU tests of the stereo stage's oracle (oracle/stereo_oracle.py): the occlusion mask against a scalar restatement in
Python floats, the padder against its formula, the model inputs against torch's pad and flip, and the depth dtype
decision (DESIGN.md section 7c)."""
import math
from argparse import Namespace

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from gs2mesh_b200 import stereo
from oracle import stereo_oracle as so
from tests import stereo_cases as sc


def scalar_mask(L2R, R2L, threshold):
    """get_occlusion_mask pixel by pixel with Python floats (IEEE double) and x86's int32 truncation rule."""
    H, W = L2R.shape
    out = np.zeros((H, W), bool)
    for y in range(H):
        for x in range(W):
            v = float(x) - float(L2R[y, x])
            if math.isnan(v) or math.isinf(v):
                xp = -2 ** 31
            else:
                xp = math.trunc(v)
                if not -2 ** 31 <= xp < 2 ** 31:
                    xp = -2 ** 31
            xc = min(max(xp, 0), W - 1)
            xr = float(xc) + float(R2L[y, xc])
            if not math.isnan(xr):
                xr = min(max(xr, 0.0), float(W - 1))
            diff = abs(float(x) - xr)
            out[y, x] = (not diff > threshold) and 0 <= xp < W
    return out


@pytest.mark.parametrize("H,W,rows,cols", [(12, 40, 12, 40), (9, 33, 32, 64), (20, 16, 32, 32)])
def test_oracle_mask_equals_scalar_restatement(H, W, rows, cols):
    L, R = sc.adversarial_disparities(H, W, rows, cols, seed=H)
    report = sc.case_report(L, R)
    assert all(report.values()), {k: v for k, v in report.items() if not v}
    for thr in sc.THRESHOLDS:
        got = so.occlusion_mask(L, R, thr)
        want = scalar_mask(L, R, thr)
        assert got.dtype == np.bool_ and got.shape == (H, W)
        np.testing.assert_array_equal(got, want, err_msg=f"threshold {thr}")


def test_fp64_subtraction_decides_truncation():
    """x - 1e-30 is x in float64 (truncates to x), and 1000 - 1e-5 is 999.99999 in float64 (truncates to 999) while the
    float32 difference would be 1000."""
    L = np.zeros((1, 1001), np.float32)
    L[0, 3] = 1e-30
    L[0, 1000] = 1e-5
    xp, _, _ = so.occlusion_terms(L, np.zeros_like(L))
    assert xp[0, 3] == 3 and xp[0, 1000] == 999
    assert np.float32(1000) - np.float32(1e-5) == np.float32(1000)
    assert so.trunc_int32([np.nan, 2.0 ** 31, -2.0 ** 31, -2.0 ** 31 - 0.5, -2.0 ** 31 - 1, -0.9, 0.9]).tolist() == \
        [-2 ** 31, -2 ** 31, -2 ** 31, -2 ** 31, -2 ** 31, 0, 0]


def _padder_formula(n):
    p = (32 - n % 32) % 32  # distance to the next multiple of 32
    return p // 2, p - p // 2


@pytest.mark.parametrize("extra", [(1200, 1600), (540, 960), (1080, 1920)])
def test_padder_matches_formula(extra):
    sizes = [(h, w) for h in range(1, 101) for w in range(1, 101)] + [extra]
    for h, w in sizes:
        l, r = _padder_formula(w)
        t, b = _padder_formula(h)
        assert so.padding(h, w) == [l, r, t, b] == stereo.padding(h, w), (h, w)
        assert stereo.padded_shape(h, w) == (h + t + b, w + l + r)
        assert (h + t + b) % 32 == 0 and (w + l + r) % 32 == 0
    assert so.padding(1200, 1600) == [0, 0, 8, 8]
    assert so.padding(304, 400) == [8, 8, 8, 8]


@pytest.mark.parametrize("H,W", [(1, 1), (1, 7), (7, 1), (31, 33), (32, 32), (33, 65)])
def test_pack_oracle_equals_torch_pad_and_flip(H, W):
    rng = np.random.default_rng(H * 100 + W)
    left, right = (rng.integers(0, 256, (H, W, 3), dtype=np.uint8) for _ in range(2))
    to = lambda u8: torch.from_numpy(u8).permute(2, 0, 1).float()[None]
    L, R = (F.pad(to(a), so.padding(H, W), mode="replicate") for a in (left, right))
    want = torch.cat([L, R, torch.flip(R, dims=[3]), torch.flip(L, dims=[3])]).numpy()
    got = so.pack(left, right)
    assert got.dtype == np.float32 and got.shape == want.shape
    np.testing.assert_array_equal(got, want)


def test_disparity_oracle_crop_and_flip():
    H, W = 30, 45
    l, r, t, b = so.padding(H, W)
    Hp, Wp = H + t + b, W + l + r
    fl = np.arange(Hp * Wp, dtype=np.float32).reshape(Hp, Wp)
    fr = -fl
    dl, dr = so.disparities(fl, fr, H, W, -1)
    assert dl.shape == (H, W) and dr.shape == (Hp, Wp)
    assert dl[0, 0] == -fl[t, l] and dl[H - 1, W - 1] == -fl[t + H - 1, l + W - 1]
    assert dr[0, 0] == fl[0, Wp - 1] and dr[Hp - 1, 0] == fl[Hp - 1, Wp - 1]


def test_depth_dtype_decision_matters():
    """fx * B / d with fx * B rounded to float32 (NumPy 1.x) differs from the float64 quotient rounded afterwards (NumPy >= 2
    with a float64 scalar) on a seeded case; both agree with an exact rational check of their own rounding."""
    from fractions import Fraction

    rng = np.random.default_rng(7)
    d = rng.uniform(0.5, 200, 100000).astype(np.float32)
    fx, B = 1440.0, 0.137
    a, b = so.depth(fx, B, d), so.depth_float64_route(fx, B, d)
    assert a.dtype == b.dtype == np.float32
    diff = a != b
    assert diff.any() and diff.mean() < 0.5
    assert np.abs(a.view(np.int32) - b.view(np.int32)).max() <= 1
    num = np.float32(fx * B)
    assert float(num) != fx * B
    for i in np.flatnonzero(diff)[:20]:
        q = Fraction(float(num)) / Fraction(float(d[i]))  # float32 division is the rounded exact quotient
        cands = np.array([a[i], b[i]], np.float32)
        errs = [abs(Fraction(float(c)) - q) for c in cands]
        assert errs[0] <= errs[1]


def test_depth_special_values():
    d = np.array([0.0, -0.0, 1e-45, -1e-45, np.nan, np.inf], np.float32)
    got = so.depth(1000.0, 0.1, d)
    assert np.isposinf(got[0]) and np.isneginf(got[1]) and np.isposinf(got[2]) and np.isneginf(got[3])
    assert np.isnan(got[4]) and got[5] == 0


def test_stereo_refuses_unsupported_model(tmp_path):
    args = Namespace(stereo_model="RAFT", stereo_warm=False, stereo_occlusion_threshold=3, stereo_shading_eps=1e-4)
    with pytest.raises(ValueError, match="not supported"):
        stereo.Stereo(str(tmp_path), None, args, device="cpu")


def test_depth_numerator_is_rounded_once():
    assert stereo.depth_numerator(1440.0, 0.137) == np.float32(1440.0 * 0.137)
    with pytest.raises(ValueError):
        stereo.depth_numerator(1e30, 1e30)


def test_entry_points_refuse_bad_frames_without_gpu(gsb_lib):
    """Frames beyond GSB_TSDF_MAX_WIDTH x GSB_TSDF_MAX_HEIGHT, empty frames and NULL buffers are refused before any launch."""
    from gs2mesh_b200 import _lib

    L = gsb_lib
    for w, h in ((65537, 4), (4, 32769), (0, 4), (4, 0)):
        assert L.gsb_stereo_pack_inputs(256, 256, w, h, 256, None) == _lib.GSB_ERR_INVALID
        assert L.gsb_stereo_disparities(256, 256, w, h, -1.0, 256, 256, None) == _lib.GSB_ERR_INVALID
        assert L.gsb_stereo_occlusion_depth(256, 256, w, h, max(w, 1), 3.0, 1.0, 256, 256, None) == _lib.GSB_ERR_INVALID
        assert b"frame" in L.gsb_last_error()
    assert L.gsb_stereo_pack_inputs(None, 256, 8, 8, 256, None) == _lib.GSB_ERR_INVALID
    assert L.gsb_stereo_disparities(256, 256, 8, 8, float("nan"), 256, 256, None) == _lib.GSB_ERR_INVALID
    assert L.gsb_stereo_occlusion_depth(256, 256, 8, 8, 7, 3.0, 1.0, 256, None, None) == _lib.GSB_ERR_INVALID  # stride < width
    assert L.gsb_stereo_occlusion_depth(256, None, 8, 8, 8, 3.0, 1.0, 256, None, None) == _lib.GSB_ERR_INVALID
    assert L.gsb_stereo_occlusion_depth(256, 256, 8, 8, 8, 3.0, 1.0, None, None, None) == _lib.GSB_ERR_INVALID
