"""Adversarial disparity fields for the stereo stage's occlusion mask and depth (shared by the CPU and GPU tests)."""
import numpy as np

from oracle import stereo_oracle as so

THRESHOLDS = (0.0, 2.5, 3.0)
SUBNORMAL = np.float32(1e-40)


def adversarial_disparities(H, W, rows_rl=None, cols_rl=None, seed=0):
    """(L2R float32 [H,W], R2L float32 [rows_rl, cols_rl]) with, at fixed pixels of every row: NaN, +-inf, +-0,
    subnormals, +-1e-30 and 1e-5 (where the float64 subtraction decides the truncation), xp = 0, -1, W-1 and W exactly,
    |d| >= 2^31, NaN read from R2L, and reprojection differences of exactly 0, 2.5 and 3.  Needs W >= 12."""
    rng = np.random.default_rng(seed)
    rows_rl = H if rows_rl is None else rows_rl
    cols_rl = W if cols_rl is None else cols_rl
    L = rng.uniform(-4, W / 3, (H, W)).astype(np.float32)
    L = np.where(rng.random((H, W)) < 0.3, np.round(rng.uniform(-4, W / 3, (H, W))), L).astype(np.float32)
    R = rng.uniform(-W / 3, 4, (rows_rl, cols_rl)).astype(np.float32)
    R = np.where(rng.random(R.shape) < 0.3, np.round(R), R).astype(np.float32)
    specials = [np.nan, np.inf, -np.inf, 0.0, -0.0, SUBNORMAL, -SUBNORMAL, 1e-30, -1e-30, 1e-5, 3e9, -3e9, 2.0 ** 31]
    for y in range(H):
        x0 = (y * 7) % max(W - len(specials), 1)
        for k, v in enumerate(specials):
            if x0 + k < W:
                L[y, x0 + k] = v
        # xp exactly 0, -1, W-1, W
        for x, xp in (((y * 3) % W, 0), ((y * 5 + 1) % W, -1), ((y * 11 + 2) % W, W - 1), ((y * 13 + 3) % W, W)):
            L[y, x] = np.float32(x - xp)
        # integer disparity D at x, R2L at the read column set for a difference of exactly 0, 2.5, 3 or a NaN
        x = W - 1 - (y % 4)
        D = min(3 + y % 5, x)
        L[y, x] = D
        R[y, x - D] = [D, D - 2.5, D - 3.0, np.nan][y % 4]  # xr = x - D + R = x, x - 2.5, x - 3, NaN
    return L.astype(np.float32), R.astype(np.float32)


def case_report(L2R, R2L):
    """Which of the adversarial situations the pair contains (names -> bool), from the oracle's intermediates."""
    xp, xr, diff = so.occlusion_terms(L2R, R2L)
    H, W = L2R.shape
    L = L2R
    in_range = (xp >= 0) & (xp < W)
    x = np.arange(W)[None, :]
    exact = x - L.astype(np.float64)
    return {
        "nan": bool(np.isnan(L).any()), "+inf": bool(np.isposinf(L).any()), "-inf": bool(np.isneginf(L).any()),
        "+0": bool(((L == 0) & ~np.signbit(L)).any()), "-0": bool(((L == 0) & np.signbit(L)).any()),
        "subnormal": bool(((L != 0) & (np.abs(L) < np.finfo(np.float32).tiny)).any()),
        "1e-30": bool((L == np.float32(1e-30)).any()),
        # the float64 difference is an integer although d != 0, so truncation keeps x instead of x - 1
        "fp64_subtraction_rounds": bool(((L > 0) & (L < 1e-4) & (exact == np.round(exact)) & (x > 0)).any()),
        "xp=0": bool((xp == 0).any()), "xp=-1": bool((xp == -1).any()), "xp=W-1": bool((xp == W - 1).any()),
        "xp=W": bool((xp == W).any()), "xp=INT32_MIN": bool((xp == so.INT32_MIN).any()),
        "nan_from_rl": bool((np.isnan(xr) & ~np.isnan(L) & in_range).any()),
        **{f"diff={t}": bool((diff == t).any()) for t in THRESHOLDS},
    }
