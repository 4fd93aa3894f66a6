"""CPU checks that every per-Gaussian geometry case of tests/raster_geometry_cases.py reaches the edge it is named for,
computed with the CPU oracle's preprocess (both FMA builds) and the float32 restatements there."""
import numpy as np
import pytest

from tests import raster_cases as rc
from tests import raster_geometry_cases as gc

F = np.float32


def _both(oracle, case, **kw):
    return gc.preprocess(oracle, case, **kw), gc.preprocess(oracle, case, fma=True, **kw)


def test_fma32_is_correctly_rounded():
    rng = np.random.default_rng(0)
    a, b, c = (rng.normal(size=20000).astype(F) for _ in range(3))
    got = gc.fma32(a, b, c)
    from fractions import Fraction

    for i in range(0, 20000, 97):
        exact = Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i]))
        lo = F(float(exact))  # within one float32 step of the exact value
        cands = [np.nextafter(lo, F(-np.inf)), lo, np.nextafter(lo, F(np.inf))]
        best = min(cands, key=lambda v: (abs(Fraction(float(v)) - exact), int(v.view(np.int32)) & 1))
        assert got[i] == best, i
    # (1 + 2^-11)(1 + 2^-13) lies on a float32 midpoint; +-2^-60 takes it off, but the float64 sum rounds back onto it,
    # where rounding to float32 would tie to even (down) both times
    a, b, base = F(1 + 2 ** -11), F(1 + 2 ** -13), 1 + 2 ** -11 + 2 ** -13
    assert gc.fma32(a, b, F(2 ** -60)) == F(base + 2 ** -23) and gc.fma32(a, b, F(-(2 ** -60))) == F(base)


def test_near_plane_depths_straddle_0_2(oracle):
    case = gc.near_plane()
    z = case.cloud.xyz[:, 2]
    assert (z.view(np.int32) - gc.NEAR.view(np.int32) == case.info["ulps"]).all()
    for pre in _both(oracle, case):
        vis = pre["radii"] > 0
        assert (vis == (z > gc.NEAR)).all()  # every Gaussian in front of the plane is drawn: nothing else decides here
        assert (vis & (case.info["ulps"] == 1)).sum() >= 3 and ((case.info["ulps"] == 0) & ~vis).sum() >= 3
        assert (case.info["ulps"] > 0).sum() >= 8 and (case.info["ulps"] < 0).sum() >= 8
    cover = case.info["covers_frame"]
    pre = gc.preprocess(oracle, case)
    r = rc.tile_rects(pre["xy"], pre["radii"], case.W, case.H)
    gx, gy = rc.grid(case.W, case.H)
    full = (r[:, 0] == 0) & (r[:, 1] == 0) & (r[:, 2] == gx) & (r[:, 3] == gy)
    assert full[cover].sum() >= 6  # 1..4 ulp in front of the plane and covering the whole frame


def test_near_plane_rotated_contraction_splits(oracle):
    case = gc.near_plane_rotated()
    vm = case.vt.world_view
    assert (np.abs(vm[:3, :3]) > 0.05).all()  # no axis-aligned row or column
    plain, late, early = gc.view_depths(case.cloud.xyz, vm)
    off = case.info["ulps"]
    for k in range(-4, 5):  # the three forms agree at 0.2f + k ulp, four Gaussians per offset
        sel = off == k
        assert sel.sum() >= 4 and (plain[sel] == late[sel]).all() and (late[sel] == early[sel]).all()
        assert (plain[sel].view(np.int32) - gc.NEAR.view(np.int32) == k).all()
    assert ((off >= 1) & (off <= 4)).sum() >= 8 and ((off >= -4) & (off <= 0)).sum() >= 8
    split = case.info["split"]
    assert len(split) >= 8
    fused_front = late[split] > gc.NEAR
    assert (fused_front == (early[split] > gc.NEAR)).all() and (fused_front != (plain[split] > gc.NEAR)).all()
    assert fused_front.sum() >= 2 and (~fused_front).sum() >= 2  # both directions of the split
    pre, pre_fma = _both(oracle, case)
    assert ((pre["radii"] > 0) == (plain > gc.NEAR)).all()  # the plainly rounded build culls by the plainly rounded depth
    assert (pre_fma["radii"][split] > 0).sum() + (pre["radii"][split] > 0).sum() > 0
    assert (pre["radii"][case.info["covers_frame"]] > 150).all()


def test_guard_band_clamp_is_active_on_visible_gaussians(oracle):
    case = gc.guard_band()
    lx, ly = gc.lim(case.vt)
    assert lx != ly
    x, y, z = (case.cloud.xyz[:, k] for k in range(3))
    txtz, tytz = x / z, y / z  # identity camera: t = xyz exactly
    cx, cy = np.abs(txtz) > lx, np.abs(tytz) > ly
    for pre in _both(oracle, case):
        vis = pre["radii"] > 0
        assert (vis & cx).sum() >= 24 and (vis & cy).sum() >= 24 and (vis & cx & cy).sum() >= 12
        assert (vis & ~cx & (np.abs(txtz) > 0.99 * lx)).sum() >= 8  # just inside the band
        assert (vis & cy & (np.abs(tytz) <= lx)).sum() >= 16  # clamped at limy, not at limx
        # just outside: within 2^-17 of the band
        assert (vis & cx & (np.abs(txtz) < lx * F(1 + 2 ** -17))).sum() >= 4
        # the footprint reaches into the frame although the centre lies outside it
        out = (pre["xy"][:, 0] < 0) | (pre["xy"][:, 0] > case.W) | (pre["xy"][:, 1] < 0) | (pre["xy"][:, 1] > case.H)
        assert (vis & out).sum() >= 48


def test_tile_edge_centres_move_a_rectangle(oracle):
    case = gc.tile_edge_centres()
    px, py = gc.identity_proj(case.cloud.xyz, case.vt)
    xd, xp, xf = gc.ndc2pix(px, case.W)
    yd, yp, yf = gc.ndc2pix(py, case.H)
    for pre in _both(oracle, case):
        assert (pre["radii"] == case.info["radius"]).all()
        np.testing.assert_array_equal(pre["xy"], np.c_[xd, yd])  # the restatement is the oracle's double ndc2Pix
        ref = rc.tile_rects(pre["xy"], pre["radii"], case.W, case.H)
        for fx, fy in ((xp, yp), (xf, yf)):
            flt = rc.tile_rects(np.c_[fx, fy], pre["radii"], case.W, case.H)
            moved = (flt != ref).any(1)
            assert moved.sum() >= 40, moved.sum()
            assert (flt[:, [0, 2]] != ref[:, [0, 2]]).any(1).sum() >= 16 and (flt[:, [1, 3]] != ref[:, [1, 3]]).any(1).sum() >= 16
            assert (pre["tiles_touched"][moved] != rc.rect_shape(flt[moved]).prod(1)).sum() >= 8  # the instance count moves


def test_degenerate_covariances(oracle):
    case = gc.degenerate_cov()
    ind, d0 = case.info["indefinite"], case.info["det0"]
    assert len(d0) >= 4
    for pre in _both(oracle, case):
        co = pre["conic_opacity"].astype(np.float64)
        inv_det = co[:, 0] * co[:, 2] - co[:, 1] ** 2  # = 1 / det of the 2-D covariance
        neg = (pre["radii"] > 0) & (inv_det < 0)
        assert neg[ind].sum() >= 16
        ex = rc.exact_rects(pre, case.W, case.H)
        ref = rc.tile_rects(pre["xy"], pre["radii"], case.W, case.H)
        assert (ex[neg] == ref[neg]).all()  # a degenerate footprint keeps its whole rectangle
        assert (pre["radii"][d0] == 0).all()  # det == 0: culled
        # a, c > 0 and a negative determinant with k < -2e4: only the determinant test marks these degenerate; read as
        # ellipses, 1 + 5e-5 k < 0 would give tau < 0 and an empty candidate rectangle
        tn = case.info["tau_negative"]
        a, b, c = (pre["conic_opacity"][tn, i] for i in range(3))
        k = gc.conic_k(pre["conic_opacity"][tn])
        trap = (pre["radii"][tn] > 0) & (a > 0) & (c > 0) & (F(a * c) - F(b * b) < 0) & (F(1) + F(5e-5) * k < 0)
        assert trap.sum() >= 12, trap.sum()
        assert (rc.rect_shape(ex[tn]).prod(1) > 0).all()
        broken = []
        for i in tn[trap]:  # the rectangle a footprint without the determinant test would keep: none
            f = dict(a=F(co[i, 0]), b=F(co[i, 1]), c=F(co[i, 2]), nb_a=F(0), nb_c=F(0), degenerate=False,
                     two_tau=F(2) * F(np.log(F(255) * F(pre["conic_opacity"][i, 3]))))
            from tests.test_exact_cull_math import shrink_rect
            x0, y0, x1, y1 = shrink_rect(tuple(int(v) for v in ref[i]), F(pre["xy"][i, 0]), F(pre["xy"][i, 1]), f)
            broken.append((x1 - x0) * (y1 - y0))
        assert (np.asarray(broken) == 0).all()
    vt = case.vt
    fx, fy = gc.focal(vt)
    for i, a in zip(d0, case.cov3D[d0]):
        z = case.cloud.xyz[i, 2]
        assert case.cloud.xyz[i, 0] == 0 and case.cloud.xyz[i, 1] == 0
        jx, jy = F(fx / z), F(fy / z)
        assert jx < 1 and jy < 1
        cxx, cyy, cxy = (a[0] * jx) * jx + F(0.3), (a[3] * jy) * jy + F(0.3), (a[1] * jy) * jx
        assert cxx == cyy == cxy and F(cxx * cxx) == float(cxx) ** 2  # a^2 exact: det = 0 under any contraction
        assert F(cxx * cyy) - F(cxy * cxy) == 0 and gc.fma32(cxx, cyy, -F(cxy * cxy)) == 0
    # the cov3D_precomp path ignores scale_modifier (on the oracle as on the reference)
    a, b = gc.preprocess(oracle, case), gc.preprocess(oracle, case, scale_modifier=0.5)
    for k in ("radii", "xy", "conic_opacity"):
        np.testing.assert_array_equal(a[k], b[k])


def test_needles_straddle_the_elongation_cut_off(oracle):
    case = gc.needles(oracle)
    pre = gc.preprocess(oracle, case)
    assert (pre["radii"] > 0).all()
    k = gc.conic_k(pre["conic_opacity"])
    kb = k.view(np.int32) - F(1000).view(np.int32)
    assert ((k < 1000) & (k > 995)).sum() >= 8 and ((k > 1000) & (k < 1005)).sum() >= 8
    assert (np.abs(kb) <= 3).sum() >= 4  # within 3 ulp of the cut-off
    assert (k >= 1e4).sum() >= 8
    ex = rc.exact_rects(pre, case.W, case.H)
    ref = rc.tile_rects(pre["xy"], pre["radii"], case.W, case.H)
    assert (ex[k > 1000] == ref[k > 1000]).all()  # above the cut-off: the reference rectangle
    shrunk = (rc.rect_shape(ex).prod(1) < rc.rect_shape(ref).prod(1))[k <= 1000]
    assert shrunk.sum() >= 8  # at or below it: the ellipse's bounding box


def test_huge_footprints(oracle):
    case = gc.huge_footprints()
    pre = gc.preprocess(oracle, case)
    r, w = pre["radii"], case.info["where"]
    assert (r >= max(case.W, case.H)).all() and r.max() >= 9e4
    for k in range(3):
        assert (r[w == k] > 0).sum() >= 24
    xy = pre["xy"]
    inside = (xy[:, 0] >= 0) & (xy[:, 0] < case.W) & (xy[:, 1] >= 0) & (xy[:, 1] < case.H)
    far = np.maximum(np.maximum(-xy[:, 0], xy[:, 0] - case.W), np.maximum(-xy[:, 1], xy[:, 1] - case.H)) > 1e4
    assert inside.sum() >= 24 and (~inside).sum() >= 48 and far.sum() >= 8
    assert int(pre["tiles_touched"].astype(np.int64).sum()) < 2e7
    gx, gy = rc.grid(case.W, case.H)
    assert (pre["tiles_touched"] == gx * gy).sum() >= 24  # the radius clamps to the whole grid


def test_opacity_edges(oracle):
    case = gc.opacity_edges()
    op = case.cloud.opacity[:, 0]
    assert set(op.tolist()) == set(gc.OPACITY_EDGES.tolist()) and len(gc.OPACITY_EDGES) == 5
    pre = gc.preprocess(oracle, case)
    assert (pre["radii"] > 0).all()
    with np.errstate(divide="ignore"):
        ex = rc.exact_rects(pre, case.W, case.H)
    area_ref = rc.rect_shape(rc.tile_rects(pre["xy"], pre["radii"], case.W, case.H)).prod(1)
    area_ex = rc.rect_shape(ex).prod(1)
    zero, faint = op == 0, op < gc.ALPHA_MIN
    assert zero.sum() >= 8 and faint.sum() >= 16 and (area_ref[faint] > 0).all()
    assert (area_ex[zero] == 0).all()  # tau = -inf: nothing can be blended, yet the reference counts the rectangle
    # one ulp below 1/255 the rounding allowance of tau still keeps a small candidate box (never blended: alpha < 1/255)
    assert (area_ex[faint & ~zero] < area_ref[faint & ~zero]).all()
    assert (area_ex[~zero] > 0).all()
    hits = rc.tile_hits(rc.tile_rects(pre["xy"], pre["radii"], case.W, case.H), case.W, case.H)
    assert hits.max() >= 10  # overlapping


def test_quaternions_are_used_as_given(oracle):
    case = gc.quaternions()
    kind, q = case.info["kind"], case.cloud.rotation
    norms = np.linalg.norm(q.astype(np.float64), axis=1)
    assert np.allclose(norms[kind == "half"], 0.5, rtol=1e-6) and np.allclose(norms[kind == "two"], 2, rtol=1e-6)
    assert (q[kind == "zero"] == 0).all()
    pre = gc.preprocess(oracle, case)
    s = case.cloud.scaling.astype(F)
    c3 = pre["cov3d"]
    zero = kind == "zero"
    np.testing.assert_array_equal(c3[zero][:, [0, 3, 5]], (s[zero] * s[zero]).astype(F))  # R = I
    assert (c3[zero][:, [1, 2, 4]] == 0).all()
    pairs = np.flatnonzero(kind == "pair")
    np.testing.assert_array_equal(c3[pairs[0::2]], c3[pairs[1::2]])  # q and -q: the same covariance, bit for bit
    unit = case.cloud.rotation / norms[:, None].clip(1e-30).astype(F)
    norm_case = gc.GeoCase(case.name, gc.gcloud(case.cloud.xyz, case.cloud.scaling, unit, case.cloud.opacity,
                                                case.cloud.features), case.vt, case.focal, 0.0)
    pre_n = gc.preprocess(oracle, norm_case)
    for kd in ("half", "two"):
        sel = kind == kd
        assert (pre["radii"][sel] != pre_n["radii"][sel]).sum() >= 8  # renormalising would change the footprint


@pytest.mark.parametrize("deg", gc.SH_DEGREES)
def test_sh_colours_reach_the_clamp(oracle, deg):
    case = gc.sh_clamp(deg)
    assert case.cloud.features.shape[1] == (deg + 1) ** 2
    for pre in _both(oracle, case):
        rgb = pre["rgb"]
        assert (pre["radii"] > 0).all()
        assert (rgb == 0).sum() >= 24 and (rgb > 1).sum() >= 24  # clamped at 0, and far above 1 (not clamped)
        on = case.info["on_axis"]
        assert ((rgb[on] == 0).any(1)).sum() >= 4
    xyz = case.cloud.xyz
    assert (xyz[case.info["on_axis"], :2] == 0).all() and (xyz[:, 0] == 0).sum() >= 32 and (xyz[:, 1] == 0).sum() >= 32


def test_colors_precomp_pass_through(oracle):
    case = gc.colors_precomp()
    pre = gc.preprocess(oracle, case)
    assert (pre["radii"] > 0).all()
    np.testing.assert_array_equal(pre["rgb"], case.colors)
    assert (case.colors < 0).sum() >= 24 and (case.colors > 1).sum() >= 24


def test_toed_in_pair_splits_visibility(oracle):
    case = gc.toed_in_pair(oracle)
    vl, vr = case.vt, case.info["right"]
    assert not (vl.world_view == vr.world_view).all(1).any() and not (vl.world_view.T == vr.world_view.T).all(1)[:3].any()
    tag = case.info["tag"]
    pl, pr = gc.preprocess(oracle, case), gc.preprocess(oracle, case, vt=vr)
    dl, dr = gc.view_depths(case.cloud.xyz, vl.world_view)[0], gc.view_depths(case.cloud.xyz, vr.world_view)[0]
    vis_l, vis_r = pl["radii"] > 0, pr["radii"] > 0
    assert ((tag == "near_left") & ~vis_l & vis_r & (dl < gc.NEAR)).sum() >= 16
    assert ((tag == "near_right") & vis_l & ~vis_r & (dr < gc.NEAR)).sum() >= 16
    assert ((tag == "off_left") & ~vis_l & vis_r & (dl > gc.NEAR)).sum() >= 16
    assert ((tag == "off_right") & vis_l & ~vis_r & (dr > gc.NEAR)).sum() >= 16
    assert (vis_l & vis_r).sum() >= 64
    assert (pl["rgb"][vis_l & vis_r] != pr["rgb"][vis_l & vis_r]).any(1).mean() > 0.9  # per-eye SH direction
