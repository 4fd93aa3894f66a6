"""The rasterizer where its kernels change path (tests/raster_cases.py builds the inputs and shows on the CPU that each
reaches its edge): depth sorts around 4M Gaussians (radix_pass_kernel<8> / <16>) and the scan's look-back window, tile
sorts from 1 tile to above 2^20 tiles (1 to 3 passes), the image-side limit, packed rectangles of 63 / 64 / 65 tiles and
clamped shapes, bitwise-equal depths and the histogram's match-all path, and the blend's chunk edges and thresholds.

Three references per case:
  * the reference rasterizer binary (oracle/_ref, skipped with the reason when it was not built): radii and instance
    counts exact, final_T bit-identical and colour within the full-size expf bar for the full-precision kernel, the ex2
    bar for the default table kernel (tests/test_gpu_pipeline.py's FULL_SIZE_BUDGET / FULL_SIZE_MAX_ERR);
  * the CUB validation path (emit in Gaussian order + one 64-bit sort): every output bit-identical, both culling modes;
  * for one > 4M-Gaussian and one > 65536-tile case, the pair entry point with a shared depth order against two single
    views, bit for bit.
The small blend cases are also checked against the CPU oracle and against a float32 restatement of the blend loop at the
pixel they were built for.  Frames are compared on the GPU; large tensors are released between cases."""
import ctypes as C

import numpy as np
import pytest

from tests import raster_cases as rc
from tests.raster_compare import compare_images

pytestmark = pytest.mark.gpu

EXPF = (1e-6, 3e-6)  # fraction of values outside 1e-4 relative, largest single error (tests/test_gpu_pipeline.py)
EX2 = (4e-5, 3e-2)
BG = np.array([0.2, 0.4, 0.6], np.float32)

CASES = {f"P{p}": (lambda p=p: rc.sort_size(p)) for p in rc.SORT_SIZES}
CASES.update(depth_ties=rc.depth_ties, keys_shared_upper=rc.keys_shared_upper, keys_spread=rc.keys_spread)
CASES.update({f"tiles_{W}x{H}": (lambda W=W, H=H: rc.tile_frame(W, H)) for W, H in rc.TILE_FRAMES})
CASES["rects"] = None  # needs the CPU oracle to pick its rectangles
BLEND = [f"hits_{W}x{H}" for W, H in rc.HIT_FRAMES] + ["alpha_threshold"] + [f"saturate_at_{k}" for k in rc.SATURATE_AT]
PAIR_CASES = [f"P{rc.SMALL_SORT + 1}", "tiles_4112x4096"]


def _build(name, oracle=None):
    if name == "rects":
        return rc.rects(oracle)
    if name in CASES:
        return CASES[name]()
    return {c.name: c for c in rc.blend_cases()}[name]


def _inputs(case, dev):
    import torch

    t = lambda a: torch.as_tensor(np.ascontiguousarray(a, dtype=np.float32)).to(dev)
    g = case.cloud
    return dict(means3D=t(g.xyz), opacities=t(g.opacity).reshape(-1), shs=t(g.features), scales=t(g.scaling),
                rotations=t(g.rotation), bg=t(BG))


def _view(vt, dev):
    import torch

    t = lambda a: torch.as_tensor(np.ascontiguousarray(a, dtype=np.float32)).to(dev)
    return dict(viewmatrix=t(vt.world_view), projmatrix=t(vt.full_proj), campos=t(vt.cam_center), tan_fovx=vt.tan_fovx,
                tan_fovy=vt.tan_fovy)


def _render(case, inp, dev, flags, vt=None, want_depth=True):
    import torch

    from gs2mesh_b200 import rasterizer as rast

    vt = case.vt if vt is None else vt
    v = _view(vt, dev)
    out = rast.rasterize_forward(means3D=inp["means3D"], opacities=inp["opacities"], viewmatrix=v["viewmatrix"],
                                 projmatrix=v["projmatrix"], campos=v["campos"], bg=inp["bg"], width=vt.width, height=vt.height,
                                 tan_fovx=v["tan_fovx"], tan_fovy=v["tan_fovy"], shs=inp["shs"], scales=inp["scales"],
                                 rotations=inp["rotations"], sh_degree=0, flags=flags, want_counts=True, want_depth=want_depth,
                                 scratch=rast.Scratch(dev))
    torch.cuda.synchronize()
    return out


def _ref(oracle, case, inp, dev):
    v = _view(case.vt, dev)
    return oracle.ref_forward_torch(inp["means3D"], inp["opacities"], v["viewmatrix"], v["projmatrix"], v["campos"], case.W, case.H,
                                    v["tan_fovx"], v["tan_fovy"], inp["bg"], shs=inp["shs"], scales=inp["scales"],
                                    rotations=inp["rotations"], sh_degree=0)


def _cmp(a, b):
    """compare_images' TRUE relative criterion on the GPU, in chunks: dict(n, n_bad, frac_bad_rel, max_err, median)
    (median: whether at least half of the values are within 1e-6)."""
    import torch

    a, b = a.reshape(-1), b.reshape(-1)
    n, bad, mx, close = a.numel(), 0, 0.0, 0
    step = 1 << 24
    for s in range(0, n, step):
        x, y = a[s:s + step].double(), b[s:s + step].double()
        d = (x - y).abs()
        err = d / y.abs().clamp(min=1.0)
        bad += int((d / y.abs().clamp(min=0.05) > 1e-4).sum())
        mx = max(mx, float(err.max()))
        close += int((err <= 1e-6).sum())
        del x, y, d, err
    torch.cuda.synchronize()
    return dict(n=n, n_bad=bad, frac_bad_rel=bad / max(n, 1), max_err=mx, median=close * 2 >= n)


def _within(r, bar, what):
    assert r["frac_bad_rel"] <= bar[0] and r["max_err"] <= bar[1] and r["median"], (what, r)


def _free():
    """Drops the case's tensors and scratch blocks and torch's cached memory: the cases differ in size by orders of
    magnitude, and the GPU is shared."""
    import gc

    import torch

    gc.collect()
    torch.cuda.empty_cache()


@pytest.mark.parametrize("name", list(CASES) + BLEND)
def test_matches_reference_binary(oracle, gsb_lib, cuda_device, name):
    import torch

    from gs2mesh_b200 import _lib

    if not oracle.ref_available():
        pytest.skip("reference rasterizer binary oracle/_ref/libref_dgr.so was not built (needs the gs2mesh sources)")
    case = _build(name, oracle)
    inp = _inputs(case, cuda_device)
    ref = _ref(oracle, case, inp, cuda_device)
    n = ref["num_rendered"]
    for flags in (0, _lib.RASTER_EXACT_TILE_CULL):  # rectangle / exact binning, full-precision expf blend
        ours = _render(case, inp, cuda_device, flags, want_depth=False)
        assert torch.equal(ours["radii"], ref["radii"]), (name, flags)
        counts = ours["counts"].tolist()
        assert counts[1] == n and counts[2] == 0, (name, flags, counts, n)
        if flags == 0:
            assert counts[0] == n, (name, counts, n)
        else:
            assert counts[0] <= n
        assert torch.equal(ours["final_T"], ref["final_T"]), (name, flags, _cmp(ours["final_T"], ref["final_T"]))
        _within(_cmp(ours["color"], ref["color"]), EXPF, (name, flags, "color"))
        del ours
    if name not in BLEND:  # tiny frames: the ex2 bar is applied to the pooled blend cases (test_blend_cases)
        ours = _render(case, inp, cuda_device, _lib.RASTER_EXACT_TILE_CULL | _lib.RASTER_FAST_EXP, want_depth=False)
        assert ours["counts"][1].item() == n
        _within(_cmp(ours["color"], ref["color"]), EX2, (name, "ex2 color"))
        _within(_cmp(ours["final_T"], ref["final_T"]), EX2, (name, "ex2 final_T"))
        del ours
    del ref, inp
    _free()


@pytest.mark.parametrize("name", list(CASES) + BLEND)
def test_cub_path_is_bit_identical(oracle, gsb_lib, cuda_device, name):
    import torch

    from gs2mesh_b200 import _lib

    case = _build(name, oracle)
    inp = _inputs(case, cuda_device)
    for flags in (0, _lib.RASTER_EXACT_TILE_CULL | _lib.RASTER_FAST_EXP):
        new = _render(case, inp, cuda_device, flags)
        ref = _render(case, inp, cuda_device, flags | _lib.RASTER_CUB_SORT)
        for k in ("color", "depth", "final_T", "radii"):
            assert torch.equal(new[k], ref[k]), (name, flags, k)
        assert torch.equal(new["counts"][:2], ref["counts"][:2]) and new["counts"][2].item() == 0, (name, flags)
        del new, ref
    del inp
    _free()


@pytest.mark.parametrize("name", PAIR_CASES)
def test_pair_in_caller_blocks_with_shared_depth_equals_two_views(oracle, gsb_lib, cuda_device, name):
    """rasterize_forward_pair with one depth sort for both eyes (the <16> sort's second gather above 4M Gaussians, a
    3-pass tile sort above 65536 tiles) against two rasterize_forward calls."""
    import torch

    from gs2mesh_b200 import rasterizer as rast

    case = _build(name, oracle)
    inp = _inputs(case, cuda_device)
    vts = [case.vt, case.right_eye(0.01 * case.tz if case.tz else 0.02)]
    singles = [_render(case, inp, cuda_device, rast.DEFAULT_FLAGS, vt) for vt in vts]
    f32 = dict(dtype=torch.float32, device=cuda_device)
    eyes = []
    for vt in vts:
        v = _view(vt, cuda_device)
        eyes.append(dict(viewmatrix=v["viewmatrix"], projmatrix=v["projmatrix"], campos=v["campos"], tan_fovx=vt.tan_fovx,
                         tan_fovy=vt.tan_fovy, out_color=torch.empty(3, case.H, case.W, **f32),
                         out_depth=torch.empty(case.H, case.W, **f32), out_final_T=torch.empty(case.H, case.W, **f32),
                         counts_out=torch.zeros(4, dtype=torch.int64, device=cuda_device)))
    streams = (torch.cuda.Stream(cuda_device), torch.cuda.Stream(cuda_device))
    need = max(int(s["counts"][0]) for s in singles)
    torch.cuda.synchronize()
    rast.rasterize_forward_pair(means3D=inp["means3D"], opacities=inp["opacities"], shs=inp["shs"], scales=inp["scales"],
                                rotations=inp["rotations"], sh_degree=0, bg=inp["bg"], width=case.W, height=case.H, eyes=eyes,
                                streams=streams, scratch=(rast.Scratch(cuda_device), rast.Scratch(cuda_device)),
                                flags=rast.DEFAULT_FLAGS, shared_depth=True, min_instances=need)
    torch.cuda.synchronize()
    for e, s in zip(eyes, singles):
        assert e["counts_out"][3].item() == 0  # the eyes' view depths agree bit for bit
        assert torch.equal(e["counts_out"][:3], s["counts"][:3])
        for k, o in (("color", "out_color"), ("depth", "out_depth"), ("final_T", "out_final_T")):
            assert torch.equal(e[o], s[k]), (name, k)
    del singles, eyes, inp
    _free()


def test_blend_cases(oracle, gsb_lib, cuda_device):
    """Per-tile hit counts around the 32-record chunks, alpha at 1/255, saturation at hits 2 / 32 / 33 / 64, ragged frames:
    the full-precision kernel against the CPU oracle and the float32 blend restatement at the centre pixel; the table
    kernel within the ex2 bar of the reference binary (or, without it, of the full-precision kernel), pooled over the
    cases, and saturating at the same hit.  ex2.approx(log2(opacity)) is a few ulp off the opacity, so on the
    alpha_threshold frame -- whose centre pixel is built to sit exactly at 1/255 -- the table kernel may take or skip the
    Gaussians there either way: that frame holds it to the largest-error bound only."""
    from gs2mesh_b200 import _lib

    pooled = {"n": 0, "n_bad": 0, "max_err": 0.0}
    for case in rc.blend_cases():
        inp = _inputs(case, cuda_device)
        exact = _render(case, inp, cuda_device, _lib.RASTER_EXACT_TILE_CULL)
        table = _render(case, inp, cuda_device, _lib.RASTER_EXACT_TILE_CULL | _lib.RASTER_FAST_EXP)
        g = case.cloud
        o = oracle.forward(g.xyz, g.opacity, case.vt.world_view, case.vt.full_proj, case.vt.cam_center, case.W, case.H,
                           case.vt.tan_fovx, case.vt.tan_fovy, bg=BG, shs=g.features, scales=g.scaling, rotations=g.rotation,
                           sh_degree=0)
        np.testing.assert_array_equal(exact["radii"].cpu().numpy(), o["radii"], err_msg=case.name)
        assert exact["counts"][1].item() == o["num_rendered"] == table["counts"][1].item(), case.name
        for k in ("color", "final_T", "depth"):
            r = compare_images(exact[k].cpu().numpy(), o[k])
            assert r["n_bad"] == 0 and r["max_err"] <= 1e-5, (case.name, k, r)
        if "centre_alphas" in case.info:
            T, hit = rc.blend_pixel(case.info["centre_alphas"])
            got = exact["final_T"][8, 8].item()
            assert np.float32(got) == T, (case.name, got, T, hit)
            if "k" in case.info:  # 1e-4 lies well between T_{k-1} and T_k: the table kernel saturates at the same hit
                assert abs(table["final_T"][8, 8].item() - float(T)) <= 1e-4 * float(T), (case.name, "table", hit)
        want = exact
        if oracle.ref_available():
            want = _ref(oracle, case, inp, cuda_device)
        for k in ("color", "final_T"):
            r = _cmp(table[k], want[k])
            if case.name == "alpha_threshold":
                assert r["max_err"] <= EX2[1], (case.name, k, r)
                continue
            pooled["n"] += r["n"]
            pooled["n_bad"] += r["n_bad"]
            pooled["max_err"] = max(pooled["max_err"], r["max_err"])
        del exact, table, want, inp
    _free()
    assert pooled["n_bad"] <= EX2[0] * pooled["n"] and pooled["max_err"] <= EX2[1], pooled


def test_workspace_exactly_at_the_instance_count(gsb_lib, cuda_device):
    """max_instances = R renders without the overflow flag; R - 1 raises it, and the frame rendered again at R is the same."""
    import torch

    from gs2mesh_b200 import _lib
    from gs2mesh_b200 import rasterizer as rast

    case = rc.tile_hit_counts(*rc.HIT_FRAMES[0])
    inp = _inputs(case, cuda_device)
    full = _render(case, inp, cuda_device, rast.DEFAULT_FLAGS)
    R = int(full["counts"][0])
    v = _view(case.vt, cuda_device)
    P, W, H = case.P, case.W, case.H

    def call(cap):
        col = torch.zeros(3, H, W, device=cuda_device)
        status = torch.zeros(4, dtype=torch.int64, device=cuda_device)
        ws = torch.empty(gsb_lib.gsb_raster_workspace_bytes(P, W, H, cap), dtype=torch.uint8, device=cuda_device)
        a = _lib.GsbRasterArgs(P=P, sh_degree=0, sh_coeffs=1, width=W, height=H, background=_lib.ptr(inp["bg"]),
                               means3D=_lib.ptr(inp["means3D"]), shs=_lib.ptr(inp["shs"]), opacities=_lib.ptr(inp["opacities"]),
                               scales=_lib.ptr(inp["scales"]), rotations=_lib.ptr(inp["rotations"]), scale_modifier=1.0,
                               viewmatrix=_lib.ptr(v["viewmatrix"]), projmatrix=_lib.ptr(v["projmatrix"]), cam_pos=_lib.ptr(v["campos"]),
                               tan_fovx=v["tan_fovx"], tan_fovy=v["tan_fovy"], flags=rast.DEFAULT_FLAGS | _lib.RASTER_ASYNC,
                               out_color=_lib.ptr(col), num_rendered=_lib.ptr(status), workspace=_lib.ptr(ws),
                               workspace_bytes=ws.numel(), max_instances=cap)
        rc_ = gsb_lib.gsb_raster_forward(C.byref(a), None)
        torch.cuda.synchronize()
        assert rc_ == _lib.GSB_OK
        return col, status.tolist()

    col, st = call(R)
    assert st[0] == R and st[2] == 0 and torch.equal(col, full["color"])
    _, st = call(R - 1)
    assert st[0] == R and st[2] == 1
    col, st = call(R)
    assert st[2] == 0 and torch.equal(col, full["color"])
    _free()
