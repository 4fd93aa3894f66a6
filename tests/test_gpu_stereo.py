"""GPU tests of the stereo stage (gs2mesh_b200/stereo.py, gsb_stereo.cu): the model inputs against torch's pad and flip,
disparities / occlusion mask / depth against oracle/stereo_oracle.py bit for bit, `Stereo.run` end to end against a
restatement of the reference's file-based loop (stereo_utils.py:93-147) with a stand-in disparity model, the TSDF fed
from memory against the TSDF fed from the files, and two known answers."""
import os

import numpy as np
import pytest

from gs2mesh_b200 import scene
from oracle import stereo_oracle as so
from tests import stereo_cases as sc

pytestmark = pytest.mark.gpu

W, H, NPTS, NVIEWS = 400, 304, 20000, 4

# A deterministic stand-in for DLNR with its call signature: mode 0 = a function of both images (disparity in
# [params[0], params[0] + params[1]]) plus a quarter of the upsampled warm start; mode 1 = constant disparity params[0];
# mode 2 = disparity (padded row^2 * params[0]) mod params[1], constant along each row.  It records every call.
STANDIN = '''
import torch
import torch.nn.functional as F


class DLNR(torch.nn.Module):
    calls = []

    def __init__(self, args):
        super().__init__()
        self.args = args
        self.register_buffer("mode", torch.zeros((), dtype=torch.int64))
        self.register_buffer("params", torch.zeros(4))

    def forward(self, image1, image2, iters=12, flow_init=None, test_mode=False):
        DLNR.calls.append((image1.cpu(), image2.cpu(), None if flow_init is None else flow_init.cpu(), iters, test_mode))
        _, _, hp, wp = image1.shape
        mode, p = int(self.mode), self.params
        if mode == 1:
            up = torch.full((1, 1, hp, wp), -float(p[0]), device=image1.device)
        elif mode == 2:
            rows = torch.arange(hp, device=image1.device, dtype=torch.float32)
            up = (-torch.remainder(rows * rows * p[0], p[1])).view(1, 1, hp, 1).expand(1, 1, hp, wp).contiguous()
        else:
            a = image1[:, 0:1] * 0.6 + image2[:, 1:2] * 0.4
            up = -(p[0] + p[1] * a / 255.0)
            if flow_init is not None:
                up = up + 0.25 * F.interpolate(flow_init[:, :1], size=(hp, wp), mode="nearest")
        low = F.avg_pool2d(up, 4)
        return torch.cat([low, torch.zeros_like(low)], dim=1), up
'''


def write_standin(base_dir, model_name, mode, params):
    import torch

    d = os.path.join(base_dir, "third_party", "DLNR")
    os.makedirs(os.path.join(d, "core"), exist_ok=True)
    os.makedirs(os.path.join(d, "pretrained"), exist_ok=True)
    open(os.path.join(d, "core", "__init__.py"), "w").close()
    with open(os.path.join(d, "core", "dlnr.py"), "w") as f:
        f.write(STANDIN)
    p = torch.zeros(4)
    p[: len(params)] = torch.tensor(params, dtype=torch.float32)
    torch.save({"module.mode": torch.tensor(mode), "module.params": p}, os.path.join(d, "pretrained", f"{model_name}.pth"))
    return base_dir


class Args:
    GS_white_background = False
    stereo_model = "DLNR_Middlebury"
    stereo_warm = True
    stereo_occlusion_threshold = 3
    stereo_shading_eps = 1e-4
    TSDF_voxel = 8
    TSDF_sdf_trunc = 0.06
    TSDF_scale = 1.0
    TSDF_min_depth_baselines = 0
    TSDF_max_depth_baselines = 1000
    TSDF_dilate = 1
    TSDF_valid = None
    TSDF_skip = None
    TSDF_use_mask = False
    TSDF_use_occlusion_mask = True


def bits_equal(a, b):
    """Equal shape, dtype and bits, except that any NaN equals any NaN."""
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    if a.dtype.kind != "f":
        return np.array_equal(a, b)
    iv = {4: np.uint32, 8: np.uint64}[a.dtype.itemsize]
    return bool(((np.isnan(a) & np.isnan(b)) | (a.view(iv) == b.view(iv))).all())


@pytest.fixture(scope="module")
def rig():
    cloud = scene.make_gaussians(NPTS, seed=5)
    rigs, baseline = scene.make_stereo_cameras(NVIEWS, W, H)
    return cloud, rigs, baseline


def _renderer(rig, cuda_device, out=None):
    from gs2mesh_b200.renderer import Renderer

    cloud, rigs, baseline = rig
    r = Renderer.from_scene(rigs, baseline, cloud, output_dir_root=out, args=Args(), device=str(cuda_device))
    r.prepare_renderer()
    return r


def _fxb(rig):
    _, rigs, baseline = rig
    return rigs[0]["left"]["fx"] * baseline


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("h,w", [(1, 1), (1, 77), (77, 1), (31, 33), (32, 32), (33, 65), (540, 960), (1200, 1600),
                                 (1080, 1920), (2163, 4099), (4, 65536), (32768, 4)])
def test_pack_equals_torch_pad_and_flip(gsb_lib, cuda_device, h, w):
    import torch
    import torch.nn.functional as F

    from gs2mesh_b200 import stereo

    g = torch.Generator(device=cuda_device).manual_seed(h * 7 + w)
    left, right = (torch.randint(0, 256, (h, w, 3), generator=g, device=cuda_device, dtype=torch.uint8) for _ in range(2))
    got = stereo.pack_inputs(left, right)
    to = lambda u8: u8.permute(2, 0, 1).float()[None]
    L, R = (F.pad(to(a), stereo.padding(h, w), mode="replicate") for a in (left, right))
    want = torch.cat([L, R, torch.flip(R, dims=[3]), torch.flip(L, dims=[3])])
    assert got.shape == want.shape == (4, 3) + stereo.padded_shape(h, w)
    assert torch.equal(got, want)
    if h * w <= 64 * 64:
        assert np.array_equal(got.cpu().numpy(), so.pack(left.cpu().numpy(), right.cpu().numpy()))


def test_frame_limits_refused(gsb_lib, cuda_device):
    import torch

    from gs2mesh_b200 import stereo

    for h, w in ((4, 65537), (32769, 4)):
        with pytest.raises(ValueError):
            stereo.pack_inputs(torch.zeros(h, w, 3, dtype=torch.uint8, device=cuda_device),
                               torch.zeros(h, w, 3, dtype=torch.uint8, device=cuda_device))


@pytest.mark.parametrize("h,w", [(64, 50), (50, 64), (37, 45), (300, 410)])  # padded in x, in y, in both
def test_disparities_mask_depth_equal_oracle(gsb_lib, cuda_device, h, w):
    import torch

    from gs2mesh_b200 import stereo

    l, r, t, b = so.padding(h, w)
    Hp, Wp = h + t + b, w + l + r
    L, R = sc.adversarial_disparities(h, w, Hp, Wp, seed=h + w)
    report = sc.case_report(L, R)
    assert all(report.values()), {k: v for k, v in report.items() if not v}
    rng = np.random.default_rng(h)
    flow_lr = rng.uniform(-50, 50, (Hp, Wp)).astype(np.float32)
    flow_lr[t:t + h, l:l + w] = -L
    flow_rl = np.ascontiguousarray(-R[:, ::-1])
    # depth cases: d = 0, -0, subnormal (overflow to inf), and a numerator that float32 rounds
    fx, B = 1440.0, 0.137
    assert float(np.float32(fx * B)) != fx * B
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda_device)[None, None]
    d_lr, d_rl = stereo.disparities(dev(flow_lr), dev(flow_rl), h, w, -1)
    want_lr, want_rl = so.disparities(flow_lr, flow_rl, h, w, -1)
    assert bits_equal(d_lr.cpu().numpy(), want_lr) and bits_equal(d_rl.cpu().numpy(), want_rl)
    assert bits_equal(want_lr, L) and bits_equal(want_rl, R)
    want_depth = so.depth(fx, B, want_lr)
    with np.errstate(over="ignore"):
        assert np.isposinf(want_depth[want_lr == sc.SUBNORMAL]).all()
    assert np.isposinf(want_depth[(want_lr == 0) & ~np.signbit(want_lr)]).all()
    assert np.isneginf(want_depth[(want_lr == 0) & np.signbit(want_lr)]).all()
    for thr in sc.THRESHOLDS:
        vis, depth = stereo.occlusion_depth(d_lr, d_rl, thr, stereo.depth_numerator(fx, B))
        want = so.occlusion_mask(want_lr, want_rl, thr)
        assert vis.dtype == torch.bool and np.array_equal(vis.cpu().numpy(), want), f"threshold {thr}"
        assert bits_equal(depth.cpu().numpy(), want_depth)
        # only the mask: no depth buffer
        vis2, none = stereo.occlusion_depth(d_lr, d_rl, thr)
        assert none is None and torch.equal(vis2, vis)


def test_get_occlusion_mask(gsb_lib, cuda_device, tmp_path):
    from gs2mesh_b200.stereo import Stereo

    st = Stereo(write_standin(str(tmp_path), "DLNR_Middlebury", 1, [3]), None, Args(), device=str(cuda_device))
    for rows, cols in ((40, 50), (64, 64), (72, 96)):
        L, R = sc.adversarial_disparities(40, 50, rows, cols, seed=rows)
        for thr in sc.THRESHOLDS:
            got = st.get_occlusion_mask(L, R, thr)
            assert got.dtype == np.bool_ and np.array_equal(got, so.occlusion_mask(L, R, thr))
    for rows, cols in ((39, 50), (40, 49)):
        with pytest.raises(IndexError):
            st.get_occlusion_mask(L, np.zeros((rows, cols), np.float32), 3)


# ---------------------------------------------------------------------------------------------------------------------
def _shading(depth, eps):
    import cv2

    gx = cv2.Sobel(depth, cv2.CV_64F, 1, 0)
    gy = cv2.Sobel(depth, cv2.CV_64F, 0, 1)
    return 1 / (np.sqrt((gx ** 2) + (gy ** 2) + eps))


def reference_loop(st, renderer, start):
    """stereo_utils.py:93-147 over the PNG files, restated: padder rebuilt from the (already padded) images for RL, the RL
    outputs flipped back, numpy mask from the oracle, depth in NumPy 1.x's float32."""
    import cv2
    import torch
    import torch.nn.functional as F

    args, sign = st.args, st.disparity_signs[st.model_name]
    with torch.no_grad():
        prev = {"LR": None, "RL": None}
        for i, cam in enumerate(renderer.left_cameras):
            if i < start:
                continue
            out_dir = renderer.render_folder_name(i)
            renderer.render_image_pair(i, visualize=False)
            image1 = st.load_image(os.path.join(out_dir, "left.png"))
            image2 = st.load_image(os.path.join(out_dir, "right.png"))
            disp = {}
            for direction in ("LR", "RL"):
                pad = so.padding(*image1.shape[-2:])
                image1, image2 = (F.pad(im, pad, mode="replicate") for im in (image1, image2))
                a, b = (image1, image2) if direction == "LR" else (torch.flip(image2, dims=[3]), torch.flip(image1, dims=[3]))
                pf, up = st.model(a, b, iters=st.model_args.valid_iters, test_mode=True,
                                  flow_init=prev[direction] if args.stereo_warm else None)
                if direction == "RL":
                    pf, up = torch.flip(pf, dims=[3]), torch.flip(up, dims=[3])
                ht, wd = up.shape[-2:]
                up = up[..., pad[2]:ht - pad[3], pad[0]:wd - pad[1]].squeeze()
                prev[direction] = pf
                disp[direction] = sign * up.cpu().numpy().squeeze()
                od = os.path.join(out_dir, f"out_{st.model_name}")
                os.makedirs(od, exist_ok=True)
                np.save(os.path.join(od, f"disparity_{direction}.npy"), disp[direction])
            occ = so.occlusion_mask(disp["LR"], disp["RL"], args.stereo_occlusion_threshold)
            depth = so.depth(cam["fx"], renderer.baseline, disp["LR"])
            np.save(os.path.join(od, "occlusion_mask.npy"), occ)
            np.save(os.path.join(od, "depth.npy"), depth)
            cv2.imwrite(os.path.join(od, "depth.png"), depth)
            cv2.imwrite(os.path.join(od, "shading.png"), _shading(depth, args.stereo_shading_eps))


FILES = ["disparity_LR.npy", "disparity_RL.npy", "occlusion_mask.npy", "depth.npy", "depth.png", "shading.png"]


@pytest.mark.parametrize("warm,start", [(True, 0), (False, 0), (True, 2), (False, 1)])
def test_run_equals_reference_loop(gsb_lib, cuda_device, rig, tmp_path, warm, start):
    import torch
    from PIL import Image

    from gs2mesh_b200.stereo import Stereo

    fxb = _fxb(rig)
    base = write_standin(str(tmp_path / "base"), "DLNR_Middlebury", 0, [fxb / 3.4, fxb / 1.4 - fxb / 3.4])
    args = Args()
    args.stereo_warm = warm
    r_mem, r_ref = _renderer(rig, cuda_device, str(tmp_path / "mem")), _renderer(rig, cuda_device, str(tmp_path / "ref"))
    st = Stereo(base, r_mem, args, device=str(cuda_device))
    st_ref = Stereo(base, r_ref, args, device=str(cuda_device))
    calls = type(st.model).calls
    calls.clear()
    st.run(start=start)
    ours = list(calls)
    calls.clear()
    reference_loop(st_ref, r_ref, start)
    theirs = list(calls)
    assert len(ours) == len(theirs) == 2 * (NVIEWS - start)
    assert r_mem.keep_frames is False  # restored after the loop
    for k, (a, b) in enumerate(zip(ours, theirs)):
        assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]), f"model inputs of call {k}"
        assert (a[2] is None) == (b[2] is None) and (a[2] is None or torch.equal(a[2], b[2])), f"flow_init of call {k}"
        assert a[3:] == b[3:]
    assert (ours[2][2] is not None) == warm  # the second view's LR call is warm-started
    n_visible = 0
    for i in range(NVIEWS):
        d_mem = os.path.join(r_mem.render_folder_name(i), "out_DLNR_Middlebury")
        d_ref = os.path.join(r_ref.render_folder_name(i), "out_DLNR_Middlebury")
        if i < start:
            assert not os.path.exists(d_mem) and r_mem.get_frame(i) is None
            continue
        for name in FILES:
            with open(os.path.join(d_mem, name), "rb") as f1, open(os.path.join(d_ref, name), "rb") as f2:
                assert f1.read() == f2.read(), f"view {i} {name}"
        frame = r_mem.get_frame(i)
        depth = np.load(os.path.join(d_mem, "depth.npy"))
        occ = np.load(os.path.join(d_mem, "occlusion_mask.npy"))
        assert depth.dtype == np.float32 and occ.dtype == np.bool_ and depth.shape == occ.shape == (H, W)
        assert np.load(os.path.join(d_mem, "disparity_RL.npy")).shape == (H + 16, W + 16)
        assert bits_equal(frame["depth"].cpu().numpy(), depth)
        assert np.array_equal(frame["occlusion_mask"].cpu().numpy(), occ)
        left = np.array(Image.open(os.path.join(r_mem.render_folder_name(i), "left.png")))
        assert np.array_equal(frame["left_u8"].cpu().numpy(), left)
        n_visible += int(occ.sum())
    assert 0 < n_visible < (NVIEWS - start) * H * W  # the mask is not trivial


def test_tsdf_from_memory_equals_tsdf_from_files(gsb_lib, cuda_device, rig, tmp_path):
    import torch

    from gs2mesh_b200.stereo import Stereo
    from gs2mesh_b200.tsdf import TSDF

    fxb = _fxb(rig)
    base = write_standin(str(tmp_path / "base"), "DLNR_SceneFlow", 0, [fxb / 3.4, fxb / 1.4 - fxb / 3.4])
    args = Args()
    args.stereo_model = "DLNR_SceneFlow"
    r = _renderer(rig, cuda_device, str(tmp_path / "out"))
    st = Stereo(base, r, args, device=str(cuda_device))
    st.run()
    mem = TSDF(r, st, args, "mem").run()
    torch.cuda.synchronize()
    assert mem.frames_integrated == NVIEWS
    r._frames = {}
    disk = TSDF(r, st, args, "disk").run()
    torch.cuda.synchronize()
    a, b = mem.export_units(), disk.export_units()
    assert len(a) == len(b) > 50
    for key in a:
        np.testing.assert_array_equal(a[key][0], b[key][0], err_msg=f"tsdf/weight of unit {key}")
        np.testing.assert_array_equal(a[key][1], b[key][1], err_msg=f"colour of unit {key}")


@pytest.mark.parametrize("D", [0, 5, 37])
def test_known_answer_constant_disparity(gsb_lib, cuda_device, rig, tmp_path, D):
    from gs2mesh_b200.stereo import Stereo

    r = _renderer(rig, cuda_device)
    st = Stereo(write_standin(str(tmp_path), "DLNR_Middlebury", 1, [D]), r, Args(), device=str(cuda_device))
    st.run()
    x = np.arange(W)[None, :].repeat(H, 0)
    with np.errstate(divide="ignore"):
        want_depth = np.full((H, W), np.float32(_fxb(rig)) / np.float32(D), np.float32)
    for i in range(NVIEWS):
        f = r.get_frame(i)
        assert np.array_equal(f["occlusion_mask"].cpu().numpy(), x >= D)
        assert bits_equal(f["depth"].cpu().numpy(), want_depth)


@pytest.mark.parametrize("thr", sc.THRESHOLDS)
def test_known_answer_row_disparity_pins_rl_offset(gsb_lib, cuda_device, rig, tmp_path, thr):
    """Disparity f(padded row) in both directions, frame padded by t = 8 rows at the top: at original row y the LR
    disparity is f(y + t) and the RL value read is f(y), so where both projections stay inside the frame a pixel is
    occluded iff |f(y + t) - f(y)| > thr."""
    from gs2mesh_b200.stereo import Stereo

    a, m = 1, 23
    f = lambda row: (row * row * a) % m
    l, _, t, _ = so.padding(H, W)
    assert t == 8
    r = _renderer(rig, cuda_device)
    args = Args()
    args.stereo_occlusion_threshold = thr
    st = Stereo(write_standin(str(tmp_path), "DLNR_Middlebury", 2, [a, m]), r, args, device=str(cuda_device))
    st.run()
    y = np.arange(H)[:, None].repeat(W, 1)
    x = np.arange(W)[None, :].repeat(H, 0)
    fl, fr = f(y + t), f(y)
    inside = (x - fl >= 0) & (x - fl <= W - 1) & (x - fl + fr >= 0) & (x - fl + fr <= W - 1)
    want = np.abs(fl - fr) <= thr
    assert inside.mean() > 0.9 and want[inside].any() and not want[inside].all()
    for i in range(NVIEWS):
        got = r.get_frame(i)["occlusion_mask"].cpu().numpy()
        assert np.array_equal(got[inside], want[inside])
        assert not got[x - fl < 0].any()
