"""GPU tests of the stereo-pair path: one fused preprocess pass (+ one shared depth sort) for both eyes must give exactly what
two independent forward calls give; scratch overflow and a wrong shared-depth claim are repaired transparently; the in-memory
hand-off to / from the stereo stage equals the file round trip of the reference (renderer_utils.py:389-391,
stereo_utils.py:100-103, tsdf_utils.py:65-67)."""
import os

import numpy as np
import pytest

from gs2mesh_b200 import scene

pytestmark = pytest.mark.gpu

W, H, NPTS, NPAIRS = 400, 304, 20000, 10  # a 10-camera ring: views 3, 4, 5, 8, 9 have eyes whose z rows differ by an ulp


class Args:
    GS_white_background = False
    TSDF_voxel = 8
    TSDF_sdf_trunc = 0.06
    TSDF_scale = 1.0
    TSDF_min_depth_baselines = 4
    TSDF_max_depth_baselines = 20
    TSDF_dilate = 1
    TSDF_valid = None
    TSDF_skip = None
    TSDF_use_mask = False
    TSDF_use_occlusion_mask = True


class StereoStub:
    model_name = "unit"


@pytest.fixture(scope="module")
def rig():
    cloud = scene.make_gaussians(NPTS, seed=3)
    rigs, baseline = scene.make_stereo_cameras(NPAIRS, W, H)
    return cloud, rigs, baseline


def _renderer(rig, cuda_device, out=None, **kw):
    from gs2mesh_b200.renderer import Renderer

    cloud, rigs, baseline = rig
    r = Renderer.from_scene(rigs, baseline, cloud, output_dir_root=out, args=Args(), device=str(cuda_device))
    for k, v in kw.items():
        setattr(r, k, v)
    r.prepare_renderer()
    return r


def _grab(out):
    import torch

    torch.cuda.synchronize()
    return {k: out[k].cpu().numpy().copy() for k in ("left", "right", "depth", "final_T", "left_u8", "right_u8")}


def test_fused_pair_equals_two_forward_calls(gsb_lib, cuda_device, rig, monkeypatch):
    """fused (shared depth sort where the eyes' z rows are bitwise equal), fused without sharing, and two separate forward
    calls: bit-identical frames for every view of the rig, which contains rigs of both kinds."""
    r = _renderer(rig, cuda_device)
    shared = list(r._shared_depth)
    assert any(shared) and not all(shared), "the synthetic rig should contain both kinds of stereo pairs"
    frames = {}
    for mode in ("fused", "noshare", "separate"):
        monkeypatch.setenv("GSB_PAIR_MODE", mode)
        frames[mode] = [_grab(r.render_image_pair(i, to_host=False)) for i in range(NPAIRS)]
        r.check_status()
    for i in range(NPAIRS):
        for k in frames["separate"][i]:
            np.testing.assert_array_equal(frames["fused"][i][k], frames["separate"][i][k], err_msg=f"fused view {i} {k} shared={shared[i]}")
            np.testing.assert_array_equal(frames["noshare"][i][k], frames["separate"][i][k], err_msg=f"noshare view {i} {k}")
    assert float(frames["fused"][0]["final_T"].mean()) < 0.9  # something was rendered


def test_wrong_shared_depth_claim_is_flagged_and_repaired(gsb_lib, cuda_device, rig):
    r = _renderer(rig, cuda_device)
    view = r._shared_depth.index(False)
    good = _grab(r.render_image_pair(view, to_host=True))
    r._shared_depth[view] = True  # lie: this rig's z rows differ by an ulp
    out = r.render_image_pair(view, to_host=True)  # synchronous path: flagged by the kernel, re-rendered without the claim
    assert r._shared_depth[view] is False
    got = _grab(out)
    for k in good:
        np.testing.assert_array_equal(got[k], good[k], err_msg=k)
    # pure device path: nothing waits, so the flag is only reported
    r._shared_depth[view] = True
    r.render_image_pair(view, to_host=False)
    import torch

    torch.cuda.synchronize()
    assert int(r._status[view, 0, 3]) == 1 and int(r._status[view, 1, 3]) == 1
    with pytest.raises(RuntimeError):
        r.check_status([view])


def test_undersized_renderer_scratch_is_repaired_transparently(gsb_lib, cuda_device, rig):
    """The reference resizes its binning buffer inside every frame (rasterizer_impl.cu:281-285); here an undersized scratch is
    detected from the frame's status word and the pair is rendered again -- on the synchronous path and on the handle of the
    asynchronous one -- instead of raising."""
    from gs2mesh_b200 import rasterizer as rast

    r = _renderer(rig, cuda_device)
    good = [_grab(r.render_image_pair(i, to_host=True)) for i in (0, 1)]
    need = int(r._status[0, :, 0].max())
    assert need > 20000

    def shrink():
        import torch

        torch.cuda.synchronize()
        for st in r._stream_sets:  # replace the grown scratch blocks with 1024-instance ones
            st.scratch = (rast.Scratch(cuda_device, max_instances=1024), rast.Scratch(cuda_device, max_instances=1024))
        r._min_instances = 1

    # synchronous call: rendered, found too small, scratch grown, rendered again -- all inside the call
    shrink()
    got = _grab(r.render_image_pair(0, to_host=True))
    for k in good[0]:
        np.testing.assert_array_equal(got[k], good[0][k], err_msg=k)
    assert r._min_instances >= need
    # asynchronous call: the handle's synchronize() repairs the pair
    shrink()
    out = r.render_image_pair(1, to_host=True, wait=False)
    out["ready"].synchronize()
    got = _grab(out)
    for k in good[1]:
        np.testing.assert_array_equal(got[k], good[1][k], err_msg=k)
    # pure device path: reported, not repaired
    shrink()
    r.render_image_pair(2, to_host=False)
    import torch

    torch.cuda.synchronize()
    assert int(r._status[2, 0, 2]) == 1
    with pytest.raises(RuntimeError):
        r.check_status([2])


def test_in_memory_handoff_equals_file_round_trip(oracle, gsb_lib, cuda_device, rig, tmp_path):
    """(a) Renderer.stereo_inputs == Stereo.load_image(left.png / right.png) bit for bit (stereo_utils.py:68-80,102-103);
    (b) TSDF.run() fed from the frame cache (rendered frames + depth / occlusion handed back with put_stereo_outputs) equals
    TSDF.run() fed from left.png / depth.npy / occlusion_mask.npy (tsdf_utils.py:65-80) bit for bit."""
    import torch
    from PIL import Image

    from gs2mesh_b200.tsdf import TSDF

    cloud, rigs, baseline = rig
    r = _renderer(rig, cuda_device, out=str(tmp_path))
    r.keep_frames = True
    views = [0, 1, 2, 5]
    occ = np.ones((H, W), bool)
    occ[:, : W // 6] = False
    for i in views:
        out = r.render_image_pair(i)
        # (a)
        l, rr = r.stereo_inputs(i)
        for name, t in (("left", l), ("right", rr)):
            img = np.array(Image.open(os.path.join(r.render_folder_name(i), f"{name}.png"))).astype(np.uint8)
            want = torch.from_numpy(img).permute(2, 0, 1).float()[None]
            assert t.shape == want.shape and t.dtype == want.dtype
            assert torch.equal(t.cpu(), want)
        # the stereo stage's outputs: here the rendered expected depth, written the way stereo_utils.py:135-137 does
        depth = r.expected_depth(out["depth"], out["final_T"])
        d = os.path.join(r.render_folder_name(i), f"out_{StereoStub.model_name}")
        os.makedirs(d, exist_ok=True)
        np.save(os.path.join(d, "depth.npy"), depth.cpu().numpy())
        np.save(os.path.join(d, "occlusion_mask.npy"), occ)
        r.put_stereo_outputs(i, depth, torch.as_tensor(occ))

    class A(Args):
        TSDF_valid = views

    mem = TSDF(r, StereoStub(), A(), "mem").run()
    torch.cuda.synchronize()
    assert mem.frames_integrated == len(views)
    r.keep_frames = False
    r._frames = {}
    disk = TSDF(r, StereoStub(), A(), "disk").run()
    torch.cuda.synchronize()
    a, b = mem.export_units(), disk.export_units()
    assert len(a) == len(b) > 50
    for key in a:
        np.testing.assert_array_equal(a[key][0], b[key][0], err_msg=f"tsdf/weight of unit {key}")
        np.testing.assert_array_equal(a[key][1], b[key][1], err_msg=f"colour of unit {key}")


@pytest.mark.parametrize("num_points,W,H,deg", [(4099, 333, 250, 3), (777, 250, 130, 1), (33, 64, 48, 0)])
def test_pair_entry_point_on_ragged_inputs_in_caller_blocks(gsb_lib, cuda_device, num_points, W, H, deg):
    """`gsb_raster_forward_pair` through the ctypes stub against two `gsb_raster_forward` calls on awkward shapes: a Gaussian
    count that is no multiple of the warp size (the last warp takes the plain-load path), ragged tile rows / columns, lower SH
    degrees; with and without a shared depth order; eyes on one stream and on two."""
    import torch

    from gs2mesh_b200 import _lib, camera as cam
    from gs2mesh_b200 import rasterizer as rast

    g = scene.make_gaussians(num_points, seed=40 + deg, sh_degree=deg)
    rigs, _ = scene.make_stereo_cameras(10, W, H)
    dev = cuda_device
    t = lambda a: torch.as_tensor(np.ascontiguousarray(a, dtype=np.float32)).to(dev)
    means, op, shs, sc, ro = t(g.xyz), t(g.opacity).reshape(-1), t(g.features), t(g.scaling), t(g.rotation)
    bg = torch.zeros(3, device=dev)
    for view in (0, 3):  # rig 0: eyes share their view depths; rig 3: the z rows differ by an ulp
        vts = [cam.view_transforms_from_camera(rigs[view][s]) for s in ("left", "right")]
        zrow = [vt.world_view.reshape(-1)[[2, 6, 10, 14]].view(np.uint32) for vt in vts]
        shared = bool(np.array_equal(zrow[0], zrow[1]))
        assert shared == (view == 0)
        recs = [t(vt.packed()) for vt in vts]
        want = []
        for vt, rec in zip(vts, recs):
            o = rast.rasterize_forward(means3D=means, opacities=op, viewmatrix=rec[0:16], projmatrix=rec[16:32], campos=rec[32:35], bg=bg,
                                       width=W, height=H, tan_fovx=vt.tan_fovx, tan_fovy=vt.tan_fovy, shs=shs, scales=sc, rotations=ro,
                                       sh_degree=deg, want_counts=True)
            want.append({k: o[k].clone() for k in ("color", "depth", "final_T", "counts")})
        main = torch.cuda.current_stream(dev)
        side = torch.cuda.Stream(dev)
        scratch = (rast.Scratch(dev), rast.Scratch(dev))
        for streams in ((main, main), (main, side)):
            for claim in ((True, False) if shared else (False,)):
                eyes = []
                for vt, rec in zip(vts, recs):
                    eyes.append(dict(viewmatrix=rec[0:16], projmatrix=rec[16:32], campos=rec[32:35], tan_fovx=vt.tan_fovx,
                                     tan_fovy=vt.tan_fovy, out_color=torch.empty(3, H, W, device=dev), out_depth=torch.empty(H, W, device=dev),
                                     out_final_T=torch.empty(H, W, device=dev), counts_out=torch.zeros(4, dtype=torch.int64, device=dev)))
                side.wait_stream(main)
                rast.rasterize_forward_pair(means3D=means, opacities=op, shs=shs, scales=sc, rotations=ro, sh_degree=deg, bg=bg,
                                            width=W, height=H, eyes=eyes, streams=streams, scratch=scratch, shared_depth=claim)
                torch.cuda.synchronize()
                for e, w in zip(eyes, want):
                    assert int(e["counts_out"][2]) == 0 and int(e["counts_out"][3]) == 0
                    assert torch.equal(e["counts_out"][:2], w["counts"][:2])
                    for k, kk in (("out_color", "color"), ("out_depth", "depth"), ("out_final_T", "final_T")):
                        assert torch.equal(e[k], w[kk]), (view, claim, k)
    # no Gaussians at all: zero-filled outputs, like rasterize_points.cu:77
    L = gsb_lib
    empty = dict(viewmatrix=recs[0][0:16], projmatrix=recs[0][16:32], campos=recs[0][32:35], tan_fovx=vts[0].tan_fovx,
                 tan_fovy=vts[0].tan_fovy)
    eyes = [dict(empty, out_color=torch.ones(3, H, W, device=dev), out_depth=None, out_final_T=None, counts_out=None) for _ in range(2)]
    rast.rasterize_forward_pair(means3D=means[:0], opacities=op[:0], shs=shs[:0], scales=sc[:0], rotations=ro[:0], sh_degree=deg, bg=bg,
                                width=W, height=H, eyes=eyes, streams=(main, main), scratch=scratch)
    torch.cuda.synchronize()
    assert all(float(e["out_color"].abs().max()) == 0.0 for e in eyes)


def test_pair_scratch_is_released_with_its_blocks(gsb_lib, cuda_device, rig):
    """The wrapper keeps nothing for the streams it ran on: once the caller drops the blocks of a pair rendered on fresh
    streams, the device memory they took is free again."""
    import gc

    import torch

    from gs2mesh_b200 import camera as cam
    from gs2mesh_b200 import rasterizer as rast

    cloud, rigs, _ = rig
    dev = cuda_device
    t = lambda a: torch.as_tensor(np.ascontiguousarray(a, dtype=np.float32)).to(dev)
    means, op, shs, sc, ro = t(cloud.xyz), t(cloud.opacity).reshape(-1), t(cloud.features), t(cloud.scaling), t(cloud.rotation)
    eyes = []
    for side in ("left", "right"):
        vt = cam.view_transforms_from_camera(rigs[0][side])
        rec = t(vt.packed())
        eyes.append(dict(viewmatrix=rec[0:16], projmatrix=rec[16:32], campos=rec[32:35], tan_fovx=vt.tan_fovx,
                         tan_fovy=vt.tan_fovy, out_color=torch.empty(3, H, W, device=dev),
                         counts_out=torch.zeros(4, dtype=torch.int64, device=dev)))
    bg = torch.zeros(3, device=dev)
    streams = (torch.cuda.Stream(dev), torch.cuda.Stream(dev))
    for st in streams:
        st.wait_stream(torch.cuda.current_stream(dev))
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated(dev)
    scratch = (rast.Scratch(dev), rast.Scratch(dev))
    rast.rasterize_forward_pair(means3D=means, opacities=op, shs=shs, scales=sc, rotations=ro, sh_degree=cloud.sh_degree, bg=bg,
                                width=W, height=H, eyes=eyes, streams=streams, scratch=scratch)
    assert torch.cuda.memory_allocated(dev) > before
    del scratch
    gc.collect()
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated(dev) == before
    assert all(int(e["counts_out"][2]) == 0 for e in eyes) and float(eyes[0]["out_color"].abs().max()) > 0
