"""Time the stereo stage at 1600x1200 with a stand-in disparity model of negligible cost, so that the numbers are the
stage around the model and not DLNR:
  - Stereo.run per view in memory (no files), and with the reference's files written;
  - a restatement of the reference's loop: render with PNGs, read them back, pad, numpy mask and depth, write the files;
  - the three gsb_stereo_* kernels alone, with CUDA events.
Every variant renders the pair first.  Prints one JSON line with the card name and power limit read in the same run.
Everything is written to a temporary directory.

    python scripts/stereo_stage_time.py [--views 20] [--points 200000]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from gs2mesh_b200 import scene, stereo  # noqa: E402
from gs2mesh_b200.renderer import Renderer  # noqa: E402
from oracle import stereo_oracle as so  # noqa: E402

STANDIN = '''
import torch


class DLNR(torch.nn.Module):
    """Constant-time stand-in: flow = -(8 + red / 32), low-res flow = zeros."""

    def __init__(self, args):
        super().__init__()
        self.register_buffer("unused", torch.zeros(1))

    def forward(self, image1, image2, iters=12, flow_init=None, test_mode=False):
        b, _, h, w = image1.shape
        return image1.new_zeros(b, 2, h // 4, w // 4), -(8.0 + image1[:, :1] / 32.0)
'''


class Args:
    GS_white_background = False
    stereo_model = "DLNR_Middlebury"
    stereo_warm = True
    stereo_occlusion_threshold = 3
    stereo_shading_eps = 1e-4


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        return float(out.strip().splitlines()[0])
    except Exception:
        return None


def reference_loop(st, r, n):
    import cv2

    for i in range(n):
        cam = r.left_cameras[i]
        out_dir = r.render_folder_name(i)
        r.render_image_pair(i)
        image1 = st.load_image(os.path.join(out_dir, "left.png"))
        image2 = st.load_image(os.path.join(out_dir, "right.png"))
        disp = {}
        for direction in ("LR", "RL"):
            pad = so.padding(*image1.shape[-2:])
            image1, image2 = (F.pad(im, pad, mode="replicate") for im in (image1, image2))
            a, b = (image1, image2) if direction == "LR" else (torch.flip(image2, dims=[3]), torch.flip(image1, dims=[3]))
            _, up = st.model(a, b, iters=10, test_mode=True)
            if direction == "RL":
                up = torch.flip(up, dims=[3])
            ht, wd = up.shape[-2:]
            disp[direction] = -1 * up[..., pad[2]:ht - pad[3], pad[0]:wd - pad[1]].squeeze().cpu().numpy()
            od = os.path.join(out_dir, f"out_{st.model_name}")
            os.makedirs(od, exist_ok=True)
            np.save(os.path.join(od, f"disparity_{direction}.npy"), disp[direction])
        occ = so.occlusion_mask(disp["LR"], disp["RL"], 3)
        depth = so.depth(cam["fx"], r.baseline, disp["LR"])
        np.save(os.path.join(od, "occlusion_mask.npy"), occ)
        np.save(os.path.join(od, "depth.npy"), depth)
        cv2.imwrite(os.path.join(od, "depth.png"), depth)
        cv2.imwrite(os.path.join(od, "shading.png"), stereo.get_shading(depth, 1e-4))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=20)
    ap.add_argument("--points", type=int, default=200000)
    ap.add_argument("--width", type=int, default=1600)
    ap.add_argument("--height", type=int, default=1200)
    a = ap.parse_args()
    W, H, n = a.width, a.height, a.views
    dev = "cuda:0"
    cloud = scene.make_gaussians(a.points, seed=0)
    rigs, baseline = scene.make_stereo_cameras(n, W, H)
    res = dict(card=torch.cuda.get_device_name(0), power_limit_w=power_limit(), width=W, height=H, views=n,
               points=a.points)
    with tempfile.TemporaryDirectory() as tmp:
        dlnr = os.path.join(tmp, "base", "third_party", "DLNR")
        os.makedirs(os.path.join(dlnr, "core"))
        os.makedirs(os.path.join(dlnr, "pretrained"))
        open(os.path.join(dlnr, "core", "__init__.py"), "w").close()
        with open(os.path.join(dlnr, "core", "dlnr.py"), "w") as f:
            f.write(STANDIN)
        torch.save({"module.unused": torch.zeros(1)}, os.path.join(dlnr, "pretrained", "DLNR_Middlebury.pth"))

        def renderer(out):
            r = Renderer.from_scene(rigs, baseline, cloud, output_dir_root=out, args=Args(), device=dev)
            r.prepare_renderer()
            return r

        def per_view(fn):
            fn()  # warm-up pass over every view
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            return (time.perf_counter() - t0) * 1e3 / n

        r_mem = renderer(None)
        st = stereo.Stereo(os.path.join(tmp, "base"), r_mem, Args(), device=dev)
        res["run_in_memory_ms_per_view"] = per_view(lambda: st.run())
        r_mem._frames.clear()
        res["render_only_ms_per_view"] = per_view(lambda: [r_mem.render_image_pair(i) for i in range(n)])
        r_files = renderer(os.path.join(tmp, "files"))
        st_files = stereo.Stereo(os.path.join(tmp, "base"), r_files, Args(), device=dev)
        res["run_with_files_ms_per_view"] = per_view(lambda: st_files.run())
        r_files._frames.clear()
        r_ref = renderer(os.path.join(tmp, "ref"))
        res["reference_loop_ms_per_view"] = per_view(lambda: reference_loop(st_files, r_ref, n))

        # the kernels alone, on one view's frames and model outputs
        r_mem.keep_frames = True
        r_mem.render_image_pair(0)
        fr = r_mem.get_frame(0)
        block = stereo.pack_inputs(fr["left_u8"], fr["right_u8"])
        _, f_lr = st.model(block[0:1], block[1:2])
        _, f_rl = st.model(block[2:3], block[3:4])
        d_lr, d_rl = stereo.disparities(f_lr, f_rl, H, W, -1)
        num = stereo.depth_numerator(rigs[0]["left"]["fx"], baseline)
        kernels = {"pack_inputs": lambda: stereo.pack_inputs(fr["left_u8"], fr["right_u8"]),
                   "disparities": lambda: stereo.disparities(f_lr, f_rl, H, W, -1),
                   "occlusion_depth": lambda: stereo.occlusion_depth(d_lr, d_rl, 3, num)}
        for name, fn in kernels.items():
            for _ in range(5):
                fn()
            times = []
            for _ in range(50):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                fn()
                e1.record()
                e1.synchronize()
                times.append(e0.elapsed_time(e1))
            res[f"{name}_ms_median"] = float(np.median(times))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
