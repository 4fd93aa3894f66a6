"""TEST INFRASTRUCTURE ONLY -- ctypes front-end of the CPU oracle (oracle/*.cpp) and of the
reference rasterizer built for sm_90a (oracle/_ref/libref_dgr.so).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / `--impl reference`
legs may import this module.  The product package gs2mesh_b200 never does.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_BUILD = os.path.join(_HERE, "_build")
_REF = os.path.join(_HERE, "_ref")

_f32p = C.POINTER(C.c_float)
_u32p = C.POINTER(C.c_uint32)
_i32p = C.POINTER(C.c_int)
_u8p = C.POINTER(C.c_uint8)
_f64p = C.POINTER(C.c_double)


def build(force: bool = False) -> None:
    """Compile the CPU oracle (always) and the reference rasterizer (only where the gs2mesh sources
    are present, $GS2MESH_REFERENCE; elsewhere a prebuilt oracle/_ref is used if there is one)."""
    need = force or not all(os.path.exists(os.path.join(_BUILD, n)) for n in ("liboracle.so", "liboracle_fma.so"))
    if not need:
        srcs = [os.path.join(_HERE, n) for n in ("raster_oracle.cpp", "tsdf_oracle.cpp", "Makefile")]
        newest = max(os.path.getmtime(s) for s in srcs)
        need = newest > min(os.path.getmtime(os.path.join(_BUILD, n)) for n in ("liboracle.so", "liboracle_fma.so"))
    if need:
        subprocess.run(["make", "-C", _HERE, "-s"], check=True)
    ref_root = os.environ.get("GS2MESH_REFERENCE", "/root/reference")
    if os.path.isdir(ref_root):
        so = os.path.join(_REF, "libref_dgr.so")
        shim = os.path.join(_HERE, "ref_dgr_capi.cu")
        if force or not os.path.exists(so) or os.path.getmtime(shim) > os.path.getmtime(so):
            subprocess.run(["bash", os.path.join(_HERE, "build_ref.sh")], check=True)


def _ptr(a, ty):
    return None if a is None else a.ctypes.data_as(ty)


def _f32(a):
    return None if a is None else np.ascontiguousarray(a, dtype=np.float32)


class _Lib:
    def __init__(self, name):
        path = os.path.join(_BUILD, name)
        if not os.path.exists(path):
            build()
        self.lib = C.CDLL(path)
        L = self.lib
        L.orc_higher_msb.restype = C.c_uint32
        L.orc_higher_msb.argtypes = [C.c_uint32]
        L.orc_preprocess.restype = None
        L.orc_preprocess.argtypes = [C.c_int, C.c_int, C.c_int, _f32p, _f32p, C.c_float, _f32p, _f32p, _f32p, _f32p, _f32p,
                                     _f32p, _f32p, _f32p, C.c_int, C.c_int, C.c_float, C.c_float, _i32p, _f32p, _f32p,
                                     _f32p, _f32p, _f32p, _u32p]
        L.orc_forward.restype = C.c_int64
        L.orc_forward.argtypes = [C.c_int, C.c_int, C.c_int, _f32p, C.c_int, C.c_int, _f32p, _f32p, _f32p, _f32p, _f32p,
                                  C.c_float, _f32p, _f32p, _f32p, _f32p, _f32p, C.c_float, C.c_float, _f32p, _f32p, _f32p,
                                  _u32p, _i32p, _u32p, C.c_int64, _u32p]


_libs = {}


def _lib(fma=False):
    key = "liboracle_fma.so" if fma else "liboracle.so"
    if key not in _libs:
        _libs[key] = _Lib(key)
    return _libs[key].lib


def higher_msb(n: int) -> int:
    return int(_lib().orc_higher_msb(n))


def _raster_inputs(means3D, opacities, shs, colors_precomp, scales, rotations, cov3D_precomp, view, proj, campos, bg):
    d = dict(means3D=_f32(means3D).reshape(-1, 3), opacities=_f32(opacities).reshape(-1), shs=_f32(shs),
             colors=_f32(colors_precomp), scales=_f32(scales), rotations=_f32(rotations), cov3D=_f32(cov3D_precomp),
             view=_f32(view).reshape(16), proj=_f32(proj).reshape(16), campos=_f32(campos).reshape(3),
             bg=_f32(bg).reshape(3) if bg is not None else None)
    if (d["shs"] is None) == (d["colors"] is None):
        raise ValueError("provide exactly one of shs / colors_precomp")
    if (d["cov3D"] is None) == (d["scales"] is None or d["rotations"] is None):
        raise ValueError("provide exactly one of (scales, rotations) / cov3D_precomp")
    return d


def preprocess(means3D, opacities, view, proj, campos, W, H, tan_fovx, tan_fovy, shs=None, colors_precomp=None, scales=None,
               rotations=None, cov3D_precomp=None, sh_degree=3, scale_modifier=1.0, fma=False):
    """Per-Gaussian stage; returns dict(radii, xy, depths, cov3d, rgb, conic_opacity, tiles_touched)."""
    d = _raster_inputs(means3D, opacities, shs, colors_precomp, scales, rotations, cov3D_precomp, view, proj, campos, None)
    P = d["means3D"].shape[0]
    M = 0 if d["shs"] is None else d["shs"].shape[1]
    out = dict(radii=np.zeros(P, np.int32), xy=np.zeros((P, 2), np.float32), depths=np.zeros(P, np.float32),
               cov3d=np.zeros((P, 6), np.float32), rgb=np.zeros((P, 3), np.float32),
               conic_opacity=np.zeros((P, 4), np.float32), tiles_touched=np.zeros(P, np.uint32))
    _lib(fma).orc_preprocess(P, sh_degree, M, _ptr(d["means3D"], _f32p), _ptr(d["scales"], _f32p), scale_modifier,
                             _ptr(d["rotations"], _f32p), _ptr(d["opacities"], _f32p), _ptr(d["shs"], _f32p),
                             _ptr(d["cov3D"], _f32p), _ptr(d["colors"], _f32p), _ptr(d["view"], _f32p),
                             _ptr(d["proj"], _f32p), _ptr(d["campos"], _f32p), W, H, tan_fovx, tan_fovy,
                             _ptr(out["radii"], _i32p), _ptr(out["xy"], _f32p), _ptr(out["depths"], _f32p),
                             _ptr(out["cov3d"], _f32p), _ptr(out["rgb"], _f32p), _ptr(out["conic_opacity"], _f32p),
                             _ptr(out["tiles_touched"], _u32p))
    return out


def forward(means3D, opacities, view, proj, campos, W, H, tan_fovx, tan_fovy, bg=(0, 0, 0), shs=None, colors_precomp=None,
            scales=None, rotations=None, cov3D_precomp=None, sh_degree=3, scale_modifier=1.0, fma=False, want_list=False):
    """Full forward; returns dict(color[3,H,W], depth[H,W], final_T[H,W], n_contrib, radii, num_rendered
    [, point_list, ranges])."""
    d = _raster_inputs(means3D, opacities, shs, colors_precomp, scales, rotations, cov3D_precomp, view, proj, campos, bg)
    P = d["means3D"].shape[0]
    M = 0 if d["shs"] is None else d["shs"].shape[1]
    ntiles = ((W + 15) // 16) * ((H + 15) // 16)
    out = dict(color=np.zeros((3, H, W), np.float32), depth=np.zeros((H, W), np.float32),
               final_T=np.zeros((H, W), np.float32), n_contrib=np.zeros((H, W), np.uint32), radii=np.zeros(P, np.int32))
    plist = ranges = None
    cap = 0
    if want_list:
        pre = preprocess(means3D, opacities, view, proj, campos, W, H, tan_fovx, tan_fovy, shs, colors_precomp, scales,
                         rotations, cov3D_precomp, sh_degree, scale_modifier, fma)
        cap = int(pre["tiles_touched"].astype(np.int64).sum())
        plist = np.zeros(max(cap, 1), np.uint32)
        ranges = np.zeros((ntiles, 2), np.uint32)
    n = _lib(fma).orc_forward(P, sh_degree, M, _ptr(d["bg"], _f32p), W, H, _ptr(d["means3D"], _f32p), _ptr(d["shs"], _f32p),
                              _ptr(d["colors"], _f32p), _ptr(d["opacities"], _f32p), _ptr(d["scales"], _f32p),
                              scale_modifier, _ptr(d["rotations"], _f32p), _ptr(d["cov3D"], _f32p), _ptr(d["view"], _f32p),
                              _ptr(d["proj"], _f32p), _ptr(d["campos"], _f32p), tan_fovx, tan_fovy,
                              _ptr(out["color"], _f32p), _ptr(out["depth"], _f32p), _ptr(out["final_T"], _f32p),
                              _ptr(out["n_contrib"], _u32p), _ptr(out["radii"], _i32p), _ptr(plist, _u32p), cap,
                              _ptr(ranges, _u32p))
    out["num_rendered"] = int(n)
    if want_list:
        out["point_list"] = plist[:cap]
        out["ranges"] = ranges
    return out


# ----------------------------------------------------------------------------- TSDF

def _tsdf_lib():
    L = _lib(False)
    if not getattr(L, "_tsdf_ready", False):
        L.orc_tsdf_create.restype = C.c_void_p
        L.orc_tsdf_create.argtypes = [C.c_double, C.c_double, C.c_int]
        L.orc_tsdf_destroy.argtypes = [C.c_void_p]
        L.orc_tsdf_set_variant.argtypes = [C.c_int]
        L.orc_tsdf_num_units.restype = C.c_int64
        L.orc_tsdf_num_units.argtypes = [C.c_void_p]
        L.orc_depth_convert.argtypes = [_f32p, C.c_int64, C.c_double, C.c_double, _f32p]
        L.orc_depth_multiplier.argtypes = [C.c_int, C.c_int, C.c_double, C.c_double, C.c_double, C.c_double, _f32p]
        L.orc_tsdf_integrate.restype = C.c_int64
        L.orc_tsdf_integrate.argtypes = [C.c_void_p, _f32p, _u8p, C.c_int, C.c_int, C.c_double, C.c_double, C.c_double,
                                         C.c_double, _f64p, C.c_int]
        L.orc_tsdf_unit_indices.argtypes = [C.c_void_p, _i32p]
        L.orc_tsdf_unit_data.argtypes = [C.c_void_p, C.c_int64, _f32p, _f32p, _f64p]
        L.orc_tsdf_export_bricks.restype = C.c_int64
        L.orc_tsdf_export_bricks.argtypes = [C.c_void_p, _i32p, _i32p, _f32p, _u8p]
        L._tsdf_ready = True
    return L


def tsdf_set_variant(bits: int) -> None:
    """Sensitivity study of the restatement's two DOUBT points (oracle/tsdf_oracle.cpp): bit 0 pairwise 4x4*4x1 sum,
    bit 1 `sdf / trunc`, bit 2 FMA-contracted product; bit 3 keeps colour as the CUDA kernel's fp32 running mean instead
    of Open3D's fp64.  0 restores the restatement.  Process-wide: reset after use."""
    _tsdf_lib().orc_tsdf_set_variant(int(bits))


def depth_convert(depth, depth_scale, depth_trunc):
    """RGBDImage.create_from_color_and_depth's depth step (T0b)."""
    src = np.ascontiguousarray(depth, dtype=np.float32)
    out = np.empty_like(src)
    _tsdf_lib().orc_depth_convert(_ptr(src, _f32p), src.size, float(depth_scale), float(depth_trunc), _ptr(out, _f32p))
    return out


def depth_multiplier(W, H, fx, fy, cx, cy):
    out = np.empty((H, W), np.float32)
    _tsdf_lib().orc_depth_multiplier(W, H, fx, fy, cx, cy, _ptr(out, _f32p))
    return out


class OracleTSDFVolume:
    """Open3D-0.17-equivalent ScalableTSDFVolume restatement (hashed 16^3 units, unbounded)."""

    def __init__(self, voxel_length, sdf_trunc, with_color=True):
        self._L = _tsdf_lib()
        self._h = self._L.orc_tsdf_create(float(voxel_length), float(sdf_trunc), int(with_color))
        self.voxel_length = float(voxel_length)
        self.sdf_trunc = float(sdf_trunc)
        self.with_color = with_color

    def __del__(self):
        if getattr(self, "_h", None):
            self._L.orc_tsdf_destroy(self._h)
            self._h = None

    def integrate(self, depth, rgb, W, H, fx, fy, cx, cy, extrinsic_w2c, depth_scale=1.0, depth_trunc=1e30, threads=1):
        """`depth` is the raw float depth handed to create_from_color_and_depth."""
        d = depth_convert(depth, depth_scale, depth_trunc).reshape(H, W)
        c = None if rgb is None else np.ascontiguousarray(rgb, dtype=np.uint8).reshape(H, W, 3)
        e = np.ascontiguousarray(extrinsic_w2c, dtype=np.float64).reshape(16)
        return int(self._L.orc_tsdf_integrate(self._h, _ptr(d, _f32p), _ptr(c, _u8p), W, H, fx, fy, cx, cy, _ptr(e, _f64p),
                                              int(threads)))

    @property
    def num_units(self):
        return int(self._L.orc_tsdf_num_units(self._h))

    def unit_indices(self):
        out = np.zeros((self.num_units, 3), np.int32)
        if self.num_units:
            self._L.orc_tsdf_unit_indices(self._h, _ptr(out, _i32p))
        return out

    def unit_data(self, i):
        t = np.empty(4096, np.float32)
        w = np.empty(4096, np.float32)
        c = np.empty((4096, 3), np.float64) if self.with_color else None
        self._L.orc_tsdf_unit_data(self._h, i, _ptr(t, _f32p), _ptr(w, _f32p), _ptr(c, _f64p))
        return t, w, c

    def export_bricks(self, brick_origin, brick_count):
        """Dense window in the CUDA path's brick layout: returns (tsdf_weight[nb,4096,2], allocated[nb], n_outside)."""
        b0 = np.ascontiguousarray(brick_origin, dtype=np.int32)
        nb = np.ascontiguousarray(brick_count, dtype=np.int32)
        total = int(np.prod(nb.astype(np.int64)))
        tw = np.zeros((total, 4096, 2), np.float32)
        alloc = np.zeros(total, np.uint8)
        outside = self._L.orc_tsdf_export_bricks(self._h, _ptr(b0, _i32p), _ptr(nb, _i32p), _ptr(tw, _f32p), _ptr(alloc, _u8p))
        return tw, alloc, int(outside)


# ----------------------------------------------------------------------------- reference rasterizer (GPU)

_ref = None


def ref_available() -> bool:
    return os.path.exists(os.path.join(_REF, "libref_dgr.so"))


def _ref_lib():
    global _ref
    if _ref is None:
        L = C.CDLL(os.path.join(_REF, "libref_dgr.so"))
        vp = C.c_void_p
        L.ref_dgr_forward.restype = C.c_int
        L.ref_dgr_forward.argtypes = [C.c_int, C.c_int, C.c_int, vp, C.c_int, C.c_int, vp, vp, vp, vp, vp, C.c_float, vp, vp,
                                      vp, vp, vp, C.c_float, C.c_float, C.c_int, vp, vp, C.c_int]
        L.ref_dgr_last_error.restype = C.c_char_p
        L.ref_dgr_last_final_T.argtypes = [C.c_int, C.c_int, vp]
        L.ref_dgr_last_geometry.argtypes = [C.c_int, vp, vp, vp, vp, vp]
        _ref = L
    return _ref


def ref_forward_torch(means3D, opacities, view, proj, campos, W, H, tan_fovx, tan_fovy, bg, shs=None, colors_precomp=None,
                      scales=None, rotations=None, cov3D_precomp=None, sh_degree=3, scale_modifier=1.0, want_geometry=False):
    """Runs the UNMODIFIED reference rasterizer (built for sm_90a) on CUDA torch tensors.
    Returns dict(color, radii, num_rendered, final_T [, depths, xy, conic_opacity, rgb, tiles_touched])."""
    import torch

    L = _ref_lib()
    dev = means3D.device
    P = means3D.shape[0]
    M = 0 if shs is None else shs.shape[1]

    def p(t):
        return None if t is None else C.c_void_p(t.data_ptr())

    keep = [t.contiguous().float() if t is not None else None
            for t in (bg, means3D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp, view, proj, campos)]
    bg_, m_, sh_, cp_, op_, sc_, ro_, c3_, v_, pr_, cam_ = keep
    color = torch.zeros(3, H, W, device=dev, dtype=torch.float32)
    radii = torch.zeros(P, device=dev, dtype=torch.int32)
    torch.cuda.synchronize()
    n = L.ref_dgr_forward(P, sh_degree, M, p(bg_), W, H, p(m_), p(sh_), p(cp_), p(op_), p(sc_), scale_modifier, p(ro_), p(c3_),
                          p(v_), p(pr_), p(cam_), tan_fovx, tan_fovy, 0, p(color), p(radii), 0)
    if n < 0:
        raise RuntimeError(L.ref_dgr_last_error().decode())
    torch.cuda.synchronize()
    out = dict(color=color, radii=radii, num_rendered=int(n))
    ft = torch.empty(H, W, device=dev, dtype=torch.float32)
    if L.ref_dgr_last_final_T(W, H, p(ft)) == 0:
        out["final_T"] = ft
    if want_geometry:
        g = dict(depths=torch.zeros(P, device=dev), xy=torch.zeros(P, 2, device=dev), conic_opacity=torch.zeros(P, 4, device=dev),
                 rgb=torch.zeros(P, 3, device=dev), tiles_touched=torch.zeros(P, device=dev, dtype=torch.int32))
        L.ref_dgr_last_geometry(P, p(g["depths"]), p(g["xy"]), p(g["conic_opacity"]), p(g["rgb"]), p(g["tiles_touched"]))
        out.update(g)
    torch.cuda.synchronize()
    return out


# ----------------------------------------------------------------------------- marching cubes (Open3D ExtractTriangleMesh)

def _mc_tables():
    import re

    text = open(os.path.join(os.path.dirname(_HERE), "include", "gsb_mc_tables.h")).read()

    def grab(name, shape):
        m = re.search(name + r"\[[^\]]*\](?:\[[^\]]*\])?\s*=\s*\{(.*?)\};", text, re.S)
        return np.array([int(v) for v in re.findall(r"-?\d+", m.group(1))]).reshape(shape)

    return grab("kMcShift", (8, 3)), grab("kMcEdgeShift", (12, 4)), grab("kMcEdgeToVert", (12, 2)), grab("kMcTriTable", (256, 16))


def extract_mesh_from_bricks(tw, brick_origin, brick_count, voxel_length, color=None):
    """CPU restatement of ScalableTSDFVolume::ExtractTriangleMesh on a dense brick window
    (tw: [n_bricks,4096,2] as returned by OracleTSDFVolume.export_bricks; unallocated units have weight 0,
    which is what Open3D's hash-map miss yields).  Returns dict(keys, vertices, colors, triangles, cubes):
    `keys[i]` = (gx,gy,gz,axis) of vertex i in window voxel coordinates, vertices fp64 like Open3D, `cubes[t]` = (x,y,z)
    of the cube triangle t came from, in window voxel coordinates.  Triangles follow the walk over the whole window in
    x, y, z order, each cube's in the case table's order."""
    shift, edge_shift, e2v, tri = _mc_tables()
    nbx, nby, nbz = (int(v) for v in brick_count)
    g = np.asarray(tw).reshape(nbx, nby, nbz, 16, 16, 16, 2).transpose(0, 3, 1, 4, 2, 5, 6).reshape(nbx * 16, nby * 16, nbz * 16, 2)
    f, w = g[..., 0], g[..., 1]
    col = None
    if color is not None:
        col = np.asarray(color).reshape(nbx, nby, nbz, 16, 16, 16, -1).transpose(0, 3, 1, 4, 2, 5, 6).reshape(
            nbx * 16, nby * 16, nbz * 16, -1)[..., :3]
    X, Y, Z = f.shape
    fp = np.pad(f, ((0, 1),) * 3)
    wp = np.pad(w, ((0, 1),) * 3)  # outside the window == unallocated == weight 0
    valid = np.ones((X, Y, Z), bool)
    case = np.zeros((X, Y, Z), np.int32)
    for i in range(8):
        sx, sy, sz = shift[i]
        valid &= wp[sx:sx + X, sy:sy + Y, sz:sz + Z] != 0
        case |= (fp[sx:sx + X, sy:sy + Y, sz:sz + Z] < 0).astype(np.int32) << i
    active = np.argwhere(valid & (case != 0) & (case != 255))
    vmap, verts, cols, tris, keys, cubes = {}, [], [], [], [], []
    half = voxel_length * 0.5
    b0 = np.asarray(brick_origin, dtype=np.int64) * 16
    for x, y, z in active:
        c = case[x, y, z]
        row = tri[c]
        idx = {}
        for e in set(int(v) for v in row if v >= 0):
            es = edge_shift[e]
            key = (int(x + es[0]), int(y + es[1]), int(z + es[2]), int(es[3]))
            if key not in vmap:
                vmap[key] = len(verts)
                c0 = np.array([x, y, z]) + shift[e2v[e][0]]
                c1 = np.array([x, y, z]) + shift[e2v[e][1]]
                f0 = abs(float(fp[tuple(c0)]))
                f1 = abs(float(fp[tuple(c1)]))
                pt = half + voxel_length * (b0 + np.array(key[:3], dtype=np.float64))
                pt[key[3]] += f0 * voxel_length / (f0 + f1)
                verts.append(pt)
                keys.append(key)
                if col is not None:
                    k0 = col[tuple(c0)].astype(np.float64) / 255.0
                    k1 = col[tuple(c1)].astype(np.float64) / 255.0
                    cols.append((f1 * k0 + f0 * k1) / (f0 + f1))
            idx[e] = vmap[key]
        for t in range(0, 15, 3):
            if row[t] < 0:
                break
            tris.append((idx[int(row[t])], idx[int(row[t + 2])], idx[int(row[t + 1])]))
            cubes.append((x, y, z))
    return dict(keys=np.array(keys, np.int64).reshape(-1, 4), vertices=np.array(verts, np.float64).reshape(-1, 3),
                colors=np.array(cols, np.float64).reshape(-1, 3) if col is not None else None,
                triangles=np.array(tris, np.int64).reshape(-1, 3), cubes=np.array(cubes, np.int64).reshape(-1, 3))


# ---------------------------------------------------------------------------------------------------------------
# T0 mask filters: numpy restatement of cv2.erode / cv2.dilate / cv2.morphologyEx(MORPH_CLOSE) with a k x k kernel of
# ones and default anchor / border, as called at gs2mesh_utils/tsdf_utils.py:73-77.  OpenCV (opencv-python 4.x, an
# un-vendored dependency of the reference) places the anchor at k/2 and ignores pixels outside the image; pinned
# against cv2 itself in tests/test_oracle_tsdf.py::test_mask_morphology_matches_cv2.
def mask_morphology(mask, k, dilate):
    m = np.asarray(mask, dtype=np.uint8)
    h, w = m.shape
    ax = k // 2
    neutral = 0 if dilate else 255
    pad = np.full((h + k - 1, w + k - 1), neutral, np.uint8)
    pad[ax:ax + h, ax:ax + w] = m
    out = np.full((h, w), neutral, np.uint8)
    op = np.maximum if dilate else np.minimum
    for dy in range(k):
        for dx in range(k):
            out = op(out, pad[dy:dy + h, dx:dx + w])
    return out


def filter_object_mask(mask, closing_k=10, erosion_k=10, invert=False):
    """tsdf_utils.py:69-77 -> bool mask."""
    m = np.asarray(mask).astype(bool)
    if invert:
        m = ~m
    closing = mask_morphology(mask_morphology(m.astype(np.uint8), closing_k, True), closing_k, False)
    return mask_morphology(closing, erosion_k, False) > 0.5
