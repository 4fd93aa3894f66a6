"""The C-ABI library builds for sm_90a, loads without a GPU and exports exactly the symbols
include/gs2mesh_b200.h declares (no compute calls here)."""
import os
import re

from gs2mesh_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    text = open(os.path.join(ROOT, "include", "gs2mesh_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(gsb_[a-z0-9_]+)\s*\(", text)))


def test_header_symbols_exported_and_bound(gsb_lib):
    names = _declared()
    assert len(names) >= 15
    for n in names:
        assert hasattr(gsb_lib, n), f"{n} declared in the header but not exported"
        assert n in _lib.SIGNATURES, f"{n} has no ctypes signature"
    assert sorted(_lib.SIGNATURES) == names


def test_version_and_host_only_queries(gsb_lib):
    assert gsb_lib.gsb_version() == 100
    assert gsb_lib.gsb_kernel_launch_count() == 0
    small = gsb_lib.gsb_raster_workspace_bytes(1000, 640, 480, 10_000)
    big = gsb_lib.gsb_raster_workspace_bytes(1_000_000, 1600, 1200, 8_000_000)
    assert 0 < small < big
    # 40 B of records + 12 B bookkeeping per Gaussian, 24 B per instance + sort scratch
    assert big >= 1_000_000 * 52 + 8_000_000 * 24


def test_argument_validation_without_gpu_reduce_reports_need(gsb_lib):
    import ctypes as C

    assert gsb_lib.gsb_raster_forward(None, None) == _lib.GSB_ERR_INVALID
    a = _lib.GsbRasterArgs(P=10, width=64, height=64)
    assert gsb_lib.gsb_raster_forward(C.byref(a), None) == _lib.GSB_ERR_INVALID
    assert b"required" in gsb_lib.gsb_last_error()
    assert gsb_lib.gsb_tsdf_create(None) is None
    # stereo-pair entry point: both argument blocks are validated before anything is enqueued
    assert gsb_lib.gsb_raster_forward_pair(C.byref(a), None, None, None) == _lib.GSB_ERR_INVALID
    # brick pool descriptor: hash_slots must be a power of two >= 2 * pool_bricks
    d = _lib.GsbVolumeDesc(voxel_length=0.01, sdf_trunc=0.04, pool_bricks=100, hash_slots=128)
    for f in ("tsdf_weight", "brick_index", "hash_keys", "hash_vals", "hash_stamp", "brick_list", "counters"):
        setattr(d, f, 256)  # any non-NULL value: create() only records the pointers
    assert gsb_lib.gsb_tsdf_create(C.byref(d)) is None and b"power of two" in gsb_lib.gsb_last_error()
    d.hash_slots = 256
    h = gsb_lib.gsb_tsdf_create(C.byref(d))
    assert h is not None
    assert gsb_lib.gsb_tsdf_reduce_scratch_bytes(h, 8, 1000) > 1000 * 4096 * 8  # (sum, w) payload of the union, no colour
    assert gsb_lib.gsb_tsdf_reduce(h, None, 8, 0, 0, None, 0, None, None) == _lib.GSB_ERR_INVALID
    # the scratch need is written only with GSB_ERR_WORKSPACE: a refused call leaves it as it was
    need = C.c_size_t(7)
    assert gsb_lib.gsb_tsdf_reduce(h, None, 8, 0, 0, None, 0, C.byref(need), None) == _lib.GSB_ERR_INVALID
    assert need.value == 7
    gsb_lib.gsb_tsdf_destroy(h)


def test_undefined_flag_bits_are_refused(gsb_lib):
    """A flags word with a bit outside the GSB_RASTER_* set fails validation, before anything is enqueued.  The blend-kernel
    (bits 8..10) and SH-staging (bits 12..13) selector fields no longer exist; a caller still passing them gets an error."""
    import ctypes as C

    P, W, H, cap = 1000, 64, 48, 4000
    need = gsb_lib.gsb_raster_workspace_bytes(P, W, H, cap)
    ok = _lib.RASTER_EXACT_TILE_CULL | _lib.RASTER_FAST_EXP

    def args(flags, workspace):
        # any non-NULL pointers: validation only checks them for NULL, nothing is dereferenced before it passes
        ptrs = {f: 256 for f in ("background", "means3D", "shs", "opacities", "scales", "rotations", "viewmatrix", "projmatrix",
                                 "cam_pos", "out_color")}
        return _lib.GsbRasterArgs(P=P, sh_degree=3, sh_coeffs=16, width=W, height=H, scale_modifier=1.0, tan_fovx=0.5,
                                  tan_fovy=0.4, flags=flags, workspace=workspace, workspace_bytes=need, max_instances=cap, **ptrs)

    for bit in (1 << 8, 1 << 9, 1 << 10, 1 << 12, 1 << 13, 1 << 31):
        msg = b"undefined bits 0x%x" % bit
        bad = args(ok | bit, 4096)
        assert gsb_lib.gsb_raster_forward(C.byref(bad), None) == _lib.GSB_ERR_INVALID
        assert msg in gsb_lib.gsb_last_error()
        good = args(ok, 8192)
        for left, right in ((bad, good), (good, bad)):
            assert gsb_lib.gsb_raster_forward_pair(C.byref(left), C.byref(right), None, None) == _lib.GSB_ERR_INVALID
            assert msg in gsb_lib.gsb_last_error()


def test_struct_layout_matches_header():
    import ctypes as C

    # 5 int32 (+4 pad) | 8 ptr | float (+4) | 3 ptr | 2 float | int32 | uint32 | 8 ptr/size fields
    assert C.sizeof(_lib.GsbRasterArgs) == 24 + 8 * 8 + 8 + 3 * 8 + 16 + 8 * 8
    # 2 double | 2 uint32 | 8 pointers
    assert C.sizeof(_lib.GsbVolumeDesc) == 16 + 8 + 8 * 8
    assert _lib.GsbVolumeDesc.tsdf_weight.offset == 24 and _lib.GsbVolumeDesc.counters.offset == 24 + 7 * 8


def test_sass_contains_bulk_tma():
    """The preprocess kernel stages parameters with 1-D bulk TMA (UBLKCP in SASS)."""
    import shutil
    import subprocess

    if shutil.which("cuobjdump") is None:
        return
    sass = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True).stdout
    assert "UBLKCP" in sass and "sm_90a" in sass
