"""The Tanks and Temples kernels (gsb_tnt.cu, gs2mesh_b200/tnt.py) at their edges: the cases of tests/tnt_cases.py, each
checked bit for bit against oracle/tnt_oracle.py (NaN-aware where NaN can appear) and against an exact reference that
shares no code with it (Fraction arithmetic, exact integer sums, math.fsum).

  transform   n around the block size, v3 = 0 and v3 < 0, -0.0 entries, subnormal products, non-finite points
  crop        polygons of 3 .. 2048 vertices (2049 refused), points on vertices, edges and exact crossings, horizontal,
              vertical, zero-length and collinear edges, a bow-tie, both windings, degenerate and signed-zero slabs,
              coordinates where (b_u - a_u) overflows, n around the block size
  voxel       one voxel (zero key bits), planar and linear clouds, 63-bit keys (64 refused), a span of exactly
              vs * INT_MAX (one voxel more refused), the benchmark's voxel sizes on half-voxel lattices tens of metres out,
              one point per voxel, duplicates, -0.0 with +0.0
  moments     n around the 65536-lane stride, no correspondence, one in the last lane, d2 = 0 and subnormal, far clouds
  ICP         with_scaling=False (and a rigid motion recovered to 1e-9), the reflection branch, src_var = 0, collinear
              correspondences, max_iteration = 0, empty source and target, an init with -0.0 entries"""
import ctypes as C

import numpy as np
import pytest

from oracle import tnt_oracle as to
from tests import tnt_cases as tc

pytestmark = pytest.mark.gpu

TRANSFORM = tc.transform_cases()
CROP = tc.crop_cases()
VOXEL = tc.voxel_cases()
MOMENTS = tc.moment_cases()
ICP = tc.icp_cases()


@pytest.fixture(scope="module", autouse=True)
def _peak_memory():
    yield
    import torch

    if torch.cuda.is_available():
        print(f"\ntest_gpu_tnt_edges: peak torch memory {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def _same(a, b):
    """Bit for bit, except that any NaN equals any NaN (the GPU's NaN payload is not the host's)."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    if a.shape != b.shape or not np.array_equal(np.isnan(a), np.isnan(b)):
        return False
    ok = ~np.isnan(a)
    return np.array_equal(_bits(a[ok]), _bits(b[ok]))


def _dev(x, device):
    import torch

    return torch.as_tensor(np.ascontiguousarray(x, dtype=np.float64).reshape(-1, 3), device=device)


# ------------------------------------------------------------------------------------------------------- transform
@pytest.mark.parametrize("name", sorted(TRANSFORM))
def test_transform_edges(gsb_lib, cuda_device, name):
    from gs2mesh_b200.tnt import transform_points

    pts, T = TRANSFORM[name]
    got = transform_points(_dev(pts, cuda_device), T).cpu().numpy()
    with np.errstate(all="ignore"):
        want = to.transform(pts, T)
    assert _same(got, want)
    if name == "w_zero":  # x / 0: +-inf, NaN for 0 / 0
        assert not np.isfinite(got).any() and np.isnan(got[:, 0]).all() and np.isinf(got[:, 1:]).any()
        return
    if name.startswith("non_finite"):  # passed through, not refused
        bad = ~np.isfinite(pts).all(1)
        assert (~np.isfinite(got[bad]).all(1)).all() and np.isfinite(got[~bad]).all()
        return
    checked, skipped = tc.transform_exact_check(pts, T, got)
    assert checked == len(pts) and skipped == 0


# ------------------------------------------------------------------------------------------------------------ crop
def _crop_mask(case, device):
    """gsb_eval_crop_polygon's keep mask."""
    import torch

    from gs2mesh_b200 import _lib
    from gs2mesh_b200.evaluate import _stream

    p, P = _dev(case["points"], device), _dev(case["polygon"], device)
    n = p.shape[0]
    keep = torch.empty(n, dtype=torch.uint8, device=device)
    counter = torch.empty(1, dtype=torch.int32, device=device)
    host = torch.empty(1, dtype=torch.int32).pin_memory()
    _lib.check(_lib.lib().gsb_eval_crop_polygon(_lib.ptr(p), n, _lib.ptr(P), len(P), "xyz".index(case["axis"].lower()),
                                                float(case["axis_min"]), float(case["axis_max"]), _lib.ptr(keep),
                                                _lib.ptr(counter), _lib.ptr(host), _stream(device)))
    return keep.cpu().numpy().astype(bool)


@pytest.mark.parametrize("name", sorted(CROP))
def test_crop_edges(gsb_lib, cuda_device, name):
    from gs2mesh_b200.tnt import SelectionPolygonVolume, crop_point_cloud

    case = CROP[name]
    pts = case["points"]
    mask = _crop_mask(case, cuda_device)
    with np.errstate(all="ignore"):
        want = to.crop_mask(pts, case["axis"], case["axis_min"], case["axis_max"], case["polygon"])
    assert np.array_equal(mask, want)
    vol = SelectionPolygonVolume(case["axis"], case["axis_min"], case["axis_max"], case["polygon"])
    assert np.array_equal(_bits(crop_point_cloud(_dev(pts, cuda_device), vol).cpu().numpy()), _bits(pts[want]))
    keep, band = tc.crop_exact(case)
    assert np.array_equal(mask[~band], keep[~band])
    print(f"\ncrop {name}: {int(band.sum())} of {len(pts)} points within 8 ulp of a crossing, {int(mask.sum())} kept")
    if name != "huge":
        assert not band.any()
    if name == "slab_reversed":
        assert not mask.any()
    if name.startswith("zero_bounds"):  # -0.0 == +0.0: both signed zeros lie inside either slab
        z = pts[:, 2] == 0
        assert np.array_equal(mask[z], keep[z]) and mask[z].any() and not mask[~z].any()


def test_crop_refuses_2049_vertices(gsb_lib, cuda_device):
    from gs2mesh_b200.tnt import SelectionPolygonVolume, crop_point_cloud

    poly = np.concatenate([tc.star(tc.MAX_POLYGON + 1), np.zeros((tc.MAX_POLYGON + 1, 1))], 1)
    with pytest.raises(ValueError, match="2049 vertices.*2048"):
        crop_point_cloud(_dev(np.zeros((4, 3)), cuda_device), SelectionPolygonVolume("z", -1, 1, poly))


# ----------------------------------------------------------------------------------------------------------- voxel
@pytest.mark.parametrize("name", sorted(VOXEL))
def test_voxel_edges(gsb_lib, cuda_device, name):
    from gs2mesh_b200.tnt import voxel_down_sample

    pts, vs, expect = VOXEL[name]
    if expect != "ok":
        with pytest.raises(ValueError, match=expect):
            voxel_down_sample(_dev(pts, cuda_device), vs)
        if expect == "too small":  # Open3D's check, which the oracle restates
            with pytest.raises(ValueError, match="too small"):
                to.voxel_down_sample(pts, vs)
        return
    got = voxel_down_sample(_dev(pts, cuda_device), vs).cpu().numpy()
    assert _same(got, to.voxel_down_sample(pts, vs)[0])
    keys, groups, n_boundary = tc.voxel_exact(pts, vs)
    assert len(got) == len(keys)
    worst = tc.voxel_mean_check(pts, groups, got)
    print(f"\nvoxel {name}: {len(got)} voxels, {n_boundary} points within an ulp of a voxel boundary, worst mean error "
          f"{worst:.3g} of the bar")
    if name.startswith("one_voxel"):
        assert len(got) == 1
    if name == "all_distinct":
        assert len(got) == len(pts)
    if name == "signed_zero":  # 0.0 + (-0.0) = +0.0
        assert _bits(got[0]).tolist()[1:] == [0, 0]


# --------------------------------------------------------------------------------------------------------- moments
@pytest.mark.parametrize("name", sorted(MOMENTS))
def test_moment_edges(gsb_lib, cuda_device, name):
    import torch

    from gs2mesh_b200.tnt import _Moments

    src, tgt, idx, d2 = MOMENTS[name]
    n = len(src)
    m = _Moments(cuda_device)
    args = (_dev(src, cuda_device), torch.as_tensor(idx, device=cuda_device),
            torch.as_tensor(d2, dtype=torch.float64, device=cuda_device), _dev(tgt, cuda_device))
    s0, c0 = m(*args, 0)
    o0, oc0 = to.moments(src, tgt, idx, d2)
    assert c0 == oc0 == int((idx >= 0).sum())
    assert np.array_equal(_bits(s0[:7]), _bits(o0))
    tc.moment_fsum_check(tc.moment_values(src, tgt, idx, d2), n, s0[:7])
    mu = np.concatenate([o0[1:4], o0[4:7]]) * (1.0 / max(oc0, 1))
    s1, c1 = m(*args, 1, mu)
    assert c1 == c0 and np.array_equal(_bits(s1), _bits(to.moments(src, tgt, idx, d2, mu)[0]))
    tc.moment_fsum_check(tc.moment_values(src, tgt, idx, d2, mu), n, s1)
    assert np.array_equal(_bits(m(*args, 1, mu)[0]), _bits(s1)) and np.array_equal(_bits(m(*args, 0)[0]), _bits(s0))
    if name == "no_correspondence":
        assert c0 == 0 and not _bits(s0).any() and not _bits(s1).any()  # every sum +0.0
    if name == "last_lane":
        i = tc.MOMENT_LANES - 1
        assert c0 == 1 and s0[0] == d2[i] and np.array_equal(s0[1:7], np.concatenate([src[i], tgt[-1]]))


# ------------------------------------------------------------------------------------------------------------- ICP
@pytest.mark.parametrize("name", sorted(ICP))
def test_icp_edges(gsb_lib, cuda_device, name):
    from gs2mesh_b200.tnt import registration_icp

    c = ICP[name]
    with np.errstate(divide="ignore", invalid="ignore"):
        T, fit, rmse, it, hist = to.registration_icp(c["source"], c["target"], c["radius"], c["init"], c["with_scaling"],
                                                     c["relative"], c["relative"], c["max_iteration"])
        got = registration_icp(_dev(c["source"], cuda_device), _dev(c["target"], cuda_device), c["radius"], c["init"],
                               c["with_scaling"], c["relative"], c["relative"], c["max_iteration"])
    assert (got.iterations, got.fitness, got.inlier_rmse) == (it, fit, rmse)
    assert len(got.transformations) == len(hist)
    for a, b in zip(got.transformations, hist):
        assert _same(a, b)
    assert _same(got.transformation, T)
    if name == "rigid":
        assert fit == 1.0 and np.abs(got.transformation - tc.RIGID).max() < 1e-9
    if name == "one_source_point":  # (1 / src_var) * (D . S) = inf * 0
        assert it == 2 and np.isnan(got.transformation).all() and fit == 0.0
    if name == "max_iteration_0":
        assert it == 0 and got.transformations == [] and np.array_equal(got.transformation, np.eye(4))
    if name.startswith("empty"):
        assert (it, fit, rmse) == (1, 0.0, 0.0) and np.array_equal(got.transformation, np.eye(4))
    if name == "negative_zero_init":  # the init counts as the identity, and its -0.0 entries go into T's product
        assert np.array_equal(_bits(hist[0]), _bits(got.transformations[0]))
