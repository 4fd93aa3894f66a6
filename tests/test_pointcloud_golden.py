"""The point-cloud oracle (tests/pointcloud_oracle.py) against Open3D 0.17.0's own ExtractPointCloud /
ExtractVoxelPointCloud, on the fixtures tests/golden/make_pointcloud_golden.py writes.  Open3D's order follows its hash
map, so the clouds are compared as sets sorted by point.  Skips while the fixtures do not exist."""
import os

import numpy as np
import pytest

from tests.golden.make_tsdf_golden import CASES, frames_from_npz

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _sorted(points, *attrs):
    order = np.lexsort(points.T[::-1])
    return [points[order]] + [a[order] for a in attrs]


@pytest.mark.parametrize("case", sorted(CASES))
def test_open3d_golden_point_clouds(oracle, case):
    path = os.path.join(GOLDEN, f"pointcloud_o3d_{case}.npz")
    if not os.path.exists(path):
        pytest.skip("no Open3D 0.17.0 point-cloud fixture: run tests/golden/make_pointcloud_golden.py where open3d 0.17.0 "
                    "imports")
    from tests.golden.make_pointcloud_golden import oracle_clouds
    from tests.golden.make_tsdf_golden import oracle_volume

    z = np.load(path)
    got = oracle_clouds(case, oracle_volume(case, frames_from_npz(z)))
    for a, b in zip(_sorted(got["points"], got["colors"], got["normals"]), _sorted(z["points"], z["colors"], z["normals"])):
        np.testing.assert_array_equal(a, b)
    for a, b in zip(_sorted(got["voxel_points"], got["voxel_colors"]), _sorted(z["voxel_points"], z["voxel_colors"])):
        np.testing.assert_array_equal(a, b)
