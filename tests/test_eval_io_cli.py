"""Host side of the mesh evaluator: PLY / .mat readers and writers, and the command line's flags, defaults and printed
line (eval.py:30-40, 157-166; parsed the way run_and_evaluate_dtu.py:57-59 does)."""
import json
import os

import numpy as np
import pytest

from gs2mesh_b200 import evaluate as ev
from gs2mesh_b200 import io as gio
from gs2mesh_b200.mesh import TriangleMesh


def _ascii_ply(path, xyz, tris, vtype, ltype):
    lines = ["ply", "format ascii 1.0", f"element vertex {len(xyz)}"] + [f"property {vtype} {c}" for c in "xyz"]
    if tris is not None:
        lines += [f"element face {len(tris)}", f"property list {ltype} vertex_indices"]
    lines += ["end_header"] + [" ".join(repr(float(v)) for v in row) for row in xyz]
    if tris is not None:
        lines += ["3 " + " ".join(str(int(v)) for v in t) for t in tris]
    with open(path, "w") as f:
        f.write("\n".join(lines) + "\n")


def _binary_ply(path, xyz, tris, vtype, ltype):
    vt = {"float": "<f4", "double": "<f8"}[vtype]
    ct, it = {"uchar int": ("u1", "<i4"), "uchar uint": ("u1", "<u4"), "int int": ("<i4", "<i4")}[ltype]
    head = ["ply", "format binary_little_endian 1.0", f"element vertex {len(xyz)}"] + [f"property {vtype} {c}" for c in "xyz"]
    head += [f"element face {len(tris)}", f"property list {ltype} vertex_indices", "end_header"]
    face = np.zeros(len(tris), dtype=[("n", ct), ("v", it, (3,))])
    face["n"], face["v"] = 3, tris
    with open(path, "wb") as f:
        f.write(("\n".join(head) + "\n").encode())
        f.write(np.asarray(xyz, vt).tobytes())
        f.write(face.tobytes())


@pytest.fixture
def mesh_data():
    rng = np.random.default_rng(0)
    return rng.normal(size=(50, 3)) * 100, rng.integers(0, 50, size=(80, 3))


@pytest.mark.parametrize("vtype", ["float", "double"])
@pytest.mark.parametrize("ltype", ["uchar int", "uchar uint", "int int"])
def test_triangle_mesh_ply_round_trip(tmp_path, mesh_data, vtype, ltype):
    xyz, tris = mesh_data
    want = xyz.astype(np.float32).astype(np.float64) if vtype == "float" else xyz
    for writer, name in ((_binary_ply, "b.ply"), (_ascii_ply, "a.ply")):
        path = str(tmp_path / name)
        writer(path, xyz, tris, vtype, ltype)
        v, t = gio.read_triangle_mesh_ply(path)
        assert np.array_equal(v, want) and np.array_equal(t, tris) and v.dtype == np.float64 and t.dtype == np.int64


def test_mesh_writer_and_point_cloud_round_trip(tmp_path, mesh_data):
    xyz, tris = mesh_data
    path = str(tmp_path / "m.ply")
    TriangleMesh(xyz, tris, vertex_colors=np.full((len(xyz), 3), 0.5)).write_ply(path)
    v, t = gio.read_triangle_mesh_ply(path)
    assert np.array_equal(v, xyz) and np.array_equal(t, tris)
    assert np.array_equal(gio.read_point_cloud_ply(path), xyz)
    cols = np.random.default_rng(1).uniform(size=(len(xyz), 3))
    gio.write_point_cloud_ply(str(tmp_path / "p.ply"), xyz, cols)
    tab = gio._read_vertex_table(str(tmp_path / "p.ply"))
    assert np.array_equal(gio.read_point_cloud_ply(str(tmp_path / "p.ply")), xyz)
    assert np.array_equal(np.stack([tab["red"], tab["green"], tab["blue"]], 1), np.rint(cols * 255).astype(np.uint8))
    _ascii_ply(str(tmp_path / "pa.ply"), xyz, None, "double", None)
    assert np.array_equal(gio.read_point_cloud_ply(str(tmp_path / "pa.ply")), xyz)


def test_non_triangle_faces_rejected(tmp_path):
    path = str(tmp_path / "q.ply")
    with open(path, "w") as f:
        f.write("ply\nformat ascii 1.0\nelement vertex 4\nproperty float x\nproperty float y\nproperty float z\n"
                "element face 1\nproperty list uchar int vertex_indices\nend_header\n0 0 0\n1 0 0\n1 1 0\n0 1 0\n4 0 1 2 3\n")
    with pytest.raises(ValueError):
        gio.read_triangle_mesh_ply(path)


def test_mat_round_trip(tmp_path):
    from scipy.io import loadmat, savemat

    obs = np.zeros((5, 6, 7), np.uint8)
    obs[1:4, 2:5, 3:6] = 1
    bb = np.array([[-10.0, -20.0, -30.0], [10.0, 20.0, 30.0]])
    savemat(str(tmp_path / "ObsMask1_10.mat"), {"ObsMask": obs, "BB": bb, "Res": np.array([[4.0]])})
    savemat(str(tmp_path / "Plane1.mat"), {"P": np.array([[0.0], [0.0], [1.0], [5.0]])})
    m = loadmat(str(tmp_path / "ObsMask1_10.mat"))
    assert np.array_equal(m["ObsMask"], obs) and np.array_equal(m["BB"], bb) and m["Res"].reshape(-1)[0] == 4.0
    assert loadmat(str(tmp_path / "Plane1.mat"))["P"].reshape(4).tolist() == [0.0, 0.0, 1.0, 5.0]


def test_cli_flags_and_defaults_match_eval_py():
    a = ev.build_parser().parse_args([])
    assert vars(a) == {"data": "data_in.ply", "scan": 1, "mode": "mesh", "dataset_dir": ".", "vis_out_dir": ".",
                       "downsample_density": 0.2, "patch_size": 60, "max_dist": 20, "visualize_threshold": 10, "seed": 0}
    a = ev.build_parser().parse_args(["--data", "x.ply", "--scan", "24", "--mode", "pcd", "--dataset_dir", "d",
                                      "--vis_out_dir", "o", "--downsample_density", "0.5", "--patch_size", "30",
                                      "--max_dist", "10", "--visualize_threshold", "5", "--seed", "3"])
    assert (a.scan, a.mode, a.downsample_density, a.patch_size, a.max_dist, a.visualize_threshold, a.seed) == \
        (24, "pcd", 0.5, 30.0, 10.0, 5.0, 3)
    with pytest.raises(SystemExit):
        ev.build_parser().parse_args(["--mode", "voxels"])


def test_printed_line_parses_like_run_and_evaluate_dtu(tmp_path, capsys):
    r = {"mean_d2s": np.float64(0.1) + np.float64(1e-17), "mean_s2d": np.float64(2.0 / 3.0)}
    r["overall"] = (r["mean_d2s"] + r["mean_s2d"]) / 2
    ev.report(r, str(tmp_path))
    output = capsys.readouterr().out
    output = output.replace(" ", ",").split(",")  # run_and_evaluate_dtu.py:58-59
    output[-1] = output[-1].strip()
    assert [float(x) for x in output] == [r["mean_d2s"], r["mean_s2d"], r["overall"]]
    with open(os.path.join(str(tmp_path), "results.json")) as f:
        assert json.load(f) == {k: float(v) for k, v in r.items()}


def test_vis_colors_follow_eval_py():
    dist = np.array([0.0, 5.0, 10.0, 15.0, np.inf])
    c = ev.vis_colors(7, np.array([0, 2, 3, 5, 6]), dist, visualize_threshold=10, max_dist=20)
    assert c[1].tolist() == [0, 0, 1] and c[4].tolist() == [0, 0, 1]  # not evaluated: blue
    assert c[0].tolist() == [1, 1, 1] and c[2].tolist() == [1, 0.5, 0.5]
    assert c[3].tolist() == [1, 0, 0] and c[5].tolist() == [1, 0, 0]  # clipped at the visualisation threshold
    assert c[6].tolist() == [0, 1, 0]  # beyond max_dist: green
