"""Loaders for the reference-signature `Renderer(base_dir, colmap_dir, output_dir_root, args, ...)`:
the COLMAP text model and the trained 3DGS point cloud, read directly into the tensors the hot path
needs (SURVEY.md section 8(f) rank 3).

The reference goes through `Scene(...)`, which loads every training image to the GPU just to reach
`GaussianModel.load_ply` (renderer_utils.py:357-358); here the PLY and the two text files are parsed
directly.  Restated (file:line in /root/reference):
  gs2mesh_utils/third_party/colmap_runner/utils/read_write_model.py:101-124  read_cameras_text
  gs2mesh_utils/third_party/colmap_runner/utils/read_write_model.py:193-221  read_images_text
  gs2mesh_utils/colmap_utils.py:26-42                                        poses_from_file
  gs2mesh_utils/third_party/visualization/camera_utils.py:188-196            Quaternion.q_to_R
  gs2mesh_utils/renderer_utils.py:69-99, 127-216                            camera sort, rig construction
  third_party/gaussian-splatting/scene/gaussian_model.py:95-115, 215-256     activations, load_ply
Checked against golden camera rigs produced by the reference's own Renderer.__init__
(tests/golden/make_rig_golden.py).
"""
from __future__ import annotations

import os
from collections import OrderedDict

import numpy as np

from . import camera as cam
from .scene import GaussianCloud


# ----------------------------------------------------------------------------- COLMAP text model
def read_cameras_text(path):
    """{camera_id: dict(model, width, height, params)} (read_write_model.py:101-124)."""
    cameras = {}
    with open(path, "r") as f:
        for line in f:
            line = line.strip()
            if not line or line[0] == "#":
                continue
            e = line.split()
            cameras[int(e[0])] = dict(id=int(e[0]), model=e[1], width=int(e[2]), height=int(e[3]),
                                      params=np.array(tuple(map(float, e[4:]))))
    return cameras


def read_images_text(path):
    """{image_id: dict(qvec, tvec, camera_id, name)}; the 2D-point line after each image is skipped
    (read_write_model.py:193-221)."""
    images = {}
    with open(path, "r") as f:
        while True:
            line = f.readline()
            if not line:
                break
            line = line.strip()
            if not line or line[0] == "#":
                continue
            e = line.split()
            images[int(e[0])] = dict(id=int(e[0]), qvec=np.array(tuple(map(float, e[1:5]))),
                                     tvec=np.array(tuple(map(float, e[5:8]))), camera_id=int(e[8]), name=e[9])
            f.readline()  # POINTS2D[] line
    return images


def quaternions_to_matrices(q):
    """[...,4] (w,x,y,z) -> [...,3,3] (camera_utils.py:188-196), float64."""
    q = np.asarray(q, dtype=np.float64)
    qa, qb, qc, qd = q[..., 0], q[..., 1], q[..., 2], q[..., 3]
    r0 = np.stack([1 - 2 * (qc ** 2 + qd ** 2), 2 * (qb * qc - qa * qd), 2 * (qa * qc + qb * qd)], -1)
    r1 = np.stack([2 * (qb * qc + qa * qd), 1 - 2 * (qb ** 2 + qd ** 2), 2 * (qc * qd - qa * qb)], -1)
    r2 = np.stack([2 * (qb * qd - qa * qc), 2 * (qa * qb + qc * qd), 1 - 2 * (qb ** 2 + qc ** 2)], -1)
    return np.stack([r0, r1, r2], -2)


def poses_from_file(images_txt):
    """[N,3,4] world->camera [R|t] in ascending image-id order (colmap_utils.py:26-42)."""
    images = OrderedDict(sorted(read_images_text(images_txt).items()))
    q = np.stack([im["qvec"] for im in images.values()])
    t = np.stack([im["tvec"] for im in images.values()])
    return np.concatenate([quaternions_to_matrices(q), t[..., None]], axis=-1)


# ----------------------------------------------------------------------------- camera ordering (renderer_utils.py:34-99)
def sort_camera_coordinates(coordinates):
    coordinates = np.asarray(coordinates)
    visited = np.zeros(len(coordinates), dtype=bool)
    order = []
    current = int(np.argmin(coordinates[:, 2]))
    while not np.all(visited):
        visited[current] = True
        order.append(current)
        if np.all(visited):
            break
        dist = np.linalg.norm(coordinates - coordinates[current], axis=1)
        dist[visited] = np.inf
        dist[current] = np.inf
        nearest = np.argsort(dist)[:2]
        if len(nearest) == 0:
            break
        z_diff = np.abs(coordinates[nearest][:, 2] - coordinates[current][2])
        pick = int(nearest[np.argmin(z_diff)])
        if visited[pick]:
            # The reference loops forever here (its candidate list still contains visited cameras once fewer than two
            # unvisited ones remain).  Deviation: fall back to the nearest unvisited camera.
            pick = int(nearest[0])
        current = pick
    return order


def build_stereo_rigs(poses, camera_params, args):
    """renderer_utils.py:132-206: camera poses -> Euler angles/positions -> baseline -> left/right dicts.
    Returns (cameras, baseline, sorted_camera_indices)."""
    poses_inv = [np.linalg.inv(np.vstack((p, np.array([0, 0, 0, 1])))) for p in poses]
    rotations = [cam.matrix_to_euler_deg(p[:3, :3]) for p in poses_inv]
    for i in range(len(rotations)):
        r = cam.euler_deg_to_matrix(rotations[i])
        r[:, 1:] *= -1
        rotations[i] = cam.matrix_to_euler_deg(r)
    locations = [p[:3, 3].tolist() for p in poses_inv]

    ids = sorted(camera_params.keys())
    plist = []
    for i in ids:
        c = camera_params[i]
        simple = c["model"] == "SIMPLE_RADIAL"
        plist.append(dict(width=c["width"], height=c["height"], fx=c["params"][0], fy=c["params"][0 if simple else 1],
                          cx=c["params"][1 if simple else 2], cy=c["params"][2 if simple else 3]))
    if len(plist) != len(locations):
        plist = [plist[0]] * len(locations)

    absolute = getattr(args, "renderer_baseline_absolute", None)
    if absolute is not None:
        baseline = absolute
    else:
        baseline = cam.scene_baseline(locations, getattr(args, "renderer_baseline_percentage", 7.0),
                                      scene_360=getattr(args, "renderer_scene_360", True),
                                      dtu_compat=getattr(args, "dataset_name", "custom") == "DTU")
    if getattr(args, "renderer_sort_cameras", False):
        order = sort_camera_coordinates(np.array(locations))
    else:
        order = list(range(len(locations)))

    rigs = []
    for i in range(len(locations)):
        k = order[i]
        p = plist[k]
        rig = cam.make_stereo_rig(rotations[k], tuple(locations[k]), baseline, p["width"], p["height"], p["fx"].item(),
                                  p["fy"].item(), p["cx"].item(), p["cy"].item())
        rigs.append(rig)
    return rigs, baseline, order


# ----------------------------------------------------------------------------- 3DGS point cloud
_PLY_TYPES = {"float": "<f4", "float32": "<f4", "double": "<f8", "float64": "<f8", "uchar": "u1", "uint8": "u1", "int": "<i4",
              "int32": "<i4", "uint": "<u4", "uint32": "<u4", "short": "<i2", "ushort": "<u2", "char": "i1"}


def _read_vertex_table(path, with_faces=False):
    """The vertex element of a binary-little-endian or ascii PLY as a structured array; with_faces also returns the face
    element's triangles (int64 [M,3], from a `property list <uchar|int> <int|uint>` of length 3), or None without one."""
    with open(path, "rb") as f:
        if f.readline().strip() != b"ply":
            raise ValueError(f"{path}: not a PLY file")
        fmt, elements = None, []  # [name, count, props]; props of a list property: ("list", count type, index type)
        while True:
            line = f.readline()
            if not line:
                raise ValueError(f"{path}: truncated PLY header")
            tok = line.decode("ascii", "replace").split()
            if not tok:
                continue
            if tok[0] == "format":
                fmt = tok[1]
            elif tok[0] == "element":
                elements.append([tok[1], int(tok[2]), []])
            elif tok[0] == "property" and elements:
                if tok[1] == "list":
                    if elements[-1][0] == "vertex":
                        raise ValueError(f"{path}: list property on the vertex element is not supported")
                    elements[-1][2].append(("list", _PLY_TYPES[tok[2]], _PLY_TYPES[tok[3]]))
                else:
                    elements[-1][2].append((tok[2], _PLY_TYPES[tok[1]]))
            elif tok[0] == "end_header":
                break
        if not elements or elements[0][0] != "vertex":
            raise ValueError(f"{path}: the first PLY element must be 'vertex'")
        _, count, props = elements[0]
        face = elements[1] if len(elements) > 1 and elements[1][0] == "face" else None
        if face is not None and (len(face[2]) != 1 or face[2][0][0] != "list"):
            raise ValueError(f"{path}: the face element must hold exactly one list property")
        if fmt == "binary_little_endian":
            vert = np.fromfile(f, dtype=np.dtype(props), count=count)
            tris = None
            if face is not None:
                _, ct, it = face[2][0]
                rec = np.fromfile(f, dtype=np.dtype([("n", ct), ("v", it, (3,))]), count=face[1])
                if len(rec) != face[1] or (rec["n"] != 3).any():
                    raise ValueError(f"{path}: only triangle faces are supported")
                tris = rec["v"].astype(np.int64)
        elif fmt == "ascii":
            lines = [ln for ln in f.read().decode("ascii").splitlines() if ln.strip()]
            raw = np.array([ln.split() for ln in lines[:count]], dtype=np.float64).reshape(count, len(props))
            vert = np.zeros(count, dtype=np.dtype(props))
            for j, (name, _) in enumerate(props):
                vert[name] = raw[:, j]
            tris = None
            if face is not None:
                rows = [ln.split() for ln in lines[count:count + face[1]]]
                if len(rows) != face[1] or any(len(r) != 4 or r[0] != "3" for r in rows):
                    raise ValueError(f"{path}: only triangle faces are supported")
                tris = np.array([r[1:] for r in rows], dtype=np.int64).reshape(-1, 3)
        else:
            raise ValueError(f"{path}: unsupported PLY format {fmt}")
        return (vert, tris) if with_faces else vert


def read_point_cloud_ply(path):
    """o3d.io.read_point_cloud(path).points (eval.py:76-77, 114-115): float64 [N,3]."""
    v = _read_vertex_table(path)
    return np.stack([v["x"], v["y"], v["z"]], axis=1).astype(np.float64)


def read_triangle_mesh_ply(path, with_colors=False):
    """o3d.io.read_triangle_mesh(path) vertices / triangles (eval.py:46-49): (float64 [N,3], int64 [M,3]).  with_colors
    adds a third item, the vertex colours as Open3D reads uchar red / green / blue (value / 255, float64 [N,3]), or None
    when the file has none."""
    v, tris = _read_vertex_table(path, with_faces=True)
    xyz = np.stack([v["x"], v["y"], v["z"]], axis=1).astype(np.float64)
    tris = np.zeros((0, 3), np.int64) if tris is None else tris
    if not with_colors:
        return xyz, tris
    names = v.dtype.names
    colors = None
    if all(c in names for c in ("red", "green", "blue")):
        colors = np.stack([v["red"], v["green"], v["blue"]], axis=1).astype(np.float64) / 255.0
    return xyz, tris, colors


def color_to_uint8(colors):
    """Open3D's utility::ColorToUint8, which its PLY writer applies to colours:
    uint8_t(std::round(std::min(1., std::max(0., c)) * 255.)).  std::round rounds halves away from zero (np.rint would
    round them to even), and std::max(0., NaN) is 0."""
    c = np.asarray(colors, dtype=np.float64)
    c = np.where(c > 0.0, c, 0.0)
    s = np.where(c < 1.0, c, 1.0) * 255.0
    lo = np.floor(s)
    return (lo + (s - lo >= 0.5)).astype(np.uint8)


def write_point_cloud_ply(path, points, colors=None, normals=None, triangles=None):
    """o3d.io.write_point_cloud (eval.py's visualisation clouds, eval.py:21-25), and with `triangles`
    o3d.io.write_triangle_mesh: binary little-endian, double xyz, double normals nx ny nz when given, uchar rgb =
    color_to_uint8(colour) when given, in Open3D's property order.  A mesh file also carries a `comment Created by
    gs2mesh_b200` header line and, after the vertices, a face element of uchar-counted uint triangles."""
    points = np.asarray(points, dtype=np.float64).reshape(-1, 3)
    props = [("x", "<f8"), ("y", "<f8"), ("z", "<f8")]
    header = ["ply", "format binary_little_endian 1.0"]
    if triangles is not None:
        header.append("comment Created by gs2mesh_b200")
    header += [f"element vertex {len(points)}", "property double x", "property double y", "property double z"]
    if normals is not None:
        props += [("nx", "<f8"), ("ny", "<f8"), ("nz", "<f8")]
        header += ["property double nx", "property double ny", "property double nz"]
    if colors is not None:
        props += [("red", "u1"), ("green", "u1"), ("blue", "u1")]
        header += ["property uchar red", "property uchar green", "property uchar blue"]
    tab = np.zeros(len(points), dtype=props)
    tab["x"], tab["y"], tab["z"] = points.T
    if normals is not None:
        tab["nx"], tab["ny"], tab["nz"] = np.asarray(normals, dtype=np.float64).reshape(-1, 3).T
    if colors is not None:
        tab["red"], tab["green"], tab["blue"] = color_to_uint8(colors).reshape(-1, 3).T
    face = np.zeros(0, dtype=[("n", "u1"), ("v", "<u4", (3,))])
    if triangles is not None:
        tris = np.asarray(triangles).reshape(-1, 3)
        face = np.zeros(len(tris), dtype=face.dtype)
        face["n"], face["v"] = 3, tris.astype(np.uint32)
        header += [f"element face {len(face)}", "property list uchar uint vertex_indices"]
    with open(path, "wb") as f:
        f.write(("\n".join(header + ["end_header"]) + "\n").encode("ascii"))
        f.write(tab.tobytes())
        f.write(face.tobytes())
    return path


def read_gaussian_ply(path, sh_degree=3) -> GaussianCloud:
    """`GaussianModel.load_ply` (gaussian_model.py:215-256) + the activations the renderer applies per view
    (gaussian_model.py:95-115: exp / normalize / sigmoid / cat), done once here in float32."""
    import torch

    v = _read_vertex_table(path)
    names = v.dtype.names
    n = len(v)
    xyz = np.stack([v["x"], v["y"], v["z"]], axis=1).astype(np.float32)
    dc = np.stack([v["f_dc_0"], v["f_dc_1"], v["f_dc_2"]], axis=1).astype(np.float32)  # [P,3]
    rest_names = sorted([p for p in names if p.startswith("f_rest_")], key=lambda s: int(s.split("_")[-1]))
    ncoef = (sh_degree + 1) ** 2
    if len(rest_names) != 3 * ncoef - 3:
        raise ValueError(f"{path}: {len(rest_names)} f_rest_* properties, expected {3 * ncoef - 3} for SH degree {sh_degree}")
    rest = np.stack([v[p] for p in rest_names], axis=1).astype(np.float32).reshape(n, 3, ncoef - 1)  # channel-major on disk
    feats = np.zeros((n, 16, 3), np.float32)
    feats[:, 0, :] = dc
    feats[:, 1:ncoef, :] = rest.transpose(0, 2, 1)
    scale_names = sorted([p for p in names if p.startswith("scale_")], key=lambda s: int(s.split("_")[-1]))
    rot_names = sorted([p for p in names if p.startswith("rot")], key=lambda s: int(s.split("_")[-1]))
    scales = torch.from_numpy(np.stack([v[p] for p in scale_names], axis=1).astype(np.float32))
    rots = torch.from_numpy(np.stack([v[p] for p in rot_names], axis=1).astype(np.float32))
    opac = torch.from_numpy(np.asarray(v["opacity"], dtype=np.float32)[:, None])
    return GaussianCloud(xyz=np.ascontiguousarray(xyz), features=feats, opacity=torch.sigmoid(opac).numpy(),
                         scaling=torch.exp(scales).numpy(), rotation=torch.nn.functional.normalize(rots).numpy(), sh_degree=sh_degree)


def write_gaussian_ply(path, cloud: GaussianCloud):
    """Inverse of read_gaussian_ply in the layout `GaussianModel.save_ply` writes (gaussian_model.py:177-207);
    used to build fixtures from synthetic scenes."""
    n = cloud.num_points
    ncoef = (cloud.sh_degree + 1) ** 2
    names = ["x", "y", "z", "nx", "ny", "nz", "f_dc_0", "f_dc_1", "f_dc_2"] + [f"f_rest_{i}" for i in range(3 * (ncoef - 1))] + \
            ["opacity", "scale_0", "scale_1", "scale_2", "rot_0", "rot_1", "rot_2", "rot_3"]
    tab = np.zeros(n, dtype=[(k, "<f4") for k in names])
    tab["x"], tab["y"], tab["z"] = cloud.xyz.T
    for c in range(3):
        tab[f"f_dc_{c}"] = cloud.features[:, 0, c]
    rest = cloud.features[:, 1:ncoef, :].transpose(0, 2, 1).reshape(n, -1)
    for i in range(rest.shape[1]):
        tab[f"f_rest_{i}"] = rest[:, i]
    o = np.clip(cloud.opacity.reshape(-1).astype(np.float64), 1e-7, 1 - 1e-7)
    tab["opacity"] = np.log(o / (1 - o))
    for c in range(3):
        tab[f"scale_{c}"] = np.log(cloud.scaling[:, c])
    for c in range(4):
        tab[f"rot_{c}"] = cloud.rotation[:, c]
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    with open(path, "wb") as f:
        f.write(("ply\nformat binary_little_endian 1.0\nelement vertex %d\n" % n).encode())
        f.write("".join(f"property float {k}\n" for k in names).encode())
        f.write(b"end_header\n")
        f.write(tab.tobytes())


def load_reference_scene(base_dir, colmap_dir, args, splatting="custom"):
    """Everything `Renderer.__init__` + `prepare_renderer` read from disk (renderer_utils.py:118-216, 316-358).
    Returns (cameras, baseline, gaussians, poses, sorted_camera_indices)."""
    poses = poses_from_file(os.path.join(colmap_dir, "sparse", "0", "images.txt"))
    params = read_cameras_text(os.path.join(colmap_dir, "sparse", "0", "cameras.txt"))
    rigs, baseline, order = build_stereo_rigs(poses, params, args)
    if getattr(args, "renderer_sort_cameras", False):
        poses = poses[np.asarray(order)]
    ply = os.path.join(base_dir, "splatting_output", splatting, getattr(args, "colmap_name"), "point_cloud",
                       f"iteration_{getattr(args, 'GS_iterations', 30000)}", "point_cloud.ply")
    return rigs, baseline, read_gaussian_ply(ply, sh_degree=3), poses, order
