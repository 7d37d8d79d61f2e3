"""On-disk formats either side of the hot path (SURVEY §8f-4): the Gaussian point cloud as an Inria-compatible binary
PLY, the sparse input points PLY, cameras.json and cfg_args — byte layout and property order as written by the reference
(GaussianModel::savePly / loadPly / saveSparsePointsPly, src/gaussian_model.cpp:838-1088; GaussianMapper::savePly /
keyframesToJson / saveModelParams, src/gaussian_mapper.cpp:1658-1753), so Inria viewers and Photo-SLAM-eval read the
files unchanged. Host-side numpy only (the reference does this on the CPU through tinyply / jsoncpp as well)."""
import json
import math
import os

import numpy as np

F_REST = lambda max_sh_degree: ((max_sh_degree + 1) ** 2 - 1) * 3


def _vertex_properties(max_sh_degree):
    names = ["x", "y", "z", "nx", "ny", "nz", "f_dc_0", "f_dc_1", "f_dc_2"]
    names += [f"f_rest_{i}" for i in range(F_REST(max_sh_degree))]
    names += ["opacity", "scale_0", "scale_1", "scale_2", "rot_0", "rot_1", "rot_2", "rot_3"]
    return names


def _header(n, props, types):
    lines = ["ply", "format binary_little_endian 1.0", f"element vertex {n}"]
    lines += [f"property {t} {p}" for p, t in zip(props, types)]
    lines.append("end_header")
    return ("\n".join(lines) + "\n").encode("ascii")


def save_ply(path, xyz, features_dc, features_rest, opacity, scaling, rotation):
    """Arrays in the reference's tensor layout: xyz [N,3], features_dc [N,1,3], features_rest [N,K,3], opacity [N,1],
    scaling [N,3], rotation [N,4] (raw, un-activated parameters). Property order and the channel-major flattening of the
    SH tensors (transpose(1,2).flatten(1)) follow gaussian_model.cpp:968-1056."""
    xyz = np.asarray(xyz, np.float32).reshape(-1, 3)
    n = xyz.shape[0]
    dc = np.asarray(features_dc, np.float32).reshape(n, -1, 3)
    rest = np.asarray(features_rest, np.float32).reshape(n, -1, 3)
    k = rest.shape[1]
    deg = int(round(math.sqrt(k + 1))) - 1
    if (deg + 1) ** 2 - 1 != k:
        raise ValueError(f"features_rest has {k} coefficients: not (d+1)^2 - 1")
    cols = [xyz, np.zeros_like(xyz), dc.transpose(0, 2, 1).reshape(n, -1), rest.transpose(0, 2, 1).reshape(n, -1),
            np.asarray(opacity, np.float32).reshape(n, 1), np.asarray(scaling, np.float32).reshape(n, 3),
            np.asarray(rotation, np.float32).reshape(n, 4)]
    table = np.ascontiguousarray(np.concatenate(cols, axis=1), dtype="<f4")
    props = _vertex_properties(deg)
    assert table.shape[1] == len(props)
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    with open(path, "wb") as f:
        f.write(_header(n, props, ["float"] * len(props)))
        f.write(table.tobytes())


_PLY_TYPES = {"float": "<f4", "float32": "<f4", "double": "<f8", "float64": "<f8", "uchar": "u1", "uint8": "u1", "char": "i1", "int8": "i1",
              "short": "<i2", "int16": "<i2", "ushort": "<u2", "uint16": "<u2", "int": "<i4", "int32": "<i4", "uint": "<u4", "uint32": "<u4"}


def _read_vertex_table(path):
    with open(path, "rb") as f:
        if f.readline().strip() != b"ply":
            raise ValueError(f"{path}: not a PLY file")
        fmt, n, props, in_vertex = None, None, [], False
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
                in_vertex = tok[1] == "vertex"
                if in_vertex:
                    n = int(tok[2])
            elif tok[0] == "property" and in_vertex:
                if tok[1] == "list":
                    raise ValueError("list properties on the vertex element are not supported")
                props.append((tok[2], _PLY_TYPES[tok[1]]))
            elif tok[0] == "end_header":
                break
        if n is None:
            raise ValueError(f"{path}: no vertex element")
        if fmt == "binary_little_endian":
            data = np.frombuffer(f.read(n * np.dtype(props).itemsize), dtype=np.dtype(props), count=n)
        elif fmt == "ascii":
            raw = np.loadtxt(f, max_rows=n, ndmin=2)
            data = np.zeros(n, dtype=np.dtype(props))
            for i, (name, _) in enumerate(props):
                data[name] = raw[:, i]
        else:
            raise ValueError(f"{path}: unsupported PLY format {fmt}")
    return data


def load_ply(path, max_sh_degree=3):
    """-> dict(xyz, features_dc [N,1,3], features_rest [N,K,3], opacity [N,1], scaling [N,3], rotation [N,4]) float32, the
    layout GaussianModel.from_numpy takes. Properties are looked up by name (gaussian_model.cpp:866-888); extra ones (normals)
    are ignored; the active SH degree becomes max_sh_degree like in the reference (:951)."""
    v = _read_vertex_table(path)
    n = v.shape[0]
    col = lambda names: np.stack([v[nm].astype(np.float32) for nm in names], axis=1)
    k3 = F_REST(max_sh_degree)
    missing = [nm for nm in ["x", "y", "z", "f_dc_0", "f_dc_1", "f_dc_2", "opacity", "scale_0", "scale_1", "scale_2", "rot_0", "rot_1", "rot_2", "rot_3"] +
               [f"f_rest_{i}" for i in range(k3)] if nm not in v.dtype.names]
    if missing:
        raise ValueError(f"{path}: missing vertex properties {missing[:4]}{'...' if len(missing) > 4 else ''}")
    return dict(
        xyz=col(["x", "y", "z"]),
        features_dc=np.ascontiguousarray(col(["f_dc_0", "f_dc_1", "f_dc_2"]).reshape(n, 3, 1).transpose(0, 2, 1)),
        features_rest=np.ascontiguousarray(col([f"f_rest_{i}" for i in range(k3)]).reshape(n, 3, k3 // 3).transpose(0, 2, 1)),
        opacity=col(["opacity"]), scaling=col(["scale_0", "scale_1", "scale_2"]), rotation=col(["rot_0", "rot_1", "rot_2", "rot_3"]))


def save_sparse_points_ply(path, xyz, color):
    """input.ply: x y z nx ny nz (float) + red green blue (uchar), colour in [0,1] scaled by 255 and truncated
    (gaussian_model.cpp:1058-1088)."""
    xyz = np.asarray(xyz, np.float32).reshape(-1, 3)
    n = xyz.shape[0]
    rgb = (np.asarray(color, np.float32).reshape(n, 3) * 255.0).astype(np.uint8)
    dt = np.dtype([(p, "<f4") for p in ("x", "y", "z", "nx", "ny", "nz")] + [(p, "u1") for p in ("red", "green", "blue")])
    rec = np.zeros(n, dtype=dt)
    rec["x"], rec["y"], rec["z"] = xyz[:, 0], xyz[:, 1], xyz[:, 2]
    rec["red"], rec["green"], rec["blue"] = rgb[:, 0], rgb[:, 1], rgb[:, 2]
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    with open(path, "wb") as f:
        f.write(_header(n, list(dt.names), ["float"] * 6 + ["uchar"] * 3))
        f.write(rec.tobytes())


def fov2focal(fov, pixels):
    """reference include/graphics_utils.h:42-45"""
    return pixels / (2.0 * math.tan(fov / 2.0))


def focal2fov(focal, pixels):
    """reference include/graphics_utils.h:47-50"""
    return 2.0 * math.atan(pixels / (2.0 * focal))


def keyframes_to_json(path, keyframes):
    """cameras.json as written by GaussianMapper::keyframesToJson (gaussian_mapper.cpp:1675-1729). keyframes: iterable of dicts with
    fid, img_name, width, height, R (3x3 world->camera rotation), t (3,), FoVx, FoVy; stored are the camera-to-world position
    and rotation (inverse of [R|t]) and the focal lengths."""
    out = []
    for kf in keyframes:
        R = np.asarray(kf["R"], np.float32).reshape(3, 3)
        t = np.asarray(kf["t"], np.float32).reshape(3)
        Rt = np.eye(4, dtype=np.float32)
        Rt[:3, :3], Rt[:3, 3] = R, t
        Twc = np.linalg.inv(Rt)
        out.append({"id": int(kf["fid"]), "img_name": str(kf["img_name"]), "width": int(kf["width"]), "height": int(kf["height"]),
                    "position": [float(x) for x in Twc[:3, 3]], "rotation": [[float(x) for x in row] for row in Twc[:3, :3]],
                    "fy": float(fov2focal(kf["FoVy"], kf["height"])), "fx": float(fov2focal(kf["FoVx"], kf["width"]))})
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    with open(path, "w") as f:
        json.dump(out, f, indent=1)
    return out


def save_model_params(path, eval_=False, images="images", model_path="", resolution=-1, sh_degree=3, source_path="", white_background=False):
    """cfg_args in the exact text form of GaussianMapper::saveModelParams (gaussian_mapper.cpp:1731-1752) — the Inria viewers eval() it."""
    txt = ("Namespace(" + f"eval={'True' if eval_ else 'False'}, images='{images}', model_path='{model_path}', resolution={resolution}, "
           f"sh_degree={sh_degree}, source_path='{source_path}', white_background={'True' if white_background else 'False'}, )")
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    with open(path, "w") as f:
        f.write(txt)
    return txt


def save_exposure(path, rows):
    """exposure.json in graphdeco's form, {"<id>": 3x4 list}: rows maps a keyframe id to its 3x4 exposure row (row-major, E[:3,:3]
    right-multiplies HWC pixels, E[:3,3] is the bias)."""
    out = {}
    for k, row in rows.items():
        a = np.asarray(row, np.float64)
        if a.shape != (3, 4):
            raise ValueError(f"exposure row {k}: want shape (3, 4), got {a.shape}")
        out[str(int(k))] = [[float(x) for x in r] for r in a]
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    with open(path, "w") as f:
        json.dump(out, f, indent=1)
    return out


def load_exposure(path):
    """exposure.json -> {keyframe id (int): float32 [3,4] array}. Keys must be integer ids."""
    with open(path) as f:
        raw = json.load(f)
    rows = {}
    for k, v in raw.items():
        try:
            kid = int(k)
        except ValueError:
            raise ValueError(f"{path}: key {k!r} is not a keyframe id") from None
        a = np.asarray(v, np.float32)
        if a.shape != (3, 4) or kid < 0:
            raise ValueError(f"{path}: entry {k!r}: want a 3x4 list under a non-negative id")
        rows[kid] = a
    return rows


def save_result_dir(result_dir, iteration, model_arrays, keyframes=(), sparse_xyz=None, sparse_color=None, **model_params):
    """Directory layout of GaussianMapper::savePly (gaussian_mapper.cpp:1658-1673): cameras.json, cfg_args,
    point_cloud/iteration_<n>/point_cloud.ply, input.ply."""
    keyframes_to_json(os.path.join(result_dir, "cameras.json"), keyframes)
    save_model_params(os.path.join(result_dir, "cfg_args"), **model_params)
    save_ply(os.path.join(result_dir, "point_cloud", f"iteration_{int(iteration)}", "point_cloud.ply"), **model_arrays)
    if sparse_xyz is not None:
        save_sparse_points_ply(os.path.join(result_dir, "input.ply"), sparse_xyz, sparse_color)
