"""Gaussian point clouds as PLY files in the layout every 3DGS code base shares, the reference included
(``litegs/io_manager/ply.py:7-45`` writes it through ``plyfile``; this is a dependency-free numpy restatement of the same
file format): ``binary_little_endian 1.0``, one ``vertex`` element of float32 properties

    x y z  nx ny nz  f_dc_0..2  f_rest_0..(3(K-1)-1)  opacity  scale_0..2  rot_0..3

with the SH rest coefficients channel-major (``f_rest_[c (K-1) + k]``), log-scales, opacity logits and (w,x,y,z) rotations
stored raw.  ``save_ply`` / ``load_ply`` keep the reference's signatures (``[C, N]`` arrays, SH as ``[1,3,N]`` / ``[K-1,3,N]``);
``params_from_ply`` / ``params_to_ply`` convert to and from this package's clustered parameter dict.  Checkpoints trained with
Mip-Splatting's 3D smoothing filter carry it as one more float property, ``filter_3D``, after ``rot_3``; it is written when given
and read (by name) into the dict's ``"filter_3D"`` entry when the file has it.
``save_mesh_ply`` / ``load_mesh_ply`` write and read triangle meshes (litegs_b200.mesh's output) in the binary layout MeshLab,
Open3D and Blender read.
"""
from __future__ import annotations

import os

import numpy as np

from . import scene

PARAM_KEYS = ("xyz", "scale", "rot", "sh_0", "sh_rest", "opacity")


def _names(n_dc: int, n_rest: int):
    return (["x", "y", "z", "nx", "ny", "nz"] + [f"f_dc_{i}" for i in range(n_dc)] + [f"f_rest_{i}" for i in range(n_rest)] + ["opacity"] +
            [f"scale_{i}" for i in range(3)] + [f"rot_{i}" for i in range(4)])


def save_ply(path: str, xyz, scale, rot, sh_0, sh_rest, opacity, filter_3d=None) -> None:
    """xyz [3,N] scale [3,N] rot [4,N] sh_0 [1,3,N] sh_rest [K-1,3,N] opacity [1,N] (raw parameters); filter_3d [1,N] or None
    (written as the last property, filter_3D)."""
    xyz = np.asarray(xyz, np.float32); n = xyz.shape[1]
    dc = np.asarray(sh_0, np.float32).transpose(2, 1, 0).reshape(n, -1)            # [N, 3]
    rest = np.asarray(sh_rest, np.float32).transpose(2, 1, 0).reshape(n, -1)       # [N, 3 (K-1)], channel-major
    cols = np.concatenate([xyz.T, np.zeros((n, 3), np.float32), dc, rest, np.asarray(opacity, np.float32).T,
                           np.asarray(scale, np.float32).T, np.asarray(rot, np.float32).T] +
                          ([] if filter_3d is None else [np.asarray(filter_3d, np.float32).reshape(1, n).T]), axis=1).astype("<f4")
    names = _names(dc.shape[1], rest.shape[1]) + ([] if filter_3d is None else ["filter_3D"])
    assert cols.shape[1] == len(names)
    header = "ply\nformat binary_little_endian 1.0\nelement vertex %d\n" % n + "".join(f"property float {a}\n" for a in names) + "end_header\n"
    d = os.path.dirname(path)
    if d:
        os.makedirs(d, exist_ok=True)
    with open(path, "wb") as f:
        f.write(header.encode("ascii"))
        f.write(np.ascontiguousarray(cols).tobytes())


def _read_vertex_table(path: str):
    with open(path, "rb") as f:
        if f.readline().strip() != b"ply":
            raise ValueError(f"{path}: not a PLY file")
        fmt, n, props, in_vertex = None, None, [], False
        while True:
            line = f.readline()
            if not line:
                raise ValueError(f"{path}: header without end_header")
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
                    raise ValueError(f"{path}: list properties in the vertex element are not a Gaussian point cloud")
                props.append((tok[2], tok[1]))
            elif tok[0] == "end_header":
                break
        if fmt not in ("binary_little_endian", "ascii") or n is None:
            raise ValueError(f"{path}: unsupported PLY (format {fmt})")
        types = {"float": "<f4", "float32": "<f4", "double": "<f8", "float64": "<f8", "uchar": "u1", "uint8": "u1", "int": "<i4", "int32": "<i4",
                 "uint": "<u4", "short": "<i2", "ushort": "<u2", "char": "i1"}
        dt = np.dtype([(name, types[t]) for name, t in props])
        if fmt == "ascii":
            raw = np.loadtxt(f, max_rows=n, ndmin=2)
            tab = np.zeros(n, dt)
            for j, (name, _) in enumerate(props):
                tab[name] = raw[:, j]
            return tab
        return np.frombuffer(f.read(dt.itemsize * n), dtype=dt, count=n)


def load_ply(path: str, sh_degree: int):
    """-> xyz [3,N], scale [3,N], rot [4,N], sh_0 [1,3,N], sh_rest [K-1,3,N], opacity [1,N]  (float32), the reference's
    return order (ply.py:47-87).  Files with fewer SH bands than sh_degree are zero-extended; more is an error."""
    return _params_of_table(_read_vertex_table(path), path, sh_degree)


def _params_of_table(t, path: str, sh_degree: int):
    n = t.shape[0]
    col = lambda name: np.asarray(t[name], np.float32)
    xyz = np.stack([col("x"), col("y"), col("z")])
    K = (sh_degree + 1) ** 2
    rest_names = sorted([a for a in t.dtype.names if a.startswith("f_rest_")], key=lambda a: int(a.split("_")[-1]))
    if len(rest_names) % 3 or len(rest_names) > 3 * (K - 1):
        raise ValueError(f"{path}: {len(rest_names)} f_rest properties do not fit sh_degree {sh_degree}")
    kf = len(rest_names) // 3
    rest = np.zeros((n, 3, K - 1), np.float32)
    if kf:
        rest[:, :, :kf] = np.stack([col(a) for a in rest_names], 1).reshape(n, 3, kf)
    sh_0 = np.stack([col("f_dc_0"), col("f_dc_1"), col("f_dc_2")])[None]                 # [1,3,N]
    scale = np.stack([col(a) for a in sorted([a for a in t.dtype.names if a.startswith("scale_")], key=lambda a: int(a.split("_")[-1]))])
    rot = np.stack([col(a) for a in sorted([a for a in t.dtype.names if a.startswith("rot_")], key=lambda a: int(a.split("_")[-1]))])
    return xyz, scale, rot, sh_0, np.ascontiguousarray(rest.transpose(2, 1, 0)), col("opacity")[None]


def params_from_ply(path: str, sh_degree: int = 3, chunk: int = 128, morton: bool = True) -> dict:
    """PLY -> clustered parameter dict (+ cluster_origin / cluster_extend, n_points), Morton sorted like scene.make_scene.
    A file with the filter_3D property also gives "filter_3D" [1,C,S]; the chunk boxes stay those of the unfiltered splats
    (scene.cluster_aabb(..., filter_3d=) gives the filtered ones)."""
    t = _read_vertex_table(path)
    vals = dict(zip(PARAM_KEYS, _params_of_table(t, path, sh_degree)))
    if "filter_3D" in t.dtype.names:
        vals["filter_3D"] = np.asarray(t["filter_3D"], np.float32)[None]
    n = vals["xyz"].shape[-1]
    order = scene.morton_order(vals["xyz"]) if morton else np.arange(n)
    out = {k: scene.cluster(np.ascontiguousarray(v[..., order]), chunk) for k, v in vals.items()}
    out["cluster_origin"], out["cluster_extend"] = scene.cluster_aabb(out["xyz"], out["scale"], out["rot"])
    out["n_points"] = n
    return out


def _numpy(a, dtype, name: str, cols: int = 3):
    a = a.detach().cpu().numpy() if hasattr(a, "detach") else np.asarray(a)
    if a.ndim != 2 or a.shape[1] != cols:
        raise ValueError(f"{name} must be [N,{cols}], got {list(a.shape)}")
    return np.ascontiguousarray(a, dtype)


def save_mesh_ply(path: str, vertices, faces, colors=None) -> None:
    """A triangle mesh as the binary little-endian PLY that MeshLab, Open3D and Blender read: element vertex (float x y z and,
    with colours, uchar red green blue), element face (list uchar int vertex_indices).  vertices f32[M,3], faces i32[F,3],
    colors u8[M,3] or None; numpy arrays or tensors of any device."""
    v = _numpy(vertices, "<f4", "vertices")
    f = _numpy(faces, "<i4", "faces")
    fields = [("x", "<f4"), ("y", "<f4"), ("z", "<f4")]
    if colors is not None:
        c = _numpy(colors, "u1", "colors")
        if c.shape[0] != v.shape[0]:
            raise ValueError(f"colors has {c.shape[0]} rows, vertices {v.shape[0]}")
        fields += [("red", "u1"), ("green", "u1"), ("blue", "u1")]
    vt = np.empty(v.shape[0], np.dtype(fields))
    vt["x"], vt["y"], vt["z"] = v[:, 0], v[:, 1], v[:, 2]
    if colors is not None:
        vt["red"], vt["green"], vt["blue"] = c[:, 0], c[:, 1], c[:, 2]
    ft = np.empty(f.shape[0], np.dtype([("n", "u1"), ("i", "<i4", (3,))]))
    ft["n"], ft["i"] = 3, f
    header = ("ply\nformat binary_little_endian 1.0\n" + f"element vertex {v.shape[0]}\n" + "".join(f"property float {a}\n" for a in "xyz")
              + ("".join(f"property uchar {a}\n" for a in ("red", "green", "blue")) if colors is not None else "")
              + f"element face {f.shape[0]}\nproperty list uchar int vertex_indices\nend_header\n")
    d = os.path.dirname(path)
    if d:
        os.makedirs(d, exist_ok=True)
    with open(path, "wb") as fh:
        fh.write(header.encode("ascii"))
        fh.write(vt.tobytes())
        fh.write(ft.tobytes())


def load_mesh_ply(path: str):
    """save_mesh_ply's layout back -> (vertices f32[M,3], faces i32[F,3], colors u8[M,3] or None), numpy.  Other layouts (ASCII,
    other vertex properties, polygons that are not triangles) are refused."""
    with open(path, "rb") as fh:
        if fh.readline().strip() != b"ply":
            raise ValueError(f"{path}: not a PLY file")
        lines = []
        while True:
            line = fh.readline()
            if not line:
                raise ValueError(f"{path}: header without end_header")
            tok = line.decode("ascii", "replace").split()
            if tok == ["end_header"]:
                break
            if tok and tok[0] != "comment":
                lines.append(tok)
        body = fh.read()
    if ["format", "binary_little_endian", "1.0"] not in lines:
        raise ValueError(f"{path}: only binary_little_endian 1.0 meshes are read")
    els, cur = {}, None
    for tok in lines:
        if tok[0] == "element":
            cur = els[tok[1]] = (int(tok[2]), [])
        elif tok[0] == "property" and cur is not None:
            cur[1].append(tuple(tok[1:]))
    xyz = [("float", a) for a in "xyz"]
    rgb = [("uchar", a) for a in ("red", "green", "blue")]
    if set(els) != {"vertex", "face"} or els["vertex"][1] not in (xyz, xyz + rgb) or els["face"][1] != [("list", "uchar", "int", "vertex_indices")]:
        raise ValueError(f"{path}: not a triangle mesh in save_mesh_ply's layout")
    has_rgb = els["vertex"][1] == xyz + rgb
    M, F = els["vertex"][0], els["face"][0]
    vdt = np.dtype([("p", "<f4", (3,))] + ([("c", "u1", (3,))] if has_rgb else []))
    fdt = np.dtype([("n", "u1"), ("i", "<i4", (3,))])
    if len(body) < M * vdt.itemsize + F * fdt.itemsize:
        raise ValueError(f"{path}: truncated")
    vt = np.frombuffer(body, vdt, count=M)
    ft = np.frombuffer(body, fdt, count=F, offset=M * vdt.itemsize)
    if F and not (ft["n"] == 3).all():
        raise ValueError(f"{path}: faces that are not triangles")
    return (np.ascontiguousarray(vt["p"]), np.ascontiguousarray(ft["i"]), np.ascontiguousarray(vt["c"]) if has_rgb else None)


def params_to_ply(path: str, params: dict, n_points: int | None = None) -> None:
    """Clustered parameter dict -> PLY; n_points drops the padding of the last chunk.  A "filter_3D" entry ([1,C,S]) is written
    as the filter_3D property."""
    keys = PARAM_KEYS + (("filter_3D",) if params.get("filter_3D") is not None else ())
    flat = {k: np.asarray(params[k]).reshape(*np.asarray(params[k]).shape[:-2], -1) for k in keys}
    n = flat["xyz"].shape[-1] if n_points is None else int(n_points)
    save_ply(path, *[flat[k][..., :n] for k in PARAM_KEYS], filter_3d=flat["filter_3D"][..., :n] if "filter_3D" in flat else None)
