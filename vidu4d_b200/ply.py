"""2DGS's vertex PLY (gs/scene/gaussian_model.py:189-268, save_ply / load_ply) with numpy alone.

The file is binary little-endian with one `vertex` element whose properties are all `float`, in
construct_list_of_attributes' order:

    x y z nx ny nz  f_dc_0..2  f_rest_0..44  opacity  scale_0..1  rot_0..3  [regist_feat_0..15]

The normals are zero; the SH rows are channel-major, features.transpose(1, 2).flatten(1), as save_ply writes them.
regist_feat_0..15, the Stage-3 registration feature, is this project's addition: the reference's load_ply selects
properties by name and ignores it.  The reader selects by name too, so it takes the reference's files with their
properties in any order and of any scalar type.
"""
from __future__ import annotations

import numpy as np
import torch

MAX_SH_DEGREE = 3
N_REST = 3 * (MAX_SH_DEGREE + 1) ** 2 - 3
N_REGIST = 16
_TYPES = {"char": "i1", "int8": "i1", "uchar": "u1", "uint8": "u1", "short": "i2", "int16": "i2", "ushort": "u2",
          "uint16": "u2", "int": "i4", "int32": "i4", "uint": "u4", "uint32": "u4", "float": "f4", "float32": "f4",
          "double": "f8", "float64": "f8"}


def attribute_names(regist_feat: bool = False) -> list[str]:
    """gaussian_model.py construct_list_of_attributes for SH degree 3, then regist_feat_0..15 if asked."""
    names = ["x", "y", "z", "nx", "ny", "nz"] + [f"f_dc_{i}" for i in range(3)] + [f"f_rest_{i}" for i in range(N_REST)]
    names += ["opacity", "scale_0", "scale_1"] + [f"rot_{i}" for i in range(4)]
    return names + ([f"regist_feat_{i}" for i in range(N_REGIST)] if regist_feat else [])


def header(names, count: int) -> bytes:
    lines = ["ply", "format binary_little_endian 1.0", f"element vertex {count}"]
    lines += [f"property float {n}" for n in names] + ["end_header"]
    return ("\n".join(lines) + "\n").encode("ascii")


def write_surfels(path, groups: dict) -> None:
    """groups: xyz (P,3), f_dc (P,1,3), f_rest (P,15,3), opacity (P,1), scaling (P,2), rotation (P,4), optional
    regist_feat (P,16) -- tensors or arrays in the reference's shapes."""
    a = {n: (v.detach().cpu().numpy() if isinstance(v, torch.Tensor) else np.asarray(v)).astype(np.float32, copy=False)
         for n, v in groups.items()}
    P = a["xyz"].shape[0]
    cols = [a["xyz"], np.zeros((P, 3), np.float32),
            a["f_dc"].transpose(0, 2, 1).reshape(P, 3), a["f_rest"].transpose(0, 2, 1).reshape(P, N_REST),
            a["opacity"].reshape(P, 1), a["scaling"], a["rotation"]]
    regist = "regist_feat" in a
    if regist:
        cols.append(a["regist_feat"])
    names = attribute_names(regist)
    body = np.ascontiguousarray(np.concatenate(cols, axis=1), dtype="<f4")
    if body.shape != (P, len(names)):
        raise ValueError(f"the surfel groups make rows of {body.shape[1]} values, the PLY layout has {len(names)}")
    with open(path, "wb") as f:
        f.write(header(names, P))
        f.write(body.tobytes())


def _parse_header(f, path):
    if f.readline().rstrip(b"\r\n") != b"ply":
        raise ValueError(f"{path}: not a PLY file")
    elements, fmt = [], None
    while True:
        raw = f.readline()
        if not raw:
            raise ValueError(f"{path}: the PLY header has no end_header")
        line = raw.decode("ascii", "replace").strip()
        words = line.split()
        if not words or words[0] in ("comment", "obj_info"):
            continue
        if words[0] == "end_header":
            return elements, fmt
        if words[0] == "format":
            if words[1:2] != ["binary_little_endian"]:
                raise ValueError(f"{path}: PLY format {' '.join(words[1:2]) or '?'} is not supported; only "
                                 f"binary_little_endian (what 2DGS's save_ply writes) is")
            fmt = words[1]
        elif words[0] == "element" and len(words) == 3:
            elements.append((words[1], int(words[2]), []))
        elif words[0] == "property" and elements:
            # a list property's row size varies; it is recorded as None and refused only in the element that is read
            if words[1] == "list" and len(words) == 5:
                elements[-1][2].append((words[4], None))
            elif len(words) == 3 and words[1] in _TYPES:
                elements[-1][2].append((words[2], "<" + _TYPES[words[1]]))
            else:
                raise ValueError(f"{path}: unsupported property line {line!r}")
        else:
            raise ValueError(f"{path}: unexpected PLY header line {line!r}")


def read_vertices(path) -> np.ndarray:
    """The vertex element of a binary little-endian PLY file as a numpy structured array (its first element; the
    elements after it, faces for instance, are not read)."""
    with open(path, "rb") as f:
        elements, fmt = _parse_header(f, path)
        if fmt is None:
            raise ValueError(f"{path}: the PLY header has no format line")
        if not elements or elements[0][0] != "vertex":
            raise ValueError(f"{path}: the first PLY element must be 'vertex', got {[e[0] for e in elements]}")
        _, count, props = elements[0]
        lists = [n for n, t in props if t is None]
        if lists:
            raise ValueError(f"{path}: the vertex element has list properties {lists}; a surfel PLY's vertex properties "
                             f"are scalars")
        dtype = np.dtype(props)
        data = f.read(count * dtype.itemsize)
    if len(data) != count * dtype.itemsize:
        raise ValueError(f"{path}: truncated: {count} vertices need {count * dtype.itemsize} bytes, the file has {len(data)}")
    return np.frombuffer(data, dtype=dtype, count=count)


def _indexed(v, prefix):
    return sorted((n for n in v.dtype.names if n.startswith(prefix)), key=lambda n: int(n.split("_")[-1]))


def read_surfels(path) -> dict:
    """gaussian_model.py load_ply's reading: properties by name, float32 tensors in the reference's shapes --
    xyz (P,3), f_dc (P,1,3), f_rest (P,15,3), opacity (P,1), scaling (P,2), rotation (P,4), and regist_feat (P,16) when
    the file has regist_feat_0..15."""
    v = read_vertices(path)
    P = v.shape[0]

    def cols(names, what):
        absent = [n for n in names if n not in v.dtype.names]
        if absent:
            raise ValueError(f"{path}: the vertex element has no {what} properties {absent}")
        return np.stack([np.asarray(v[n], dtype=np.float32) for n in names], axis=1).reshape(P, len(names))

    rest, scale, rot = _indexed(v, "f_rest_"), _indexed(v, "scale_"), _indexed(v, "rot")
    if len(rest) != N_REST:
        raise ValueError(f"{path}: {len(rest)} f_rest properties, SH degree {MAX_SH_DEGREE} has {N_REST} "
                         f"(gaussian_model.py:242)")
    if len(scale) != 2 or len(rot) != 4:
        raise ValueError(f"{path}: a surfel has 2 scale_ and 4 rot properties, the file {len(scale)} and {len(rot)}")
    t = torch.from_numpy
    out = {"xyz": t(cols(["x", "y", "z"], "position")),
           "f_dc": t(cols([f"f_dc_{i}" for i in range(3)], "f_dc")).view(P, 1, 3),
           "f_rest": t(cols(rest, "f_rest")).view(P, 3, N_REST // 3).transpose(1, 2).contiguous(),
           "opacity": t(cols(["opacity"], "opacity")), "scaling": t(cols(scale, "scale")),
           "rotation": t(cols(rot, "rot"))}
    regist = _indexed(v, "regist_feat_")
    if regist:
        if len(regist) != N_REGIST:
            raise ValueError(f"{path}: {len(regist)} regist_feat properties, the registration feature has {N_REGIST}")
        out["regist_feat"] = t(cols(regist, "regist_feat"))
    return out
