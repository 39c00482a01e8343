"""Point-cloud file formats on the input side of the hot path.

* binary PLY (little/big endian) as read by the reference evaluation driver (/root/reference/evaluation/eval_kitti.py:117-241,
  element ``vertex`` with scalar properties, optional triangular ``face`` element with ``uchar int`` lists),
* ASCII PLY with 6 columns ``x y z r g b`` as read by the demo (/root/reference/demo/utils.py:4-30),
* the two input normalisations (eval_kitti.py:73-88, demo/app.py:124-127).

Own implementation: the header is parsed into a numpy structured dtype and the payload is mapped in one read."""
from __future__ import annotations

import io
from typing import Dict, List, Optional, Sequence, Tuple, Union

import numpy as np

_SCALARS = {"char": "i1", "int8": "i1", "uchar": "u1", "uint8": "u1", "short": "i2", "int16": "i2", "ushort": "u2",
            "uint16": "u2", "int": "i4", "int32": "i4", "uint": "u4", "uint32": "u4", "float": "f4", "float32": "f4",
            "double": "f8", "float64": "f8"}
_ENDIAN = {"binary_little_endian": "<", "binary_big_endian": ">", "ascii": "="}


class PlyHeader:
    def __init__(self):
        self.format = None
        self.elements: List[Tuple[str, int, List[Tuple[str, ...]]]] = []  # (name, count, [(kind, ...)])

    def element(self, name: str):
        for e in self.elements:
            if e[0] == name:
                return e
        return None


def parse_header(f) -> PlyHeader:
    first = f.readline()
    if first.strip() != b"ply":
        raise ValueError("The file does not start with the word ply")
    h = PlyHeader()
    while True:
        line = f.readline()
        if line == b"":
            raise ValueError("unterminated PLY header")
        tok = line.split()
        if not tok or tok[0] in (b"comment", b"obj_info"):
            continue
        if tok[0] == b"format":
            h.format = tok[1].decode()
            if h.format not in _ENDIAN:
                raise ValueError(f"unknown PLY format {h.format}")
        elif tok[0] == b"element":
            h.elements.append((tok[1].decode(), int(tok[2]), []))
        elif tok[0] == b"property":
            if not h.elements:
                raise ValueError("property before element")
            if tok[1] == b"list":
                h.elements[-1][2].append(("list", tok[2].decode(), tok[3].decode(), tok[4].decode()))
            else:
                h.elements[-1][2].append(("scalar", tok[1].decode(), tok[2].decode()))
        elif tok[0] == b"end_header":
            break
    if h.format is None:
        raise ValueError("PLY header without a format line")
    return h


def _vertex_dtype(props, ext) -> np.dtype:
    fields = []
    for p in props:
        if p[0] != "scalar":
            raise ValueError("list properties are not supported on the vertex element")
        if p[1] not in _SCALARS:
            raise ValueError(f"unsupported PLY scalar type {p[1]}")
        fields.append((p[2], ext + _SCALARS[p[1]]))
    return np.dtype(fields)


def read_ply(filename, triangular_mesh: bool = False, allow_ascii: bool = False):
    """Structured array of the vertex element (fields named as in the header: x, y, z, R, G, B, label ...).
    ``triangular_mesh=True`` returns ``[vertex_data, faces[int32, F x 3]]`` like the reference reader.  ASCII files are
    refused unless ``allow_ascii`` (the reference evaluation reader raises on them, eval_kitti.py:207-208)."""
    with open(filename, "rb") as f:
        h = parse_header(f)
        if h.format == "ascii" and not allow_ascii:
            raise ValueError("The file is not binary")
        ext = _ENDIAN[h.format]
        v = h.element("vertex") or (h.elements[0] if h.elements else None)
        if v is None:
            raise ValueError("PLY file without elements")
        dt = _vertex_dtype(v[2], ext)
        if h.format == "ascii":
            rows = np.loadtxt(io.BytesIO(b"".join(f.readline() for _ in range(v[1]))), dtype=np.float64, ndmin=2)
            data = np.empty(v[1], dtype=dt)
            for i, name in enumerate(dt.names):
                data[name] = rows[:, i]
        else:
            data = np.fromfile(f, dtype=dt, count=v[1])
            if data.shape[0] != v[1]:
                raise ValueError(f"truncated PLY payload: {data.shape[0]} of {v[1]} vertices")
        if not triangular_mesh:
            return data
        fe = h.element("face")
        nf = fe[1] if fe else 0
        if h.format == "ascii":
            fr = np.loadtxt(io.BytesIO(b"".join(f.readline() for _ in range(nf))), dtype=np.int64, ndmin=2)
            faces = fr[:, 1:4].astype(np.int32)
        else:
            fdt = np.dtype([("k", ext + "u1"), ("v1", ext + "i4"), ("v2", ext + "i4"), ("v3", ext + "i4")])
            fd = np.fromfile(f, dtype=fdt, count=nf)
            faces = np.stack([fd["v1"], fd["v2"], fd["v3"]], axis=1).astype(np.int32)
        return [data, faces]


def vertex_count(filename) -> int:
    """Number of vertices from the header alone (the payload is not read): the ``vertex`` element's count, or the first
    element's as read_ply uses it."""
    with open(filename, "rb") as f:
        h = parse_header(f)
    v = h.element("vertex") or (h.elements[0] if h.elements else None)
    if v is None:
        raise ValueError("PLY file without elements")
    return v[1]


def write_ply(filename, fields: Dict[str, np.ndarray], fmt: str = "binary_little_endian"):
    """Writer used by the tests and by ``save`` of the demo session: one scalar property per dict entry."""
    names = list(fields)
    n = len(fields[names[0]])
    inv = {"i1": "char", "u1": "uchar", "i2": "short", "u2": "ushort", "i4": "int", "u4": "uint", "f4": "float", "f8": "double"}
    ext = _ENDIAN[fmt]
    head = ["ply", f"format {fmt} 1.0", f"element vertex {n}"]
    dt = []
    for k in names:
        a = np.asarray(fields[k])
        code = a.dtype.str[1:]
        if code not in inv:
            raise ValueError(f"unsupported dtype {a.dtype} for PLY property {k}")
        head.append(f"property {inv[code]} {k}")
        dt.append((k, ext + code))
    head.append("end_header")
    rec = np.empty(n, dtype=np.dtype(dt))
    for k in names:
        rec[k] = fields[k]
    with open(filename, "wb") as f:
        f.write(("\n".join(head) + "\n").encode())
        if fmt == "ascii":
            for r in rec:
                f.write((" ".join(repr(x.item()) if rec.dtype[i].kind == "f" else str(x.item()) for i, x in enumerate(r)) + "\n").encode())
        else:
            rec.tofile(f)


def load_ply(filename) -> np.ndarray:
    """demo/utils.py:4-30: ASCII PLY with exactly 6 columns -> float64 [n, 6] (x y z r g b, colours 0..255)."""
    with open(filename, "rb") as f:
        h = parse_header(f)
        if h.format != "ascii":
            raise NotImplementedError("demo loader reads ASCII PLY only")
        n = h.element("vertex")[1]
        pts = np.loadtxt(io.BytesIO(b"".join(f.readline() for _ in range(n))), dtype=np.float64, ndmin=2)
    assert pts.shape == (n, 6), pts.shape
    return pts


def normalize_points(points: np.ndarray) -> np.ndarray:
    """eval_kitti.py:82-88 - centre on the centroid, scale so the farthest point has norm 1."""
    assert points.ndim == 2 and points.shape[1] == 3, points.shape
    points = points - np.mean(points, axis=0)
    return points / np.max(np.linalg.norm(points, ord=2, axis=1))


def normalize_colors(features: np.ndarray, mean: Optional[float] = 0.5, std: Optional[float] = 0.5) -> np.ndarray:
    """eval_kitti.py:73-79 - 0..255 colours -> [-1, 1]."""
    features = features / 255
    if mean is not None:
        features = features - mean
    if std is not None:
        features = features / std
    return features
