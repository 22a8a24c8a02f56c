"""CAD model vertices for the LINEMOD metrics: a small PLY reader standing in for the reference's
``load_points_from_cad`` / ``model_diameter_from_bbox`` (src/utils/sample_points_on_cad.py:47-82,
which read the mesh with open3d's ``read_triangle_mesh``).

Reads ``ascii``, ``binary_little_endian`` and ``binary_big_endian`` files whose first element is
``vertex`` with scalar properties, of which ``x``, ``y`` and ``z`` are the coordinates.  Other
scalar vertex properties (normals, colours) are skipped; elements after ``vertex`` (faces, ...)
are ignored.  Anything else raises a ``ValueError`` naming the file."""
import numpy as np

__all__ = ["read_ply_vertices", "load_points_from_cad", "model_diameter_from_bbox"]

_TYPES = {"char": "i1", "int8": "i1", "uchar": "u1", "uint8": "u1", "short": "i2", "int16": "i2",
          "ushort": "u2", "uint16": "u2", "int": "i4", "int32": "i4", "uint": "u4", "uint32": "u4",
          "float": "f4", "float32": "f4", "double": "f8", "float64": "f8"}
_FORMATS = {"ascii": None, "binary_little_endian": "<", "binary_big_endian": ">"}


def _parse_header(path, raw):
    end = raw.find(b"end_header")
    if not raw.startswith(b"ply") or end < 0:
        raise ValueError(f"{path}: not a PLY file (no 'ply' magic or 'end_header')")
    nl = raw.find(b"\n", end)
    body = len(raw) if nl < 0 else nl + 1
    fmt, count, props, element = None, None, [], None
    for line in raw[:end].decode("ascii", errors="replace").splitlines()[1:]:
        tok = line.split()
        if not tok or tok[0] in ("comment", "obj_info"):
            continue
        if tok[0] == "format":
            if len(tok) < 2 or tok[1] not in _FORMATS:
                raise ValueError(f"{path}: unsupported PLY format line {line!r}")
            fmt = tok[1]
        elif tok[0] == "element":
            if element is None and (len(tok) != 3 or tok[1] != "vertex"):
                raise ValueError(f"{path}: the first PLY element must be 'vertex', got {line!r}")
            element = tok[1] if element is None else "after-vertex"
            if element == "vertex":
                try:
                    count = int(tok[2])
                except ValueError:
                    raise ValueError(f"{path}: bad vertex count in {line!r}") from None
        elif tok[0] == "property":
            if element == "vertex":
                if len(tok) != 3 or tok[1] not in _TYPES:
                    raise ValueError(f"{path}: unsupported vertex property {line!r} (scalar properties only)")
                props.append((tok[2], _TYPES[tok[1]]))
            elif element is None:
                raise ValueError(f"{path}: property before any element: {line!r}")
        else:
            raise ValueError(f"{path}: unexpected PLY header line {line!r}")
    if fmt is None or count is None or count < 0:
        raise ValueError(f"{path}: PLY header lacks a format line or a vertex element")
    names = [n for n, _ in props]
    if any(names.count(n) > 1 for n in names) or not {"x", "y", "z"} <= set(names):
        raise ValueError(f"{path}: vertex element needs one each of x, y, z properties, got {names}")
    return fmt, count, props, body


def read_ply_vertices(path):
    """Vertex coordinates of a PLY file in file order, as float64 [V, 3] (values exactly as stored;
    ascii values as parsed to double)."""
    with open(path, "rb") as f:
        raw = f.read()
    fmt, count, props, body = _parse_header(path, raw)
    names = [n for n, _ in props]
    cols = [names.index(c) for c in "xyz"]
    if fmt == "ascii":
        lines = raw[body:].decode("ascii", errors="replace").splitlines()
        lines = [ln for ln in lines if ln.strip()][:count]
        if len(lines) < count:
            raise ValueError(f"{path}: {len(lines)} vertex lines, header declares {count}")
        try:
            rows = [[float(v) for v in ln.split()] for ln in lines]
        except ValueError as e:
            raise ValueError(f"{path}: bad ascii vertex value ({e})") from None
        if any(len(r) != len(props) for r in rows):
            raise ValueError(f"{path}: ascii vertex line with other than {len(props)} values")
        v = np.array(rows, dtype=np.float64).reshape(count, len(props))
        return np.ascontiguousarray(v[:, cols])
    dt = np.dtype([(n, _FORMATS[fmt] + t) for n, t in props])
    if len(raw) - body < count * dt.itemsize:
        raise ValueError(f"{path}: truncated: {count} vertices of {dt.itemsize} bytes declared, "
                         f"{len(raw) - body} bytes of data")
    rec = np.frombuffer(raw, dtype=dt, count=count, offset=body)
    return np.stack([rec[c].astype(np.float64) for c in "xyz"], axis=-1)


def load_points_from_cad(path):
    """sample_points_on_cad.py:47-75 with max_num = -1: (vertices fp32 [V, 3], the 8 bounding-box
    corners followed by their centre, fp32 [9, 3])."""
    v = read_ply_vertices(path)
    if v.shape[0] == 0:
        raise ValueError(f"{path}: the model has no vertices")
    lo, hi = v.min(0), v.max(0)
    corners = np.array([[x, y, z] for x in (lo[0], hi[0]) for y in (lo[1], hi[1]) for z in (lo[2], hi[2])])
    centre = (corners.max(0, keepdims=True) + corners.min(0, keepdims=True)) / 2
    return v.astype(np.float32), np.concatenate([corners, centre], 0).astype(np.float32)


def model_diameter_from_bbox(bbox):
    """sample_points_on_cad.py:77-84: |max corner - min corner| of a 8x3 or 9x3 corner array."""
    return np.linalg.norm(bbox[7] - bbox[0])
