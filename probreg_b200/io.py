"""Caller-side helpers so that scripts written against the reference run without open3d:
readers for the point-cloud files the reference ships (ASCII ``.pcd``, binary/ASCII ``.ply``, whitespace ``.txt``) and a
voxel-grid down-sampler in the spirit of ``open3d.geometry.PointCloud.voxel_down_sample`` (per-voxel mean; the
reference's examples/utils.py:20 and tests/test_cpd.py:12 use open3d's).  Plain numpy on the host -- this is data
preparation before ``registration_cpd``, not part of the EM path."""
import numpy as np

_PLY_TYPES = {"char": "i1", "int8": "i1", "uchar": "u1", "uint8": "u1", "short": "i2", "int16": "i2", "ushort": "u2",
              "uint16": "u2", "int": "i4", "int32": "i4", "uint": "u4", "uint32": "u4", "float": "f4", "float32": "f4",
              "double": "f8", "float64": "f8"}


def read_pcd(path):
    """x, y, z (and nothing else) of an ASCII ``.pcd`` file -> (n, 3) float64."""
    fields, data_start = None, None
    with open(path, "r") as f:
        lines = f.read().splitlines()
    for i, line in enumerate(lines):
        tok = line.split()
        if not tok or tok[0].startswith("#"):
            continue
        if tok[0] == "FIELDS":
            fields = tok[1:]
        elif tok[0] == "DATA":
            if tok[1].lower() != "ascii":
                raise ValueError("only ASCII .pcd files are supported, got DATA %s" % tok[1])
            data_start = i + 1
            break
    if fields is None or data_start is None:
        raise ValueError("%s: not a PCD file" % path)
    cols = [fields.index(c) for c in ("x", "y", "z")]
    rows = [l.split() for l in lines[data_start:] if l.strip()]
    return np.array([[float(r[c]) for c in cols] for r in rows], dtype=np.float64)


def read_ply(path):
    """Vertex x, y, z of a ``.ply`` file (ascii, binary_little_endian or binary_big_endian) -> (n, 3) float64."""
    with open(path, "rb") as f:
        if f.readline().strip() != b"ply":
            raise ValueError("%s: not a PLY file" % path)
        fmt, n_vertex, props, in_vertex = None, 0, [], False
        before = []          # elements declared BEFORE the vertex element: (count, [(name, type) or ("list", count type, item type)])
        while True:
            line = f.readline()
            if not line:
                raise ValueError("%s: unterminated PLY header" % path)
            tok = line.decode("ascii", "replace").split()
            if not tok:
                continue
            if tok[0] == "format":
                fmt = tok[1]
            elif tok[0] == "element":
                in_vertex = tok[1] == "vertex"
                if in_vertex:
                    n_vertex = int(tok[2])
                elif n_vertex == 0:
                    before.append((int(tok[2]), []))
            elif tok[0] == "property" and in_vertex:
                if tok[1] == "list":
                    raise ValueError("list properties on vertices are not supported")
                props.append((tok[2], _PLY_TYPES[tok[1]]))
            elif tok[0] == "property" and before and n_vertex == 0:
                before[-1][1].append(tuple(tok[1:]))
            elif tok[0] == "end_header":
                break
        names = [p[0] for p in props]
        if n_vertex == 0 or not all(c in names for c in ("x", "y", "z")):
            raise ValueError("%s: no vertex element with x, y, z properties" % path)
        # skip whatever the file stores in front of the vertices (rare, but legal PLY)
        for count, eprops in before:
            if fmt == "ascii":
                for _ in range(count):
                    f.readline()
            elif any(p[0] == "list" for p in eprops):
                raise ValueError("%s: a list-valued element precedes the vertices in a binary file" % path)
            else:
                f.read(count * sum(np.dtype(_PLY_TYPES[p[0]]).itemsize for p in eprops))
        if fmt == "ascii":
            rows = [f.readline().split() for _ in range(n_vertex)]
            return np.array([[float(r[names.index(c)]) for c in ("x", "y", "z")] for r in rows], dtype=np.float64)
        order = {"binary_little_endian": "<", "binary_big_endian": ">"}[fmt]
        dt = np.dtype([(nm, order + tp) for nm, tp in props])
        v = np.frombuffer(f.read(dt.itemsize * n_vertex), dtype=dt, count=n_vertex)
        return np.stack([v["x"], v["y"], v["z"]], axis=1).astype(np.float64)


def read_points(path):
    """Dispatch on the extension: .pcd, .ply, anything else via numpy.loadtxt."""
    low = path.lower()
    if low.endswith(".pcd"):
        return read_pcd(path)
    if low.endswith(".ply"):
        return read_ply(path)
    return np.atleast_2d(np.loadtxt(path)).astype(np.float64)


def voxel_down_sample(points, voxel_size):
    """One point per occupied voxel of edge ``voxel_size``: the mean of the points inside (voxel grid anchored at the
    cloud's minimum corner, like open3d's; the order of the output follows the voxel index)."""
    pts = np.asarray(points, dtype=np.float64)
    if voxel_size <= 0:
        raise ValueError("voxel_size must be positive")
    key = np.floor((pts - pts.min(axis=0)) / voxel_size).astype(np.int64)
    _, inv, cnt = np.unique(key, axis=0, return_inverse=True, return_counts=True)
    inv = inv.ravel()
    out = np.zeros((cnt.shape[0], pts.shape[1]))
    np.add.at(out, inv, pts)
    return out / cnt[:, None]
