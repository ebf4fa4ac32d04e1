"""The 3DGS .ply files at both ends of SuGaR's pipeline (torch, numpy and the standard library only).

    save_gaussians_ply(path, raw)                   # GaussianModel.save_ply: point_cloud/iteration_N/point_cloud.ply
    raw = load_gaussians_ply(path, sh_degree=3)     # GaussianModel.load_ply: what SuGaR's train.py -c reads
    points, colors = read_sfm_points(path)          # dataset_readers.fetchPly of a COLMAP points3D.ply
    export_refined_ply(path, raw, mesh)             # refine.py --export_ply: convert_refined_sugar_into_gaussians

`raw` is steps.activate's dict (points [P,3], sh_dc [P,1,3], sh_rest [P,M-1,3], densities [P,1] logit, scales [P,3]
log, quaternions [P,4] unnormalised), vanilla's _xyz, _features_dc, _features_rest, _opacity, _scaling, _rotation one
to one.  The vertex element holds x y z nx ny nz f_dc_0..2 f_rest_0.. opacity scale_0.. rot_0..3, all float32,
normals zero, f_rest channel-major (sh_rest.transpose(1, 2).flatten(1)).  The header is the one plyfile writes for
PlyElement.describe(elements, 'vertex') as its source reads: ASCII lines joined by '\\n' -- `ply`,
`format binary_little_endian 1.0`, `element vertex N`, one `property float <name>` per property, `end_header` --
then the rows.  plyfile itself was not run against this writer.
"""
import os

import numpy as np
import torch

_PLY_TYPES = {"float": "<f4", "float32": "<f4", "double": "<f8", "float64": "<f8", "uchar": "u1", "uint8": "u1"}


def _header(n, names):
    lines = ["ply", "format binary_little_endian 1.0", f"element vertex {n}"]
    lines += [f"property float {name}" for name in names] + ["end_header"]
    return ("\n".join(lines) + "\n").encode("ascii")


def _write(path, columns):
    """columns: [(name, float32 [P] array)] -> the vertex-only binary little-endian file."""
    P = columns[0][1].shape[0] if columns else 0
    rows = np.empty(P, dtype=[(name, "<f4") for name, _ in columns])
    for name, v in columns:
        rows[name] = v
    d = os.path.dirname(path)
    if d:
        os.makedirs(d, exist_ok=True)
    with open(path, "wb") as f:
        f.write(_header(P, [name for name, _ in columns]))
        f.write(rows.tobytes())


def gaussian_columns(points, sh_dc, sh_rest, densities, scales, quaternions):
    """-> [(property name, float32 [P] column)] in construct_list_of_attributes' order."""
    f = lambda t: t.detach().float().cpu().numpy()
    P = points.shape[0]
    xyz = f(points).reshape(P, 3)
    f_dc = f(sh_dc.transpose(1, 2).flatten(1)).reshape(P, -1)
    f_rest = f(sh_rest.transpose(1, 2).flatten(1)).reshape(P, -1)
    opac, scl, rot = f(densities).reshape(P, -1), f(scales).reshape(P, -1), f(quaternions).reshape(P, -1)
    cols = [(a, xyz[:, i]) for i, a in enumerate("xyz")] + [(a, np.zeros(P, np.float32)) for a in ("nx", "ny", "nz")]
    cols += [(f"f_dc_{i}", f_dc[:, i]) for i in range(f_dc.shape[1])]
    cols += [(f"f_rest_{i}", f_rest[:, i]) for i in range(f_rest.shape[1])]
    cols += [("opacity", opac[:, 0])]
    cols += [(f"scale_{i}", scl[:, i]) for i in range(scl.shape[1])]
    cols += [(f"rot_{i}", rot[:, i]) for i in range(rot.shape[1])]
    return cols


def save_gaussians_ply(path, raw):
    """GaussianModel.save_ply (gaussian_model.py:191-208) of `raw` (see the module docstring)."""
    _write(path, gaussian_columns(raw["points"], raw["sh_dc"], raw["sh_rest"], raw["densities"], raw["scales"],
                                  raw["quaternions"]))


def read_ply(path):
    """-> (element name, {property: numpy array}) of a binary little-endian .ply with one element whose properties
    are float, double or uchar scalars.  Raises ValueError on anything else (ASCII or big-endian data, list
    properties, other types, a short file)."""
    with open(path, "rb") as f:
        data = f.read()
    end = data.find(b"end_header")
    if not data.startswith(b"ply") or end < 0:
        raise ValueError(f"{path}: not a .ply file (no 'ply' magic or no end_header)")
    nl = data.find(b"\n", end)
    body = data[nl + 1:] if nl >= 0 else b""
    lines = [ln.strip() for ln in data[:end].decode("ascii", errors="replace").splitlines()]
    fmt, elements = None, []
    for ln in lines[1:]:
        tok = ln.split()
        if not tok or tok[0] in ("comment", "obj_info"):
            continue
        if tok[0] == "format":
            fmt = tok[1] if len(tok) > 1 else None
        elif tok[0] == "element":
            elements.append((tok[1], int(tok[2]), []))
        elif tok[0] == "property":
            if not elements:
                raise ValueError(f"{path}: property before any element")
            if tok[1] == "list" or tok[1] not in _PLY_TYPES:
                raise ValueError(f"{path}: property {' '.join(tok[1:])!r} is not a float, double or uchar scalar")
            elements[-1][2].append((tok[2], _PLY_TYPES[tok[1]]))
    if fmt != "binary_little_endian":
        raise ValueError(f"{path}: format {fmt!r} is not supported (binary_little_endian only)")
    if len(elements) != 1:
        raise ValueError(f"{path}: expected one element, found {len(elements)}")
    name, n, props = elements[0]
    dtype = np.dtype(props)
    if len(body) < n * dtype.itemsize:
        raise ValueError(f"{path}: {len(body)} bytes of data for {n} rows of {dtype.itemsize} bytes")
    rows = np.frombuffer(body, dtype=dtype, count=n)
    return name, {p: rows[p] for p, _ in props}


def _sorted_names(props, prefix):
    return sorted((p for p in props if p.startswith(prefix)), key=lambda x: int(x.split("_")[-1]))


def load_gaussians_ply(path, sh_degree=3, device="cuda"):
    """GaussianModel.load_ply (gaussian_model.py:215-256): -> the raw dict of float32 leaf tensors on `device`.
    Properties are found by name in any order; f_rest_*, scale_* and rot_* are sorted by their numeric suffix; the
    f_rest count must be 3 (sh_degree + 1)^2 - 3 (ValueError otherwise)."""
    _, props = read_ply(path)
    need = ["x", "y", "z", "opacity", "f_dc_0", "f_dc_1", "f_dc_2"]
    missing = [p for p in need if p not in props]
    if missing:
        raise ValueError(f"{path}: missing properties {missing}")
    col = lambda names: np.stack([np.asarray(props[p], dtype=np.float64) for p in names], axis=1)
    xyz = col(["x", "y", "z"])
    P = xyz.shape[0]
    extra = _sorted_names(props, "f_rest_")
    want = 3 * (sh_degree + 1) ** 2 - 3
    if len(extra) != want:
        raise ValueError(f"{path}: {len(extra)} f_rest properties, sh_degree {sh_degree} needs {want}")
    M1 = (sh_degree + 1) ** 2 - 1
    f_rest = col(extra) if extra else np.zeros((P, 0))
    scales = col(_sorted_names(props, "scale_"))
    rots = col(_sorted_names(props, "rot"))
    t = lambda a: torch.tensor(a, dtype=torch.float, device=device)
    return dict(points=t(xyz).requires_grad_(True),
                sh_dc=t(col(["f_dc_0", "f_dc_1", "f_dc_2"]).reshape(P, 3, 1)).transpose(1, 2).contiguous()
                .requires_grad_(True),
                sh_rest=t(f_rest.reshape(P, 3, M1)).transpose(1, 2).contiguous().requires_grad_(True),
                densities=t(col(["opacity"])).requires_grad_(True), scales=t(scales).requires_grad_(True),
                quaternions=t(rots).requires_grad_(True))


def read_sfm_points(path):
    """dataset_readers.fetchPly of a points3D.ply (storePly's layout: x y z nx ny nz float, red green blue uchar):
    -> (points float32 [P,3], colors float64 [P,3] = uint8 / 255), numpy arrays as the reference's BasicPointCloud
    holds them."""
    _, props = read_ply(path)
    missing = [p for p in ("x", "y", "z", "red", "green", "blue") if p not in props]
    if missing:
        raise ValueError(f"{path}: missing properties {missing}")
    positions = np.vstack([props["x"], props["y"], props["z"]]).T
    colors = np.vstack([props["red"], props["green"], props["blue"]]).T / 255.0
    return positions, colors


def export_refined_ply(path, raw, mesh):
    """refine.py's --export_ply (convert_refined_sugar_into_gaussians + save_ply) of a refined model: `raw` and `mesh`
    as steps.refine_step takes them.  Points, scales (log of the bound scaling, thickness axis included) and
    quaternions come from meshbind.bind_to_mesh; densities and the SH columns are the raw tensors."""
    from . import meshbind
    with torch.no_grad():
        a = meshbind.bind_to_mesh(raw["verts"], mesh.faces, mesh.bary, raw["scales"], raw["quaternions"],
                                  mesh.thickness)
        _write(path, gaussian_columns(a.points, raw["sh_dc"], raw["sh_rest"], raw["densities"],
                                      torch.log(a.scaling), a.quaternions))
