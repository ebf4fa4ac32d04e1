"""Quadric decimation and clean-up of an extracted mesh (csrc/sgr_decimate.cu).

Both coarse-mesh extraction branches of the reference end with open3d (sugar_extractors/coarse_mesh.py:433-463,
:716-744):

    decimated = mesh.simplify_quadric_decimation(decimation_target)
    decimated.remove_degenerate_triangles(); decimated.remove_duplicated_triangles()
    decimated.remove_duplicated_vertices();  decimated.remove_non_manifold_edges()

Here, without open3d:

    m = simplify_quadric_decimation(verts, faces, target, colors, normals)      # rounds of parallel edge collapses
    m = clean_mesh(m["verts"], m["faces"], m["colors"], m["normals"])           # the four passes, in that order

The rules are restated from open3d's published algorithm in oracle/decimate_oracle.py (not checked against open3d,
which is not available here), and the op equals its `decimate_rounds` array for array.  Deliberate differences from
open3d: the collapses run in rounds of independent edges (each round takes every edge whose key is least in its
two-ring, so the order differs from one heap; quality is measured against the sequential loop in the tests); equal
costs go to the lower (a, b); an edge counts only while a live face holds it; vertices no face references are dropped;
colours and normals are averaged in float64; the non-manifold pass visits edges in ascending (a, b) order.
"""
import numpy as np
import torch

from ._lib import check, lib, ptr, require_cuda, scratch, stream, tensor


def simplify_quadric_decimation(verts, faces, target, colors=None, normals=None):
    """open3d's simplify_quadric_decimation(target) (maximum_error = inf, boundary_weight = 1) for a CUDA mesh:
    verts float32 [V,3], faces int64 [F,3] (no face repeats a vertex), optional per-vertex colors / normals float32
    [V,3].  -> {"verts" f32 [V',3], "faces" i64 [F',3], "colors", "normals" (None when not given), "rounds": int,
    "last_removed": faces removed by the collapse that reached the target (0 if it was not reached)}.
    F' <= target unless no edge can be collapsed; the vertices are those the faces reference, in their order."""
    require_cuda("decimate", verts)
    dev = verts.device
    verts = tensor(verts, "verts", torch.float32, ("V", 3))
    faces = tensor(faces, "faces", torch.int64, ("F", 3), dev)
    target = int(target)
    if target < 0:
        raise ValueError(f"target = {target}: must be >= 0")
    V, F = verts.shape[0], faces.shape[0]
    colors = None if colors is None else tensor(colors, "colors", torch.float32, (V, 3), dev)
    normals = None if normals is None else tensor(normals, "normals", torch.float32, (V, 3), dev)
    with torch.cuda.device(dev):
        ws = scratch(lib.sgr_decimate_scratch_bytes(V, F), dev)
        vo, fo = torch.empty_like(verts), torch.empty_like(faces)
        co = None if colors is None else torch.empty_like(colors)
        no = None if normals is None else torch.empty_like(normals)
        res = np.zeros(4, np.int64)
        check(lib.sgr_decimate(V, F, target, ptr(verts), ptr(faces), ptr(colors), ptr(normals), ptr(vo), ptr(fo),
                               ptr(co), ptr(no), res.ctypes.data, ws.data_ptr(), stream(dev)))
    nv, nf = int(res[0]), int(res[1])
    cut = lambda t, n: None if t is None else t[:n].clone()
    return {"verts": cut(vo, nv), "faces": cut(fo, nf), "colors": cut(co, nv), "normals": cut(no, nv),
            "rounds": int(res[2]), "last_removed": int(res[3])}


def _first_of_groups(rows):
    """-> (index of the first row equal to each row, mask of first occurrences) for a 2-D tensor."""
    n = rows.shape[0]
    ar = torch.arange(n, device=rows.device)
    _, inv = torch.unique(rows, dim=0, return_inverse=True)
    first = torch.full((n,), n, dtype=torch.int64, device=rows.device).scatter_reduce(0, inv, ar, "amin")[inv]
    return first, first == ar


def _areas(verts, faces):
    """0.5 |(p1 - p0) x (p2 - p0)| in float64, one rounding per operation (the oracle's arithmetic)."""
    v = verts.double()
    p0, p1, p2 = v[faces[:, 0]], v[faces[:, 1]], v[faces[:, 2]]
    u, w = p1 - p0, p2 - p0
    nx = u[:, 1] * w[:, 2] - u[:, 2] * w[:, 1]
    ny = u[:, 2] * w[:, 0] - u[:, 0] * w[:, 2]
    nz = u[:, 0] * w[:, 1] - u[:, 1] * w[:, 0]
    return 0.5 * ((nx * nx + ny * ny) + nz * nz).sqrt()


def clean_mesh(verts, faces, colors=None, normals=None):
    """open3d's remove_degenerate_triangles, remove_duplicated_triangles, remove_duplicated_vertices and
    remove_non_manifold_edges, in that order (the rules of oracle/decimate_oracle.py), on any device.
    -> {"verts", "faces", "colors", "normals"}; vertices that no face references are kept, as in open3d."""
    dev = faces.device
    f = faces
    f = f[(f[:, 0] != f[:, 1]) & (f[:, 1] != f[:, 2]) & (f[:, 0] != f[:, 2])]
    if f.shape[0]:
        rot = (f.argmin(dim=1, keepdim=True) + torch.arange(3, device=dev)) % 3
        f = f[_first_of_groups(f.gather(1, rot))[1]]
    if verts.shape[0]:
        first, keep = _first_of_groups(verts.double() + 0.0)     # + 0.0: -0 and +0 are one coordinate
        remap = torch.cumsum(keep.long(), 0) - 1
        f = remap[first][f]
        verts = verts[keep]
        colors = None if colors is None else colors[keep]
        normals = None if normals is None else normals[keep]
    while f.shape[0]:
        e = torch.sort(torch.stack([f, f.roll(-1, 1)], 2).reshape(-1, 2), dim=1)[0]
        _, inv, cnt = torch.unique(e, dim=0, return_inverse=True, return_counts=True)
        slots = torch.nonzero(cnt[inv] > 2)[:, 0]
        if not slots.numel():
            break
        # few edges: visit them in ascending (a, b) order (torch.unique sorts) on the host
        groups, fids = inv[slots].cpu().numpy(), (slots // 3).cpu().numpy()
        area = _areas(verts, f[torch.from_numpy(np.unique(fids)).to(dev)]).cpu().numpy()
        area_of = dict(zip(np.unique(fids).tolist(), area.tolist()))
        order = np.lexsort((fids, groups))
        groups, fids = groups[order], fids[order]
        starts = np.unique(groups, return_index=True)[1].tolist() + [len(groups)]
        dead = set()
        for s, e in zip(starts[:-1], starts[1:]):
            fs = [t for t in fids[s:e].tolist() if t not in dead]
            fs.sort(key=lambda t: (area_of[t], t))
            dead.update(fs[:max(len(fs) - 2, 0)])
        keep = torch.ones(f.shape[0], dtype=torch.bool, device=dev)
        keep[torch.tensor(sorted(dead), dtype=torch.int64, device=dev)] = False
        f = f[keep]
    return {"verts": verts, "faces": f, "colors": colors, "normals": normals}
