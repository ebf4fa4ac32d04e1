"""CPU restatement of the splatted mesh and the nearest-face z-buffer -- TEST INFRASTRUCTURE ONLY.

Follows, op for op in PyTorch (float64 here):
    SuGaR.triangle_vertices, primitive 'diamond'   sugar_scene/sugar_model.py:481-514
    SuGaR.splat_mesh, mode 'perspective'           sugar_scene/sugar_model.py:695-728
    SuGaR.triangles                                sugar_scene/sugar_model.py:254-256, 523-528
with pytorch3d's quaternion_to_matrix / quaternion_apply from oracle/field_oracle.py and matrix_to_quaternion from
oracle/meshbind_oracle.py.  The camera is this package's (the rasterizer's transposed world->view matrix as a
row-vector transform, its inverse for the way back), standing in for get_world_to_view_transform().

`rasterize` restates pytorch3d 0.7.4's MeshRasterizer as the extraction configures it (blur_radius 0, perspective-correct
barycentrics, no culling) read at its first face per pixel, by brute force over every face's pixel box, in float64, in
this package's pixel convention (the sample of pixel (i, j) at ndc (2i+1)/S - 1, vertices through viewmatrix for the
view z and through projmatrix / (w + 1e-7)).  A face is skipped when max z < 0, its screen area is <= 1e-8 in
pytorch3d's NDC units (2 / min(W, H) per pixel) or a vertex is not finite; it covers a pixel when every b'_i > 0 and
pz >= 0, with w_i = b_i z_j z_k, b' = w / max(sum w, 1e-8), pz = sum b'_i z_i.  The pixel keeps the least pz (equal pz:
the lower face id).  Besides the winner it reports the margins a float32 implementation can disagree within:
`min_bary` (the winner's least b'), `bary_margin` (over every face tested at the pixel, the least |min_i b'_i|: how
close the pixel is to some face's edge) and `depth_gap` (runner-up pz minus the winner's; inf with fewer than two).
"""
import numpy as np
import torch

from oracle import field_oracle as fo
from oracle import meshbind_oracle as mbo

DIAMOND = [[0.0, -1.0, 0.0], [0.0, 0.0, 1.0], [0.0, 1.0, 0.0], [0.0, 0.0, -1.0]]   # sugar_model.py:242-245
TRIANGLES = [[0, 2, 1], [0, 3, 2]]                                                    # sugar_model.py:254-256


def triangle_vertices(points, scaling, quaternions, triangle_scale=2.0):
    """[4P,3]: the diamond of every Gaussian in its frame with the smallest axis first (ties: lowest index)."""
    a0 = scaling.argmin(dim=-1)
    perm = torch.stack([a0, (a0 + 1) % 3, (a0 + 2) % 3], dim=-1)                     # :494-496
    scale_sort = scaling.gather(dim=1, index=perm)                                     # :502
    rot = fo.quaternion_to_matrix(quaternions)
    rot_sort = rot.gather(dim=2, index=perm[..., None, :].expand(-1, 3, -1))           # :506
    q_sort = mbo.matrix_to_quaternion(rot_sort)                                        # :507
    prim = torch.tensor(DIAMOND, dtype=points.dtype)[None]
    v = points.unsqueeze(1) + fo.quaternion_apply(q_sort.unsqueeze(1), prim * triangle_scale * scale_sort.unsqueeze(1))
    return v.reshape(-1, 3)


def splat_mesh(points, scaling, quaternions, viewmatrix, triangle_scale=2.0):
    """(verts [4P,3], faces [2P,3] int64) of SuGaR.splat_mesh; viewmatrix [4,4] transposed world->view."""
    view = viewmatrix.to(points.dtype)
    inv = torch.linalg.inv(view)
    to_view = lambda p: p @ view[:3, :3] + view[3, :3]
    n = points.shape[0]
    v = to_view(triangle_vertices(points, scaling, quaternions, triangle_scale)).reshape(n, 4, 3)   # :704
    c = to_view(points).reshape(n, 1, 3)                                                              # :705
    d = torch.nn.functional.normalize(c, dim=-1)                                                      # :710
    v = ((c * d).sum(-1, keepdim=True) / (v * d).sum(-1, keepdim=True)) * v                         # :711-713
    verts = v.reshape(-1, 3) @ inv[:3, :3] + inv[3, :3]                                              # :715
    faces = (4 * torch.arange(n)[:, None, None] + torch.tensor(TRIANGLES)[None]).reshape(-1, 3)      # :524-528
    return verts, faces


def project(verts, viewmatrix, projmatrix, W, H):
    """-> pixel x, y (ndc2pix units) and view z of every vertex, float64."""
    v = np.asarray(verts, np.float64)
    vm, pm = np.asarray(viewmatrix, np.float64), np.asarray(projmatrix, np.float64)
    z = v @ vm[:3, 2] + vm[3, 2]
    hom = v @ pm[:3, :] + pm[3, :]
    with np.errstate(all="ignore"):
        ndc = hom[:, :2] / (hom[:, 3:4] + 1e-7)
    return ((ndc[:, 0] + 1.0) * W - 1.0) * 0.5, ((ndc[:, 1] + 1.0) * H - 1.0) * 0.5, z


def rasterize(verts, faces, viewmatrix, projmatrix, W, H, chunk_pairs=4_000_000):
    """-> dict of [H,W] arrays: pix_to_face (int64, -1 empty), zbuf (-1 empty), min_bary, bary_margin, depth_gap."""
    x, y, z = project(verts, viewmatrix, projmatrix, W, H)
    f = np.asarray(faces, np.int64)
    F = f.shape[0]
    inb = ((f >= 0) & (f < len(x))).all(1)
    fs = np.where(inb[:, None], f, 0)
    X, Y, Z = x[fs], y[fs], z[fs]
    half = 0.5 * min(W, H)
    with np.errstate(all="ignore"):
        area = (X[:, 2] - X[:, 0]) * (Y[:, 1] - Y[:, 0]) - (Y[:, 2] - Y[:, 0]) * (X[:, 1] - X[:, 0])
        ok = inb & np.isfinite(X).all(1) & np.isfinite(Y).all(1) & np.isfinite(Z).all(1)
        ok &= Z.max(1) >= 0.0
        ok &= np.abs(area) > 1e-8 * half * half
        x0 = np.ceil(np.clip(X.min(1), 0, W)).astype(np.int64)
        x1 = np.floor(np.clip(X.max(1), -1, W - 1)).astype(np.int64)
        y0 = np.ceil(np.clip(Y.min(1), 0, H)).astype(np.int64)
        y1 = np.floor(np.clip(Y.max(1), -1, H - 1)).astype(np.int64)
    ok &= (x0 <= x1) & (y0 <= y1)
    ids = np.nonzero(ok)[0]
    bw, bh = (x1 - x0 + 1)[ids], (y1 - y0 + 1)[ids]
    counts = bw * bh
    margin = np.full(W * H, np.inf)
    hits = []
    start = 0
    while start < len(ids):
        stop = start + max(1, int(np.searchsorted(np.cumsum(counts[start:]), chunk_pairs)))
        sel = np.arange(start, min(stop, len(ids)))
        start = sel[-1] + 1
        c = counts[sel]
        fi = np.repeat(sel, c)
        k = np.arange(c.sum()) - np.repeat(np.cumsum(c) - c, c)
        face = ids[fi]
        px = x0[face] + k % bw[fi]
        py = y0[face] + k // bw[fi]
        Xf, Yf, Zf = X[face], Y[face], Z[face]
        b = np.empty((len(face), 3))
        for e in range(3):
            a_, b_ = (e + 1) % 3, (e + 2) % 3
            b[:, e] = ((px - Xf[:, a_]) * (Yf[:, b_] - Yf[:, a_]) - (py - Yf[:, a_]) * (Xf[:, b_] - Xf[:, a_])) / area[face]
        w = b * np.stack([Zf[:, 1] * Zf[:, 2], Zf[:, 0] * Zf[:, 2], Zf[:, 0] * Zf[:, 1]], 1)
        bp = w / np.maximum(w.sum(1), 1e-8)[:, None]
        pz = (bp * Zf).sum(1)
        mb = bp.min(1)
        pix = py * W + px
        np.minimum.at(margin, pix, np.abs(mb))
        cov = (mb > 0) & (pz >= 0) & np.isfinite(pz)
        hits.append((pix[cov], pz[cov], face[cov], mb[cov]))
    p2f = np.full(W * H, -1, np.int64)
    zbuf = np.full(W * H, -1.0)
    min_bary = np.full(W * H, np.nan)
    gap = np.full(W * H, np.inf)
    if hits:
        pix, pz, face, mb = (np.concatenate(v) for v in zip(*hits))
        order = np.lexsort((face, pz, pix))
        pix, pz, face, mb = pix[order], pz[order], face[order], mb[order]
        first = np.ones(len(pix), bool)
        first[1:] = pix[1:] != pix[:-1]
        w = np.nonzero(first)[0]
        p2f[pix[w]], zbuf[pix[w]], min_bary[pix[w]] = face[w], pz[w], mb[w]
        second = w + 1
        has2 = second < len(pix)
        has2[has2] = ~first[second[has2]]
        gap[pix[w[has2]]] = pz[second[has2]] - pz[w[has2]]
    shape = (H, W)
    return dict(pix_to_face=p2f.reshape(shape), zbuf=zbuf.reshape(shape), min_bary=min_bary.reshape(shape),
                bary_margin=margin.reshape(shape), depth_gap=gap.reshape(shape))
