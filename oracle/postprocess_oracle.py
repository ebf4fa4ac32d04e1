"""CPU restatement of the refined mesh's post-processing -- TEST INFRASTRUCTURE ONLY (see raster_oracle.c).

Follows sugar_extractors/refined_mesh.py:128-162 (the `--postprocess_mesh` branch) op for op, per face:
    edge entries (0,1), (1,2), (2,0) of each face, vertex ids sorted                     :132-136
    erosion: K = 2 nearest neighbours of the live entries' float32 vertex-id pairs;
             a live face stays iff all three second-nearest squared distances are < 0.01   :139-147
    re-admission: density of the bound model at the eroded faces' centres > threshold     :149-152
    compaction of the faces and the face-major per-Gaussian blocks                         :155-162
with the bound Gaussians of oracle/meshbind_oracle.py and the density of oracle/field_oracle.py over the 16 nearest
Gaussians.  pytorch3d's knn_points is restated as an exact K-NN on squared distances (float64 from the float32
inputs), ties to the lower index.  The reference's initial mask has P = F n entries, so its branch raises at n > 1;
here a face starts live iff all n of its strengths are > -1, which at n = 1 is the reference's mask.

Parity pinning: tests/golden/postprocess_*.npz come from the reference's own lines (make_postprocess_golden.py).
"""
from types import SimpleNamespace

import numpy as np
import torch

from oracle import field_oracle as fo
from oracle import meshbind_oracle as mbo
from sugar_b200.meshbind import bary_coords

KNN_K = 16


def knn_points(p1, p2, K):
    """pytorch3d.ops.knn_points for one cloud pair, exact: -> (squared distances float64 [N,K], idx int64 [N,K]),
    ascending, ties to the lower index; columns past len(p2) are inf / -1."""
    d2 = ((p1.double()[:, None, :] - p2.double()[None, :, :]) ** 2).sum(-1)
    order = torch.argsort(d2, dim=1, stable=True)[:, :K]
    d2 = torch.gather(d2, 1, order)
    pad = K - order.shape[1]
    return (torch.nn.functional.pad(d2, (0, pad), value=float("inf")),
            torch.nn.functional.pad(order, (0, pad), value=-1))


def edge_entries(faces):
    """faces int64 [F,3] -> [F,3,2]: edges (0,1), (1,2), (2,0), each pair sorted (refined_mesh.py:133-136)."""
    e = torch.stack([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]], 1)
    return e.sort(dim=-1)[0]


def erode(faces, iterations, face_mask=None):
    """The erosion rounds (:139-147) from `face_mask` (bool [F], default all) -> bool [F]."""
    faces = torch.as_tensor(faces).long()
    F = faces.shape[0]
    mask = torch.ones(F, dtype=torch.bool) if face_mask is None else torch.as_tensor(face_mask).clone()
    entries = edge_entries(faces)
    for _ in range(iterations):
        if not mask.any():
            break
        live = entries[mask].view(-1, 2).float()
        d2, _ = knn_points(live, live, 2)
        mask[mask.clone()] = (d2[:, 1] < 0.01).view(-1, 3).all(-1)
    return mask


def erode_by_counting(faces, iterations, face_mask=None):
    """The per-face rule stated directly: a live face stays iff each of its edges occurs at least twice among the live
    faces' (face, edge) entries."""
    faces = np.asarray(faces, np.int64)
    mask = np.ones(len(faces), bool) if face_mask is None else np.array(face_mask, bool)
    edges = [[tuple(sorted((int(f[a]), int(f[b])))) for a, b in ((0, 1), (1, 2), (2, 0))] for f in faces]
    for _ in range(iterations):
        count = {}
        for f in np.nonzero(mask)[0]:
            for e in edges[f]:
                count[e] = count.get(e, 0) + 1
        mask = mask & np.array([all(count.get(e, 0) >= 2 for e in es) for es in edges], bool)
    return mask


def density(centres, points, scaling, quaternions, strengths):
    """Density of the Gaussians at `centres` over their 16 nearest, density factor 1 (sugar_model.py:1335-1368).
    -> (density float32 [R], the 16th and 17th squared neighbour distances float64 [R,2] (inf past P))."""
    d2, idx = knn_points(centres, points, KNN_K + 1)
    rho = fo.field_values_torch(centres, idx[:, :KNN_K], points, scaling, quaternions, strengths.view(-1, 1),
                                density_factor=1.0)["density"]
    return rho, d2[:, KNN_K - 1:KNN_K + 1]


def postprocess_mesh(verts, faces, n, scales_raw, complex_raw, densities_raw, sh_dc, sh_rest, thickness,
                     density_threshold=0.1, iterations=5):
    """Steps 1-5 per face, on float32 CPU tensors as sugar_b200.postprocess.postprocess_mesh takes them.
    -> namespace(faces, scales, quaternions, densities, sh_dc, sh_rest, face_mask, eroded, eroded_density,
    knn_d2 (the eroded faces' 16th and 17th squared neighbour distances))."""
    faces = faces.long()
    F = faces.shape[0]
    strengths = torch.sigmoid(densities_raw.view(-1, 1))
    mask = erode(faces, iterations, (strengths.view(F, n) > -1.0).all(1))
    eroded = torch.nonzero(~mask)[:, 0]
    points, scaling, quats = mbo.bind_to_mesh_torch(verts, faces, bary_coords(n), scales_raw, complex_raw, thickness)
    centres = verts[faces].mean(-2)[eroded]
    rho, knn_d2 = density(centres, points.float(), scaling.float(), quats.float(), strengths)
    mask[eroded] = rho > density_threshold
    rows = lambda t: t.reshape(F, n, *t.shape[1:])[mask].reshape(-1, *t.shape[1:])
    return SimpleNamespace(faces=faces[mask], scales=rows(scales_raw), quaternions=rows(complex_raw),
                           densities=rows(densities_raw), sh_dc=rows(sh_dc), sh_rest=rows(sh_rest), face_mask=mask,
                           eroded=eroded, eroded_density=rho, knn_d2=knn_d2)


def ambiguous(out, density_threshold, rel_density=1e-4, rel_knn=1e-6):
    """The eroded faces whose outcome a float32 evaluation in another order could flip: density within `rel_density`
    of float32(threshold), or 16th and 17th neighbour distances within `rel_knn` of each other.  -> bool [R]."""
    thr = float(np.float32(density_threshold))
    near_thr = (out.eroded_density.double() - thr).abs() <= rel_density * thr
    d16, d17 = out.knn_d2[:, 0], out.knn_d2[:, 1]
    return near_thr | ((d17 - d16) <= rel_knn * d17)
