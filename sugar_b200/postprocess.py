"""Post-processing of the refined mesh: the reference's `--postprocess_mesh` (sugar_extractors/refined_mesh.py:125-187).

The option erodes the refined mesh's open borders and keeps the eroded faces that still sit in dense Gaussians, which
the reference recommends when an object is seen from one side only.  With the bound model's raw state:

    out = postprocess_mesh(verts, faces, n, scales_raw, complex_raw, densities_raw, sh_dc, sh_rest, thickness)
    # out.faces, out.scales, out.quaternions, out.densities, out.sh_dc, out.sh_rest: the model on the kept faces

1. erosion (:132-147): `iterations` rounds; a live face stays iff each of its three edges occurs at least twice among
   the live faces' (face, edge) entries.  One csrc/sgr_postprocess.cu launch per round over an edge-run table built
   once on the device with torch's sort (`erode_border_faces`);
2. re-admission (:150-152): an eroded face comes back when the density of the full bound model at its centre
   (verts[faces].mean(-2); K = 16 nearest Gaussians, density factor 1) is > density_threshold, compared in float32;
3. compaction (:155-162): the kept faces and the face-major blocks of the per-Gaussian tensors.  All vertices stay.

Edges are exact integer keys lo * V + hi; the reference searches float32 vertex ids, which merge distinct ids only
above 2^24 vertices, so below that the two agree.  Everything runs on the GPU only, under no_grad.
"""
from types import SimpleNamespace

import torch

from . import field, knn, meshbind
from ._lib import check, check_ids, lib, require_cuda, same_device, stream, tensor

INT32_MAX = 2 ** 31 - 1
KNN_K = 16              # SuGaR.get_gaussians_closest_to_samples without knn_to_track (sugar_model.py:1337-1340)


def _faces(faces, n_verts):
    faces = tensor(faces, "faces", torch.int64, ("F", 3))
    V, F = int(n_verts), faces.shape[0]
    if V <= 0 or V > INT32_MAX or 3 * F > INT32_MAX:
        raise ValueError(f"{V} vertices / {F} faces: need 0 < V <= 2^31 - 1 and 3F <= 2^31 - 1")
    return faces, V


def _iterations(iterations):
    if isinstance(iterations, bool) or int(iterations) != iterations or not 0 <= iterations <= INT32_MAX:
        raise ValueError(f"iterations must be an integer in [0, 2^31 - 1], got {iterations!r}")
    return int(iterations)


def _edge_runs(faces, V):
    """-> (entry_run int32 [3F], run_ptr int32 [3F+1], run_faces int32 [3F]): entry 3 f + m is edge m of face f,
    (0,1), (1,2), (2,0); equal unordered edges form one run, in key order.  run_ptr has an entry for every possible
    run; those past the last run are 3F.  No host synchronisation."""
    n, dev = 3 * faces.shape[0], faces.device
    ea, eb = faces[:, [0, 1, 2]].reshape(-1), faces[:, [1, 2, 0]].reshape(-1)
    key, order = torch.sort(torch.minimum(ea, eb) * V + torch.maximum(ea, eb), stable=True)
    starts = torch.ones(n, dtype=torch.bool, device=dev)
    starts[1:] = key[1:] != key[:-1]
    run = torch.cumsum(starts, 0) - 1
    entry_run = torch.empty(n, dtype=torch.int32, device=dev)
    entry_run[order] = run.int()
    run_ptr = torch.searchsorted(run, torch.arange(n + 1, device=dev)).int()
    return entry_run, run_ptr, (order // 3).int()


def _erode(faces, V, iterations, live):
    """The erosion on checked arguments: faces int64 [F,3] with ids in [0, V), live bool [F] -> bool [F]."""
    F, dev = faces.shape[0], faces.device
    if F == 0 or iterations == 0:
        return live.clone()
    with torch.cuda.device(dev):
        entry_run, run_ptr, run_faces = _edge_runs(faces, V)
        mask = live.to(torch.uint8)
        tmp = torch.empty_like(mask)
        check(lib.sgr_border_peel(F, iterations, entry_run.data_ptr(), run_ptr.data_ptr(), run_faces.data_ptr(),
                                  mask.data_ptr(), tmp.data_ptr(), stream(dev)))
    return mask.bool()


def erode_border_faces(faces, n_verts, iterations=5, face_mask=None):
    """The reference's border erosion (refined_mesh.py:132-147).  faces int64 [F,3] (CUDA) over `n_verts` vertices,
    face_mask bool [F] of the faces live at the start (default: all).  In each of `iterations` rounds a live face stays
    iff each of its three edges occurs at least twice among the live faces' edges; faces removed once stay removed.
    -> bool [F], the faces alive after the rounds.  One host read (the face-id range check, ValueError)."""
    faces, V = _faces(faces, n_verts)
    iterations = _iterations(iterations)
    F, dev = faces.shape[0], faces.device
    if face_mask is None:
        face_mask = torch.ones(F, dtype=torch.bool, device=dev)
    face_mask = tensor(face_mask, "face_mask", torch.bool, (F,), dev, "faces")
    require_cuda("postprocess", faces, face_mask)
    check_ids((faces, 0, V, "face vertex ids"))
    with torch.no_grad():
        return _erode(faces, V, iterations, face_mask)


def postprocess_mesh(verts, faces, n, scales_raw, complex_raw, densities_raw, sh_dc, sh_rest, thickness,
                     density_threshold=0.1, iterations=5):
    """The reference's mesh post-processing (refined_mesh.py:125-187) from a refined model's raw state: verts float32
    [V,3] (_points), faces int64 [F,3], n Gaussians per face (1, 3, 4 or 6), and face-major per-Gaussian tensors of
    P = F n rows: scales_raw [P,2] (_scales), complex_raw [P,2] (_quaternions), densities_raw [P,1] (all_densities),
    sh_dc [P,1,3] (_sh_coordinates_dc), sh_rest [P,M,3] (_sh_coordinates_rest); thickness (surface_mesh_thickness).

    A face starts live iff all of its n strengths sigmoid(densities_raw) are > -1 (not NaN); `erode_border_faces` runs
    `iterations` rounds; the density of the full bound model (meshbind.bind_to_mesh) at each eroded face's centre,
    over its 16 nearest Gaussians at density factor 1 (knn.knn_points, field.compute_density), re-admits the face when
    > density_threshold (in float32).  At n = 1 this is the reference exactly.  At n > 1 the reference raises an
    IndexError (its mask has P entries, its edge list F); here the rule is applied per face, as its reshapes intend.

    -> SimpleNamespace(faces, scales, quaternions, densities, sh_dc, sh_rest: the kept faces and their Gaussians' rows;
    face_mask bool [F]: the kept faces; eroded int64 [R]: the faces the erosion removed, ascending; eroded_density
    float32 [R]: the density at their centres).  verts is unchanged and every vertex stays.  Raises ValueError when
    P < 16 (the exact 16-NN needs 16 Gaussians).  Host reads: the face-id range check, the eroded-face count and, when
    a face was eroded, the kept-face count; nothing is launched for re-admission when no face was eroded."""
    dev = verts.device
    verts = tensor(verts, "verts", torch.float32, ("V", 3))
    faces, V = _faces(faces, verts.shape[0])
    iterations = _iterations(iterations)
    if n not in (1, 3, 4, 6):
        raise ValueError(f"n must be 1, 3, 4 or 6 Gaussians per face, got {n!r}")
    F = faces.shape[0]
    P = F * n
    scales_raw = tensor(scales_raw, "scales_raw", torch.float32, (P, 2), dev)
    complex_raw = tensor(complex_raw, "complex_raw", torch.float32, (P, 2), dev)
    densities_raw = tensor(densities_raw, "densities_raw", torch.float32, (P, 1), dev)
    sh_dc = tensor(sh_dc, "sh_dc", torch.float32, (P, 1, 3), dev)
    sh_rest = tensor(sh_rest, "sh_rest", torch.float32, (P, "M", 3), dev)
    same_device(dev, faces=faces)
    if 0 < P < KNN_K:
        raise ValueError(f"{P} Gaussians: the density re-admission needs at least {KNN_K}")
    require_cuda("postprocess", verts, faces)
    M = sh_rest.shape[1]
    if F == 0:
        return SimpleNamespace(faces=faces.clone(), scales=scales_raw.clone(), quaternions=complex_raw.clone(),
                               densities=densities_raw.clone(), sh_dc=sh_dc.clone(), sh_rest=sh_rest.clone(),
                               face_mask=torch.zeros(0, dtype=torch.bool, device=dev),
                               eroded=torch.zeros(0, dtype=torch.int64, device=dev),
                               eroded_density=torch.zeros(0, dtype=torch.float32, device=dev))
    check_ids((faces, 0, V, "face vertex ids"))
    with torch.no_grad(), torch.cuda.device(dev):
        strengths = torch.sigmoid(densities_raw)
        live = (strengths.view(F, n) > -1.0).all(1)
        mask = _erode(faces, V, iterations, live)
        eroded = torch.nonzero(~mask)[:, 0]                                  # host read: the eroded-face count
        density = torch.zeros(0, dtype=torch.float32, device=dev)
        if eroded.numel():
            b = meshbind.bind_to_mesh(verts, faces, meshbind.bary_coords(n, dev), scales_raw, complex_raw, thickness)
            centres = verts[faces[eroded]].mean(-2)
            _, idx = knn.knn_points(centres, b.points, KNN_K)
            density = field.compute_density(centres, idx, b.points, b.scaling, b.quaternions, strengths,
                                            density_factor=1.0)
            mask[eroded] = density > float(density_threshold)
            keep = torch.nonzero(mask)[:, 0]                                 # host read: the kept-face count
            rows = lambda t, *shape: t.view(F, n, *shape)[keep].reshape(keep.numel() * n, *shape)
            faces, scales_raw, complex_raw = faces[keep], rows(scales_raw, 2), rows(complex_raw, 2)
            densities_raw, sh_dc, sh_rest = rows(densities_raw, 1), rows(sh_dc, 1, 3), rows(sh_rest, M, 3)
        else:
            faces, scales_raw, complex_raw, densities_raw, sh_dc, sh_rest = (
                t.clone() for t in (faces, scales_raw, complex_raw, densities_raw, sh_dc, sh_rest))
    return SimpleNamespace(faces=faces, scales=scales_raw, quaternions=complex_raw, densities=densities_raw,
                           sh_dc=sh_dc, sh_rest=sh_rest, face_mask=mask, eroded=eroded, eroded_density=density)
