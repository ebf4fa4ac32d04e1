"""CPU restatement of an EDITABLE mesh-bound SuGaR model and of the compositor's rotated SH colours -- TEST
INFRASTRUCTURE ONLY.

Follows, op for op in PyTorch (any float dtype; float64 for per-Gaussian references):
    SuGaR.get_edited_quaternions_and_scales   sugar_scene/sugar_model.py:572-667   (use_old_method = False, :22)
    SuGaR.scaling / .quaternions (editable)   sugar_scene/sugar_model.py:415-479
    SuGaRCompositor's sh_rotations colour     sugar_scene/sugar_compositor.py:146-150: get_points_rgb(directions=
                                              normalize(p - campos) @ R) with eval_sh (sugar_utils/spherical_harmonics.py)
pytorch3d's face normal and matrix_to_quaternion are oracle/meshbind_oracle.py's restatements.  Parity pinning:
tests/golden/editmesh_*.npz come from the reference's own property code (tests/golden/make_editmesh_golden.py).
"""
import math

import numpy as np
import torch

from oracle import meshbind_oracle as mo

_normalize = torch.nn.functional.normalize


def edited_bind_torch(verts, reference_verts, faces, bary, scales_raw, complex_raw, thickness):
    """bary [n,3]; returns (points [F*n,3], scaling [F*n,3], quaternions [F*n,4]) of the model made editable at
    `reference_verts` and deformed to `verts`."""
    F, n = faces.shape[0], bary.shape[0]
    bary_coords = bary.reshape(n, 3, 1)
    reference = reference_verts[faces]
    faces_verts = verts[faces]
    faces_normals = mo.faces_normals(verts, faces)
    points = (faces_verts[:, None] * bary_coords[None]).sum(dim=-2)
    R_0 = _normalize(faces_normals, dim=-1)
    base_R_1 = _normalize(faces_verts[:, 0] - faces_verts[:, 1], dim=-1)
    base_R_2 = _normalize(torch.cross(R_0, base_R_1, dim=-1))
    # rotation adjustment (:597-621)
    reference_base = _normalize(reference[:, 0:1] - reference[:, 1:2], dim=-1)
    reference_axis = _normalize(reference - reference.mean(dim=-2, keepdim=True), dim=-1)
    reference_axis[:, 2] = -reference_axis[:, 2]
    faces_base = _normalize(faces_verts[:, 0:1] - faces_verts[:, 1:2], dim=-1)
    faces_axis = _normalize(faces_verts - faces_verts.mean(dim=-2, keepdim=True), dim=-1)
    faces_axis[:, 2] = -faces_axis[:, 2]
    reference_angles = torch.arccos((reference_axis * reference_base).sum(dim=-1, keepdim=True).clamp(min=-1., max=1.))
    faces_angles = torch.arccos((faces_axis * faces_base).sum(dim=-1, keepdim=True).clamp(min=-1., max=1.))
    angles = faces_angles - reference_angles
    point_angles = (angles[:, None] * bary_coords[None]).sum(dim=-2)
    adjust = torch.cat([torch.cos(point_angles), torch.sin(point_angles)], dim=-1)
    cplx = _normalize(complex_raw, dim=-1).view(F, n, 2)
    x, y = cplx[..., 0].clone(), cplx[..., 1].clone()
    a, b = adjust[..., 0], adjust[..., 1]
    cplx[..., 0] = x * a - y * b
    cplx[..., 1] = x * b + y * a
    R_1 = cplx[..., 0:1] * base_R_1[:, None] + cplx[..., 1:2] * base_R_2[:, None]
    R_2 = -cplx[..., 1:2] * base_R_1[:, None] + cplx[..., 0:1] * base_R_2[:, None]
    R = torch.cat([R_0[:, None, ..., None].expand(-1, n, -1, -1).clone(), R_1[..., None], R_2[..., None]], dim=-1)
    quaternions = mo.matrix_to_quaternion(R)
    # scale adjustment (:635-660)
    faces_axis_s = faces_verts.mean(dim=-2, keepdim=True) - faces_verts
    faces_axis_norm = torch.norm(faces_axis_s, dim=-1, keepdim=True)
    faces_axis_s = _normalize(faces_axis_s, dim=-1)
    faces_orthos = torch.cross(faces_axis_s, faces_normals[:, None], dim=-1)
    reference_axis_s = reference.mean(dim=-2, keepdim=True) - reference
    reference_axis_norm = torch.norm(reference_axis_s, dim=-1, keepdim=True)
    axis_proj_1 = (R_1[..., None, :] * faces_axis_s[:, None]).sum(dim=-1, keepdim=True)
    ortho_proj_1 = (R_1[..., None, :] * faces_orthos[:, None]).sum(dim=-1, keepdim=True)
    side_proj_2 = (R_2[..., None, :] * faces_axis_s[:, None]).sum(dim=-1, keepdim=True)
    ortho_proj_2 = (R_2[..., None, :] * faces_orthos[:, None]).sum(dim=-1, keepdim=True)
    scaling_1 = torch.sqrt((axis_proj_1 * faces_axis_norm[:, None] / reference_axis_norm[:, None]) ** 2 + ortho_proj_1 ** 2)
    scaling_2 = torch.sqrt((side_proj_2 * faces_axis_norm[:, None] / reference_axis_norm[:, None]) ** 2 + ortho_proj_2 ** 2)
    scaling_1 = (scaling_1 * bary_coords[None]).sum(dim=-2)
    scaling_2 = (scaling_2 * bary_coords[None]).sum(dim=-2)
    plane = torch.exp(scales_raw).view(-1, n, 2)
    plane[..., 0:1] = plane[..., 0:1] * scaling_1
    plane[..., 1:2] = plane[..., 1:2] * scaling_2
    scales = torch.cat([thickness * torch.ones(len(scales_raw), 1, dtype=plane.dtype, device=plane.device), plane.view(-1, 2)], dim=-1)
    return points.reshape(F * n, 3), scales, _normalize(quaternions, dim=-1).reshape(F * n, 4)


_C0 = 0.28209479177387814
_C1 = 0.4886025119029199
_C2 = (1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396)
_C3 = (-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658,
       1.445305721320277, -0.5900435899266435)


def eval_sh(deg, sh, dirs):
    """eval_sh (sugar_utils/spherical_harmonics.py) for degree <= 3: sh [..., C, (deg+1)^2], dirs [..., 3]."""
    result = _C0 * sh[..., 0]
    if deg > 0:
        x, y, z = dirs[..., 0:1], dirs[..., 1:2], dirs[..., 2:3]
        result = result - _C1 * y * sh[..., 1] + _C1 * z * sh[..., 2] - _C1 * x * sh[..., 3]
        if deg > 1:
            xx, yy, zz = x * x, y * y, z * z
            xy, yz, xz = x * y, y * z, x * z
            result = (result + _C2[0] * xy * sh[..., 4] + _C2[1] * yz * sh[..., 5] +
                      _C2[2] * (2.0 * zz - xx - yy) * sh[..., 6] + _C2[3] * xz * sh[..., 7] +
                      _C2[4] * (xx - yy) * sh[..., 8])
            if deg > 2:
                result = (result + _C3[0] * y * (3 * xx - yy) * sh[..., 9] + _C3[1] * xy * z * sh[..., 10] +
                          _C3[2] * y * (4 * zz - xx - yy) * sh[..., 11] +
                          _C3[3] * z * (2 * zz - 3 * xx - 3 * yy) * sh[..., 12] +
                          _C3[4] * x * (4 * zz - xx - yy) * sh[..., 13] + _C3[5] * z * (xx - yy) * sh[..., 14] +
                          _C3[6] * x * (xx - 3 * yy) * sh[..., 15])
    return result


def rotated_colors(points, sh, campos, R, sh_degree):
    """The compositor's colour of one model with sh_rotation R: get_points_rgb(directions=normalize(p - campos) @ R).
    points [P,3], sh [P,M,3], campos [3], R [3,3] -> [P,3]."""
    d = (_normalize(points - campos.reshape(1, 3), dim=-1).unsqueeze(1) @ R)[..., 0, :]
    L = (sh_degree + 1) ** 2
    shs_view = sh[:, :L].transpose(-1, -2).reshape(-1, 3, L)
    return torch.clamp_min(eval_sh(sh_degree, shs_view, d) + 0.5, 0.0).view(-1, 3)


def rotation(axis, angle, dtype=torch.float32):
    """3x3 rotation about `axis` by `angle` (Rodrigues), computed in float64."""
    k = np.asarray(axis, np.float64)
    k = k / np.linalg.norm(k)
    K = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return torch.tensor(np.eye(3) + math.sin(angle) * K + (1 - math.cos(angle)) * (K @ K), dtype=dtype)


def well_shaped_soup(F, seed):
    """F separate triangles (V = 3F) with random centres, orientations and sizes, each vertex at 120 +- 25 degrees from
    the last and 0.6-1.4 of the face's radius from its centre: every vertex-axis / base dot stays inside
    |dot| <= 0.999, where arccos is well conditioned, also after a 10 % jitter."""
    rng = np.random.Generator(np.random.PCG64(seed))
    centres = rng.uniform(-3, 3, (F, 1, 3))
    size = rng.uniform(0.05, 0.3, (F, 1, 1))
    phi = np.cumsum(np.concatenate([rng.uniform(0, 2 * math.pi, (F, 1)),
                                    math.radians(120) + rng.uniform(-1, 1, (F, 2)) * math.radians(25)], 1), 1)
    rad = rng.uniform(0.6, 1.4, (F, 3))
    local = np.stack([rad * np.cos(phi), rad * np.sin(phi), np.zeros((F, 3))], -1)
    q, _ = np.linalg.qr(rng.normal(size=(F, 3, 3)))
    verts = (centres + size * np.einsum("fij,fkj->fki", q, local)).reshape(-1, 3)
    return verts, np.arange(3 * F, dtype=np.int64).reshape(F, 3)


def deform(kind, reference, faces, seed):
    """Current vertices for an edit of `kind` applied to `reference` (float64 numpy [V,3])."""
    rng = np.random.Generator(np.random.PCG64(1000 + seed))
    if kind == "identity":
        return reference.copy()
    if kind == "rigid":
        return reference @ rotation([0.3, -0.5, 0.8], 1.1, torch.float64).numpy().T + np.array([0.4, -1.2, 0.7])
    if kind == "jitter":        # about 10 % of each vertex's mean incident edge length
        e = np.linalg.norm(reference[faces] - reference[faces[:, [1, 2, 0]]], axis=-1)
        per_vertex = np.zeros(len(reference))
        np.add.at(per_vertex, faces.ravel(), np.repeat(e.mean(1), 3))
        per_vertex /= np.maximum(np.bincount(faces.ravel(), minlength=len(reference)), 1)
        return reference + 0.1 * per_vertex[:, None] * rng.normal(size=reference.shape) / math.sqrt(3)
    if kind == "stretch":       # 2x along x
        return reference * np.array([2.0, 1.0, 1.0])
    if kind == "bent":          # the unit square rolled up onto a cylinder of radius 0.6 about the axis x = 0, z = 0.6
        th = (reference[:, 0] - 0.5) / 0.6
        r = 0.6 - reference[:, 2]
        return np.stack([r * np.sin(th), reference[:, 1], 0.6 - r * np.cos(th)], 1)
    raise ValueError(kind)


def make_case(kind, F=200, n_per=6, seed=0, mesh="soup", dtype=torch.float32):
    """A seeded editable bound model: reference vertices, current vertices after the edit `kind`, raw scales and
    in-plane rotations.  mesh: "soup" (well_shaped_soup) or "height" (scenes.height_field_mesh, ~F faces)."""
    if mesh == "soup":
        ref, faces = well_shaped_soup(F, seed)
    else:
        from sugar_b200.scenes import height_field_mesh
        nx = max(2, int(round(math.sqrt(F / 2))) + 1)
        ref, faces = height_field_mesh(nx, nx, seed=seed)
        ref = ref.astype(np.float64)
    cur = deform(kind, ref, faces, seed)
    g = torch.Generator().manual_seed(seed)
    P = faces.shape[0] * n_per
    scales_raw = torch.randn(P, 2, generator=g, dtype=dtype) * 0.4 - 2.0
    complex_raw = torch.randn(P, 2, generator=g, dtype=dtype) * 1.5
    return dict(verts=torch.tensor(cur, dtype=dtype), reference_verts=torch.tensor(ref, dtype=dtype),
                faces=torch.from_numpy(np.ascontiguousarray(faces)), bary=mo.make_case(F=1, V=3, n_per=n_per)["bary"].to(dtype),
                scales_raw=scales_raw, complex_raw=complex_raw, thickness=1e-5)


def max_axis_dot(verts, faces):
    """max |<angle axis k, base>| over faces and k: how close any arccos argument is to +-1."""
    v = torch.as_tensor(verts, dtype=torch.float64)[torch.as_tensor(faces)]
    base = _normalize(v[:, 0:1] - v[:, 1:2], dim=-1)
    axis = _normalize(v - v.mean(dim=-2, keepdim=True), dim=-1)
    return float((axis * base).sum(-1).abs().max())


def edited_values(case, dtype=None):
    """edited_bind_torch on a make_case dict, optionally cast to `dtype` -> numpy dict."""
    c = {k: (v.to(dtype) if dtype is not None and torch.is_tensor(v) and v.is_floating_point() else v)
         for k, v in case.items()}
    p, s, q = edited_bind_torch(c["verts"], c["reference_verts"], c["faces"], c["bary"], c["scales_raw"],
                                c["complex_raw"], c["thickness"])
    return dict(points=p.numpy(), scaling=s.numpy(), quaternions=q.numpy())
