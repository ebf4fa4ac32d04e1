"""Gaussians bound to a triangle mesh: the per-step prologue of SuGaR's refinement stage, fused.

A mesh-bound `SuGaR` model derives every Gaussian from its triangle (sugar_scene/sugar_model.py):

    points       :384-398   barycentric combination of the face's vertices (n Gaussians per face, :172-214)
    scaling      :415-441   (surface_mesh_thickness, exp(_scales[:, 0]), exp(_scales[:, 1]))
    quaternions  :443-479   R = [face normal | first edge rotated in-plane by the learned complex number |
                            their cross product] -> matrix_to_quaternion -> normalize

as ~40 PyTorch kernels with [F, n, 3, 3] temporaries and their autograd.  `bind_to_mesh` computes the three
tensors with one CUDA kernel and one for the backward (sgr_meshbind.cu, one thread per face), gradients to the
vertices, `_scales` and `_quaternions`.

    b = bind_to_mesh(verts, faces, bary, scales_raw, complex_raw, thickness)
    b.points [F*n,3], b.scaling [F*n,3], b.quaternions [F*n,4]

`bind_to_edited_mesh` is the editable model (make_editable / get_edited_quaternions_and_scales, :562-667): the mesh
moved away from the vertices it was made editable at, forward only, one kernel (sgr_meshbind_edited_forward).
"""
import math
from types import SimpleNamespace

import torch

from ._lib import check, lib, require_cuda, stream, tensor


def bary_coords(n_gaussians_per_surface_triangle: int, device=None) -> torch.Tensor:
    """surface_triangle_bary_coords of the reference (sugar_model.py:172-214), as [n,3]."""
    tables = {1: [[1 / 3, 1 / 3, 1 / 3]],
              3: [[1 / 2, 1 / 4, 1 / 4], [1 / 4, 1 / 2, 1 / 4], [1 / 4, 1 / 4, 1 / 2]],
              4: [[1 / 3, 1 / 3, 1 / 3], [2 / 3, 1 / 6, 1 / 6], [1 / 6, 2 / 3, 1 / 6], [1 / 6, 1 / 6, 2 / 3]],
              6: [[2 / 3, 1 / 6, 1 / 6], [1 / 6, 2 / 3, 1 / 6], [1 / 6, 1 / 6, 2 / 3], [1 / 6, 5 / 12, 5 / 12],
                  [5 / 12, 1 / 6, 5 / 12], [5 / 12, 5 / 12, 1 / 6]]}
    return torch.tensor(tables[n_gaussians_per_surface_triangle], dtype=torch.float32, device=device)


class _MeshBind(torch.autograd.Function):
    @staticmethod
    def forward(ctx, verts, faces, bary, scales_raw, complex_raw, thickness):
        dev = verts.device
        verts = tensor(verts.float(), "verts", torch.float32, ("V", 3))
        faces = tensor(faces.long(), "faces", torch.int64, ("F", 3), dev)
        bary = bary.float()
        if bary.dim() == 3 and bary.shape[2] == 1:      # the reference's [n,3,1]
            bary = bary[..., 0]
        bary = tensor(bary, "bary", torch.float32, ("n", 3), dev)
        F, n, V = faces.shape[0], bary.shape[0], verts.shape[0]
        P = F * n
        scales_raw, complex_raw = scales_raw.float(), complex_raw.float()
        if scales_raw.shape != (P, 2) or complex_raw.shape != (P, 2):
            raise RuntimeError(f"_scales / _quaternions of a mesh-bound model must be [{P}, 2]")
        scales_raw = tensor(scales_raw, "scales_raw", torch.float32, (P, 2), dev)
        complex_raw = tensor(complex_raw, "complex_raw", torch.float32, (P, 2), dev)
        require_cuda("meshbind", verts)
        with torch.cuda.device(dev):
            points = torch.empty((P, 3), device=dev)
            scaling = torch.empty((P, 3), device=dev)
            quats = torch.empty((P, 4), device=dev)
            check(lib.sgr_meshbind_forward(F, n, V, verts.data_ptr(), faces.data_ptr(), bary.data_ptr(),
                                           scales_raw.data_ptr(), complex_raw.data_ptr(), float(thickness),
                                           points.data_ptr(), scaling.data_ptr(), quats.data_ptr(), stream(dev)))
        ctx.save_for_backward(verts, faces, bary, scales_raw, complex_raw)
        ctx.mark_non_differentiable(faces)
        return points, scaling, quats

    @staticmethod
    def backward(ctx, g_points, g_scaling, g_quats):
        verts, faces, bary, scales_raw, complex_raw = ctx.saved_tensors
        F, n, V = faces.shape[0], bary.shape[0], verts.shape[0]
        dev = verts.device
        z = lambda g, ref: torch.zeros_like(ref) if g is None else g.contiguous().float()
        with torch.cuda.device(dev):
            g_points = z(g_points, torch.empty((F * n, 3), device=dev))
            g_scaling = z(g_scaling, torch.empty((F * n, 3), device=dev))
            g_quats = z(g_quats, torch.empty((F * n, 4), device=dev))
            g_verts = torch.empty_like(verts)
            g_s = torch.empty_like(scales_raw)
            g_c = torch.empty_like(complex_raw)
            check(lib.sgr_meshbind_backward(F, n, V, verts.data_ptr(), faces.data_ptr(), bary.data_ptr(),
                                            scales_raw.data_ptr(), complex_raw.data_ptr(), g_points.data_ptr(),
                                            g_scaling.data_ptr(), g_quats.data_ptr(), g_verts.data_ptr(), g_s.data_ptr(),
                                            g_c.data_ptr(), stream(dev)))
        return g_verts, None, None, g_s, g_c, None


def bind_to_mesh(verts, faces, bary, scales_raw, complex_raw, thickness):
    """verts [V,3] (SuGaR._points of a bound model), faces [F,3] int64 (_surface_mesh_faces), bary [n,3] or the
    reference's [n,3,1], scales_raw [F*n,2] (_scales), complex_raw [F*n,2] (_quaternions), thickness (float:
    surface_mesh_thickness).  Returns namespace(points, scaling, quaternions).  Shapes, dtypes and devices are checked
    (ValueError); face ids are not range-checked, which would cost a host synchronisation per step."""
    points, scaling, quats = _MeshBind.apply(verts, faces, bary, scales_raw, complex_raw, float(thickness))
    return SimpleNamespace(points=points, scaling=scaling, quaternions=quats)


def edited_args(verts, reference_verts, faces, bary, scales_raw, complex_raw, thickness):
    """The checked arguments of one sgr_meshbind_edited_forward launch -> SimpleNamespace (F, n, V, P, tensors as
    the kernel reads them).  ValueError on a wrong shape, dtype or device, or, under grad mode, on an input that
    requires grad: the edited binding is forward only."""
    verts = tensor(verts, "verts", torch.float32, ("V", 3))
    dev = verts.device
    V = verts.shape[0]
    reference_verts = tensor(reference_verts, "reference_verts", torch.float32, (V, 3), dev)
    faces = tensor(faces, "faces", torch.int64, ("F", 3), dev)
    if torch.is_tensor(bary) and bary.dim() == 3 and bary.shape[2] == 1:      # the reference's [n,3,1]
        bary = bary[..., 0]
    bary = tensor(bary, "bary", torch.float32, ("n", 3), dev)
    F, n = faces.shape[0], bary.shape[0]
    scales_raw = tensor(scales_raw, "scales_raw", torch.float32, (F * n, 2), dev)
    complex_raw = tensor(complex_raw, "complex_raw", torch.float32, (F * n, 2), dev)
    if torch.is_grad_enabled() and any(t.requires_grad for t in (verts, reference_verts, bary, scales_raw, complex_raw)):
        raise ValueError("the edited binding is forward only: detach its inputs or run it under torch.no_grad()")
    return SimpleNamespace(F=F, n=n, V=V, P=F * n, verts=verts, reference_verts=reference_verts, faces=faces, bary=bary,
                           scales_raw=scales_raw, complex_raw=complex_raw, thickness=float(thickness))


def edited_launch(a, points, scaling, quats, out_rows=None):
    """One sgr_meshbind_edited_forward launch of checked arguments `a` (edited_args) into float32 CUDA buffers, at row
    g, or at row out_rows[g] (int64 [P], negative: skipped) when given."""
    require_cuda("meshbind", a.verts)
    with torch.cuda.device(a.verts.device):
        check(lib.sgr_meshbind_edited_forward(
            a.F, a.n, a.V, a.verts.data_ptr(), a.reference_verts.data_ptr(), a.faces.data_ptr(), a.bary.data_ptr(),
            a.scales_raw.data_ptr(), a.complex_raw.data_ptr(), a.thickness,
            None if out_rows is None else out_rows.data_ptr(), points.data_ptr(), scaling.data_ptr(),
            quats.data_ptr(), stream(a.verts.device)))


def bind_to_edited_mesh(verts, reference_verts, faces, bary, scales_raw, complex_raw, thickness):
    """The Gaussians of an EDITABLE bound model: SuGaR.points / .scaling / .quaternions after make_editable() was
    called with the mesh at `reference_verts` [V,3] and the mesh then moved to `verts` [V,3] (sugar_model.py:562-667).
    Each Gaussian's in-plane rotation turns with the change in angle of its face's vertex axes, and its two plane
    scales stretch with their change in length.  Other arguments as bind_to_mesh.  Forward only (ValueError when an
    input requires grad under grad mode).  Returns namespace(points, scaling, quaternions), each [F*n, .]."""
    a = edited_args(verts, reference_verts, faces, bary, scales_raw, complex_raw, thickness)
    require_cuda("meshbind", a.verts)
    dev = a.verts.device
    points = torch.empty((a.P, 3), device=dev)
    scaling = torch.empty((a.P, 3), device=dev)
    quats = torch.empty((a.P, 4), device=dev)
    edited_launch(a, points, scaling, quats)
    return SimpleNamespace(points=points, scaling=scaling, quaternions=quats)
