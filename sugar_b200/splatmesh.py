"""The splatted "diamond" mesh of the Gaussians and a nearest-face triangle z-buffer (csrc/sgr_splatmesh.cu).

The reference's default depth source for mesh extraction (compute_level_surface_points_from_camera_fast with
use_gaussian_depth=False, sugar_scene/sugar_model.py:1880-1968) turns every Gaussian into a view-facing diamond of two
triangles and z-buffers them with pytorch3d's MeshRasterizer:

    verts, faces = splat_mesh(points, scaling, quaternions, cam)     # SuGaR.splat_mesh(p3d_camera): verts/faces_packed
    zbuf, pix_to_face = rasterize_mesh(verts, faces, cam)            # fragments.zbuf / pix_to_face [0, ..., 0]
    gaussian_idx = pix_to_face // 2                                  # where pix_to_face >= 0

`cam` is the namespace `steps.camera_from_scene` builds (viewmatrix / projmatrix device tensors in the rasterizer's
transposed convention, width, height).  Pixels follow this package's rasterizer convention, not pytorch3d's NDC, so the
back-projection of `levelset` matches the depth.  Neither op is differentiable (the extraction runs under no_grad);
both run on the GPU only.
"""
import torch

from ._lib import check, lib

INT32_MAX = 2 ** 31 - 1
TRIANGLES = ((0, 2, 1), (0, 3, 2))   # the two faces of a diamond (sugar_model.py:254-256)


def _stream(dev):
    return torch.cuda.current_stream(dev).cuda_stream


def _require_cuda(*ts):
    for t in ts:
        if not t.is_cuda:
            raise RuntimeError("sugar_b200.splatmesh needs CUDA tensors: there is no CPU fallback")


def _cam_matrix(m, dev, name):
    if not torch.is_tensor(m) or m.shape != (4, 4) or m.dtype != torch.float32:
        raise ValueError(f"cam.{name} must be a float32 [4,4] tensor")
    if m.device != dev:
        raise ValueError(f"cam.{name} on {m.device}, the mesh on {dev}")
    return m.contiguous()


def _vec3(t, name, n=None):
    if t.dtype != torch.float32 or t.dim() != 2 or t.shape[1] != 3 or (n is not None and t.shape[0] != n):
        want = f"[{n},3]" if n is not None else "[N,3]"
        raise ValueError(f"{name} must be float32 {want}, got {t.dtype} {tuple(t.shape)}")
    return t.contiguous()


def splat_mesh(points, scaling, quaternions, cam, triangle_scale=2.0):
    """SuGaR.splat_mesh(camera) for primitive 'diamond', mode 'perspective' (sugar_model.py:481-514, 695-728).

    points, scaling (activated) float32 [P,3], quaternions float32 [P,4] (normalised, w first) on one CUDA device.
    -> verts float32 [4P,3] (every vertex moved along its view ray onto the plane through the Gaussian's centre
    perpendicular to the centre's ray), faces int64 [2P,3] = 4g + (0, 2, 1), 4g + (0, 3, 2)."""
    P, dev = points.shape[0], points.device
    points = _vec3(points, "points")
    scaling = _vec3(scaling, "scaling", P)
    if quaternions.dtype != torch.float32 or quaternions.shape != (P, 4):
        raise ValueError(f"quaternions must be float32 [{P},4], got {quaternions.dtype} {tuple(quaternions.shape)}")
    if scaling.device != dev or quaternions.device != dev:
        raise ValueError("points, scaling and quaternions must be on one device")
    if 4 * P > INT32_MAX:
        raise ValueError(f"{P} Gaussians: at most (2^31 - 1) / 4")
    view = _cam_matrix(cam.viewmatrix, dev, "viewmatrix")
    _require_cuda(points, scaling, quaternions)
    quaternions = quaternions.contiguous()
    if quaternions.data_ptr() % 16:                  # the kernel loads one float4 per Gaussian
        quaternions = quaternions.clone()
    with torch.no_grad(), torch.cuda.device(dev):
        verts = torch.empty((4 * P, 3), dtype=torch.float32, device=dev)
        faces = (4 * torch.arange(P, device=dev)[:, None, None] +
                 torch.tensor(TRIANGLES, device=dev)[None]).reshape(-1, 3)
        if P:
            view_inv = torch.linalg.inv(view.double()).float().contiguous()
            check(lib.sgr_splat_mesh(P, points.data_ptr(), scaling.data_ptr(), quaternions.data_ptr(), view.data_ptr(),
                                     view_inv.data_ptr(), float(triangle_scale), verts.data_ptr(), _stream(dev)))
    return verts, faces


def rasterize_mesh(verts, faces, cam):
    """Nearest-face z-buffer of the mesh: pytorch3d's MeshRasterizer (blur_radius 0, perspective-correct, no culling)
    read at faces_per_pixel index 0, without the coarse pass's per-bin face limit (the result is complete).

    verts float32 [V,3], faces int64 [F,3] with ids in [0, V) (checked with one host read), on one CUDA device.
    -> zbuf float32 [H,W] (view-space depth of the nearest covering face, -1 where none), pix_to_face int64 [H,W]
    (its index, -1 where none; equal depths resolve to the lower index), identical from run to run."""
    dev = verts.device
    verts = _vec3(verts, "verts")
    if faces.dtype != torch.int64 or faces.dim() != 2 or faces.shape[1] != 3:
        raise ValueError(f"faces must be int64 [F,3], got {faces.dtype} {tuple(faces.shape)}")
    if faces.device != dev:
        raise ValueError(f"faces on {faces.device}, verts on {dev}")
    V, F = verts.shape[0], faces.shape[0]
    if V > INT32_MAX or F > INT32_MAX:
        raise ValueError(f"{V} vertices / {F} faces: at most 2^31 - 1 each (the face id is packed in 32 bits)")
    H, W = int(cam.height), int(cam.width)
    if not (0 < W <= 65535 and 0 < H <= 65535 and W * H <= INT32_MAX):
        raise ValueError(f"image {W}x{H}: need 0 < W, H <= 65535 and W*H <= 2^31 - 1")
    view = _cam_matrix(cam.viewmatrix, dev, "viewmatrix")
    proj = _cam_matrix(cam.projmatrix, dev, "projmatrix")
    faces = faces.contiguous()
    n_bad = int(((faces < 0) | (faces >= V)).sum()) if F else 0             # the one host read
    if n_bad:
        raise ValueError(f"{n_bad} face vertex ids outside [0, {V})")
    _require_cuda(verts, faces)
    with torch.no_grad(), torch.cuda.device(dev):
        if F == 0:
            return (torch.full((H, W), -1.0, device=dev), torch.full((H, W), -1, dtype=torch.int64, device=dev))
        zbuf = torch.empty((H, W), dtype=torch.float32, device=dev)
        pix_to_face = torch.empty((H, W), dtype=torch.int64, device=dev)
        scratch = torch.empty(lib.sgr_mesh_raster_scratch_bytes(F, W, H), dtype=torch.uint8, device=dev)
        check(lib.sgr_mesh_raster(V, F, verts.data_ptr(), faces.data_ptr(), view.data_ptr(), proj.data_ptr(), W, H,
                                  zbuf.data_ptr(), pix_to_face.data_ptr(), scratch.data_ptr(), _stream(dev)))
    return zbuf, pix_to_face
