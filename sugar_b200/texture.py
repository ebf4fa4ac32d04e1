"""UV texture of the refined mesh from its bound Gaussians (csrc/sgr_texture.cu).

The reference's last stage (extract_refined_mesh_with_texture.py) calls extract_texture_image_and_uv_from_gaussians
(sugar_scene/sugar_model.py:2464-2677) with n_sh=1 and texture_with_gaussian_renders=True.  Here, without pytorch3d:

    verts_uv, faces_uv, T = uv_layout(F, square_size)              # :2486-2535, plain torch
    init = initial_texture(verts, faces, points, scaling, quaternions, sh_dc, square_size)   # :2537-2605, one kernel
    state = new_bake_state(init)
    for cam in cams:                                               # :2648-2672
        image = <render of the bound Gaussians, sh degree 0, black background>   # [3,H,W]
        zbuf, pix_to_face = splatmesh.rasterize_mesh(verts, faces, cam)
        bake_view(state, verts, faces, verts_uv, faces_uv, cam, image, zbuf, pix_to_face)  # two kernels over H*W
    texture = finish(state)                                        # :2674-2675

or all of it as `extract_texture_image_and_uv_from_gaussians`.  Square k = (k // n_sq, k % n_sq) of the T x T map
(T = square_size * n_sq, n_sq = int(sqrt(F // 2 + 1) + 1)) holds face 2k (its bottom triangle) and 2k + 1 (its top).

What each view does, per pixel with pix_to_face >= 0 and zbuf > 0: the face's perspective-correct barycentrics at the
pixel (in this package's pixel convention, as the z-buffer samples it), the UV interpolated in float32, and the texel
TexturesUV(sampling_mode='nearest') returns from the reference's index map (grid_sample, align_corners, border padding,
the map flipped in y, round half to even): col = round(u (T-1)), row = (T-1) - round(v (T-1)).  The texel adds the
pixel's clamp(0, 1) colour and 1 to its counter; finish() divides, and texels no view reached keep their initial value.

Two places where this differs from the reference on purpose:
  * several pixels of one view on one texel: the reference's index_put does not accumulate, so one of them contributes
    and which one is unspecified.  Here the pixel of highest row-major index does, the same one on every run (the
    reference can also produce that outcome).  The counter still grows by one per view.
  * the shader's far plane: the reference's SoftPhongShader blends with pytorch3d's default zfar = 100, so pixels whose
    face lies beyond 100 scene units blend to the black background and their colour lands on texel (0, 0) (pixels
    within about 0.1 of that plane get a rounded mix).  Here every pixel with zbuf > 0 goes to its own texel.
The initial texels follow the reference's float32 arithmetic as its CPU evaluation orders it; where two Gaussians'
densities at a texel are within rounding of each other (argmax near-ties) the chosen Gaussian can differ.

Not built: n_sh > 1 (inconsistent with texture_with_gaussian_renders in the reference), postprocess_mesh's border-face
removal (off by default) and the .obj / .mtl / .png writers.  Everything runs on the GPU only, under no_grad.
"""
import math
from types import SimpleNamespace

import torch

from ._lib import check, lib
from .splatmesh import _cam_matrix, _require_cuda, _stream, _vec3

INT32_MAX = 2 ** 31 - 1
SH_C0 = 0.28209479177387814


def texture_size(n_faces, square_size=10):
    """T of the layout: square_size * int(sqrt(n_faces // 2 + 1) + 1)."""
    return square_size * int(math.sqrt(n_faces // 2 + 1) + 1)


def uv_layout(n_faces, square_size=10, device=None):
    """-> (verts_uv float32 [6 n_sq^2, 2], faces_uv int64 [F,3], texture_size), the reference's lines (:2486-2535)
    evaluated on the CPU (exact division by T) and moved to `device`."""
    if square_size < 3:
        raise ValueError("square_size must be >= 3")
    F = int(n_faces)
    if F < 0:
        raise ValueError(f"n_faces must be >= 0, got {F}")
    n_sq = int(math.sqrt(F // 2 + 1) + 1)
    T = square_size * n_sq
    if T * T > INT32_MAX:
        raise ValueError(f"{F} faces at square size {square_size}: texture {T}x{T} has more than 2^31 - 1 texels")
    faces_uv = torch.arange(3 * F).view(F, 3)
    vuv = torch.cartesian_prod(torch.arange(n_sq), torch.arange(n_sq))[:, None]
    u_shift = torch.tensor([[1, 0]], dtype=torch.int32)[:, None]
    v_shift = torch.tensor([[0, 1]], dtype=torch.int32)[:, None]
    bottom = torch.cat([vuv + u_shift, vuv, vuv + u_shift + v_shift], dim=1)
    top = torch.cat([vuv + v_shift, vuv, vuv + u_shift + v_shift], dim=1)
    verts_uv = torch.cat([bottom, top], dim=1) * square_size
    for c, off in enumerate(([-2, 1], [2, 1], [-2, -3], [1, -1], [1, 3], [-3, -1])):
        verts_uv[:, c] = verts_uv[:, c] + torch.tensor([off])
    verts_uv = verts_uv.reshape(-1, 2) / T
    return verts_uv.to(device), faces_uv.to(device), T


def _faces(faces, V):
    if faces.dtype != torch.int64 or faces.dim() != 2 or faces.shape[1] != 3:
        raise ValueError(f"faces must be int64 [F,3], got {faces.dtype} {tuple(faces.shape)}")
    if faces.shape[0] > INT32_MAX // 3:
        raise ValueError(f"{faces.shape[0]} faces: at most (2^31 - 1) / 3")
    return faces.contiguous()


def _same_device(dev, **ts):
    for name, t in ts.items():
        if t.device != dev:
            raise ValueError(f"{name} on {t.device}, verts on {dev}")


def _n_bad(*conds):
    """Counts of the given bool tensors with one host read."""
    if not conds:
        return []
    return torch.stack([c.sum() for c in conds]).tolist()


def initial_texture(verts, faces, points, scaling, quaternions, sh_dc, square_size=10):
    """The reference's initial texels (:2537-2605) for n = P / F Gaussians per face (face-major, as meshbind lays them
    out).  verts float32 [V,3], faces int64 [F,3], points / scaling (activated) float32 [P,3], quaternions float32 [P,4]
    (w first), sh_dc float32 [P,3] or [P,1,3] (the DC SH coefficients).  -> float32 [T,T,3]: SH2RGB of the densest
    Gaussian's DC at every texel a face owns, 0.5 elsewhere."""
    if square_size < 3:
        raise ValueError("square_size must be >= 3")
    dev = verts.device
    verts = _vec3(verts, "verts")
    V = verts.shape[0]
    faces = _faces(faces, V)
    F = faces.shape[0]
    P = points.shape[0]
    points = _vec3(points, "points")
    scaling = _vec3(scaling, "scaling", P)
    if quaternions.dtype != torch.float32 or quaternions.shape != (P, 4):
        raise ValueError(f"quaternions must be float32 [{P},4], got {quaternions.dtype} {tuple(quaternions.shape)}")
    if sh_dc.dtype != torch.float32 or tuple(sh_dc.shape) not in ((P, 3), (P, 1, 3)):
        raise ValueError(f"sh_dc must be float32 [{P},3] or [{P},1,3], got {sh_dc.dtype} {tuple(sh_dc.shape)}")
    if (F == 0 and P != 0) or (F > 0 and (P == 0 or P % F)):
        raise ValueError(f"{P} Gaussians on {F} faces: need n >= 1 Gaussians per face, P = F * n")
    if P > INT32_MAX:
        raise ValueError(f"{P} Gaussians: at most 2^31 - 1")
    n = P // F if F else 1
    _same_device(dev, faces=faces, points=points, scaling=scaling, quaternions=quaternions, sh_dc=sh_dc)
    T = texture_size(F, square_size)
    if T * T > INT32_MAX:
        raise ValueError(f"{F} faces at square size {square_size}: texture {T}x{T} has more than 2^31 - 1 texels")
    (bad,) = _n_bad((faces < 0) | (faces >= V)) if F else [0]
    if bad:
        raise ValueError(f"{bad} face vertex ids outside [0, {V})")
    _require_cuda(verts, faces, points, scaling, quaternions, sh_dc)
    quaternions = quaternions.contiguous()
    if quaternions.data_ptr() % 16:                  # the kernel loads one float4 per Gaussian
        quaternions = quaternions.clone()
    sh_dc = sh_dc.reshape(P, 3).contiguous()
    with torch.no_grad(), torch.cuda.device(dev):
        tex = torch.empty((T, T, 3), dtype=torch.float32, device=dev)
        check(lib.sgr_texture_init(F, n, V, square_size, T, verts.data_ptr(), faces.data_ptr(), points.data_ptr(),
                                   scaling.data_ptr(), quaternions.data_ptr(), sh_dc.data_ptr(), tex.data_ptr(),
                                   _stream(dev)))
    return tex


def new_bake_state(init_texture):
    """-> namespace(sum float32 [T,T,3], count int32 [T,T], owner int32 [T,T] all -1, init): the accumulators of the
    per-view bake, starting from the initial texture `init_texture` [T,T,3] (kept for finish)."""
    if init_texture.dtype != torch.float32 or init_texture.dim() != 3 or init_texture.shape[2] != 3 or \
            init_texture.shape[0] != init_texture.shape[1]:
        raise ValueError(f"init_texture must be float32 [T,T,3], got {init_texture.dtype} {tuple(init_texture.shape)}")
    _require_cuda(init_texture)
    T, dev = init_texture.shape[0], init_texture.device
    return SimpleNamespace(sum=torch.zeros((T, T, 3), dtype=torch.float32, device=dev),
                           count=torch.zeros((T, T), dtype=torch.int32, device=dev),
                           owner=torch.full((T, T), -1, dtype=torch.int32, device=dev), init=init_texture)


def _check_view(state, verts, faces, verts_uv, faces_uv, cam, image, zbuf, pix_to_face):
    dev = verts.device
    verts = _vec3(verts, "verts")
    faces = _faces(faces, verts.shape[0])
    if verts_uv.dtype != torch.float32 or verts_uv.dim() != 2 or verts_uv.shape[1] != 2:
        raise ValueError(f"verts_uv must be float32 [N,2], got {verts_uv.dtype} {tuple(verts_uv.shape)}")
    F = faces.shape[0]
    if faces_uv.dtype != torch.int64 or faces_uv.shape != (F, 3):
        raise ValueError(f"faces_uv must be int64 [{F},3], got {faces_uv.dtype} {tuple(faces_uv.shape)}")
    H, W = int(cam.height), int(cam.width)
    if not (0 < W and 0 < H and W * H <= INT32_MAX):
        raise ValueError(f"image {W}x{H}: need 0 < W, H and W*H <= 2^31 - 1")
    if image.dtype != torch.float32 or image.shape != (3, H, W):
        raise ValueError(f"image must be float32 [3,{H},{W}], got {image.dtype} {tuple(image.shape)}")
    if zbuf.dtype != torch.float32 or zbuf.shape != (H, W):
        raise ValueError(f"zbuf must be float32 [{H},{W}], got {zbuf.dtype} {tuple(zbuf.shape)}")
    if pix_to_face.dtype != torch.int64 or pix_to_face.shape != (H, W):
        raise ValueError(f"pix_to_face must be int64 [{H},{W}], got {pix_to_face.dtype} {tuple(pix_to_face.shape)}")
    T = state.sum.shape[0]
    if state.sum.shape != (T, T, 3) or state.count.shape != (T, T) or state.owner.shape != (T, T) or \
            state.count.dtype != torch.int32 or state.owner.dtype != torch.int32:
        raise ValueError("state must come from new_bake_state")
    _same_device(dev, faces=faces, verts_uv=verts_uv, faces_uv=faces_uv, image=image, zbuf=zbuf,
                 pix_to_face=pix_to_face, state=state.sum)
    _cam_matrix(cam.viewmatrix, dev, "viewmatrix")
    _cam_matrix(cam.projmatrix, dev, "projmatrix")
    V, n_uv = verts.shape[0], verts_uv.shape[0]
    if V > INT32_MAX or n_uv > INT32_MAX:
        raise ValueError(f"{V} vertices / {n_uv} UV vertices: at most 2^31 - 1 each")
    bad = _n_bad((faces < 0) | (faces >= V), (faces_uv < 0) | (faces_uv >= n_uv),
                 (pix_to_face < -1) | (pix_to_face >= F))
    for count, what in zip(bad, (f"face vertex ids outside [0, {V})", f"faces_uv ids outside [0, {n_uv})",
                                 f"pix_to_face values outside [-1, {F})")):
        if count:
            raise ValueError(f"{count} {what}")
    _require_cuda(verts, faces, verts_uv, faces_uv, image, zbuf, pix_to_face, state.sum)


def _bake(state, verts, faces, verts_uv, faces_uv, cam, image, zbuf, pix_to_face):
    dev = verts.device
    H, W = int(cam.height), int(cam.width)
    T = state.sum.shape[0]
    verts, faces, verts_uv, faces_uv = (t.contiguous() for t in (verts, faces, verts_uv, faces_uv))
    if verts_uv.data_ptr() % 8:                      # the kernel loads one float2 per UV vertex
        verts_uv = verts_uv.clone()
    image, zbuf, pix_to_face = image.contiguous(), zbuf.contiguous(), pix_to_face.contiguous()
    view, proj = cam.viewmatrix.contiguous(), cam.projmatrix.contiguous()
    with torch.no_grad(), torch.cuda.device(dev):
        pix_texel = torch.empty((H, W), dtype=torch.int32, device=dev)
        check(lib.sgr_texture_bake_view(verts.shape[0], faces.shape[0], verts_uv.shape[0], T, verts.data_ptr(),
                                        faces.data_ptr(), verts_uv.data_ptr(), faces_uv.data_ptr(), view.data_ptr(),
                                        proj.data_ptr(), W, H, image.data_ptr(), zbuf.data_ptr(),
                                        pix_to_face.data_ptr(), state.sum.data_ptr(), state.count.data_ptr(),
                                        state.owner.data_ptr(), pix_texel.data_ptr(), _stream(dev)))


def bake_view(state, verts, faces, verts_uv, faces_uv, cam, image, zbuf, pix_to_face):
    """Add one view to `state` (new_bake_state): `image` float32 [3,H,W] (the render, clamped to [0, 1] here), `zbuf`
    float32 [H,W] and `pix_to_face` int64 [H,W] of splatmesh.rasterize_mesh(verts, faces, cam); `cam` as
    steps.camera_from_scene builds it.  Ids are checked with one host read."""
    _check_view(state, verts, faces, verts_uv, faces_uv, cam, image, zbuf, pix_to_face)
    _bake(state, verts, faces, verts_uv, faces_uv, cam, image, zbuf, pix_to_face)
    return state


def finish(state):
    """-> float32 [T,T,3]: the mean baked colour of every texel some view reached, the initial texel elsewhere."""
    with torch.no_grad():
        return torch.where(state.count[..., None] > 0, state.sum / state.count[..., None].float(), state.init)


def extract_texture_image_and_uv_from_gaussians(verts, faces, points, scaling, quaternions, strengths, sh_dc, cams,
                                                square_size=10):
    """The reference's texture extraction (n_sh=1, texture_with_gaussian_renders=True) over the views `cams`
    (steps.camera_from_scene namespaces).  verts / faces: the refined surface mesh; points, scaling, quaternions,
    strengths [P] or [P,1] (activated opacities) and sh_dc [P,3] or [P,1,3]: its bound Gaussians, n = P / F per face,
    face-major.  Each view renders the Gaussians at sh degree 0 on a black background with this package's rasterizer,
    z-buffers the mesh and bakes.  -> (verts_uv, faces_uv, texture float32 [T,T,3]), the reference's return order."""
    from .diff_gaussian_rasterization import GaussianRasterizationSettings, GaussianRasterizer
    from . import splatmesh
    dev = verts.device
    P = points.shape[0]
    if strengths.dtype != torch.float32 or tuple(strengths.shape) not in ((P,), (P, 1)):
        raise ValueError(f"strengths must be float32 [{P}] or [{P},1], got {strengths.dtype} {tuple(strengths.shape)}")
    _same_device(dev, strengths=strengths)
    with torch.no_grad():
        init = initial_texture(verts, faces, points, scaling, quaternions, sh_dc, square_size)
        verts_uv, faces_uv, _ = uv_layout(faces.shape[0], square_size, dev)
        state = new_bake_state(init)
        opac = strengths.reshape(P, 1)
        shs = sh_dc.reshape(P, 1, 3)
        bg = torch.zeros(3, device=dev)
        for cam in cams:
            H, W = int(cam.height), int(cam.width)
            st = GaussianRasterizationSettings(image_height=H, image_width=W, tanfovx=cam.tanfovx,
                                               tanfovy=cam.tanfovy, bg=bg, scale_modifier=1.0,
                                               viewmatrix=cam.viewmatrix, projmatrix=cam.projmatrix, sh_degree=0,
                                               campos=cam.campos, prefiltered=False, debug=False)
            image = GaussianRasterizer(st)(means3D=points, means2D=torch.zeros_like(points), opacities=opac, shs=shs,
                                           scales=scaling, rotations=quaternions)[0]
            zbuf, pix_to_face = splatmesh.rasterize_mesh(verts, faces, cam)
            # faces were checked by initial_texture, the layout's ids and rasterize_mesh's output are in range
            _bake(state, verts, faces, verts_uv, faces_uv, cam, image, zbuf, pix_to_face)
        return verts_uv, faces_uv, finish(state)
