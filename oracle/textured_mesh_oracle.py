"""CPU restatement of the textured mesh's render -- TEST INFRASTRUCTURE ONLY.

Restates metrics.py --use_uv_texture (metrics.py:260-300, 370-372) from pytorch3d 0.7.4's published algorithm
(pytorch3d is not installed): MeshRasterizer with one face per pixel and blur 0, then SoftPhongShader with
AmbientLights and a background colour:
    interpolate_face_attributes   UV = sum_k b'_k uv_k with the perspective-correct barycentrics of texture_oracle
    TexturesUV.sample_textures    torch.nn.functional.grid_sample itself, on the map flipped in y at uv * 2 - 1,
                                  align_corners=True, border padding
    phong_shading                 AmbientLights and default Materials: the colour is the texel
    softmax_rgb_blend             K = 1, sigma = gamma = 1e-4, with the edge weight prob taken as 1 (the z-buffer has
                                  no dists), in float32 as torch evaluates it on the GPU
"""
import numpy as np
import torch

from oracle.texture_oracle import pixel_barycentrics

# the shader constants of metrics.py's SoftPhongShader (BlendParams sigma = gamma = 1e-4) and softmax_rgb_blend's eps
BLEND_EPS = 1e-10
BLEND_GAMMA = 1e-4


def sample_texture(uv, texture, mode):
    """TexturesUV.sample_textures at float32 UVs [N,2] of the float32 map [Ht,Wt,3]: grid_sample on the map flipped in
    y at uv * 2 - 1, align_corners=True, border padding -- the reference's own op.  -> float32 [N,3] (torch, on the
    inputs' device)."""
    grid = (uv * 2.0 - 1.0).reshape(1, 1, -1, 2)
    maps = torch.flip(texture.permute(2, 0, 1)[None], [2])
    return torch.nn.functional.grid_sample(maps, grid, mode=mode, align_corners=True, padding_mode="border")[0, :, 0].T


def blend(colors, zbuf, mask, background, znear=1e-4, zfar=100.0):
    """softmax_rgb_blend at K = 1 with prob = 1 where `mask`, 0 elsewhere, in float32 as torch evaluates it on the GPU
    (a division by a Python number multiplies by its float32 reciprocal).  colors float32 [N,3], zbuf [N], mask bool
    [N] (numpy) -> float32 [N,3]."""
    f32 = np.float32
    m = np.asarray(mask, bool)
    z = np.asarray(zbuf, f32)
    c = np.where(m[:, None], np.asarray(colors, f32), f32(0.0))
    inv_range, inv_gamma, eps = f32(1.0) / f32(zfar - znear), f32(1.0) / f32(BLEND_GAMMA), f32(BLEND_EPS)
    with np.errstate(over="ignore", invalid="ignore"):
        z_inv = np.where(m, (f32(zfar) - z) * inv_range, f32(0.0))
        z_max = np.where(z_inv < eps, eps, z_inv)                                  # clamp(min=eps) keeps NaN
        w = np.where(m, np.exp((z_inv - z_max) * inv_gamma), f32(0.0))            # prob * exp(...)
        delta = np.exp((eps - z_max) * inv_gamma)
        delta = np.where(delta < eps, eps, delta)
        bg = np.asarray(background, f32)
        return ((w[:, None] * c + delta[:, None] * bg) / (w + delta)[:, None]).astype(f32)


def render_view(verts, faces, verts_uv, faces_uv, texture, viewmatrix, projmatrix, W, H, zbuf, pix_to_face,
                sampling_mode="bilinear", background=(0.0, 0.0, 0.0), znear=1e-4, zfar=100.0):
    """The textured mesh's image over a given z-buffer: float64 barycentrics (pixel_barycentrics), the UV in float64
    rounded once to float32, sample_texture, blend.  texture float32 torch [Ht,Wt,3]; the rest numpy.  -> dict: image
    float32 [3,H,W], uv float64 [H*W,2] (NaN where no face), colour float32 [H*W,3] (the sampled texel, 0 where no
    face), mask bool [H*W]."""
    p2f = np.asarray(pix_to_face).reshape(-1)
    mask = p2f >= 0
    b = pixel_barycentrics(verts, faces, viewmatrix, projmatrix, W, H, p2f)
    uv = np.full((W * H, 2), np.nan)
    uv[mask] = (b[mask][:, :, None] * np.asarray(verts_uv, np.float64)[np.asarray(faces_uv)[p2f[mask]]]).sum(1)
    colour = np.zeros((W * H, 3), np.float32)
    if mask.any():
        t = torch.from_numpy(uv[mask].astype(np.float32)).to(texture.device)
        colour[mask] = sample_texture(t, texture, sampling_mode).cpu().numpy()
    image = blend(colour, np.asarray(zbuf).reshape(-1), mask, background, znear, zfar)
    return dict(image=image.T.reshape(3, H, W), uv=uv, colour=colour, mask=mask)
