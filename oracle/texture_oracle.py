"""CPU restatement of the UV texture extraction -- TEST INFRASTRUCTURE ONLY.

Restates extract_texture_image_and_uv_from_gaussians (sugar_scene/sugar_model.py:2464-2677, n_sh 1,
texture_with_gaussian_renders=True):
    layout           :2486-2535   squares of side s on an n_sq x n_sq grid, T = s n_sq, faces 2k / 2k+1 in square k
    initial texels   :2537-2605   with get_covariance(return_sqrt, inverse_scales) :730-736, in float32 torch ops as
                                  the reference evaluates them (so the CPU result is the reference's own)
and, per view, pytorch3d 0.7.4's published algorithm as the reference uses it (pytorch3d is not installed):
    interpolate_face_attributes   UV = sum_k b'_k uv_k with the perspective-correct, unclipped barycentrics (blur 0)
    TexturesUV nearest            grid_sample, align_corners=True, border padding, the map flipped in y, nearbyint:
                                  col = round(u (T-1)), row = (T-1) - round(v (T-1)) (round half to even)
    SoftPhongShader, AmbientLights, blend   pass the index texel through; then .round()
    index_put (:2668-2672)        of several pixels of one view on one texel the highest row-major index is kept
The barycentrics come from splatmesh_oracle's projection, in float64, for the face the given pix_to_face names.
Every baked pixel also reports its margin: the distance of u (T-1) and v (T-1) from a half-integer (the lesser).
"""
import math

import numpy as np
import torch

from oracle import field_oracle as fo
from oracle import splatmesh_oracle as smo

SH_C0 = 0.28209479177387814


def layout(n_faces, square_size):
    """-> (verts_uv float32 [6 n_sq^2, 2], faces_uv int64 [F,3], T)."""
    if square_size < 3:
        raise ValueError("square_size must be >= 3")
    s, F = square_size, n_faces
    n_sq = int(math.sqrt(F // 2 + 1) + 1)
    T = s * n_sq
    ab = torch.stack(torch.meshgrid(torch.arange(n_sq), torch.arange(n_sq), indexing="ij"), -1).reshape(-1, 1, 2)
    # per square: bottom (a+1, b), (a, b), (a+1, b+1); top (a, b+1), (a, b), (a+1, b+1); then the texel offsets
    corner = torch.tensor([[1, 0], [0, 0], [1, 1], [0, 1], [0, 0], [1, 1]])
    offset = torch.tensor([[-2, 1], [2, 1], [-2, -3], [1, -1], [1, 3], [-3, -1]])
    uv = (ab + corner[None]) * s + offset[None]
    return uv.reshape(-1, 2) / T, torch.arange(3 * F).view(F, 3), T


def owned_texels(square_size):
    """-> ((ti, tj) int64 [s(s-1)/2, 2] of the bottom face, same of the top face), in the reference's order."""
    s = square_size
    bottom = [(i, j) for i in range(s - 1) for j in range(i + 1)]
    top = [(i, j) for i in range(s) for j in range(i + 1, s)]
    return torch.tensor(bottom), torch.tensor(top)


def texel_barycentrics(square_size):
    """-> float32 [2, s(s-1)/2, 3]: the fixed weights of the bottom and top faces' texels."""
    s = square_size
    bottom, top = (t.float() for t in owned_texels(s))
    b = torch.stack([(s - 2) - bottom[:, 0], bottom[:, 1] - 1], -1) / (s - 3)
    t = torch.stack([top[:, 0] - 1, (s - 1) - top[:, 1]], -1) / (s - 3)
    return torch.stack([torch.cat([1.0 - w.sum(-1, keepdim=True), w], -1) for w in (b, t)])


def initial_texture(verts, faces, points, scaling, quaternions, sh_dc, square_size, margins=True):
    """-> (texture float32 [T,T,3], d2 [T,T,2] float64: the two least squared Mahalanobis distances of each owned
    texel's point to its face's Gaussians, inf where unowned or with one Gaussian, owned bool [T,T]; both None without
    `margins`).  Inputs are float32 torch tensors on one device: sh_dc [P,3]; n = P / F."""
    s, F, dev = square_size, faces.shape[0], verts.device
    n = points.shape[0] // F
    _, _, T = layout(F, s)
    n_sq = T // s
    bottom, top = (t.to(dev) for t in owned_texels(s))
    m = bottom.shape[0]
    face_id = torch.arange(F, device=dev)
    k = face_id // 2
    sq = torch.stack([k // n_sq, k % n_sq], -1)                                    # the face's square (a, b)
    local = torch.where((face_id % 2 == 0)[:, None, None], bottom[None], top[None])   # [F,m,2]
    ij = sq[:, None] * s + local                                                   # pre-transpose texel (i, j)
    bary = texel_barycentrics(s).to(dev)[face_id % 2]                             # [F,m,3]
    x = (bary[..., None] * verts[faces][:, None]).sum(dim=-2)                      # [F,m,3]
    mu = points.reshape(F, 1, n, 3)
    M = fo.quaternion_to_matrix(quaternions) * (1.0 / scaling.clamp(min=1e-8))[:, None]
    M = M.reshape(F, 1, n, 3, 3)
    w = M.transpose(-1, -2) @ (x[:, :, None] - mu)[..., None]
    d = (w[..., 0] * w[..., 0]).sum(dim=-1).clamp(min=0.0, max=1e8)               # [F,m,n]
    best = torch.exp(-0.5 * d).argmax(dim=-1)                                      # NaN first, ties to the first
    feat = sh_dc.reshape(F, n, 3).gather(1, best[..., None].expand(-1, -1, 3))   # [F,m,3]
    tex = torch.zeros(T, T, 3, device=dev)
    tex[ij[..., 0], ij[..., 1]] = feat
    tex = (tex.transpose(0, 1).flip(0) * SH_C0 + 0.5)
    if not margins:
        return tex, None, None
    # argmax margins, in float64
    d64 = d.double().sort(dim=-1).values
    two = torch.full((F, m, 2), math.inf, dtype=torch.float64)
    two[..., :min(n, 2)] = d64[..., :2]
    d2 = torch.full((T, T, 2), math.inf, dtype=torch.float64)
    d2[T - 1 - ij[..., 1], ij[..., 0]] = two
    owned = torch.zeros(T, T, dtype=torch.bool)
    owned[T - 1 - ij[..., 1], ij[..., 0]] = True
    return tex, d2, owned


def round_half_even(x):
    return np.rint(x)


def texel_of_uv(u, v, T):
    """TexturesUV(sampling_mode='nearest') over the reference's index map: -> (row, col) int64, and the margin (float64:
    the lesser distance of u (T-1), v (T-1) from a half-integer)."""
    x = np.clip(np.asarray(u, np.float64) * (T - 1), 0, T - 1)
    y = np.clip(np.asarray(v, np.float64) * (T - 1), 0, T - 1)
    margin = np.minimum(np.abs(np.abs(x - np.floor(x)) - 0.5), np.abs(np.abs(y - np.floor(y)) - 0.5))
    return (T - 1) - round_half_even(y).astype(np.int64), round_half_even(x).astype(np.int64), margin


def pixel_barycentrics(verts, faces, viewmatrix, projmatrix, W, H, pix_to_face):
    """Perspective-correct barycentrics (float64 [H*W,3], NaN where pix_to_face < 0) of the named face at every pixel's
    sample point, in the z-buffer's convention (splatmesh_oracle)."""
    x, y, z = smo.project(verts, viewmatrix, projmatrix, W, H)
    p2f = np.asarray(pix_to_face).reshape(-1)
    pix = np.nonzero(p2f >= 0)[0]
    f = np.asarray(faces, np.int64)[p2f[pix]]
    X, Y, Z = x[f], y[f], z[f]
    px, py = (pix % W).astype(np.float64), (pix // W).astype(np.float64)
    area = (X[:, 2] - X[:, 0]) * (Y[:, 1] - Y[:, 0]) - (Y[:, 2] - Y[:, 0]) * (X[:, 1] - X[:, 0])
    b = np.empty((len(pix), 3))
    for e in range(3):
        a_, c_ = (e + 1) % 3, (e + 2) % 3
        b[:, e] = ((px - X[:, a_]) * (Y[:, c_] - Y[:, a_]) - (py - Y[:, a_]) * (X[:, c_] - X[:, a_])) / area
    w = b * np.stack([Z[:, 1] * Z[:, 2], Z[:, 0] * Z[:, 2], Z[:, 0] * Z[:, 1]], 1)
    out = np.full((W * H, 3), np.nan)
    out[pix] = w / np.maximum(w.sum(1), 1e-8)[:, None]
    return out


def bake_view(tex_sum, count, verts, faces, verts_uv, faces_uv, viewmatrix, projmatrix, image, zbuf, pix_to_face):
    """One view, in place on tex_sum float32 [T,T,3] / count int64 [T,T] (numpy).  image float32 [3,H,W], zbuf [H,W],
    pix_to_face int64 [H,W].  -> dict: texel int64 [H,W] (row * T + col, -1 for pixels not baked), margin [H,W]
    (inf for pixels not baked), winner bool [H,W] (the pixel that added to its texel)."""
    T = tex_sum.shape[0]
    _, H, W = image.shape
    p2f = np.asarray(pix_to_face).reshape(-1)
    bake = (p2f >= 0) & (np.asarray(zbuf).reshape(-1) > 0)
    b = pixel_barycentrics(verts, faces, viewmatrix, projmatrix, W, H, np.where(bake, p2f, -1))
    pix = np.nonzero(bake)[0]
    uv = np.asarray(verts_uv, np.float64)[np.asarray(faces_uv)[p2f[pix]]]      # [n,3,2]
    uvp = (b[pix][:, :, None] * uv).sum(1)
    row, col, m = texel_of_uv(uvp[:, 0], uvp[:, 1], T)
    texel = np.full(W * H, -1, np.int64)
    texel[pix] = row * T + col
    margin = np.full(W * H, np.inf)
    margin[pix] = m
    # highest row-major pixel per texel
    owner = np.full(T * T, -1, np.int64)
    np.maximum.at(owner, texel[pix], pix)
    won = owner[owner >= 0]
    t = texel[won]
    rgb = np.clip(np.asarray(image, np.float32).reshape(3, -1)[:, won].T, 0.0, 1.0)
    flat = tex_sum.reshape(-1, 3)
    flat[t] = flat[t] + rgb                                                       # float32, one add per texel
    count.reshape(-1)[t] += 1
    winner = np.zeros(W * H, bool)
    winner[won] = True
    return dict(texel=texel.reshape(H, W), margin=margin.reshape(H, W), winner=winner.reshape(H, W))


def finish(tex_sum, count, init):
    c = count[..., None]
    return np.where(c > 0, tex_sum / np.maximum(c, 1).astype(np.float32), init)
