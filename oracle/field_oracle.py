"""CPU restatement of SuGaR's density / SDF field -- TEST INFRASTRUCTURE ONLY (see raster_oracle.c).

Follows, op for op in PyTorch on the CPU:
    get_covariance(return_full_matrix, return_sqrt, inverse_scales)   sugar_scene/sugar_model.py:730-750
    get_beta, beta_mode == 'average'                                 sugar_scene/sugar_model.py:1192-1195
    get_field_values                                                 sugar_scene/sugar_model.py:1247-1316
    compute_density                                                  sugar_scene/sugar_model.py:1345-1368
    sample_points_in_gaussians                                       sugar_scene/sugar_model.py:885-928
    get_smallest_axis / get_normals(estimate_from_points=False)      sugar_scene/sugar_model.py:930-968
    "better normal" loss (inline in the trainers)                    sugar_trainers/coarse_sdf.py:688-716
    level-set points along camera rays (per-ray part)                sugar_scene/sugar_model.py:1970-2081
Third-party arithmetic that is NOT under /root/reference (pytorch3d 0.7.4, environment.yml:161) is
restated from its published algorithm: quaternion_to_matrix / quaternion_apply (real-first) and
knn_points (exact K-NN on squared distances; restated with cdist + topk).

Parity pinning: tests/golden/field_*.npz were produced by running the reference's OWN
SuGaR.get_field_values code (imported from /root/reference with the missing third-party modules
stubbed, tests/golden/make_field_golden.py); tests/test_field_oracle.py checks this file against them.
tests/golden/normal_*.npz likewise: normals from the reference's SuGaR.get_normals, loss from the
trainer's own source lines executed as they stand (tests/golden/make_normal_golden.py);
tests/golden/levelset_*.npz from lines 1970-2081 of compute_level_surface_points_from_camera_fast executed
as they stand (tests/golden/make_levelset_golden.py).
"""
import numpy as np
import torch

# The clamp bounds as the float32 constants the reference's float32 tensors compare against (torch casts a Python
# scalar to the tensor's dtype), so a float64 run clamps at exactly the same inputs as the float32 one.
_f32 = lambda v: float(np.float32(v))

def quaternion_to_matrix(q: torch.Tensor) -> torch.Tensor:
    """pytorch3d.transforms.quaternion_to_matrix (0.7.4): real part first, two_s = 2/|q|^2."""
    r, i, j, k = torch.unbind(q, -1)
    two_s = 2.0 / (q * q).sum(-1)
    o = torch.stack((1 - two_s * (j * j + k * k), two_s * (i * j - k * r), two_s * (i * k + j * r),
                     two_s * (i * j + k * r), 1 - two_s * (i * i + k * k), two_s * (j * k - i * r),
                     two_s * (i * k - j * r), two_s * (j * k + i * r), 1 - two_s * (i * i + j * j)), -1)
    return o.reshape(q.shape[:-1] + (3, 3))


def quaternion_apply(q: torch.Tensor, p: torch.Tensor) -> torch.Tensor:
    """pytorch3d.transforms.quaternion_apply: rotate points by (unit) quaternions."""
    return (quaternion_to_matrix(q) @ p[..., None])[..., 0]


def knn_idx(points: torch.Tensor, K: int, queries: torch.Tensor = None) -> torch.Tensor:
    """pytorch3d.ops.knn_points(...).idx for one cloud: exact K nearest by squared distance."""
    q = points if queries is None else queries
    d = torch.cdist(q.double(), points.double())
    return d.topk(K, dim=1, largest=False).indices


def field_values_torch(x, nbr_idx, points, scaling, quaternions, strengths, density_factor=1.0,
                       density_threshold=1.0, opacity_min_clamp=1e-16, return_sdf_grad=False, sdf_grad_max_value=10.0):
    """get_field_values with closest_gaussians_idx given; tensors may require grad."""
    opacity_min_clamp = _f32(opacity_min_clamp)
    s = 1.0 / scaling.clamp(min=_f32(1e-8))
    inv_scaled_rot = quaternion_to_matrix(quaternions) * s[:, None]          # :730-735
    c_centers = points[nbr_idx]
    c_isr = inv_scaled_rot[nbr_idx]
    c_str = strengths.view(-1, 1)[nbr_idx]
    shift = x[:, None] - c_centers
    warped = c_isr.transpose(-1, -2) @ shift[..., None]
    nb = (warped[..., 0] * warped[..., 0]).sum(dim=-1).clamp(min=0.0, max=1e8)
    nb = density_factor * c_str[..., 0] * torch.exp(-1.0 / 2 * nb)
    densities = nb.sum(dim=-1)
    out = {"density": densities.clone(), "closest_gaussian_opacities": nb}
    mask = densities >= 1.0
    densities = torch.where(mask, densities / (densities.detach() + 1e-12), densities)   # :1280-1281
    beta = scaling.min(dim=-1)[0][nbr_idx].mean(dim=1)                                   # :1195
    clamped = densities.clamp(min=opacity_min_clamp)
    out["beta"] = beta
    out["sdf"] = beta * (torch.sqrt(-2.0 * torch.log(clamped)) - np.sqrt(-2.0 * np.log(min(density_threshold, 1.0))))
    if return_sdf_grad:                                                                    # :1307-1314
        g = (nb[..., None] * (c_isr @ warped)[..., 0]).sum(dim=-2)
        g = (beta / (clamped * torch.sqrt(-2.0 * torch.log(clamped))).clamp(min=opacity_min_clamp))[..., None] * g
        out["sdf_grad"] = g.clamp(min=-sdf_grad_max_value, max=sdf_grad_max_value)
    return out


# sugar_utils/spherical_harmonics.py:1-40 (constants), :117-172 (eval_sh)
_C0 = 0.28209479177387814
_C1 = 0.4886025119029199
_C2 = [1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396]
_C3 = [-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658,
       1.445305721320277, -0.5900435899266435]


def eval_sh(deg, sh, dirs):
    """eval_sh (sugar_utils/spherical_harmonics.py:117-172), degrees 0-3: sh [..., C, (deg+1)^2], dirs [..., 3]."""
    result = _C0 * sh[..., 0]
    if deg > 0:
        x, y, z = dirs[..., 0:1], dirs[..., 1:2], dirs[..., 2:3]
        result = (result - _C1 * y * sh[..., 1] + _C1 * z * sh[..., 2] - _C1 * x * sh[..., 3])
        if deg > 1:
            xx, yy, zz = x * x, y * y, z * z
            xy, yz, xz = x * y, y * z, x * z
            result = (result + _C2[0] * xy * sh[..., 4] + _C2[1] * yz * sh[..., 5] +
                      _C2[2] * (2.0 * zz - xx - yy) * sh[..., 6] + _C2[3] * xz * sh[..., 7] + _C2[4] * (xx - yy) * sh[..., 8])
            if deg > 2:
                result = (result + _C3[0] * y * (3 * xx - yy) * sh[..., 9] + _C3[1] * xy * z * sh[..., 10] +
                          _C3[2] * y * (4 * zz - xx - yy) * sh[..., 11] + _C3[3] * z * (2 * zz - 3 * xx - 3 * yy) * sh[..., 12] +
                          _C3[4] * x * (4 * zz - xx - yy) * sh[..., 13] + _C3[5] * z * (xx - yy) * sh[..., 14] +
                          _C3[6] * x * (xx - 3 * yy) * sh[..., 15])
    return result


def points_rgb_torch(positions, sh_coordinates, camera_center, sh_levels):
    """SuGaR.get_points_rgb (sugar_model.py:839-883): the trainers' python colour path
    (compute_color_in_rasterizer=False, coarse_sdf.py:51)."""
    dirs = torch.nn.functional.normalize(positions - camera_center.reshape(1, 3), dim=-1)
    shs_view = sh_coordinates[:, :sh_levels ** 2].transpose(-1, -2).reshape(-1, 3, sh_levels ** 2)
    return torch.clamp_min(eval_sh(sh_levels - 1, shs_view, dirs) + 0.5, 0.0).view(-1, 3)


def smallest_axis(scaling, quaternions):
    """get_smallest_axis (sugar_model.py:930-945): the column of R(q) along the smallest scale."""
    rot = quaternion_to_matrix(quaternions)
    col = scaling.min(dim=-1)[1][..., None, None].expand(-1, 3, -1)
    return rot.gather(2, col).squeeze(dim=2)


def better_normal_loss_torch(x, gaussian_idx, nbr_idx, points, scaling, quaternions, nbr_opacity):
    """Per-sample "better normal" loss, coarse_sdf.py:688-716 with the trainers' only setting
    sdf_better_normal_gradient_through_normal_only=True (coarse_sdf.py:144): weights and signs are
    detached, gradients reach the quaternions through the normals only.  Returns [N]."""
    normals = smallest_axis(scaling, quaternions)
    min_scaling = scaling.min(dim=-1)[0][nbr_idx].detach().view(len(x), -1)                       # :693
    c_normals = normals[nbr_idx]                                                                 # :696
    s_normals = normals[gaussian_idx]                                                            # :697
    c_normals = c_normals * torch.sign((c_normals * s_normals[:, None]).sum(dim=-1, keepdim=True)).detach()  # :698-700
    w = ((x[:, None] - points[nbr_idx]) * c_normals).sum(dim=-1).abs().detach()                  # :704-706
    w = nbr_opacity.detach() * w / min_scaling.clamp(min=_f32(1e-6)) ** 2                              # :707
    w = w / w.sum(dim=-1).detach().unsqueeze(-1).clamp(min=_f32(1e-6))                                 # :710-711
    return (s_normals - (w[..., None] * c_normals).sum(dim=-2)).pow(2).sum(dim=-1)               # :714-715


def level_surface_points_torch(world_points, camera_center, closest_gaussians_idx, points, scaling, quaternions,
                               strengths, surface_levels=(0.1, 0.3, 0.5), n_points_in_range=21, range_size=3.0,
                               density_factor=1.0, return_normals=True):
    """Per-ray part of compute_level_surface_points_from_camera_fast (sugar_model.py:1970-2081), default flags
    (compute_intersection_for_flat_gaussian=False, compute_flat_normals=False, just_use_depth_as_level=False)."""
    cam = camera_center.reshape(1, 3)
    to_cam = torch.nn.functional.normalize(cam - points, dim=-1)                                            # :1971
    q_inv = quaternions * quaternions.new_tensor([1.0, -1.0, -1.0, -1.0])
    stds = (scaling * quaternion_apply(q_inv, to_cam)).norm(dim=-1)                                         # :1972
    points_stds = stds[closest_gaussians_idx[..., 0]]
    rng = torch.linspace(-range_size, range_size, n_points_in_range).to(points).view(1, -1, 1)              # :1976
    rng = rng * points_stds[..., None, None].expand(-1, n_points_in_range, 1)
    cam_to_samples = torch.nn.functional.normalize(world_points - cam, dim=-1)
    samples = (world_points[:, None, :] + rng * cam_to_samples[:, None, :]).view(-1, 3)
    K = closest_gaussians_idx.shape[1]
    s_idx = closest_gaussians_idx[:, None, :].expand(-1, n_points_in_range, -1).reshape(-1, K)
    isr = quaternion_to_matrix(quaternions) * (1.0 / scaling.clamp(min=_f32(1e-8)))[:, None]                      # :1986
    str_ = strengths.view(-1, 1)

    def opac(x, idx):
        shift = x[:, None] - points[idx]
        warped = isr[idx].transpose(-1, -2) @ shift[..., None]
        o = (warped[..., 0] * warped[..., 0]).sum(dim=-1).clamp(min=0.0, max=1e8)
        return density_factor * str_[idx][..., 0] * torch.exp(-1.0 / 2 * o), warped
    dens = opac(samples, s_idx)[0].sum(dim=-1)
    m = dens >= 1.0
    dens = torch.where(m, dens / (dens + 1e-12), dens).reshape(-1, n_points_in_range)                       # :2007-2011
    out = {}
    for level in surface_levels:
        under, above = dens - level < 0, dens - level > 0
        _, first = above.max(dim=-1, keepdim=True)
        empty = ~under[..., 0] + (first[..., 0] == 0)
        vd, vr, fa = dens[~empty], rng[~empty][..., 0], first[~empty]
        v1, v0 = vd.gather(-1, fa).view(-1), vd.gather(-1, fa - 1).view(-1)
        t1, t0 = vr.gather(-1, fa).view(-1), vr.gather(-1, fa - 1).view(-1)
        t = (level - v0) / (v1 - v0) * (t1 - t0) + t0
        inter = world_points[~empty] + t[:, None] * cam_to_samples[~empty]
        res = {"intersection_points": inter, "valid": ~empty}
        if return_normals:
            idx = closest_gaussians_idx[~empty]
            o, warped = opac(inter, idx)
            grad = (o[..., None] * (isr[idx] @ warped)[..., 0]).sum(dim=-2)                                 # :2065
            res["normals"] = -torch.nn.functional.normalize(grad, dim=-1)                                  # :2075
        out[level] = res
    return out


def field_values(x, nbr_idx, points, scaling, quaternions, strengths, density_factor=1.0, density_threshold=1.0,
                 opacity_min_clamp=1e-16, **_):
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a))
    with torch.no_grad():
        o = field_values_torch(t(x), t(nbr_idx), t(points), t(scaling), t(quaternions), t(strengths), density_factor,
                               density_threshold, opacity_min_clamp)
    return {k: v.numpy() for k, v in o.items()}


def make_case(P=1000, N=2000, K=16, seed=0, density_factor=1.0 / 16.0, density_threshold=1.0):
    """Seeded cloud + samples drawn like sample_points_in_gaussians(:885-928): multinomial over
    volumes, x = mu + R(q) (1.5 * s * N(0,1)); neighbours = knn_idx[gaussian_idx]."""
    g = torch.Generator().manual_seed(seed)
    points = torch.randn(P, 3, generator=g)
    scaling = torch.exp(torch.randn(P, 3, generator=g) * 0.5 - 2.3)
    q = torch.nn.functional.normalize(torch.randn(P, 4, generator=g), dim=-1)
    strengths = torch.sigmoid(torch.randn(P, generator=g) * 2.0)
    nn_idx = knn_idx(points, K)
    areas = (scaling[:, 0] * scaling[:, 1] * scaling[:, 2]).abs()
    gi = torch.multinomial(areas / areas.sum(), N, replacement=True, generator=g)
    x = points[gi] + quaternion_apply(q[gi], 1.5 * scaling[gi] * torch.randn(N, 3, generator=g))
    f = lambda a: np.ascontiguousarray(a.numpy())
    return dict(x=f(x.float()), nbr_idx=f(nn_idx[gi]), gaussian_idx=f(gi), points=f(points), scaling=f(scaling), quaternions=f(q),
                strengths=f(strengths), density_factor=density_factor, density_threshold=density_threshold)
