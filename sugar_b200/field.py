"""Fused SuGaR density / SDF field (the surface-regularisation inner loop).

Mirrors the semantics of `SuGaR.get_field_values` and `SuGaR.compute_density`
(sugar_scene/sugar_model.py:1247-1316, 1345-1368; beta_mode 'average', :1192-1195) for given
neighbour indices: the K-neighbour gather, L^-1 = R(q) diag(1/s) (get_covariance, :730-750),
the Gaussian opacities, their sum, the straight-through clamp, beta and the SDF run in ONE CUDA
kernel (sgr_field_forward), and the backward (sgr_field_backward) scatters gradients to points,
scaling, quaternions, strengths and the samples.

    fields = field_values(x, closest_gaussians_idx, points, scaling, quaternions, strengths,
                          density_factor=1/16, density_threshold=1., return_sdf=True, ...)
    fields['density'], fields['sdf'], fields['beta'], fields['closest_gaussian_opacities']

`quaternions` are the normalised (w,x,y,z) quaternions SuGaR.quaternions returns; gradients are
taken through pytorch3d's quaternion_to_matrix (two_s = 2/|q|^2) exactly like the reference.
"""
import ctypes as C

import torch

from ._lib import SgrFieldParams, check, lib, ptr, require_cuda, scratch, stream, tensor


def _params(N, K, P, density_factor, density_threshold, opacity_min_clamp, group=1):
    p = SgrFieldParams()
    p.samples_per_idx_row = int(group)
    p.N, p.K, p.P = int(N), int(K), int(P)
    p.density_factor = float(density_factor)
    p.density_threshold = float(density_threshold)
    p.opacity_min_clamp = float(opacity_min_clamp)
    return p


def _gaussians(dev, points, scaling, quaternions):
    """The Gaussians' float32 [P,3] centres, [P,3] scales and [P,4] quaternions on the samples' device."""
    points = tensor(points.float(), "points", torch.float32, ("P", 3), dev, "x")
    P = points.shape[0]
    return (points, tensor(scaling.float(), "scaling", torch.float32, (P, 3), dev, "x"),
            tensor(quaternions.float(), "quaternions", torch.float32, (P, 4), dev, "x"))


class _Field(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, nbr_idx, points, scaling, quaternions, strengths, density_factor, density_threshold,
                opacity_min_clamp, group=1, outputs=7):
        """outputs: bit 0 nbr_opacity, bit 1 beta, bit 2 sdf -- unrequested ones are neither allocated nor
        written (they come back as empty tensors)."""
        dev = x.device
        x = tensor(x.float(), "x", torch.float32, ("N", 3))
        points, scaling, quaternions = _gaussians(dev, points, scaling, quaternions)
        N, P = x.shape[0], points.shape[0]
        strengths = strengths.float()
        if tuple(strengths.shape) not in ((P,), (P, 1)):
            raise ValueError(f"strengths must be float32 [{P}] or [{P},1], got {tuple(strengths.shape)}")
        strengths = tensor(strengths, "strengths", torch.float32, strengths.shape, dev, "x")
        nbr_idx = tensor(nbr_idx.long(), "closest_gaussians_idx", torch.int64, ("M", "K"), dev, "x")
        K = nbr_idx.shape[1]
        if nbr_idx.shape[0] * group < N:
            raise RuntimeError("closest_gaussians_idx has too few rows for the samples")
        require_cuda("field", x)
        with torch.cuda.device(dev):
            density = torch.empty(N, device=dev)
            nbr = torch.empty((N, K) if outputs & 1 else (0, K), device=dev)
            beta = torch.empty(N if outputs & 2 else 0, device=dev)
            sdf = torch.empty(N if outputs & 4 else 0, device=dev)
            ws = scratch(lib.sgr_field_scratch_bytes(P), dev)
            p = _params(N, K, P, density_factor, density_threshold, opacity_min_clamp, group)
            check(lib.sgr_field_forward(C.byref(p), ptr(x), ptr(nbr_idx), ptr(points), ptr(scaling), ptr(quaternions),
                                        ptr(strengths), ptr(density), ptr(nbr) if outputs & 1 else None,
                                        ptr(beta) if outputs & 2 else None, ptr(sdf) if outputs & 4 else None,
                                        ptr(ws), stream(dev)))
        ctx.save_for_backward(x, nbr_idx, points, scaling, quaternions, strengths)
        ctx.cfg = (density_factor, density_threshold, opacity_min_clamp, strengths.shape, group, outputs)
        ctx.mark_non_differentiable(nbr_idx)
        return density, nbr, beta, sdf

    @staticmethod
    def backward(ctx, g_density, g_nbr, g_beta, g_sdf):
        x, nbr_idx, points, scaling, quaternions, strengths = ctx.saved_tensors
        density_factor, density_threshold, opacity_min_clamp, s_shape, group, outputs = ctx.cfg
        N, K, P = x.shape[0], nbr_idx.shape[1], points.shape[0]
        dev = x.device
        c = lambda g: None if g is None else g.contiguous().float()
        g_density, g_nbr, g_beta, g_sdf = map(c, (g_density, g_nbr if outputs & 1 else None,
                                                  g_beta if outputs & 2 else None, g_sdf if outputs & 4 else None))
        with torch.cuda.device(dev):
            g_x = torch.empty_like(x)
            g_points = torch.empty_like(points)
            g_scaling = torch.empty_like(scaling)
            g_quat = torch.empty_like(quaternions)
            g_str = torch.empty(P, device=dev)
            ws = scratch(lib.sgr_field_scratch_bytes(P), dev)
            p = _params(N, K, P, density_factor, density_threshold, opacity_min_clamp, group)
            check(lib.sgr_field_backward(C.byref(p), ptr(x), ptr(nbr_idx), ptr(points), ptr(scaling),
                                         ptr(quaternions), ptr(strengths), ptr(g_density), ptr(g_nbr), ptr(g_beta),
                                         ptr(g_sdf), ptr(g_x), ptr(g_points), ptr(g_scaling), ptr(g_quat),
                                         ptr(g_str), ptr(ws), stream(dev)))
        return g_x, None, g_points, g_scaling, g_quat, g_str.view(s_shape), None, None, None, None, None


class _DensityEstimation(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, gaussian_idx, nbr_idx, points, scaling, quaternions, strengths, density_factor, with_opacity):
        dev = x.device
        # floating inputs are taken as float32 and integer indices as int64; anything else fails tensor()'s dtype check
        f32 = lambda t: t.float() if torch.is_tensor(t) and t.is_floating_point() else t
        i64 = lambda t: t.long() if torch.is_tensor(t) and not t.is_floating_point() and t.dtype != torch.bool else t
        x = tensor(f32(x), "x", torch.float32, ("N", 3))
        points = tensor(f32(points), "points", torch.float32, ("P", 3), dev, "x")
        N, P = x.shape[0], points.shape[0]
        scaling = tensor(f32(scaling), "scaling", torch.float32, (P, 3), dev, "x")
        quaternions = tensor(f32(quaternions), "quaternions", torch.float32, (P, 4), dev, "x")
        strengths = f32(strengths)
        one_d = torch.is_tensor(strengths) and strengths.dim() == 1
        strengths = tensor(strengths, "strengths", torch.float32, (P,) if one_d else (P, 1), dev, "x")
        gaussian_idx = tensor(i64(gaussian_idx), "gaussian_idx", torch.int64, (N,), dev, "x")
        nbr_idx = tensor(i64(nbr_idx), "closest_gaussians_idx", torch.int64, (N, "K"), dev, "x")
        K = nbr_idx.shape[1]
        require_cuda("field", x)
        with torch.cuda.device(dev):
            loss = torch.empty(N, device=dev)
            nbr = torch.empty((N, K) if with_opacity else (0, K), device=dev)
            ws = scratch(lib.sgr_field_scratch_bytes(P), dev)
            p = _params(N, K, P, density_factor, 1.0, 1e-16)
            check(lib.sgr_density_estimation_forward(C.byref(p), ptr(x), ptr(gaussian_idx), ptr(nbr_idx), ptr(points),
                                                     ptr(scaling), ptr(quaternions), ptr(strengths), ptr(loss),
                                                     ptr(nbr), ptr(ws), stream(dev)))
        ctx.save_for_backward(x, gaussian_idx, nbr_idx, points, scaling, quaternions, strengths)
        ctx.cfg = (density_factor, strengths.shape)
        ctx.mark_non_differentiable(nbr)
        return loss, nbr

    @staticmethod
    def backward(ctx, g_loss, _g_nbr):
        x, gaussian_idx, nbr_idx, points, scaling, quaternions, strengths = ctx.saved_tensors
        density_factor, s_shape = ctx.cfg
        N, K, P = x.shape[0], nbr_idx.shape[1], points.shape[0]
        dev = x.device
        with torch.cuda.device(dev):
            g_loss = g_loss.contiguous().float()
            g_x = torch.empty_like(x)
            g_points = torch.empty_like(points)
            g_scaling = torch.empty_like(scaling)
            g_quat = torch.empty_like(quaternions)
            g_str = torch.empty(P, device=dev)
            ws = scratch(lib.sgr_field_scratch_bytes(P), dev)
            p = _params(N, K, P, density_factor, 1.0, 1e-16)
            check(lib.sgr_density_estimation_backward(C.byref(p), ptr(x), ptr(gaussian_idx), ptr(nbr_idx), ptr(points),
                                                      ptr(scaling), ptr(quaternions), ptr(strengths), ptr(g_loss),
                                                      ptr(g_x), ptr(g_points), ptr(g_scaling), ptr(g_quat), ptr(g_str),
                                                      ptr(ws), stream(dev)))
        return g_x, None, None, g_points, g_scaling, g_quat, g_str.view(s_shape), None, None


class _NormalLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, gaussian_idx, nbr_idx, points, scaling, quaternions, nbr_opacity):
        dev = x.device
        x = tensor(x.detach().float(), "x", torch.float32, ("N", 3))
        points, scaling, quaternions = _gaussians(dev, points.detach(), scaling.detach(), quaternions.detach())
        N, P = x.shape[0], points.shape[0]
        gaussian_idx = tensor(gaussian_idx.long(), "gaussian_idx", torch.int64, (N,), dev, "x")
        nbr_idx = tensor(nbr_idx.long(), "closest_gaussians_idx", torch.int64, (N, "K"), dev, "x")
        K = nbr_idx.shape[1]
        nbr_opacity = tensor(nbr_opacity.detach().float(), "closest_gaussian_opacities", torch.float32, (N, K), dev,
                             "x")
        require_cuda("field", x)
        with torch.cuda.device(dev):
            loss = torch.empty(N, device=dev)
            ws = scratch(lib.sgr_normal_scratch_bytes(P), dev)
            check(lib.sgr_normal_loss_forward(N, K, P, ptr(x), ptr(gaussian_idx), ptr(nbr_idx), ptr(points),
                                              ptr(scaling), ptr(quaternions), ptr(nbr_opacity), ptr(loss), ptr(ws),
                                              stream(dev)))
        ctx.save_for_backward(x, gaussian_idx, nbr_idx, points, scaling, quaternions, nbr_opacity)
        return loss

    @staticmethod
    def backward(ctx, g_loss):
        x, gaussian_idx, nbr_idx, points, scaling, quaternions, nbr_opacity = ctx.saved_tensors
        N, K, P = x.shape[0], nbr_idx.shape[1], points.shape[0]
        dev = x.device
        with torch.cuda.device(dev):
            g_quat = torch.empty_like(quaternions)
            ws = scratch(lib.sgr_normal_scratch_bytes(P), dev)
            check(lib.sgr_normal_loss_backward(N, K, P, ptr(x), ptr(gaussian_idx), ptr(nbr_idx), ptr(points),
                                               ptr(scaling), ptr(quaternions), ptr(nbr_opacity),
                                               ptr(g_loss.contiguous().float()), ptr(g_quat), ptr(ws), stream(dev)))
        return None, None, None, None, None, g_quat, None


def better_normal_loss(x, gaussian_idx, closest_gaussians_idx, points, scaling, quaternions,
                       closest_gaussian_opacities, gradient_through_normal_only=True):
    """Per-sample "better normal" loss of the trainers (sugar_trainers/coarse_sdf.py:688-716): returns
    `sdf_better_normal_loss` [N]; the caller adds `factor * loss.mean()` (coarse_sdf.py:716).

    x = sdf_samples, gaussian_idx = sdf_gaussian_idx, closest_gaussians_idx = knn_idx[gaussian_idx],
    closest_gaussian_opacities = fields['closest_gaussian_opacities'] (detached by the reference, :703).
    Normals are SuGaR.get_normals(estimate_from_points=False) of an unbound model, i.e. the smallest
    axis of each Gaussian (sugar_model.py:930-968).  Only the trainers' setting
    sdf_better_normal_gradient_through_normal_only=True (coarse_sdf.py:144) is implemented: gradients
    flow to `quaternions` alone.  Shapes, dtypes and devices are checked (ValueError); index ranges are not, which
    would cost a host synchronisation per step."""
    if not gradient_through_normal_only:
        raise NotImplementedError("only sdf_better_normal_gradient_through_normal_only=True (the reference "
                                  "trainers' fixed setting, coarse_sdf.py:144) is implemented")
    return _NormalLoss.apply(x, gaussian_idx, closest_gaussians_idx, points, scaling, quaternions,
                             closest_gaussian_opacities)


def density_estimation_loss(x, gaussian_idx, closest_gaussians_idx, points, scaling, quaternions, strengths,
                            density_factor=1.0, return_closest_gaussian_opacities=False):
    """Per-sample density estimation loss of the coarse_density trainer in projection mode
    (sugar_trainers/coarse_density.py:642-656, 684-691): returns `sdf_estimation_loss` [N]; the caller adds
    `factor * loss.mean()` over all samples (:691).

        rho    = field_values(...)['density'] at x, before the straight-through clamp (sugar_model.py:1279)
        beta   = mean of the K neighbours' smallest scales ('average' beta, :1192-1195)
        e      = <x - points[gaussian_idx], n>, n the smallest axis of the sample's own Gaussian (get_normals)
        loss   = | rho - exp(-0.5 e^2 / beta^2) |

    x = sdf_samples, gaussian_idx = sdf_gaussian_idx, closest_gaussians_idx = knn_idx[gaussian_idx].  One fused
    kernel evaluates it; the backward reaches x, points, scaling, quaternions and strengths (no gradient through
    the argmin picking the normal's column).  With return_closest_gaussian_opacities, also returns the field's
    [N, K] neighbour opacities (non-differentiable, for better_normal_loss), bit for bit those of field_values.
    Shapes, dtypes and devices are checked (ValueError); index ranges are not, which would cost a host
    synchronisation per step."""
    loss, nbr = _DensityEstimation.apply(x, gaussian_idx, closest_gaussians_idx, points, scaling, quaternions,
                                         strengths, density_factor, bool(return_closest_gaussian_opacities))
    return (loss, nbr) if return_closest_gaussian_opacities else loss


def field_values(x, closest_gaussians_idx, points, scaling, quaternions, strengths, density_factor=1.,
                 density_threshold=1., opacity_min_clamp=1e-16, return_sdf=True,
                 return_closest_gaussian_opacities=False, return_beta=False, return_sdf_grad=False,
                 sdf_grad_max_value=10., beta_mode="average"):
    """SuGaR.get_field_values for explicit neighbour indices (closest_gaussians_idx = knn_idx[gaussian_idx]).

    beta_mode: only 'average' (the mean of the neighbours' smallest scales, sugar_model.py:1192-1195) -- the one
    mode every trainer and extractor of the reference constructs its model with; 'learnable' / 'weighted_average'
    raise.  `return_sdf_grad` adds fields['sdf_grad'] (:1307-1314) as a VALUE (detached, clamped to
    +-sdf_grad_max_value): it is beta / (rho sqrt(-2 ln rho)) times minus the density's spatial gradient, which the
    fused backward kernel delivers; no caller of the reference differentiates through it.  Shapes, dtypes and devices
    are checked (ValueError); index ranges are not, which would cost a host synchronisation per step."""
    if beta_mode != "average":
        raise NotImplementedError(f"beta_mode={beta_mode!r}: only 'average' is implemented (sugar_model.py:1192-1195)")
    density, nbr, beta, sdf = _Field.apply(x, closest_gaussians_idx, points, scaling, quaternions, strengths,
                                           density_factor, density_threshold, opacity_min_clamp, 1, 7)
    fields = {"density": density}
    if return_sdf_grad:
        with torch.enable_grad():
            xg = x.detach().clone().requires_grad_(True)
            d = _Field.apply(xg, closest_gaussians_idx, points.detach(), scaling.detach(), quaternions.detach(),
                             strengths.detach(), density_factor, density_threshold, opacity_min_clamp, 1, 0)[0]
            (gx,) = torch.autograd.grad(d.sum(), xg)      # d rho / d x = -sum_k o_k Sigma_k^-1 (x - mu_k)
        with torch.no_grad():
            rho = torch.where(d >= 1.0, d / (d + 1e-12), d).clamp(min=opacity_min_clamp)   # :1280-1281, :1296
            coef = beta.detach() / (rho * torch.sqrt(-2.0 * torch.log(rho))).clamp(min=opacity_min_clamp)
            fields["sdf_grad"] = (coef[:, None] * (-gx)).clamp(min=-sdf_grad_max_value, max=sdf_grad_max_value)
    if return_closest_gaussian_opacities:
        fields["closest_gaussian_opacities"] = nbr
    if return_beta:
        fields["beta"] = beta
    if return_sdf:
        fields["sdf"] = sdf
    return fields


def compute_density(x, closest_gaussians_idx, points, scaling, quaternions, strengths, density_factor=1.,
                    return_closest_gaussian_opacities=False, samples_per_idx_row=1):
    """SuGaR.compute_density (sugar_model.py:1345-1368) for given neighbour indices.  With
    `samples_per_idx_row` = g > 1, row n // g of `closest_gaussians_idx` serves sample n (consecutive ray
    samples sharing their pixel's neighbours) so the index table need not be replicated."""
    density, nbr, _, _ = _Field.apply(x, closest_gaussians_idx, points, scaling, quaternions, strengths,
                                      density_factor, 1.0, 1e-16, samples_per_idx_row,
                                      1 if return_closest_gaussian_opacities else 0)
    return (density, nbr) if return_closest_gaussian_opacities else density


def quaternion_apply(q: torch.Tensor, p: torch.Tensor) -> torch.Tensor:
    """Rotate points p by quaternions q (real part first), as pytorch3d.transforms.quaternion_apply."""
    r, i, j, k = torch.unbind(q, -1)
    two_s = 2.0 / (q * q).sum(-1)
    R = torch.stack((1 - two_s * (j * j + k * k), two_s * (i * j - k * r), two_s * (i * k + j * r),
                     two_s * (i * j + k * r), 1 - two_s * (i * i + k * k), two_s * (j * k - i * r),
                     two_s * (i * k - j * r), two_s * (j * k + i * r), 1 - two_s * (i * i + j * j)), -1)
    return (R.reshape(q.shape[:-1] + (3, 3)) @ p[..., None])[..., 0]


def sample_points_in_gaussians(points, scaling, quaternions, strengths, num_samples, sampling_scale_factor=1.,
                               mask=None, probabilities_proportional_to_opacity=False,
                               probabilities_proportional_to_volume=True, generator=None):
    """SuGaR.sample_points_in_gaussians (sugar_scene/sugar_model.py:885-928): multinomial over volume (x opacity)
    weights, then x = mu + R(q) (scale_factor * s * N(0,1)).  Kept in PyTorch on purpose: it is RNG-bound and this
    keeps the reference's random streams (SURVEY 8a, a16).  Returns (samples [N,3], gaussian indices [N])."""
    sc = scaling if mask is None else scaling[mask]
    areas = sc[..., 0] * sc[..., 1] * sc[..., 2] if probabilities_proportional_to_volume else torch.ones_like(sc[..., 0])
    if probabilities_proportional_to_opacity:
        st = strengths.view(-1)
        areas = areas * (st if mask is None else st[mask])
    areas = areas.abs()
    idx = torch.multinomial(areas / areas.sum(dim=-1, keepdim=True), num_samples=num_samples, replacement=True,
                            generator=generator)
    if mask is not None:
        idx = torch.arange(points.shape[0], device=points.device)[mask][idx]
    noise = torch.randn(points[idx].shape, device=points.device, dtype=points.dtype, generator=generator)
    x = points[idx] + quaternion_apply(quaternions[idx], sampling_scale_factor * scaling[idx] * noise)
    return x, idx
