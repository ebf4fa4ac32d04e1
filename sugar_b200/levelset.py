"""Level-set points along camera rays for mesh extraction (SURVEY.md section 8 f3).

The per-ray part of `SuGaR.compute_level_surface_points_from_camera_fast`
(sugar_scene/sugar_model.py:1970-2081, called per training view by
sugar_extractors/coarse_mesh.py:246-327): given the back-projected depth points of a view and the
Gaussian each one fell on, sample `n_points_in_range` (21) positions per ray within +-`range_size`
standard deviations, evaluate the density at every sample from the K tracked neighbours, find the
first crossing of each surface level and interpolate it; optionally the normals there.

`level_surface_points_from_camera` is the whole per-view call with either depth source in front:
  use_gaussian_depth=True (this function's default; :1898-1909, 1926-1964): depth render of the view with this
    package's rasterizer (colours = view-space z, background -1), back-projection of every covered pixel, K nearest
    Gaussians of each point with the grid K-NN (get_gaussians_closest_to_samples, :1335-1343);
  use_gaussian_depth=False (the reference's default, which the extraction driver keeps; :1912-1928, 1965-1968): the
    splatted diamond mesh z-buffered by `splatmesh.rasterize_mesh`, back-projection, and the ray's Gaussian
    pix_to_face // 2 with its neighbours from the model's knn_idx table (no per-point K-NN search).
The density evaluation -- in the reference 2M-point passes of gathered N x K x 3 x 3 matrices -- is ONE launch of the
fused field kernel (sgr_field_forward) over all n_points * 21 samples; normals come from its backward (d density / d x).
"""
import torch

from . import field


def _quaternion_invert(q):
    return q * q.new_tensor([1.0, -1.0, -1.0, -1.0])


def level_surface_points(world_points, camera_center, closest_gaussians_idx, points, scaling, quaternions, strengths,
                         surface_levels=(0.1, 0.3, 0.5), n_points_in_range=21, range_size=3.0, density_factor=1.0,
                         return_normals=False):
    """Returns {level: {'intersection_points' [n_valid,3], 'valid' bool[n_points] (= ~empty_pixels), 'normals'}}.

    world_points [n,3]: back-projected depth points (all_world_points, :1955); camera_center [3] or [1,3];
    closest_gaussians_idx i64[n,K] = knn_idx[gaussian_idx] (:1967); points/scaling/quaternions/strengths as in
    `field.field_values` (strengths [P] or [P,1])."""
    cam = camera_center.reshape(1, 3)
    n, K = closest_gaussians_idx.shape
    with torch.no_grad():
        # standard deviation of each Gaussian along its direction to the camera (:1971-1973)
        to_cam = torch.nn.functional.normalize(cam - points, dim=-1)
        stds = (scaling * field.quaternion_apply(_quaternion_invert(quaternions), to_cam)).norm(dim=-1)
        points_stds = stds[closest_gaussians_idx[..., 0]]
        # ray samples (:1976-1980)
        points_range = torch.linspace(-range_size, range_size, n_points_in_range, device=world_points.device).view(1, -1, 1)
        points_range = points_range * points_stds[..., None, None].expand(-1, n_points_in_range, 1)
        cam_to_samples = torch.nn.functional.normalize(world_points - cam, dim=-1)
        samples = (world_points[:, None, :] + points_range * cam_to_samples[:, None, :]).view(-1, 3)
        # densities of all samples (:1983-2011): fused kernel, then the straight-through clamp's value.  The
        # reference replicates the neighbour table per sample (n x 21 x K int64, :1980); here the kernel maps
        # sample -> pixel row itself
        dens = field.compute_density(samples, closest_gaussians_idx, points, scaling, quaternions, strengths,
                                     density_factor=density_factor, samples_per_idx_row=n_points_in_range)
        dens = torch.where(dens >= 1.0, dens / (dens + 1e-12), dens).reshape(-1, n_points_in_range)
    out = {}
    for level in surface_levels:
        with torch.no_grad():
            under = (dens - level < 0)
            above = (dens - level > 0)
            _, first_above = above.max(dim=-1, keepdim=True)                       # :2021
            empty = ~under[..., 0] + (first_above[..., 0] == 0)                    # :2022
            vd = dens[~empty]
            vr = points_range[~empty][..., 0]
            fa = first_above[~empty]
            v1 = vd.gather(-1, fa).view(-1)
            v0 = vd.gather(-1, fa - 1).view(-1)
            t1 = vr.gather(-1, fa).view(-1)
            t0 = vr.gather(-1, fa - 1).view(-1)
            t = (level - v0) / (v1 - v0) * (t1 - t0) + t0                          # :2036
            inter = world_points[~empty] + t[:, None] * cam_to_samples[~empty]
        res = {"intersection_points": inter, "valid": ~empty}
        if return_normals:
            # reference: -normalize(sum_k o_k Sigma_k^-1 (x - mu_k)) = normalize(d density / d x)  (:2048-2078)
            x = inter.detach().clone().requires_grad_(True)
            d = field.compute_density(x, closest_gaussians_idx[~empty], points.detach(), scaling.detach(),
                                      quaternions.detach(), strengths.detach(), density_factor=density_factor)
            (g,) = torch.autograd.grad(d.sum(), x)
            res["normals"] = torch.nn.functional.normalize(g, dim=-1)
        out[level] = res
    return out


def level_surface_points_from_camera(points, scaling, quaternions, strengths, cam, surface_levels=(0.1, 0.3, 0.5),
                                     n_surface_points=-1, n_points_in_range=21, range_size=3.0, density_factor=1.0,
                                     knn_to_track=16, return_normals=False, return_pixel_idx=False, generator=None,
                                     use_gaussian_depth=True, knn_idx=None, triangle_scale=2.0, return_gaussian_idx=False):
    """compute_level_surface_points_from_camera_fast for one view (sugar_scene/sugar_model.py:1848-2083; driver loop:
    sugar_extractors/coarse_mesh.py:246-327).

    `cam`: namespace with viewmatrix / projmatrix / campos device tensors (the rasterizer's transposed matrices) and
    width, height, tanfovx, tanfovy (sugar_b200.steps.camera_from_scene).  `use_gaussian_depth` keeps the reference's
    flag name; True (the default here) renders the Gaussians' blended depth and searches the `knn_to_track` nearest
    Gaussians of every back-projected point; False z-buffers the splatted mesh (`triangle_scale`, 2 in the
    extraction) and takes the neighbours of the pixel's Gaussian from `knn_idx` (int64 [P,K], the model's
    knn.reset_neighbors(points, K)[1] table; required there).  Returns the dict of `level_surface_points` plus, per
    level, 'pixel_idx' (flat index of each valid ray's pixel) and 'gaussian_idx' (each valid ray's Gaussian: the
    nearest one on the blended-depth branch, pix_to_face // 2 on the mesh branch) when asked."""
    from . import knn
    from .diff_gaussian_rasterization import GaussianRasterizationSettings, GaussianRasterizer
    dev = points.device
    H, W = int(cam.height), int(cam.width)
    if not use_gaussian_depth:
        if knn_idx is None:
            raise ValueError("use_gaussian_depth=False takes the neighbours from the model's table: pass knn_idx "
                             "(knn.reset_neighbors(points, K)[1])")
        if knn_idx.dtype != torch.int64 or knn_idx.dim() != 2 or knn_idx.shape[0] != points.shape[0]:
            raise ValueError(f"knn_idx must be int64 [{points.shape[0]},K], got {knn_idx.dtype} {tuple(knn_idx.shape)}")
        if knn_idx.device != dev:
            raise ValueError(f"knn_idx on {knn_idx.device}, points on {dev}")
    with torch.no_grad():
        if use_gaussian_depth:
            # splatted depth (:1898-1909): colours = view-space z, background -1 marks uncovered pixels
            view = points @ cam.viewmatrix[:3, :3] + cam.viewmatrix[3, :3]
            st = GaussianRasterizationSettings(image_height=H, image_width=W, tanfovx=cam.tanfovx, tanfovy=cam.tanfovy,
                                               bg=-torch.ones(3, device=dev), scale_modifier=1.0,
                                               viewmatrix=cam.viewmatrix, projmatrix=cam.projmatrix, sh_degree=0,
                                               campos=cam.campos, prefiltered=False, debug=False)
            depth = GaussianRasterizer(st)(means3D=points, means2D=torch.zeros_like(points),
                                           opacities=strengths.view(-1, 1),
                                           colors_precomp=view[:, 2:].expand(-1, 3).contiguous(), scales=scaling,
                                           rotations=quaternions)[0][0]
        else:
            # splatted diamond mesh, nearest face per pixel (:1920-1928)
            from . import splatmesh
            verts, faces = splatmesh.splat_mesh(points, scaling, quaternions, cam, triangle_scale=triangle_scale)
            depth, pix_to_face = splatmesh.rasterize_mesh(verts, faces, cam)
        no_depth = depth < 0.0                                                       # :1929
        depth = torch.where(no_depth, depth.max() * 1.05, depth)                     # :1930
        # back-projection of the covered pixels (:1932-1959) in the rasterizer's pixel convention
        # (ndc2Pix, auxiliary.h:41-44: pixel = ((ndc + 1) S - 1) / 2)
        keep = (~no_depth).view(-1).nonzero()[:, 0]
        if n_surface_points != -1 and n_surface_points < keep.numel():               # :1952-1958
            keep = keep[torch.randperm(keep.numel(), device=dev, generator=generator)[:n_surface_points]]
        py, px = (keep // W).float(), (keep % W).float()
        z = depth.view(-1)[keep]
        xv = ((2.0 * px + 1.0) / W - 1.0) * cam.tanfovx * z
        yv = ((2.0 * py + 1.0) / H - 1.0) * cam.tanfovy * z
        Rt, t = cam.viewmatrix[:3, :3], cam.viewmatrix[3, :3]                        # p_view = p_world @ Rt + t
        world = (torch.stack([xv, yv, z], dim=1) - t) @ Rt.transpose(0, 1)
        if use_gaussian_depth:
            # the K Gaussians around every point (:1962-1964)
            closest = knn.knn_points(world, points, knn_to_track)[1]
            gaussian_idx = closest[:, 0]
        else:
            # the pixel's Gaussian and its neighbours from the model's table (:1965-1968)
            gaussian_idx = pix_to_face.view(-1)[keep] // 2
            closest = knn_idx[gaussian_idx]
    out = level_surface_points(world, cam.campos, closest, points, scaling, quaternions, strengths,
                               surface_levels=surface_levels, n_points_in_range=n_points_in_range,
                               range_size=range_size, density_factor=density_factor, return_normals=return_normals)
    for res in out.values():
        if return_pixel_idx:
            res["pixel_idx"] = keep[res["valid"]]
        if return_gaussian_idx:
            res["gaussian_idx"] = gaussian_idx[res["valid"]]                        # :2048-2049
    return out
