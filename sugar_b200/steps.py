"""The trainers' per-iteration work around the hot path, composed from this package's operators.

`coarse_sdf_step` follows the regularised phase of the reference's coarse training loop
(sugar_trainers/coarse_sdf.py:506-716, iteration > 9000, the file's default switches):

    1. RGB render of the view                                   coarse_sdf.py:506-536  (render_image_gaussian_rasterizer)
    2. depth render: colours = view-space z, background = max z  :578-590  (backpropagate_gradients_through_depth=True)
    3. Gaussians close to the rendered surface (no grad)         :603-620  (sample_only_in_gaussians_close_to_surface)
    4. 1M samples inside those Gaussians                         :622-629  (sample_points_in_gaussians, scale 1.5)
    5. density / SDF field at the samples, K = 16 neighbours     :631-639  (get_field_values, 'sdf' mode, 'average' beta)
    6. SDF estimation loss against the depth map                 :641-668
    7. "better normal" loss                                      :688-716
    8. one backward through all of it

`coarse_density_step` is the same phase of the other coarse trainer (sugar_trainers/coarse_density.py, the
`-r density` choice of train.py): no depth render, and the density estimation loss in place of steps 2-6.

`refine_step` is the refinement loop's render (sugar_trainers/refine.py) for Gaussians bound to a mesh:
barycentric centres, flat scales and face-normal-aligned rotations (sugar_model.py:384-398, 415-479, see
sugar_b200/meshbind.py) followed by the RGB render and one backward.

The operators are passed in as an `ops` namespace so that bench.py can time the same recipe over this package's
fused kernels and over the reference's own building blocks (its CUDA rasterizer build + its PyTorch op chain):

    ops.rasterizer            module exposing GaussianRasterizationSettings / GaussianRasterizer
    ops.colors(points, sh, campos, sh_deg) -> colors_precomp or None (None: pass `shs` to the rasterizer)
    ops.field_values(x, nbr_idx, points, scaling, quaternions, strengths, **kw) -> dict
    ops.better_normal_loss(x, idx, nbr_idx, points, scaling, quaternions, nbr_opacity) -> [N]
    ops.density_estimation_loss(x, idx, nbr_idx, points, scaling, quaternions, strengths, density_factor=,
                                return_closest_gaussian_opacities=True) -> ([N], [N,K])   (coarse_density_step)
    ops.l1_dssim(pred, gt, dssim_factor) -> scalar   (only called with dssim_factor > 0)
    ops.mesh_normal_consistency(verts, faces, topology) -> scalar   (only called with normal_consistency_factor > 0)
    ops.rasterize_with_depth   sugar_b200.depth.rasterize_with_depth (only called with fused_depth=True; the
                               reference has no counterpart)

The photometric term is plain L1 by default (dssim_factor=0.0, what bench.py times); dssim_factor=0.2 gives the
trainers' (1 - 0.2) L1 + 0.2 (1 - SSIM) (coarse_sdf.py:101-103, 452-457, refine.py:103-105, 499-504).  What is NOT
reproduced: the camera is this package's pinhole convention (scenes.py) rather than pytorch3d's.
"""
import math
from types import SimpleNamespace

import torch


def activate(raw):
    """SuGaR's parameter activations (sugar_model.py:400-479, unbound model): strengths = sigmoid(all_densities),
    scaling = exp(_scales), quaternions = normalize(_quaternions), sh = cat(dc, rest)."""
    return SimpleNamespace(points=raw["points"], strengths=torch.sigmoid(raw["densities"]).view(-1, 1),
                           scaling=torch.exp(raw["scales"]),
                           quaternions=torch.nn.functional.normalize(raw["quaternions"], dim=-1),
                           sh=torch.cat([raw["sh_dc"], raw["sh_rest"]], dim=1))


def world_to_view(points, viewmatrix):
    """Row-vector convention: `viewmatrix` is the transposed world->view matrix (sugar_model.py:2149-2152)."""
    return points @ viewmatrix[:3, :3] + viewmatrix[3, :3]


def depth_lookup(depth, points_world, projmatrix):
    """SuGaR.get_points_depth_in_depth_map (sugar_model.py:1318-1333): bilinear lookup of the rendered depth at
    the points' projections, border padding.  NDC of the rasterizer (`ndc2Pix`, auxiliary.h:41-44: pixel =
    ((ndc + 1) S - 1) / 2) is grid_sample's own coordinate with align_corners=False."""
    hom = points_world @ projmatrix[:3, :] + projmatrix[3, :]
    ndc = hom[:, :2] / (hom[:, 3:4] + 1e-7)
    return torch.nn.functional.grid_sample(depth[None, None], ndc.view(1, -1, 1, 2), mode="bilinear",
                                           padding_mode="border", align_corners=False)[0, 0, :, 0]


def quaternion_apply_inverse(q, v):
    """quaternion_apply(quaternion_invert(q), v) for unit q (coarse_sdf.py:611): R(q)^T v."""
    r, i, j, k = torch.unbind(q, -1)
    two_s = 2.0 / (q * q).sum(-1)
    R = torch.stack((1 - two_s * (j * j + k * k), two_s * (i * j - k * r), two_s * (i * k + j * r),
                     two_s * (i * j + k * r), 1 - two_s * (i * i + k * k), two_s * (j * k - i * r),
                     two_s * (i * k - j * r), two_s * (j * k + i * r), 1 - two_s * (i * i + j * j)), -1)
    return (R.reshape(q.shape[:-1] + (3, 3)).transpose(-1, -2) @ v[..., None])[..., 0]


def render(ops, a, cam, bg, sh_deg, point_colors=None):
    """One rasterizer call in the trainers' form (sugar_model.py:2165-2278)."""
    R = ops.rasterizer
    st = R.GaussianRasterizationSettings(image_height=cam.height, image_width=cam.width, tanfovx=cam.tanfovx,
                                         tanfovy=cam.tanfovy, bg=bg, scale_modifier=1.0, viewmatrix=cam.viewmatrix,
                                         projmatrix=cam.projmatrix, sh_degree=sh_deg, campos=cam.campos,
                                         prefiltered=False, debug=False)
    means2D = torch.zeros_like(a.points, requires_grad=True)
    if point_colors is None:
        point_colors = ops.colors(a.points, a.sh, cam.campos, sh_deg)
    kw = dict(colors_precomp=point_colors) if point_colors is not None else dict(shs=a.sh)
    image, radii = R.GaussianRasterizer(st)(means3D=a.points, means2D=means2D, opacities=a.strengths, scales=a.scaling,
                                            rotations=a.quaternions, **kw)
    return image, radii, means2D


def render_with_depth(ops, a, cam, bg, sh_deg, point_values, depth_bg):
    """`render` and the depth render of the same view in one call: ops.rasterize_with_depth, colours as `render`
    picks them, `point_values` [P] blended over `depth_bg`.  -> (image, depth [H,W], radii)."""
    st = ops.rasterizer.GaussianRasterizationSettings(
        image_height=cam.height, image_width=cam.width, tanfovx=cam.tanfovx, tanfovy=cam.tanfovy, bg=bg,
        scale_modifier=1.0, viewmatrix=cam.viewmatrix, projmatrix=cam.projmatrix, sh_degree=sh_deg, campos=cam.campos,
        prefiltered=False, debug=False)
    means2D = torch.zeros_like(a.points, requires_grad=True)
    point_colors = ops.colors(a.points, a.sh, cam.campos, sh_deg)
    kw = dict(colors_precomp=point_colors) if point_colors is not None else dict(shs=a.sh)
    return ops.rasterize_with_depth(a.points, means2D, a.strengths, point_values, st, depth_bg, scales=a.scaling,
                                    rotations=a.quaternions, **kw)


def photometric_loss(ops, image, gt_rgb, dssim_factor):
    """Plain L1 when dssim_factor == 0, else the trainers' (1 - f) L1 + f (1 - SSIM) through ops.l1_dssim."""
    if dssim_factor == 0.0:
        return (image - gt_rgb).abs().mean()
    return ops.l1_dssim(image, gt_rgb, dssim_factor)


def coarse_sdf_step(raw, cam, gt_rgb, knn_idx, ops, n_samples=1_000_000, density_factor=1.0 / 16.0,
                    density_threshold=1.0, sdf_estimation_factor=0.2, sdf_better_normal_factor=0.2,
                    close_gaussian_threshold=2.0, sampling_scale_factor=1.5, spatial_extent=10.0, znear=0.01,
                    generator=None, backward=True, dssim_factor=0.0, fused_depth=False):
    """One regularised coarse-training iteration.  `raw`: dict of the model's raw parameter tensors (points,
    sh_dc [P,1,3], sh_rest [P,15,3], densities [P,1], scales [P,3], quaternions [P,4]); `cam`: namespace with
    viewmatrix / projmatrix / campos device tensors and width, height, tanfovx, tanfovy; `knn_idx` [P,16].
    fused_depth=True renders steps 1 and 2 with one ops.rasterize_with_depth call instead of two rasterizer calls:
    the same image, depth map and loss, one rasterization fewer."""
    from .field import sample_points_in_gaussians
    a = activate(raw)
    dev = a.points.device
    if fused_depth:
        if getattr(ops, "rasterize_with_depth", None) is None:
            raise ValueError("fused_depth=True needs ops.rasterize_with_depth")
        # 1. + 2. RGB and depth in one rasterizer call
        point_depth = world_to_view(a.points, cam.viewmatrix)[:, 2]
        max_depth = point_depth.max()
        image, depth, radii = render_with_depth(ops, a, cam, torch.zeros(3, device=dev), 3, point_depth,
                                                max_depth.detach())
        loss = photometric_loss(ops, image, gt_rgb, dssim_factor)
        vis = radii > 0
    else:
        # 1. RGB
        image, radii, viewspace = render(ops, a, cam, torch.zeros(3, device=dev), sh_deg=3)
        loss = photometric_loss(ops, image, gt_rgb, dssim_factor)
        vis = radii > 0
        # 2. depth, with gradient
        point_depth = world_to_view(a.points, cam.viewmatrix)[:, 2:].expand(-1, 3)
        max_depth = point_depth.max()
        depth = render(ops, a, cam, max_depth.detach() + torch.zeros(3, device=dev), sh_deg=0,
                       point_colors=point_depth)[0][0]
    # 3. which Gaussians sit on the rendered surface
    with torch.no_grad():
        to_cam = torch.nn.functional.normalize(cam.campos.view(1, 3) - a.points, dim=-1)
        centers_z = world_to_view(a.points, cam.viewmatrix)[:, 2]
        map_z = depth_lookup(depth, a.points, cam.projmatrix)
        std = (a.scaling * quaternion_apply_inverse(a.quaternions, to_cam)).norm(dim=-1)
        mask = vis & ((map_z - centers_z).abs() < close_gaussian_threshold * std)
    stats = {"visible": int(vis.sum()), "sampled_gaussians": int(mask.sum())}
    if stats["sampled_gaussians"] > 0:
        # 4. samples
        x, idx = sample_points_in_gaussians(a.points, a.scaling, a.quaternions, a.strengths, n_samples,
                                            sampling_scale_factor=sampling_scale_factor, mask=mask,
                                            probabilities_proportional_to_volume=False, generator=generator)
        nbr = knn_idx[idx]
        # 5. fields
        fields = ops.field_values(x, nbr, a.points, a.scaling, a.quaternions, a.strengths,
                                  density_factor=density_factor, density_threshold=density_threshold,
                                  return_sdf=True, return_closest_gaussian_opacities=True)
        # 6. SDF estimation from the depth map
        x_z = world_to_view(x, cam.viewmatrix)[:, 2]
        proj_mask = x_z > znear
        est = depth_lookup(depth, x[proj_mask], cam.projmatrix) - x_z[proj_mask]
        sdf_std = spatial_extent / 10.0
        est_loss = ((fields["sdf"][proj_mask] - est.abs()).abs() / sdf_std).clamp(max=10.0 * spatial_extent)
        loss = loss + sdf_estimation_factor * est_loss.mean()
        # 7. better normal
        nl = ops.better_normal_loss(x, idx, nbr, a.points, a.scaling, a.quaternions,
                                    fields["closest_gaussian_opacities"].detach())
        loss = loss + sdf_better_normal_factor * nl.mean()
    if backward:
        loss.backward()
    return loss.detach(), stats


def coarse_density_step(raw, cam, gt_rgb, knn_idx, ops, n_samples=1_000_000, density_factor=1.0,
                        sdf_estimation_factor=0.2, sdf_better_normal_factor=0.2, sampling_scale_factor=1.5,
                        generator=None, backward=True, dssim_factor=0.0):
    """One regularised iteration of the coarse_density trainer (sugar_trainers/coarse_density.py:510-730, iteration
    > 9000, the file's default switches: sdf_estimation_mode='density', use_projection_as_estimation=True,
    density_factor = 1, sdf_sampling_proportional_to_volume=False):

        1. RGB render of the view                                  :510-540
        2. visible Gaussians (radii > 0): the sampling mask        :574 (projection mode samples in all of them)
        3. n_samples inside them, uniformly per Gaussian, scale 1.5 :632-638
        4. density estimation loss, K = 16 neighbours              :642-656, 684-691 (ops.density_estimation_loss)
        5. "better normal" loss with the field's opacities         :702-730
        6. one backward through all of it

    Same arguments as coarse_sdf_step; no depth render.  Stats: visible and sampled_gaussians (the same Gaussians
    in projection mode)."""
    from .field import sample_points_in_gaussians
    a = activate(raw)
    dev = a.points.device
    image, radii, _ = render(ops, a, cam, torch.zeros(3, device=dev), sh_deg=3)
    loss = photometric_loss(ops, image, gt_rgb, dssim_factor)
    vis = radii > 0
    n_vis = int(vis.sum())
    stats = {"visible": n_vis, "sampled_gaussians": n_vis}
    if n_vis > 0:
        x, idx = sample_points_in_gaussians(a.points, a.scaling, a.quaternions, a.strengths, n_samples,
                                            sampling_scale_factor=sampling_scale_factor, mask=vis,
                                            probabilities_proportional_to_volume=False, generator=generator)
        nbr = knn_idx[idx]
        est, opac = ops.density_estimation_loss(x, idx, nbr, a.points, a.scaling, a.quaternions, a.strengths,
                                                density_factor=density_factor, return_closest_gaussian_opacities=True)
        loss = loss + sdf_estimation_factor * est.mean()
        nl = ops.better_normal_loss(x, idx, nbr, a.points, a.scaling, a.quaternions, opac.detach())
        loss = loss + sdf_better_normal_factor * nl.mean()
    if backward:
        loss.backward()
    return loss.detach(), stats


def refine_step(raw, mesh, cam, gt_rgb, ops, backward=True, dssim_factor=0.0, normal_consistency_factor=0.0, sh_deg=3):
    """One refinement iteration's render for mesh-bound Gaussians (sugar_trainers/refine.py; model properties
    sugar_model.py:384-398 points, :415-441 scaling, :443-479 quaternions).  `raw`: verts [V,3], sh_dc, sh_rest,
    densities [P,1], scales [P,2] (in-plane), quaternions [P,2] (the learned 2-D rotation as a complex number);
    `mesh`: faces [F,3] int64, bary [n,3,1], thickness, optionally `topology` (meshloss.mesh_topology of the faces,
    built once); P = F * n.  normal_consistency_factor > 0 adds the surface mesh's normal consistency
    (refine.py:775-783, 0.1 in the trainers) through ops.mesh_normal_consistency.  `sh_deg`: the SH degree rendered
    (the refinement's warm-up raises it from 0 to 3, train.refine_sh_degree)."""
    a = ops.bind_to_mesh(raw["verts"], mesh.faces, mesh.bary, raw["scales"], raw["quaternions"], mesh.thickness)
    b = SimpleNamespace(points=a.points, scaling=a.scaling, quaternions=a.quaternions,
                        strengths=torch.sigmoid(raw["densities"]).view(-1, 1),
                        sh=torch.cat([raw["sh_dc"], raw["sh_rest"]], dim=1))
    image, radii, _ = render(ops, b, cam, torch.zeros(3, device=b.points.device), sh_deg=sh_deg)
    loss = photometric_loss(ops, image, gt_rgb, dssim_factor)
    if normal_consistency_factor > 0.0:
        loss = loss + normal_consistency_factor * ops.mesh_normal_consistency(raw["verts"], mesh.faces,
                                                                              getattr(mesh, "topology", None))
    if backward:
        loss.backward()
    return loss.detach(), {"visible": int((radii > 0).sum())}


def camera_from_scene(sc, device):
    """scenes.Scene -> the namespace the steps take."""
    t = lambda v: torch.from_numpy(v).to(device)
    return SimpleNamespace(viewmatrix=t(sc.viewmatrix), projmatrix=t(sc.projmatrix), campos=t(sc.campos),
                           width=sc.width, height=sc.height, tanfovx=sc.tanfovx, tanfovy=sc.tanfovy)


def ours_ops():
    """This package's operators: in-kernel SH colours, fused field / normal-loss / density-estimation kernels, fused
    mesh binding, fused L1 + D-SSIM loss, fused mesh normal consistency, colour + depth in one rasterizer call."""
    from . import diff_gaussian_rasterization as dgr
    from . import depth, field, loss, meshbind, meshloss
    return SimpleNamespace(rasterizer=dgr, colors=lambda points, sh, campos, deg: None,
                           rasterize_with_depth=depth.rasterize_with_depth,
                           field_values=field.field_values, better_normal_loss=field.better_normal_loss,
                           density_estimation_loss=field.density_estimation_loss,
                           bind_to_mesh=meshbind.bind_to_mesh, l1_dssim=loss.l1_dssim_loss,
                           mesh_normal_consistency=meshloss.mesh_normal_consistency)
