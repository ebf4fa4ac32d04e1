"""The trainers' iteration schedules over this package's steps and optimizer.

    opt = train_coarse(raw, views, knn_idx, mode="sdf", spatial_extent=extent)     # coarse_sdf.py / coarse_density.py
    opt = train_refined(raw, mesh, views, spatial_lr_scale=refine_spatial_lr_scale(n_vertices, extent))   # refine.py

`train_coarse` is the `initialize_from_trained_3dgs=True` path of the coarse trainers (coarse_sdf.py:466-800,
coarse_density.py:475-815), where densification is off (coarse_sdf.py:71-73) and the SH degree stays at 3.  Each
iteration `it`:

    1. a CPU randperm of the views at the start of each epoch
    2. the points group's learning rate from the exponential schedule
    3. when it - 1 is in prune_at: prune the Gaussians with strength < prune_threshold (Densifier.prune_points), and
       reset the K-NN table if it > regularize_from                                        coarse_sdf.py:486-499
    4. K-NN reset when it > regularize_from and (it == regularize_from + 1 or it % reset_neighbors_every == 0)
                                                                                           :554-561
    5. it > sdf_from (and > regularize_from): steps.coarse_sdf_step / coarse_density_step, which run the backward;
       otherwise the RGB render, the photometric loss, plus entropy_factor * the mean binary entropy of the visible
       Gaussians' strengths when entropy_window[0] < it < entropy_window[1] (:538-551), and the backward
    6. optimizer.step(), zero_grad(set_to_none=True)

The reference starts its trained-3DGS runs at iteration 7000 (coarse_sdf.py:476-477); `first_iteration=7000` does the
same, the default 1 runs the whole schedule.  `train_refined` is refine.py:518-850: steps.refine_step with the SH
degree min(3, (it - 1) // sh_warmup_every) (the warm-up, :849-851), then the optimizer.

`train_3dgs` is the vanilla 3DGS trainer SuGaR starts from (gaussian_splatting/train.py:51-128), from an SfM point
cloud (gsply.read_sfm_points) through `init_from_points` (create_from_pcd), with `spatial_extent` =
mcubes.nerfpp_radius of the camera centres.  Each iteration: the position lr, the SH degree (gs_phase), a view popped
at random from a refilled stack, the background, the render, (1 - 0.2) L1 + 0.2 (1 - SSIM) and its backward, then per
gs_phase the densification statistics, densify-and-prune (Densifier(rotation="vanilla"), min opacity 0.005), the
opacity reset and the optimizer step, which the reference skips at the last iteration.  Its model is what
gsply.save_gaussians_ply writes as point_cloud/iteration_N/point_cloud.ply.  SuGaR's coarse trainers start from
such a file at iteration 7000:

    raw = gsply.load_gaussians_ply("point_cloud/iteration_7000/point_cloud.ply")
    train_coarse(raw, views, knn.reset_neighbors(raw["points"].detach())[1], spatial_extent=extent, first_iteration=7000)

`views` is a sequence of (cam, gt_rgb [3,H,W]) with `cam` from steps.camera_from_scene.  Both functions update `raw`
in place and return the optimizer (a SugarOptimizer; its state_dict() and raw are a checkpoint; pass one in as
`optimizer=` to reach it during the loop or to resume).  `on_iteration(it, loss, events)` is called after each
optimizer step with the loss as a device tensor and `events`, the dict that coarse_phase / refine_phase return.
Nothing is read back to the host beyond what the reference reads: the prune's scan and the sampled-Gaussian counts
the steps read.  `generator` (a CPU torch.Generator, or None for the default one) draws the view order; the SDF
samples come from the default CUDA generator, as in the reference.

`init_refined_from_mesh` builds refine.py's starting model from an extracted mesh (SuGaR's bound constructor), the
(raw, mesh) pair train_refined takes.
"""
import random

import numpy as np
import torch

from . import knn, steps
from .densify import Densifier
from .optim import SugarOptimizer, group_table


def coarse_phase(it, regularize_from=7000, entropy_window=(7000, 9000), prune_at=(9000,), reset_neighbors_every=500,
                 sdf_from=9000):
    """-> the coarse trainers' decisions at iteration `it` (>= 1), as a dict: "sh_degree" (always 3), and "prune",
    "reset_neighbors", "entropy", "sdf" present (True) when they happen.  A pure function of the schedule."""
    ev = {"sh_degree": 3}
    prune = (it - 1) in prune_at
    if prune:
        ev["prune"] = True
    if (prune and it >= regularize_from + 1) or \
            (it > regularize_from and (it == regularize_from + 1 or it % reset_neighbors_every == 0)):
        ev["reset_neighbors"] = True
    if entropy_window[0] < it < entropy_window[1]:
        ev["entropy"] = True
    if it > regularize_from and it > sdf_from:
        ev["sdf"] = True
    return ev


def refine_sh_degree(it, sh_warmup_every=1000):
    """The refinement's SH degree at iteration `it` (>= 1): 0 at first, one more every sh_warmup_every, at most 3."""
    return min(3, (it - 1) // sh_warmup_every)


def refine_phase(it, sh_warmup_every=1000):
    """-> the refinement's events at iteration `it`: {"sh_degree": refine_sh_degree(it)}."""
    return {"sh_degree": refine_sh_degree(it, sh_warmup_every)}


def refine_spatial_lr_scale(n_vertices_in_fg, spatial_extent=None, fg_bbox=None):
    """refine.py:452-459: 10 * bbox_radius / sqrt(n_vertices_in_fg), bbox_radius half the diagonal of `fg_bbox`
    ((min xyz, max xyz)) when given, else the cameras' spatial extent (mcubes.camera_spatial_extent).  The square root
    and the bounding-box norm are float32, as the reference's tensors compute them."""
    if fg_bbox is not None:
        lo, hi = fg_bbox
        bbox_radius = ((torch.tensor(hi) - torch.tensor(lo)).norm(dim=-1) / 2.0).item()
    elif spatial_extent is not None:
        bbox_radius = spatial_extent
    else:
        raise ValueError("refine_spatial_lr_scale needs spatial_extent or fg_bbox")
    return 10.0 * bbox_radius / torch.tensor(n_vertices_in_fg).pow(1 / 2).item()


def entropy_loss(strengths, visible):
    """Mean of -o log(o + 1e-10) - (1 - o) log(1 - o + 1e-10) over the visible Gaussians' strengths o, without a host
    read: a masked sum over the visible count (nan when none is visible, as the reference's empty mean)."""
    o = strengths.view(-1)
    h = -o * torch.log(o + 1e-10) - (1 - o) * torch.log(1 - o + 1e-10)
    return torch.where(visible, h, torch.zeros_like(h)).sum() / visible.sum()


def _optimizer(optimizer, raw, spatial_lr_scale, bound):
    """A new SugarOptimizer over `raw`, or the caller's after checking that its groups hold raw's tensors."""
    if optimizer is None:
        return SugarOptimizer(raw, spatial_lr_scale=spatial_lr_scale, bound=bound)
    keys = {name: key for name, key, _ in group_table(1.0, bound)}
    if not isinstance(optimizer, SugarOptimizer) or len(optimizer.param_groups) != len(keys) or \
            any(g["params"][0] is not raw[keys[g["name"]]] for g in optimizer.param_groups):
        raise ValueError(f"optimizer must be a SugarOptimizer over raw's tensors (bound={bound})")
    return optimizer


def _epochs(n_views, generator):
    while True:
        yield from torch.randperm(n_views, generator=generator).tolist()


def train_coarse(raw, views, knn_idx, mode="sdf", spatial_extent=None, num_iterations=15_000, regularize_from=7000,
                 entropy_window=(7000, 9000), entropy_factor=0.1, prune_at=(9000,), prune_threshold=0.5,
                 reset_neighbors_every=500, sdf_from=9000, dssim_factor=0.2, n_samples=1_000_000, generator=None,
                 on_iteration=None, first_iteration=1, optimizer=None):
    """The coarse trainer's loop (see the module docstring).  `raw`: steps.activate's dict of leaf tensors (updated in
    place, replaced by the prune); `knn_idx` [P,K] the K-NN table of raw["points"]; `spatial_extent` the cameras'
    (mcubes.camera_spatial_extent): the points' learning-rate scale, the Densifier's scene extent and the SDF
    normalisation.  `optimizer`: a SugarOptimizer over `raw` to continue (one the caller keeps, e.g. to save its
    state_dict from on_iteration, or one loaded from a checkpoint with first_iteration after it); by default a new one.
    -> the SugarOptimizer."""
    if mode not in ("sdf", "density"):
        raise ValueError(f"mode must be 'sdf' or 'density', got {mode!r}")
    if spatial_extent is None or not spatial_extent > 0:
        raise ValueError(f"spatial_extent must be > 0 (mcubes.camera_spatial_extent), got {spatial_extent}")
    if len(views) == 0:
        raise ValueError("views is empty")
    if first_iteration < 1:
        raise ValueError(f"first_iteration must be >= 1, got {first_iteration}")
    if entropy_window[1] > max(sdf_from, regularize_from) + 1:
        raise ValueError(f"entropy_window {tuple(entropy_window)} overlaps the SDF phase (it > {sdf_from}): the "
                         "regularised steps do not add the entropy term")
    K = knn_idx.shape[1]
    ops = steps.ours_ops()
    optimizer = _optimizer(optimizer, raw, spatial_extent, bound=False)
    densifier = Densifier(raw, optimizer, scene_extent=spatial_extent)
    order = _epochs(len(views), generator)
    dev = raw["points"].device
    bg = torch.zeros(3, device=dev)
    for it in range(first_iteration, num_iterations + 1):
        cam, gt = views[next(order)]
        optimizer.update_learning_rate(it)
        ev = coarse_phase(it, regularize_from, entropy_window, prune_at, reset_neighbors_every, sdf_from)
        if "prune" in ev:
            densifier.prune_points(torch.sigmoid(raw["densities"].detach()).view(-1) < prune_threshold)
        if "reset_neighbors" in ev:
            knn_idx = knn.reset_neighbors(raw["points"].detach(), K)[1]
        if "sdf" in ev:
            if mode == "sdf":
                loss, _ = steps.coarse_sdf_step(raw, cam, gt, knn_idx, ops, n_samples=n_samples,
                                                spatial_extent=spatial_extent, dssim_factor=dssim_factor,
                                                fused_depth=True)
            else:
                loss, _ = steps.coarse_density_step(raw, cam, gt, knn_idx, ops, n_samples=n_samples,
                                                    dssim_factor=dssim_factor)
        else:
            a = steps.activate(raw)
            image, radii, _ = steps.render(ops, a, cam, bg, sh_deg=3)
            loss = steps.photometric_loss(ops, image, gt, dssim_factor)
            if "entropy" in ev:
                loss = loss + entropy_factor * entropy_loss(a.strengths, radii > 0)
            loss.backward()
            loss = loss.detach()
        optimizer.step()
        optimizer.zero_grad(set_to_none=True)
        if on_iteration is not None:
            on_iteration(it, loss, ev)
    return optimizer


def train_refined(raw, mesh, views, spatial_lr_scale, num_iterations=15_000, dssim_factor=0.2,
                  normal_consistency_factor=0.1, sh_warmup_every=1000, generator=None, on_iteration=None,
                  first_iteration=1, optimizer=None, laplacian_smoothing_factor=0.0,
                  laplacian_smoothing_method="uniform"):
    """The refinement's loop (see the module docstring).  `raw`: steps.refine_step's dict (verts, sh_dc, sh_rest,
    densities, scales [P,2], quaternions [P,2]; leaf tensors, updated in place); `mesh` as refine_step takes it (give it
    a `topology` to build the edge table once, a `laplacian_topology` for the Laplacian lists); `spatial_lr_scale` from
    refine_spatial_lr_scale; `first_iteration` and `optimizer` (a bound SugarOptimizer over `raw`) as train_coarse takes
    them; laplacian_smoothing_factor / _method as refine_step takes them (refine.py's switch, off by default).
    -> the SugarOptimizer (bound)."""
    if len(views) == 0:
        raise ValueError("views is empty")
    if not spatial_lr_scale > 0:
        raise ValueError(f"spatial_lr_scale must be > 0, got {spatial_lr_scale}")
    if first_iteration < 1:
        raise ValueError(f"first_iteration must be >= 1, got {first_iteration}")
    ops = steps.ours_ops()
    optimizer = _optimizer(optimizer, raw, spatial_lr_scale, bound=True)
    order = _epochs(len(views), generator)
    for it in range(first_iteration, num_iterations + 1):
        cam, gt = views[next(order)]
        optimizer.update_learning_rate(it)
        ev = refine_phase(it, sh_warmup_every)
        loss, _ = steps.refine_step(raw, mesh, cam, gt, ops, dssim_factor=dssim_factor,
                                    normal_consistency_factor=normal_consistency_factor, sh_deg=ev["sh_degree"],
                                    laplacian_smoothing_factor=laplacian_smoothing_factor,
                                    laplacian_smoothing_method=laplacian_smoothing_method)
        optimizer.step()
        optimizer.zero_grad(set_to_none=True)
        if on_iteration is not None:
            on_iteration(it, loss, ev)
    return optimizer


# OptimizationParams' defaults (gaussian_splatting/arguments/__init__.py:73-89) that the vanilla loop reads
GS_SCHEDULE = dict(densify_from_iter=500, densify_until_iter=15_000, densification_interval=100,
                   opacity_reset_interval=3000)
SH_C0 = 0.28209479177387814


def gs_phase(it, num_iterations=30_000, sh_degree=3, sh_every=1000, densify_from_iter=500, densify_until_iter=15_000,
             densification_interval=100, opacity_reset_interval=3000, white_background=False):
    """-> the vanilla trainer's decisions at iteration `it` (>= 1; gaussian_splatting/train.py:69-128), as a dict:
    "sh_degree" min(sh_degree, it // sh_every) (oneupSHdegree runs before the render when it % 1000 == 0), and present
    (True) when they happen: "stats" (it < densify_until_iter), "densify" (it > densify_from_iter and
    it % densification_interval == 0; then "size_threshold" is 20 when it > opacity_reset_interval, else None),
    "reset_opacity" (within the statistics window, it % opacity_reset_interval == 0, or it == densify_from_iter with a
    white background) and "step" (every iteration but the last).  A pure function of the schedule."""
    ev = {"sh_degree": min(sh_degree, it // sh_every)}
    if it < densify_until_iter:
        ev["stats"] = True
        if it > densify_from_iter and it % densification_interval == 0:
            ev["densify"] = True
            ev["size_threshold"] = 20 if it > opacity_reset_interval else None
        if it % opacity_reset_interval == 0 or (white_background and it == densify_from_iter):
            ev["reset_opacity"] = True
    if it < num_iterations:
        ev["step"] = True
    return ev


def init_from_points(points, colors, sh_degree=3):
    """GaussianModel.create_from_pcd (gaussian_model.py:124-147) -> steps.activate's raw dict of leaf tensors on
    points' device: points = the cloud as float32; scales = log(sqrt(clamp_min(dist_cuda2, 1e-7))) on all three axes;
    quaternions (1, 0, 0, 0); densities logit(0.1); sh_dc = RGB2SH(colors) [P,1,3]; sh_rest zeros
    [P,(sh_degree+1)^2-1,3].  `points` [P,3] a CUDA tensor, `colors` [P,3] in [0, 1] (gsply.read_sfm_points)."""
    xyz = points.float()
    dev = xyz.device
    color = (torch.as_tensor(colors).float().to(dev) - 0.5) / SH_C0
    P = xyz.shape[0]
    features = torch.zeros((P, 3, (sh_degree + 1) ** 2), device=dev)
    features[:, :3, 0] = color
    dist2 = torch.clamp_min(knn.dist_cuda2(xyz), 0.0000001)
    scales = torch.log(torch.sqrt(dist2))[..., None].repeat(1, 3)
    rots = torch.zeros((P, 4), device=dev)
    rots[:, 0] = 1
    opacity = 0.1 * torch.ones((P, 1), dtype=torch.float, device=dev)
    densities = torch.log(opacity / (1 - opacity))        # inverse_sigmoid
    leaf = lambda t: t.contiguous().requires_grad_(True)
    return dict(points=leaf(xyz.detach().clone()), sh_dc=leaf(features[:, :, 0:1].transpose(1, 2)),
                sh_rest=leaf(features[:, :, 1:].transpose(1, 2)), densities=leaf(densities), scales=leaf(scales),
                quaternions=leaf(rots))


# surface_triangle_circle_radius of SuGaR's constructor (sugar_model.py:172-212), float64 as numpy computes it
CIRCLE_RADIUS = {1: 1.0 / 2.0 / np.sqrt(3.0), 3: 1.0 / 2.0 / (np.sqrt(3.0) + 1.0), 4: 1.0 / (4.0 * np.sqrt(3.0)),
                 6: 1.0 / (4.0 + 2.0 * np.sqrt(3.0))}


def init_refined_from_mesh(verts, faces, vertex_colors, n_gaussians_per_surface_triangle, thickness, sh_degree=3):
    """The refined model bound to a mesh, as SuGaR's constructor builds it for refine.py (sugar_model.py:149-361,
    learning positions, opacities and scales) -> (raw, mesh): `raw` refine_step's dict of float32 leaf tensors on the
    vertices' device, `mesh` checkpoint.mesh_namespace's (faces int64, bary, thickness, n, topology).

    verts [V,3] (rounded to float32), faces [F,3] integer, vertex_colors [V,3] in [0, 1] (mcubes.read_mesh_ply's uint8
    / 255); n Gaussians per face, 1, 3, 4 or 6 (ValueError otherwise); thickness the camera extent / 1e6 in the
    reference.  In its float32 operation order: scales = log(clamp_min(min edge length * circle radius, 1e-7)) on
    both in-plane axes of the face's n Gaussians; the complex numbers (1, 0); densities logit(0.1); sh_dc =
    RGB2SH(the barycentric mix of the face's vertex colours); sh_rest zeros [P,(sh_degree+1)^2-1,3]."""
    from . import meshbind
    from .checkpoint import mesh_namespace
    n = n_gaussians_per_surface_triangle
    if n not in CIRCLE_RADIUS:
        raise ValueError(f"n_gaussians_per_surface_triangle must be 1, 3, 4 or 6, got {n!r}")
    points = torch.as_tensor(verts).float()
    dev = points.device
    faces = torch.as_tensor(faces).to(dev)
    if faces.dim() != 2 or faces.shape[1] != 3 or faces.dtype.is_floating_point:
        raise ValueError(f"faces must be an integer [F,3] tensor, got {faces.dtype} {tuple(faces.shape)}")
    colors_v = torch.as_tensor(vertex_colors).float().to(dev)
    F, P = faces.shape[0], faces.shape[0] * n
    bary = meshbind.bary_coords(n, dev)[..., None]                     # [n,3,1]
    colors = (colors_v[faces][:, None] * bary[None]).sum(dim=-2).reshape(-1, 3)
    fv = points[faces]
    scales = (fv - fv[:, [1, 2, 0]]).norm(dim=-1).min(dim=-1)[0] * CIRCLE_RADIUS[n]
    scales = scales.clamp_min(0.0000001).reshape(F, -1, 1).expand(-1, n, 2).clone().reshape(-1, 2)
    complex_numbers = torch.zeros(P, 2, device=dev)
    complex_numbers[:, 0] = 1.0
    opacity = 0.1 * torch.ones((P, 1), dtype=torch.float, device=dev)
    leaf = lambda t: t.contiguous().requires_grad_(True)
    raw = dict(verts=leaf(points.detach().clone()), densities=leaf(torch.log(opacity / (1 - opacity))),
               scales=leaf(torch.log(scales)), quaternions=leaf(complex_numbers),
               sh_dc=leaf(((colors - 0.5) / SH_C0).unsqueeze(dim=1)),
               sh_rest=leaf(torch.zeros(P, (sh_degree + 1) ** 2 - 1, 3, device=dev)))
    return raw, mesh_namespace(faces, n, thickness, points.shape[0])


def train_3dgs(raw, views, spatial_extent, num_iterations=30_000, sh_degree=3, sh_every=1000,
               densify_from_iter=500, densify_until_iter=15_000, densification_interval=100,
               opacity_reset_interval=3000, densify_grad_threshold=0.0002, percent_dense=0.01, lambda_dssim=0.2,
               white_background=False, random_background=False, rng=None, generator=None, on_iteration=None,
               first_iteration=1, optimizer=None):
    """The vanilla 3DGS trainer's loop (see the module docstring).  `raw`: init_from_points' (or
    gsply.load_gaussians_ply's) dict of leaf tensors, updated in place and replaced by densification; `views`:
    (cam, gt_rgb [3,H,W]) pairs; `spatial_extent`: mcubes.nerfpp_radius of the camera centres, the position lr scale
    and the densifier's extent.  `rng`: the random.Random that pops the views (the reference's module-level randint;
    default a new Random(0)); `generator`: the CUDA generator of the split's normal draw (None: the default one, as in
    the reference), which also draws random backgrounds.  `optimizer`: a SugarOptimizer over raw (its six groups and
    learning rates are GaussianModel.training_setup's) to continue; by default a new one.  on_iteration(it, loss,
    events) gets the loss as a device tensor and gs_phase's events.  Nothing is read back to the host but the
    Densifier's one read per densification.  -> the SugarOptimizer."""
    if spatial_extent is None or not spatial_extent > 0:
        raise ValueError(f"spatial_extent must be > 0 (mcubes.nerfpp_radius), got {spatial_extent}")
    if len(views) == 0:
        raise ValueError("views is empty")
    if first_iteration < 1:
        raise ValueError(f"first_iteration must be >= 1, got {first_iteration}")
    M = raw["sh_dc"].shape[1] + raw["sh_rest"].shape[1]
    if M < (sh_degree + 1) ** 2:
        raise ValueError(f"raw holds {M} SH coefficients, sh_degree {sh_degree} needs {(sh_degree + 1) ** 2}")
    rng = random.Random(0) if rng is None else rng
    ops = steps.ours_ops()
    optimizer = _optimizer(optimizer, raw, spatial_extent, bound=False)
    densifier = Densifier(raw, optimizer, scene_extent=spatial_extent, percent_dense=percent_dense,
                          rotation="vanilla")
    dev = raw["points"].device
    background = torch.full((3,), 1.0 if white_background else 0.0, dtype=torch.float32, device=dev)
    stack = []
    for it in range(first_iteration, num_iterations + 1):
        optimizer.update_learning_rate(it)
        ev = gs_phase(it, num_iterations, sh_degree, sh_every, densify_from_iter, densify_until_iter,
                      densification_interval, opacity_reset_interval, white_background)
        if not stack:
            stack = list(range(len(views)))
        cam, gt = views[stack.pop(rng.randint(0, len(stack) - 1))]
        bg = torch.rand((3,), device=dev, generator=generator) if random_background else background
        a = steps.activate(raw)
        image, radii, viewspace = steps.render(ops, a, cam, bg, sh_deg=ev["sh_degree"])
        loss = ops.l1_dssim(image, gt, lambda_dssim)
        loss.backward()
        loss = loss.detach()
        with torch.no_grad():
            if "stats" in ev:
                densifier.update_densification_stats(viewspace, radii, radii > 0)
                if "densify" in ev:
                    densifier.densify_and_prune(densify_grad_threshold, 0.005, spatial_extent, ev["size_threshold"],
                                                generator=generator)
                if "reset_opacity" in ev:
                    densifier.reset_opacity()
            if "step" in ev:
                optimizer.step()
                optimizer.zero_grad(set_to_none=True)
        if on_iteration is not None:
            on_iteration(it, loss, ev)
    return optimizer
