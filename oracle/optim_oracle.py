"""SuGaROptimizer (sugar_scene/sugar_optimizer.py) and the trainers' per-iteration decisions restated, for the tests of
sugar_b200/optim.py and sugar_b200/train.py.

  - `optimizer_groups`: SuGaROptimizer's group list (:63-85) for a model that learns every parameter, as (name, raw
    key, lr); `OracleOptimizer` is that list in torch.optim.Adam(groups, lr=0.0, eps=1e-15) with update_learning_rate
    (:100-108).  The schedule function is sugar_b200.optim.expon_lr, which tests/golden/optim_expon_lr.npz holds to
    the reference's own values.
  - `coarse_events(iteration, ...)`: the coarse trainers' statements at one iteration, with the reference's switch
    names and conditions (coarse_sdf.py:486-499 prune, :538-551 entropy, :553-561 neighbour reset, :563 SDF phase;
    coarse_density.py has the same lines at :490-565).
  - `refine_sh_degrees(n, ...)`: the refinement's SH-levels counter run for n iterations (refine.py:540-560 render
    degree, :849-851 warm-up), not the closed form train.py uses.
  - `coarse_loop` / `refine_loop`: those loops in the reference's shape (epochs of a CPU randperm, an iteration
    counter, the decisions above) over this package's per-iteration steps and torch.optim.Adam; the prune is
    SuGaRDensifier's (sugar_densifier.py prune_points: index every group's tensor and Adam moments, re-key the state).
    `coarse_iteration` is one pass of the coarse loop's body, so a test can also run it from a given state.
"""
import torch

from sugar_b200 import knn, steps
from sugar_b200.optim import expon_lr


def optimizer_groups(spatial_lr_scale, bound=False, position_lr_init=0.00016, feature_lr=0.0025, opacity_lr=0.05,
                     scaling_lr=0.005, rotation_lr=0.001):
    """-> [(name, raw key, lr)] in the reference's order; a bound model's "points" are the mesh vertices."""
    l = [("points", "verts" if bound else "points", position_lr_init * spatial_lr_scale)]
    l = l + [("sh_coordinates_dc", "sh_dc", feature_lr), ("sh_coordinates_rest", "sh_rest", feature_lr / 20.0)]
    l = l + [("all_densities", "densities", opacity_lr)]
    l = l + [("scales", "scales", scaling_lr)]
    l = l + [("quaternions", "quaternions", rotation_lr)]
    return l


class OracleOptimizer:
    def __init__(self, raw, spatial_lr_scale, bound=False, position_lr_init=0.00016, position_lr_final=0.0000016,
                 position_lr_delay_mult=0.01, position_lr_max_steps=30_000, **lrs):
        groups = optimizer_groups(spatial_lr_scale, bound, position_lr_init=position_lr_init, **lrs)
        self.optimizer = torch.optim.Adam([{"params": [raw[k]], "lr": lr, "name": n} for n, k, lr in groups], lr=0.0,
                                          eps=1e-15)
        self.position_sheduler_func = expon_lr(lr_init=position_lr_init * spatial_lr_scale,
                                               lr_final=position_lr_final * spatial_lr_scale,
                                               lr_delay_mult=position_lr_delay_mult, max_steps=position_lr_max_steps)

    def update_learning_rate(self, iteration):
        lr = 0.
        for param_group in self.optimizer.param_groups:
            if param_group["name"] == "points":
                lr = self.position_sheduler_func(iteration)
                param_group["lr"] = lr
        return lr


def coarse_events(iteration, regularize_from=7000, start_entropy_regularization_from=7000,
                  end_entropy_regularization_at=9000, prune_low_opacity_gaussians_at=(9000,), reset_neighbors_every=500,
                  start_sdf_regularization_from=9000):
    """-> the list of what the coarse trainer does at `iteration`, in its order ("reset_neighbors" may appear after the
    prune and again in the regularisation block)."""
    regularize = True
    prune_when_starting_regularization = False
    enforce_entropy_regularization = True
    regularize_sdf = True
    start_reset_neighbors_from = regularize_from + 1
    out = []
    if (regularize and prune_when_starting_regularization and iteration == regularize_from + 1) or (
            (iteration - 1) in prune_low_opacity_gaussians_at):
        out.append("prune")
        if regularize and iteration >= start_reset_neighbors_from:
            out.append("reset_neighbors")
    if enforce_entropy_regularization and iteration > start_entropy_regularization_from and \
            iteration < end_entropy_regularization_at:
        out.append("entropy")
    if regularize and iteration > regularize_from:
        if (iteration >= start_reset_neighbors_from) and ((iteration == regularize_from + 1) or
                                                          (iteration % reset_neighbors_every == 0)):
            out.append("reset_neighbors")
        if regularize_sdf and iteration > start_sdf_regularization_from:
            out.append("sdf")
    return out


def refine_sh_degrees(num_iterations, sh_warmup_every=1000, sh_levels=4):
    """-> [the SH degree rendered at iteration 1, 2, ..., num_iterations]."""
    current_sh_levels = 1
    out = []
    for iteration in range(1, num_iterations + 1):
        out.append(current_sh_levels - 1)
        if (iteration > 0) and (current_sh_levels < sh_levels) and (iteration % sh_warmup_every == 0):
            current_sh_levels += 1
    return out


def prune_points(raw, optimizer, mask):
    """SuGaRDensifier.prune_points over `raw` (the unbound keys) and a torch Adam with one tensor per group."""
    valid = ~mask
    for group in optimizer.param_groups:
        old = group["params"][0]
        key = next(k for k, v in raw.items() if v is old)
        state = optimizer.state.get(old, None)
        new = torch.nn.Parameter(old[valid].requires_grad_(True))
        if state is not None:
            state["exp_avg"] = state["exp_avg"][valid]
            state["exp_avg_sq"] = state["exp_avg_sq"][valid]
            del optimizer.state[old]
            optimizer.state[new] = state
        group["params"][0] = new
        raw[key] = new


def coarse_iteration(raw, optimizer, knn_idx, cam, gt, events, mode, spatial_extent, entropy_factor, prune_threshold,
                     dssim_factor, n_samples, ops):
    """One iteration of the coarse loop with its decisions `events` (coarse_events) -> (loss, knn_idx)."""
    if "prune" in events:
        with torch.no_grad():
            prune_mask = (torch.sigmoid(raw["densities"]) < prune_threshold).squeeze()
        prune_points(raw, optimizer.optimizer, prune_mask)
    if "reset_neighbors" in events:
        knn_idx = knn.reset_neighbors(raw["points"].detach(), knn_idx.shape[1])[1]
    if "sdf" in events:
        step = steps.coarse_sdf_step if mode == "sdf" else steps.coarse_density_step
        kw = dict(spatial_extent=spatial_extent, fused_depth=True) if mode == "sdf" else {}
        loss, _ = step(raw, cam, gt, knn_idx, ops, n_samples=n_samples, dssim_factor=dssim_factor, **kw)
    else:
        a = steps.activate(raw)
        image, radii, _ = steps.render(ops, a, cam, torch.zeros(3, device=gt.device), sh_deg=3)
        loss = steps.photometric_loss(ops, image, gt, dssim_factor)
        if "entropy" in events:
            vis_opacities = a.strengths[radii > 0]
            loss = loss + entropy_factor * (
                - vis_opacities * torch.log(vis_opacities + 1e-10)
                - (1 - vis_opacities) * torch.log(1 - vis_opacities + 1e-10)).mean()
        loss.backward()
    optimizer.optimizer.step()
    optimizer.optimizer.zero_grad(set_to_none=True)
    return loss.detach(), knn_idx


def coarse_loop(raw, views, knn_idx, mode, spatial_extent, num_iterations, regularize_from, entropy_window,
                entropy_factor, prune_at, prune_threshold, reset_neighbors_every, sdf_from, dssim_factor, n_samples,
                on_iteration=None):
    """The coarse loop on `raw` (updated in place) -> the OracleOptimizer."""
    ops = steps.ours_ops()
    optimizer = OracleOptimizer(raw, spatial_lr_scale=spatial_extent)
    sched = dict(regularize_from=regularize_from, start_entropy_regularization_from=entropy_window[0],
                 end_entropy_regularization_at=entropy_window[1], prune_low_opacity_gaussians_at=prune_at,
                 reset_neighbors_every=reset_neighbors_every, start_sdf_regularization_from=sdf_from)
    iteration = 0
    for batch in range(9_999_999):
        if iteration >= num_iterations:
            break
        shuffled_idx = torch.randperm(len(views))
        for i in range(len(shuffled_idx)):
            iteration += 1
            optimizer.update_learning_rate(iteration)
            events = coarse_events(iteration, **sched)
            cam, gt = views[shuffled_idx[i].item()]
            loss, knn_idx = coarse_iteration(raw, optimizer, knn_idx, cam, gt, events, mode, spatial_extent,
                                             entropy_factor, prune_threshold, dssim_factor, n_samples, ops)
            if on_iteration is not None:
                on_iteration(iteration, loss, events)
            if iteration >= num_iterations:
                break
    return optimizer


def refine_loop(raw, mesh, views, spatial_lr_scale, num_iterations, dssim_factor, normal_consistency_factor,
                sh_warmup_every, on_iteration=None):
    """The refinement loop on `raw` (updated in place) -> the OracleOptimizer."""
    ops = steps.ours_ops()
    optimizer = OracleOptimizer(raw, spatial_lr_scale=spatial_lr_scale, bound=True)
    sh_levels = 4
    current_sh_levels = 1
    iteration = 0
    for batch in range(9_999_999):
        if iteration >= num_iterations:
            break
        shuffled_idx = torch.randperm(len(views))
        for i in range(len(shuffled_idx)):
            iteration += 1
            optimizer.update_learning_rate(iteration)
            cam, gt = views[shuffled_idx[i].item()]
            loss, _ = steps.refine_step(raw, mesh, cam, gt, ops, dssim_factor=dssim_factor,
                                        normal_consistency_factor=normal_consistency_factor,
                                        sh_deg=current_sh_levels - 1)
            optimizer.optimizer.step()
            optimizer.optimizer.zero_grad(set_to_none=True)
            if on_iteration is not None:
                on_iteration(iteration, loss, current_sh_levels - 1)
            if iteration >= num_iterations:
                break
            if (iteration > 0) and (current_sh_levels < sh_levels) and (iteration % sh_warmup_every == 0):
                current_sh_levels += 1
    return optimizer
