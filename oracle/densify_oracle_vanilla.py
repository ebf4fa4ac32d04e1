"""Vanilla 3DGS's densification (gaussian_splatting/scene/gaussian_model.py:273-410) restated as a torch program
that runs on any device, over densify_oracle.py's state (params, moments, stats).

GaussianModel and SuGaRDensifier are the same program statement for statement: densify_and_prune takes grads =
accum / denom with NaN -> 0, clones, then splits over the grown set with the clones' gradients padded by 0, then
prunes; densification_postfix resets xyz_gradient_accum, denom and max_radii2D to zeros after each append, so the
screen-size clause compares zeros, as in SuGaR; prune_points and cat_tensors_to_optimizer carry and zero the Adam
moments as SuGaRDensifier's do; reset_opacity is inverse_sigmoid(min(sigmoid(opacity), 0.01)) with that group's
moments zeroed.  The one difference is the split's rotation: build_rotation (utils/general_utils.py:78-99) of the RAW
quaternion, restated below, where SuGaR takes pytorch3d's quaternion_to_matrix of the normalised one.
"""
import torch

from oracle import densify_oracle as do

prune_points, reset_opacity, update_stats, zero_stats = do.prune_points, do.reset_opacity, do.update_stats, do.zero_stats


def build_rotation(r):
    """general_utils.build_rotation: one torch op per arithmetic operation, left to right, no epsilon."""
    norm = torch.sqrt(r[:, 0] * r[:, 0] + r[:, 1] * r[:, 1] + r[:, 2] * r[:, 2] + r[:, 3] * r[:, 3])
    q = r / norm[:, None]
    R = torch.zeros((q.size(0), 3, 3), device=r.device)
    r, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    R[:, 0, 0] = 1 - 2 * (y * y + z * z)
    R[:, 0, 1] = 2 * (x * y - r * z)
    R[:, 0, 2] = 2 * (x * z + r * y)
    R[:, 1, 0] = 2 * (x * y + r * z)
    R[:, 1, 1] = 1 - 2 * (x * x + z * z)
    R[:, 1, 2] = 2 * (y * z - r * x)
    R[:, 2, 0] = 2 * (x * z - r * y)
    R[:, 2, 1] = 2 * (y * z + r * x)
    R[:, 2, 2] = 1 - 2 * (x * x + y * y)
    return R


def densify_and_prune(params, moments, stats, max_grad, min_opacity, extent, max_screen_size, percent_dense=0.01,
                      generator=None):
    """GaussianModel.densify_and_prune.  -> (params, moments, stats, info) as densify_oracle.densify_and_prune."""
    dev = params["points"].device
    grads = stats["accum"] / stats["denom"]
    grads[grads.isnan()] = 0.0

    # densify_and_clone
    clone = torch.where(torch.norm(grads, dim=-1) >= max_grad, True, False)
    clone = torch.logical_and(clone, torch.max(torch.exp(params["scales"]), dim=1).values <= percent_dense * extent)
    params, moments, stats = do._append(params, moments, {k: v[clone] for k, v in params.items()})

    # densify_and_split, N = 2
    n = params["points"].shape[0]
    padded = torch.zeros((n,), device=dev)
    padded[:grads.shape[0]] = grads.squeeze()
    split = torch.where(padded >= max_grad, True, False)
    scaling = torch.exp(params["scales"])
    split = torch.logical_and(split, torch.max(scaling, dim=1).values > percent_dense * extent)
    stds = scaling[split].repeat(2, 1)
    samples = torch.normal(mean=torch.zeros((stds.size(0), 3), device=dev), std=stds, generator=generator)
    rots = build_rotation(params["quaternions"][split]).repeat(2, 1, 1)
    new = {"points": torch.bmm(rots, samples.unsqueeze(-1)).squeeze(-1) + params["points"][split].repeat(2, 1),
           "scales": torch.log(scaling[split].repeat(2, 1) / (0.8 * 2))}
    for k in ("densities", "quaternions"):
        new[k] = params[k][split].repeat(2, 1)
    for k in ("sh_dc", "sh_rest"):
        new[k] = params[k][split].repeat(2, 1, 1)
    params, moments, stats = do._append(params, moments, new)
    S = int(split.sum())
    params, moments, stats = do._select(params, moments, stats,
                                        ~torch.cat((split, torch.zeros(2 * S, device=dev, dtype=torch.bool))))

    prune = (torch.sigmoid(params["densities"].view(-1, 1)) < min_opacity).squeeze()
    if max_screen_size:
        big_vs = stats["max_radii"] > max_screen_size
        big_ws = torch.exp(params["scales"]).max(dim=1).values > 0.1 * extent
        prune = torch.logical_or(torch.logical_or(prune, big_vs), big_ws)
    params, moments, stats = do._select(params, moments, stats, ~prune)
    return params, moments, stats, {"clone": clone, "split": split, "prune": prune, "samples": samples}
