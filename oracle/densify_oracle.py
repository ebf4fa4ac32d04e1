"""SuGaRDensifier (sugar_scene/sugar_densifier.py) restated as a torch program that runs on any device.

State, as sugar_b200.densify keeps it:
    params   {"points" [P,3], "densities" [P,1], "scales" [P,3] (log), "quaternions" [P,4], "sh_dc" [P,1,3],
              "sh_rest" [P,15,3]}: float32 raw parameters
    moments  {key: (exp_avg, exp_avg_sq)} for the keys that have Adam state (none before the first optimizer step)
    stats    {"accum" [P,1], "denom" [P,1], "max_radii" [P]}

The statements follow the reference's order, each with the same torch operation, so on one device every decision and
every copied value has the reference's bits:
  1. statistics for rows where `vis` is set: max_radii = max(max_radii, float(radii)), accum += |grad[:, :2]|,
     denom += 1;
  2. grads = accum / denom, NaN -> 0;
  3. clone rows with |grads| >= max_grad and max(exp(scales)) <= percent_dense * extent, appended in index order; the
     statistics are reset to zeros of the new size;
  4. split rows of the grown set with padded grads >= max_grad (clones pad with 0) and max scale > percent_dense *
     extent: S rows, samples = normal(0, std = scale[sel].repeat(2, 1)) (copy 0 of all S rows, then copy 1),
     children at R(q / |q|) sample + point with log(scale / 1.6) and the parent's other fields, appended; statistics
     reset again; then the S parents are removed;
  5. prune rows with sigmoid(densities) < min_opacity, and when max_screen_size is truthy also those with
     max_radii > max_screen_size (never: the statistics are zeros after step 4) or max scale > 0.1 * extent.
Appended rows start with zero moments; removed rows take theirs with them.
"""
import torch
import torch.nn.functional as F

KEYS = ("points", "densities", "scales", "quaternions", "sh_dc", "sh_rest")


def zero_stats(P, device):
    return {"accum": torch.zeros((P, 1), device=device), "denom": torch.zeros((P, 1), device=device),
            "max_radii": torch.zeros((P,), device=device)}


def update_stats(stats, grad_means2D, radii, vis):
    """Step 1, in place (boolean-mask reads and writes, as the reference)."""
    stats["max_radii"][vis] = torch.max(stats["max_radii"][vis], radii[vis])
    stats["accum"][vis] += torch.norm(grad_means2D[vis, :2], dim=-1, keepdim=True)
    stats["denom"][vis] += 1


def quaternion_to_matrix(q):
    """pytorch3d's quaternion_to_matrix (real part first)."""
    r, i, j, k = torch.unbind(q, -1)
    two_s = 2.0 / (q * q).sum(-1)
    o = torch.stack((1 - two_s * (j * j + k * k), two_s * (i * j - k * r), two_s * (i * k + j * r),
                     two_s * (i * j + k * r), 1 - two_s * (i * i + k * k), two_s * (j * k - i * r),
                     two_s * (i * k - j * r), two_s * (j * k + i * r), 1 - two_s * (i * i + j * j)), -1)
    return o.reshape(q.shape[:-1] + (3, 3))


def _select(params, moments, stats, keep):
    params = {k: v[keep] for k, v in params.items()}
    moments = {k: (a[keep], b[keep]) for k, (a, b) in moments.items()}
    stats = {k: v[keep] for k, v in stats.items()}
    return params, moments, stats


def _append(params, moments, new):
    P = params["points"].shape[0] + new["points"].shape[0]
    moments = {k: (torch.cat((a, torch.zeros_like(new[k]))), torch.cat((b, torch.zeros_like(new[k]))))
               for k, (a, b) in moments.items()}
    params = {k: torch.cat((v, new[k])) for k, v in params.items()}
    return params, moments, zero_stats(P, params["points"].device)


def prune_points(params, moments, stats, mask):
    """Keep the rows where ~mask."""
    return _select(params, moments, stats, ~mask)


def reset_opacity(params, moments):
    """densities = logit(min(sigmoid(densities), 0.01)); that group's moments are zeroed."""
    d = params["densities"]
    op = torch.sigmoid(d.view(-1, 1))
    v = torch.min(op, torch.ones_like(d.view(-1, 1)) * 0.01)
    params = dict(params, densities=torch.log(v / (1 - v)).view_as(d))
    if "densities" in moments:
        moments = dict(moments, densities=(torch.zeros_like(d), torch.zeros_like(d)))
    return params, moments


def densify_and_prune(params, moments, stats, max_grad, min_opacity, extent, max_screen_size, percent_dense=0.01,
                      generator=None):
    """Steps 2-5.  -> (params, moments, stats, info) with info the masks that decided: clone [P], split [P + n_clone],
    prune [P'']."""
    dev = params["points"].device
    grads = stats["accum"] / stats["denom"]
    grads[grads.isnan()] = 0.0

    clone = torch.where(torch.norm(grads, dim=-1) >= max_grad, True, False)
    clone = torch.logical_and(clone, torch.max(torch.exp(params["scales"]), dim=1).values <= percent_dense * extent)
    params, moments, stats = _append(params, moments, {k: v[clone] for k, v in params.items()})

    n = params["points"].shape[0]
    padded = torch.zeros((n,), device=dev)
    padded[:grads.shape[0]] = grads.squeeze()
    split = torch.where(padded >= max_grad, True, False)
    scaling = torch.exp(params["scales"])
    split = torch.logical_and(split, torch.max(scaling, dim=1).values > percent_dense * extent)
    stds = scaling[split].repeat(2, 1)
    samples = torch.normal(mean=torch.zeros((stds.size(0), 3), device=dev), std=stds, generator=generator)
    rots = quaternion_to_matrix(F.normalize(params["quaternions"], dim=-1)[split]).repeat(2, 1, 1)
    new = {"points": torch.bmm(rots, samples.unsqueeze(-1)).squeeze(-1) + params["points"][split].repeat(2, 1),
           "scales": torch.log(scaling[split].repeat(2, 1) / (0.8 * 2))}
    for k in ("densities", "quaternions"):
        new[k] = params[k][split].repeat(2, 1)
    for k in ("sh_dc", "sh_rest"):
        new[k] = params[k][split].repeat(2, 1, 1)
    params, moments, stats = _append(params, moments, new)
    S = int(split.sum())
    params, moments, stats = _select(params, moments, stats,
                                     ~torch.cat((split, torch.zeros(2 * S, device=dev, dtype=torch.bool))))

    prune = (torch.sigmoid(params["densities"].view(-1, 1)) < min_opacity).squeeze()
    if max_screen_size:
        big_vs = stats["max_radii"] > max_screen_size
        big_ws = torch.exp(params["scales"]).max(dim=1).values > 0.1 * extent
        prune = torch.logical_or(torch.logical_or(prune, big_vs), big_ws)
    params, moments, stats = _select(params, moments, stats, ~prune)
    return params, moments, stats, {"clone": clone, "split": split, "prune": prune, "samples": samples}
