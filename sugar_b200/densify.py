"""Densification and pruning of the coarse model's Gaussians on the GPU (csrc/sgr_densify.cu).

A drop-in for the reference's SuGaRDensifier (sugar_scene/sugar_densifier.py) over this package's raw parameter dict
(`points, densities, scales, quaternions, sh_dc, sh_rest`, as steps.py uses it) and a torch optimizer with one tensor
per group (SuGaROptimizer's Adam):

    dens = Densifier(raw, optimizer, scene_extent=extent)
    dens.update_densification_stats(viewspace_points, radii, radii > 0)      # every step; no host synchronisation
    dens.densify_and_prune(max_grad, min_opacity, extent, max_screen_size)   # every 100 iterations
    dens.reset_opacity()                                                     # every 3000
    dens.prune_points(strengths < 0.5)                                       # once, when training from a 3DGS model
    knn_idx = knn.reset_neighbors(raw["points"].detach(), 16)[1]             # the K-NN table is stale after each

`raw` and the optimizer are updated in place: each parameter is replaced by a new tensor and the optimizer's groups and
state are re-keyed to it.  The decisions and copied values are the reference's bit for bit (oracle/densify_oracle.py
restates it); children's positions agree to a few ulps, the reference's bmm order being unspecified.  As in the
reference, `densify_and_prune` applies the screen-size clause only when its own `max_screen_size` argument is truthy,
and that clause compares statistics that the appends have reset to zero.

With `group` (a torch.distributed process group, one rank per GPU holding replicated parameters), `densify_and_prune`
sums accum and denom and takes the maximum of max_radii2D over the ranks before deciding, and the split's normals are
drawn on the group's first rank and broadcast, so every rank makes the same decisions.  The per-step statistics stay
local between densifications and are never part of the gradient exchange.

`rotation="vanilla"` makes it vanilla 3DGS's GaussianModel densification (gaussian_splatting/scene/gaussian_model.py:
273-410, as train.train_3dgs uses it).  Every statement there is SuGaRDensifier's except the split's rotation, which is
build_rotation of the raw quaternion (norm = sqrt(((r*r + x*x) + y*y) + z*z), no epsilon, a true division, then the
nine entries as written) instead of pytorch3d's quaternion_to_matrix of the normalised one; oracle/densify_oracle_vanilla.py
restates it.  Mesh-bound models are out of scope (the refinement never densifies).
"""
import numpy as np
import torch

from ._lib import (SGR_DENSIFY_COPY, SGR_DENSIFY_POINTS, SGR_DENSIFY_POINTS_VANILLA, SGR_DENSIFY_SCALES,
                   SGR_DENSIFY_ZERO_NEW, SgrDensifyColumn, SgrDensifyGates, check, lib, ptr, require_cuda, stream,
                   tensor)

KEYS = ("points", "densities", "scales", "quaternions", "sh_dc", "sh_rest")
# the split's R: quaternion_to_matrix / build_rotation
ROTATIONS = {"sugar": SGR_DENSIFY_POINTS, "vanilla": SGR_DENSIFY_POINTS_VANILLA}
INV_SPLIT = float(np.float32(1.0) / np.float32(0.8 * 2))   # torch's scalar division on CUDA: x * (1 / float(1.6))


def reduce_statistics(accum, denom, max_radii, group):
    """Sum accum and denom, and take the maximum of max_radii, over `group` (in place)."""
    import torch.distributed as dist
    dist.all_reduce(accum, op=dist.ReduceOp.SUM, group=group)
    dist.all_reduce(denom, op=dist.ReduceOp.SUM, group=group)
    dist.all_reduce(max_radii, op=dist.ReduceOp.MAX, group=group)


def split_normals(S, device, generator=None, group=None):
    """randn(2S, 3) from `generator`: the reference's normal(0, std) draw before it is scaled.  With `group`, drawn on
    the group's first rank and broadcast to the others."""
    import torch.distributed as dist
    first = group is None or dist.get_rank(group) == 0
    z = torch.randn(2 * S, 3, generator=generator, device=device) if first else \
        torch.empty(2 * S, 3, device=device)
    if group is not None and S:
        dist.broadcast(z, src=dist.get_global_rank(group, 0), group=group)
    return z


class Densifier:
    """SuGaRDensifier over `raw` and `optimizer`, or vanilla 3DGS's with rotation="vanilla" (see the module
    docstring)."""

    def __init__(self, raw, optimizer, max_grad=2e-4, min_opacity=0.005, max_screen_size=20, scene_extent=None,
                 percent_dense=0.01, group=None, rotation="sugar"):
        if scene_extent is None:
            raise ValueError("scene_extent is required (the reference's get_cameras_spatial_extent())")
        if rotation not in ROTATIONS:
            raise ValueError(f"rotation must be 'sugar' or 'vanilla', got {rotation!r}")
        self.points_kind = ROTATIONS[rotation]
        self.raw, self.optimizer, self.group = raw, optimizer, group
        self.max_grad, self.min_opacity, self.max_screen_size = max_grad, min_opacity, max_screen_size
        self.scene_extent, self.percent_dense = scene_extent, percent_dense
        self.groups = {}
        for k in KEYS:
            hits = [g for g in optimizer.param_groups if any(p is raw[k] for p in g["params"])]
            if len(hits) != 1 or len(hits[0]["params"]) != 1:
                raise ValueError(f"raw[{k!r}] must be the one tensor of exactly one optimizer group")
            self.groups[k] = hits[0]
        p = raw["points"]
        require_cuda("densify", p)
        self._reset_stats(p.shape[0])

    def _reset_stats(self, P):
        dev = self.raw["points"].device
        self.accum = torch.zeros((P, 1), device=dev)
        self.denom = torch.zeros((P, 1), device=dev)
        self.max_radii2D = torch.zeros((P,), device=dev)

    def update_densification_stats(self, viewspace_points, radii, visibility_filter):
        """For rows where visibility_filter (any boolean [P]): max_radii2D = max(max_radii2D, radii), accum +=
        |viewspace_points.grad[:, :2]|, denom += 1.  One kernel, no host synchronisation."""
        P = self.accum.shape[0]
        dev = self.accum.device
        g = viewspace_points.grad if torch.is_tensor(getattr(viewspace_points, "grad", None)) else viewspace_points
        require_cuda("densify", g, radii, visibility_filter)
        if g.dim() != 2 or g.shape[0] != P or g.shape[1] < 2 or g.dtype != torch.float32 or g.device != dev:
            raise ValueError(f"viewspace gradient must be float32 [{P},>=2] on {dev}, got {g.dtype} {tuple(g.shape)}")
        if g.stride(1) != 1:
            g = g.contiguous()
        radii = tensor(radii, "radii", torch.int32, (P,), dev, "points")
        vis = tensor(visibility_filter, "visibility_filter", torch.bool, (P,), dev, "points")
        with torch.cuda.device(dev):
            check(lib.sgr_densify_stats(P, ptr(g), g.stride(0), ptr(radii), ptr(vis), ptr(self.accum),
                                        ptr(self.denom), ptr(self.max_radii2D), stream(dev)))

    def _emit(self, scan, counts, normals, stats_too):
        P = self.accum.shape[0]
        n_keep, n_clone, S, n_child = counts
        P_out = n_keep + n_clone + 2 * n_child
        dev = self.raw["points"].device
        cols, new = [], {}
        alive = []   # tensors the column table points into, held until the launch is enqueued
        for k in KEYS:
            src = self.raw[k].detach().contiguous()
            alive.append(src)
            dst = torch.empty((P_out,) + tuple(src.shape[1:]), device=dev)
            width = int(np.prod(src.shape[1:]))
            kind = self.points_kind if k == "points" else SGR_DENSIFY_SCALES if k == "scales" else SGR_DENSIFY_COPY
            cols.append((src, dst, width, kind))
            st = self.optimizer.state.get(self.raw[k], None)
            mom = None
            if st is not None and "exp_avg" in st:
                mom = []
                for name in ("exp_avg", "exp_avg_sq"):
                    m = st[name].contiguous()
                    alive.append(m)
                    md = torch.empty_like(dst)
                    cols.append((m, md, width, SGR_DENSIFY_ZERO_NEW))
                    mom.append(md)
            new[k] = (dst, mom)
        stats = None
        if stats_too:
            stats = (torch.empty((P_out, 1), device=dev), torch.empty((P_out, 1), device=dev),
                     torch.empty((P_out,), device=dev))
            for s, d in zip((self.accum, self.denom, self.max_radii2D), stats):
                cols.append((s, d, 1, SGR_DENSIFY_COPY))
        tab = (SgrDensifyColumn * len(cols))(*[SgrDensifyColumn(ptr(s), ptr(d), w, kd) for s, d, w, kd in cols])
        src_row = torch.empty((P_out,), dtype=torch.int32, device=dev)
        pts, scl, q = (self.raw[k].detach().contiguous() for k in ("points", "scales", "quaternions"))
        q = tensor(q, "quaternions", torch.float32, (P, 4), align=16)
        alive += [pts, scl, q]
        with torch.cuda.device(dev):
            check(lib.sgr_densify_emit(P, n_keep, n_clone, S, n_child, ptr(scan), len(cols), tab, ptr(pts), ptr(scl),
                                       ptr(q), ptr(normals), INV_SPLIT, ptr(src_row), stream(dev)))
        self._install(new)
        return stats

    def _install(self, new):
        """Replace each parameter by its new tensor and re-key the optimizer's group and state to it."""
        for k, (dst, mom) in new.items():
            old = self.raw[k]
            p = torch.nn.Parameter(dst, requires_grad=True)
            st = self.optimizer.state.pop(old, None)
            if st is not None and mom is not None:
                st["exp_avg"], st["exp_avg_sq"] = mom
            if st is not None:
                self.optimizer.state[p] = st
            self.groups[k]["params"][0] = p
            self.raw[k] = p

    def _scan(self, flags):
        """-> (inclusive scans i32 [4,P], the four totals): the one host read."""
        P = flags.shape[1]
        scan = torch.cumsum(flags, dim=1, dtype=torch.int32)
        counts = scan[:, -1].tolist() if P else [0, 0, 0, 0]
        return scan, counts

    def densify_and_prune(self, max_grad=None, min_opacity=None, extent=None, max_screen_size=None, generator=None):
        """The reference's densify_and_prune: clone, split (normals from `generator`, a CUDA generator or None for the
        default one), then prune; one pass decides every row and one launch writes the new parameters and Adam moments.
        The statistics are zeros of the new size afterwards.  max_screen_size=None (or 0) skips the screen and world
        size clauses, as in the reference, which does not substitute its own value here."""
        dev = self.raw["points"].device
        if self.group is not None:
            reduce_statistics(self.accum, self.denom, self.max_radii2D, self.group)
        flags = self.classify(max_grad, min_opacity, extent, max_screen_size)
        scan, counts = self._scan(flags)
        normals = split_normals(counts[2], dev, generator, self.group)
        self._emit(scan, counts, normals, stats_too=False)
        self._reset_stats(self.raw["points"].shape[0])

    def classify(self, max_grad=None, min_opacity=None, extent=None, max_screen_size=None):
        """-> flags u8 [4,P] of densify_and_prune from the current statistics: keep (an original row neither split nor
        pruned), clone_kept, split, children_kept (include/sugar_b200.h, sgr_densify_classify)."""
        max_grad = self.max_grad if max_grad is None else max_grad
        min_opacity = self.min_opacity if min_opacity is None else min_opacity
        extent = self.scene_extent if extent is None else extent
        dev = self.raw["points"].device
        P = self.accum.shape[0]
        f32 = lambda x: float(np.float32(x))     # torch compares a float32 tensor with a Python float in float32
        gates = SgrDensifyGates(f32(max_grad), f32(self.percent_dense * extent), f32(0.1 * extent), f32(min_opacity),
                                f32(max_screen_size or 0), INV_SPLIT, int(bool(max_screen_size)))
        scales = tensor(self.raw["scales"].detach(), "scales", torch.float32, (P, 3), dev, "points")
        dens = tensor(self.raw["densities"].detach(), "densities", torch.float32, (P, 1), dev, "points")
        flags = torch.empty((4, P), dtype=torch.uint8, device=dev)
        with torch.cuda.device(dev):
            check(lib.sgr_densify_classify(P, ptr(self.accum), ptr(self.denom), ptr(scales), ptr(dens), gates,
                                           ptr(flags), stream(dev)))
        return flags

    def prune_points(self, mask):
        """Keep the rows where ~mask (any boolean [P]); statistics and Adam moments follow their rows."""
        P = self.accum.shape[0]
        dev = self.raw["points"].device
        mask = tensor(mask, "mask", torch.bool, (P,), dev, "points")
        flags = torch.zeros((4, P), dtype=torch.uint8, device=dev)
        flags[0] = ~mask
        scan, counts = self._scan(flags)
        stats = self._emit(scan, counts, None, stats_too=True)
        self.accum, self.denom, self.max_radii2D = stats

    def reset_opacity(self):
        """densities = logit(min(sigmoid(densities), 0.01)), with that group's Adam moments zeroed."""
        d = self.raw["densities"].detach()
        op = torch.sigmoid(d.view(-1, 1))
        v = torch.min(op, torch.ones_like(d.view(-1, 1)) * 0.01)
        new = torch.log(v / (1 - v)).view_as(d)
        st = self.optimizer.state.get(self.raw["densities"], None)
        mom = None if st is None or "exp_avg" not in st else [torch.zeros_like(new), torch.zeros_like(new)]
        self._install({"densities": (new, mom)})
