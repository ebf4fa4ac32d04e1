"""sugar_b200.train on the GPU against the oracle's loops (oracle/optim_oracle.py: the reference's loop shape and
decisions over this package's steps and torch.optim.Adam), on a scaled-down schedule: the events iteration by
iteration, the prune's survivors, and the final parameters within a tolerance (the rasterizer's backward accumulates
with atomics, so two runs of the same loop are not bit-identical)."""
import copy
import math
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import optim_oracle as oo  # noqa: E402
from sugar_b200 import knn, mcubes, meshbind, meshloss, optim, render, scenes, steps, train  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SCHED = dict(num_iterations=40, regularize_from=10, entropy_window=(10, 20), prune_at=(20,), sdf_from=20,
             reset_neighbors_every=500)


def coarse_setup(P=3000, W=160, H=120):
    sc = scenes.make_scene(P, W, H, seed=3, camera="posed")
    g = torch.Generator().manual_seed(5)
    views = []
    for yaw, shift in ((0.0, (0, 0, 0)), (0.08, (0.2, 0, 0)), (-0.08, (-0.2, 0.1, 0)), (0.04, (0, -0.2, 0.3))):
        v = scenes.with_camera_offset(sc, yaw, shift)
        views.append((steps.camera_from_scene(v, DEV), torch.rand(3, H, W, generator=g).to(DEV)))
    extent = mcubes.camera_spatial_extent(torch.stack([c.campos.cpu() for c, _ in views]))
    raw0 = dict(points=torch.from_numpy(sc.means3D), sh_dc=torch.from_numpy(sc.shs[:, :1].copy()),
                sh_rest=torch.from_numpy(sc.shs[:, 1:].copy()),
                densities=torch.logit(torch.from_numpy(sc.opacities).clamp(1e-4, 1 - 1e-4)),
                scales=torch.from_numpy(sc.scales).log(), quaternions=torch.from_numpy(sc.rotations) * 1.3)
    return raw0, views, extent


def leaf_copy(raw0):
    return {k: v.to(DEV).clone().requires_grad_(True) for k, v in raw0.items()}


def close(ours, ref, lrs, iterations, label):
    """Per group: 99.5% of the entries within 1e-4 + 1e-4 relative + 1% of the furthest Adam moves an entry in these
    iterations (lr per step), and every entry within twice that distance: an entry whose gradient cancels to nearly
    zero takes a full-size Adam step whose sign follows the atomics' rounding, so the two runs can differ by whole
    steps there and nowhere else."""
    for k, lr in lrs.items():
        a, b = ours[k].detach(), ref[k].detach()
        assert a.shape == b.shape, (label, k)
        d = (a - b).abs()
        tol = 1e-4 + 1e-4 * b.abs() + 1e-2 * lr * iterations
        share = float((d > tol).float().mean())
        print(f"{label} {k}: max |diff| {float(d.max()):.3g}, share over the tolerance {share:.2e}")
        assert share <= 5e-3, (label, k, share)
        assert float(d.max()) <= 2.0 * lr * iterations + 1e-5, (label, k, float(d.max()))


def view_order(seed, n_views, iterations):
    """The view index of each iteration 1..iterations: both loops draw one CPU randperm per epoch and nothing else
    from the CPU generator."""
    torch.manual_seed(seed)
    order = []
    while len(order) < iterations:
        order += torch.randperm(n_views).tolist()
    return order[:iterations]


@pytest.mark.parametrize("mode", ["sdf", "density"])
def test_train_coarse_matches_the_oracle_loop(mode):
    """The whole 40-iteration loop against the oracle's, and each SDF-phase iteration against the oracle's iteration
    from the same state.  The SDF phase samples in Gaussians picked by threshold tests on the rendered depth and
    visibility; a last-bit difference from the backward's atomics can flip one of them, after which the two runs draw
    different samples.  So the runs are compared as wholes up to the prune (continuous ops only) and through the SDF
    phase iteration by iteration, with the CUDA generator's state, the view and the optimizer state restored."""
    raw0, views, extent = coarse_setup()
    kw = dict(mode=mode, spatial_extent=extent, entropy_factor=0.1, prune_threshold=0.5, dssim_factor=0.2,
              n_samples=20_000, **SCHED)
    knn0 = knn.reset_neighbors(raw0["points"].to(DEV), 16)[1]

    raw_a = leaf_copy(raw0)
    opt = optim.SugarOptimizer(raw_a, spatial_lr_scale=extent)
    got, survivors, losses_a, snaps = {}, {}, {}, {}

    def hook(it, loss, ev):
        got[it] = ev
        losses_a[it] = loss
        assert loss.is_cuda and loss.dim() == 0
        if it == 20:
            survivors["want"] = int((torch.sigmoid(raw_a["densities"].detach()) >= 0.5).sum())
        if it == 21:
            survivors["got"] = raw_a["points"].shape[0]
        if it >= 20:
            snaps[it] = ({k: v.detach().clone() for k, v in raw_a.items()}, copy.deepcopy(opt.state_dict()),
                         torch.cuda.get_rng_state())
    torch.manual_seed(123)
    assert train.train_coarse(raw_a, views, knn0, on_iteration=hook, optimizer=opt, **kw) is opt

    raw_b = leaf_copy(raw0)
    want, losses_b, at20 = {}, {}, {}

    def oracle_hook(it, loss, names):
        want[it] = names
        losses_b[it] = loss
        if it == 20:
            at20.update({k: v.detach().clone() for k, v in raw_b.items()})
    torch.manual_seed(123)
    ref = oo.coarse_loop(raw_b, views, knn0, mode, extent, SCHED["num_iterations"], SCHED["regularize_from"],
                         SCHED["entropy_window"], 0.1, SCHED["prune_at"], 0.5, SCHED["reset_neighbors_every"],
                         SCHED["sdf_from"], 0.2, 20_000, on_iteration=oracle_hook)

    assert sorted(got) == sorted(want) == list(range(1, 41))
    for it in got:
        assert got[it] == dict({"sh_degree": 3}, **{n: True for n in want[it]}), it
    assert [it for it in got if "sdf" in got[it]] == list(range(21, 41))
    P0 = raw0["points"].shape[0]
    assert 0 < survivors["got"] == survivors["want"] < P0, survivors
    # the optimizer state follows the pruned rows, and the schedule set the position lr
    assert opt.param_groups[0]["lr"] == ref.optimizer.param_groups[0]["lr"] == \
        optim.expon_lr(1.6e-4 * extent, 1.6e-6 * extent, max_steps=30_000)(40)
    for k in raw_a:
        st = opt.state[raw_a[k]]
        assert st["exp_avg"].shape == raw_a[k].shape and float(st["step"]) == 40
    lrs = {k: lr for _, k, lr in optim.group_table(extent)}
    la = torch.stack([losses_a[i] for i in range(1, 21)]).cpu().numpy()
    lb = torch.stack([losses_b[i] for i in range(1, 21)]).cpu().numpy()
    print(f"{mode}: losses 1-20 max rel diff {float(np.max(np.abs(la - lb) / np.abs(lb))):.3g}")
    assert np.all(np.isfinite(la)) and np.allclose(la, lb, rtol=1e-4, atol=0)
    close(snaps[20][0], at20, lrs, 20, f"{mode} iteration 20")

    # the SDF phase, one iteration at a time from this run's state
    order = view_order(123, len(views), 40)
    sched = dict(regularize_from=SCHED["regularize_from"], start_entropy_regularization_from=SCHED["entropy_window"][0],
                 end_entropy_regularization_at=SCHED["entropy_window"][1],
                 prune_low_opacity_gaussians_at=SCHED["prune_at"], reset_neighbors_every=SCHED["reset_neighbors_every"],
                 start_sdf_regularization_from=SCHED["sdf_from"])
    ops = steps.ours_ops()
    knn_r = knn0
    for it in range(21, 41):
        params, state, rng = snaps[it - 1]
        raw_r = {k: v.clone().requires_grad_(True) for k, v in params.items()}
        opt_r = oo.OracleOptimizer(raw_r, spatial_lr_scale=extent)
        opt_r.optimizer.load_state_dict(copy.deepcopy(state))
        opt_r.update_learning_rate(it)
        torch.cuda.set_rng_state(rng)
        cam, gt = views[order[it - 1]]
        loss, knn_r = oo.coarse_iteration(raw_r, opt_r, knn_r, cam, gt, oo.coarse_events(it, **sched), mode, extent,
                                          0.1, 0.5, 0.2, 20_000, ops)
        assert raw_r["points"].shape == snaps[it][0]["points"].shape, it
        assert torch.allclose(loss, losses_a[it], rtol=1e-5, atol=0), (it, float(loss), float(losses_a[it]))
        close(snaps[it][0], raw_r, lrs, 1, f"{mode} iteration {it}")


def look_at(pos, W, H, fov_x=0.9, target=(0.5, 0.5, 0.0)):
    p = torch.tensor(pos, dtype=torch.float32)
    z = p - torch.tensor(target, dtype=torch.float32)
    z = z / z.norm()
    up = torch.tensor([0.0, 1.0, 0.0])
    x = torch.linalg.cross(up, z)
    x = x / x.norm()
    y = torch.linalg.cross(z, x)
    c2w = torch.stack([x, y, z, p], 1).to(DEV)
    fov_y = 2 * math.atan(math.tan(fov_x / 2) * H / W)
    view, proj, center = render.camera_matrices(c2w, fov_x, fov_y)
    return SimpleNamespace(viewmatrix=view, projmatrix=proj, campos=center, width=W, height=H,
                           tanfovx=math.tan(fov_x / 2), tanfovy=math.tan(fov_y / 2))


def test_train_refined_matches_the_oracle_loop():
    W, H, n, iters, every = 128, 96, 6, 12, 4
    v, f = scenes.height_field_mesh(12, 12, seed=2)
    verts, faces = torch.from_numpy(v).to(DEV), torch.from_numpy(f).to(DEV)
    F, V = faces.shape[0], verts.shape[0]
    P = F * n
    g = torch.Generator().manual_seed(8)
    views = [(look_at(pos, W, H), torch.rand(3, H, W, generator=g).to(DEV))
             for pos in ((0.5, 0.4, 1.6), (0.8, 0.3, 1.4), (0.2, 0.6, 1.5))]
    raw0 = dict(verts=verts.cpu(), sh_dc=0.5 * torch.randn(P, 1, 3, generator=g),
                sh_rest=0.1 * torch.randn(P, 15, 3, generator=g), densities=torch.randn(P, 1, generator=g) + 1.0,
                scales=torch.randn(P, 2, generator=g) * 0.2 - 3.0, quaternions=torch.randn(P, 2, generator=g))
    mesh = SimpleNamespace(faces=faces, bary=meshbind.bary_coords(n, DEV), thickness=1e-5,
                           topology=meshloss.mesh_topology(faces, V))
    extent = mcubes.camera_spatial_extent(torch.stack([c.campos.cpu() for c, _ in views]))
    scale = train.refine_spatial_lr_scale(V, spatial_extent=extent)

    raw_a = leaf_copy(raw0)
    got, la = {}, {}

    def hook(it, loss, ev):
        got[it], la[it] = ev, loss
    torch.manual_seed(7)
    opt = train.train_refined(raw_a, mesh, views, scale, num_iterations=iters, sh_warmup_every=every,
                              on_iteration=hook)
    raw_b = leaf_copy(raw0)
    want, lb = {}, {}

    def oracle_hook(it, loss, deg):
        want[it], lb[it] = deg, loss
    torch.manual_seed(7)
    ref = oo.refine_loop(raw_b, mesh, views, scale, iters, 0.2, 0.1, every, on_iteration=oracle_hook)

    assert [got[i]["sh_degree"] for i in range(1, iters + 1)] == [want[i] for i in range(1, iters + 1)] == \
        [0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2]
    assert [g["name"] for g in opt.param_groups][0] == "points" and opt.param_groups[0]["params"][0] is raw_a["verts"]
    assert opt.param_groups[0]["lr"] == ref.optimizer.param_groups[0]["lr"]
    a = torch.stack([la[i] for i in range(1, iters + 1)]).cpu().numpy()
    b = torch.stack([lb[i] for i in range(1, iters + 1)]).cpu().numpy()
    print(f"refine: losses {a[0]:.6f} -> {a[-1]:.6f}, max rel diff {float(np.max(np.abs(a - b) / np.abs(b))):.3g}")
    assert np.all(np.isfinite(a)) and np.allclose(a, b, rtol=1e-3, atol=0)
    lrs = {k: lr for _, k, lr in optim.group_table(scale, bound=True)}
    close(raw_a, raw_b, lrs, iters, "refine")
    with pytest.raises(ValueError, match="optimizer"):
        train.train_refined(raw_a, mesh, views, scale, num_iterations=1, optimizer=optim.Adam([raw_a["verts"]]))
