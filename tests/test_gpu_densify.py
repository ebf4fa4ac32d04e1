"""Densification and pruning on the GPU (csrc/sgr_densify.cu, sugar_b200/densify.py) against the reference's statements
restated in oracle/densify_oracle.py, run on the same device: the statistics, every decision and every copied value
bit for bit; children's positions within a few ulps (the reference's bmm has no specified summation order)."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import densify_oracle as do  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
KEYS = do.KEYS


def ulp_steps(x, k):
    """float32 x moved k ulps (k may be negative)."""
    a = np.array([x], np.float32)
    for _ in range(abs(k)):
        a = np.nextafter(a, np.float32(np.inf if k > 0 else -np.inf))
    return float(a[0])


def make_model(P, seed, extent=1.0, max_grad=2e-4, min_opacity=0.005):
    """Raw parameters and statistics with about 4% clone, 4% split and 1% prune, plus rows on, and one ulp either side
    of, every gate."""
    g = torch.Generator().manual_seed(seed)
    thr = 0.01 * extent
    sc = torch.where(torch.rand(P, generator=g) < 0.5, thr * 0.5, thr * 2.0) * (0.8 + 0.4 * torch.rand(P, 3, generator=g)).T
    raw = {"points": torch.randn(P, 3, generator=g), "densities": torch.randn(P, 1, generator=g) + 2.0,
           "scales": torch.log(sc.T.contiguous()), "quaternions": torch.randn(P, 4, generator=g),
           "sh_dc": torch.randn(P, 1, 3, generator=g), "sh_rest": torch.randn(P, 15, 3, generator=g)}
    r = torch.rand(P, generator=g)
    raw["densities"][r < 0.01] = -9.0                                          # pruned by opacity
    denom = torch.randint(0, 5, (P, 1), generator=g).float()
    accum = denom * torch.where(torch.rand(P, 1, generator=g) < 0.08, 4e-4, 1e-5) * (0.8 + 0.4 * torch.rand(P, 1, generator=g))
    # rows on the gates: grads at max_grad +- 1 ulp; max scale, opacity, big scale and the children's big scale near
    # their thresholds (the log / logit stepped by ulps around the inverse, so exp / sigmoid land on both sides)
    n = min(P // 8, 7 * 5)
    steps = [k for k in range(-3, 4)]
    i = 0
    for kind in ("grad", "scale", "opacity", "big", "child"):
        for k in steps[:n // 5]:
            row = P - 1 - i
            i += 1
            accum[row], denom[row] = (1e-6 if kind in ("big", "opacity") else 4e-4), 1.0
            if kind == "grad":
                accum[row] = ulp_steps(max_grad, k)
            elif kind == "scale":
                raw["scales"][row] = ulp_steps(float(np.log(np.float32(thr))), k)
            elif kind == "opacity":
                raw["densities"][row] = ulp_steps(float(np.log(min_opacity / (1 - min_opacity))), k)
            elif kind == "big":
                raw["scales"][row] = ulp_steps(float(np.log(np.float32(0.1 * extent))), k)
            else:
                raw["scales"][row] = ulp_steps(float(np.log(np.float32(0.1 * extent) * np.float32(1.6))), k)
    stats = {"accum": accum, "denom": denom, "max_radii": torch.rand(P, generator=g) * 50}
    return raw, stats


def build(raw0, stats, moments=True, lr=1e-3):
    raw = {k: torch.nn.Parameter(v.clone().to(DEV)) for k, v in raw0.items()}
    opt = torch.optim.Adam([{"params": [raw[k]], "name": k, "lr": lr} for k in KEYS], eps=1e-15)
    if moments:
        for k in KEYS:
            raw[k].grad = torch.randn_like(raw[k]) * 1e-3
        opt.step()
        opt.zero_grad()
    from sugar_b200 import densify
    d = densify.Densifier(raw, opt, scene_extent=1.0)
    d.accum.copy_(stats["accum"]), d.denom.copy_(stats["denom"]), d.max_radii2D.copy_(stats["max_radii"])
    return raw, opt, d


def oracle_state(raw, opt, d):
    params = {k: raw[k].detach().clone() for k in KEYS}
    mom = {k: (opt.state[raw[k]]["exp_avg"].clone(), opt.state[raw[k]]["exp_avg_sq"].clone())
           for k in KEYS if raw[k] in opt.state}
    stats = {"accum": d.accum.clone(), "denom": d.denom.clone(), "max_radii": d.max_radii2D.clone()}
    return params, mom, stats


def child_bound(ref_points, samples, first_child):
    """|ours - ref| per coordinate <= 2^-20 (|point| + |sample|_1): a few ulps of the largest term of R s + p, since
    |R| entries are <= 1 and the rotation itself carries a few ulps."""
    s = samples.abs().sum(1, keepdim=True)
    return 2.0 ** -20 * (ref_points[first_child:].abs() + s)


def compare(raw, opt, d, params, mom, flags, info, S_kept):
    P_out = params["points"].shape[0]
    assert raw["points"].shape[0] == P_out
    first_child = P_out - 2 * S_kept
    for k in KEYS:
        ours = raw[k].detach()
        if k == "points":
            assert torch.equal(ours[:first_child], params[k][:first_child])
            err = (ours[first_child:] - params[k][first_child:]).abs()
            assert err.shape[0] == 2 * S_kept
            samples = info["samples_kept"]
            assert bool((err <= child_bound(params[k], samples, first_child)).all()), float(err.max())
        else:
            assert torch.equal(ours, params[k]), k
        if k in mom:
            st = opt.state[raw[k]]
            assert torch.equal(st["exp_avg"], mom[k][0]) and torch.equal(st["exp_avg_sq"], mom[k][1]), k
        else:
            assert raw[k] not in opt.state or "exp_avg" not in opt.state[raw[k]]
    assert all(g["params"][0] is raw[g["name"]] for g in opt.param_groups)


def run_both(raw, opt, d, seed, max_screen_size=20, **kw):
    """One densify_and_prune on both sides from the same state and generator seed; returns the flags."""
    params, mom, stats = oracle_state(raw, opt, d)
    flags = d.classify(max_screen_size=max_screen_size, **kw).cpu()
    P = params["points"].shape[0]
    ga = torch.Generator(device=DEV).manual_seed(seed)
    gb = torch.Generator(device=DEV).manual_seed(seed)
    args = dict(max_grad=kw.get("max_grad", d.max_grad), min_opacity=kw.get("min_opacity", d.min_opacity),
                extent=kw.get("extent", d.scene_extent), max_screen_size=max_screen_size)
    p2, m2, s2, info = do.densify_and_prune(params, mom, stats, percent_dense=d.percent_dense, generator=gb, **args)
    d.densify_and_prune(generator=ga, **args)
    split = info["split"][:P].cpu()
    assert torch.equal(split, flags[2].bool())
    S = int(split.sum())
    ck = flags[3].bool()
    info["samples_kept"] = torch.cat([info["samples"][:S][ck[split].to(DEV)], info["samples"][S:][ck[split].to(DEV)]])
    compare(raw, opt, d, p2, m2, flags, info, int(ck.sum()))
    assert not d.accum.any() and d.accum.shape[0] == p2["points"].shape[0]
    return flags


@pytest.mark.parametrize("P", [1000, 100_000, 1_000_000])
def test_densify_and_prune_matches_oracle(P):
    raw0, stats = make_model(P, seed=P)
    raw, opt, d = build(raw0, stats)
    flags = run_both(raw, opt, d, seed=5)
    frac = flags.float().mean(1)
    assert frac[2] > 0.02 and flags[1].sum() > 0 and (flags[0] + flags[2]).lt(1).any()   # splits, clones, prunes
    # the optimizer steps on the new tensors
    for k in KEYS:
        raw[k].grad = torch.ones_like(raw[k])
    opt.step()
    assert all(opt.state[raw[k]]["exp_avg"].shape == raw[k].shape for k in KEYS)


@pytest.mark.parametrize("mss", [None, 0, 20, -1])
def test_screen_size_and_no_state(mss):
    raw0, stats = make_model(5000, seed=11)
    raw, opt, d = build(raw0, stats, moments=False)
    run_both(raw, opt, d, seed=6, max_screen_size=mss)
    assert not opt.state


def test_no_split_and_all_pruned():
    raw0, stats = make_model(3000, seed=12)
    raw, opt, d = build(raw0, stats)
    flags = run_both(raw, opt, d, seed=7, max_grad=1e9)
    assert flags[2].sum() == 0
    raw, opt, d = build(raw0, stats)
    run_both(raw, opt, d, seed=7, min_opacity=1.0)
    assert raw["points"].shape[0] == 0


def test_prune_points_and_reset_opacity_match_oracle():
    raw0, stats = make_model(20_000, seed=13)
    raw, opt, d = build(raw0, stats)
    params, mom, st = oracle_state(raw, opt, d)
    mask = torch.sigmoid(raw["densities"].detach()).squeeze(1) < 0.5
    p2, m2, s2 = do.prune_points(params, mom, st, mask)
    d.prune_points(mask)
    for k in KEYS:
        assert torch.equal(raw[k].detach(), p2[k]), k
        assert torch.equal(opt.state[raw[k]]["exp_avg"], m2[k][0]) and torch.equal(opt.state[raw[k]]["exp_avg_sq"], m2[k][1])
    assert torch.equal(d.accum, s2["accum"]) and torch.equal(d.denom, s2["denom"]) and torch.equal(d.max_radii2D, s2["max_radii"])
    p3, m3 = do.reset_opacity(p2, m2)
    d.reset_opacity()
    assert torch.equal(raw["densities"].detach(), p3["densities"])
    assert not opt.state[raw["densities"]]["exp_avg"].any()


def test_statistics_match_reference_without_host_sync():
    P = 100_000
    g = torch.Generator(device=DEV).manual_seed(3)
    raw0, _ = make_model(P, seed=14)
    raw, opt, d = build(raw0, {"accum": torch.zeros(P, 1), "denom": torch.zeros(P, 1), "max_radii": torch.zeros(P)})
    ref = {"accum": torch.zeros(P, 1, device=DEV), "denom": torch.zeros(P, 1, device=DEV),
           "max_radii": torch.zeros(P, device=DEV)}
    for view in range(6):
        grad = torch.randn(P, 3, generator=g, device=DEV) * torch.exp(torch.randn(P, 1, generator=g, device=DEV) * 3)
        radii = torch.randint(0, 40, (P,), generator=g, device=DEV, dtype=torch.int32)
        vis = radii > 0 if view % 2 == 0 else torch.rand(P, generator=g, device=DEV) < 0.5   # any mask
        means2D = torch.zeros(P, 3, device=DEV, requires_grad=True)
        means2D.grad = grad
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            d.update_densification_stats(means2D, radii, vis)
        finally:
            torch.cuda.set_sync_debug_mode("default")
        do.update_stats(ref, grad, radii, vis)
    assert torch.equal(d.max_radii2D, ref["max_radii"])
    assert torch.equal(d.denom, ref["denom"])
    bad = (d.accum != ref["accum"]).sum().item()
    assert bad == 0, f"{bad} accum rows differ, largest {(d.accum - ref['accum']).abs().max().item()}"


def test_training_loop_against_oracle():
    """A short loop on a synthetic scene: render, L1, Adam, statistics, prune_points(strengths < 0.5) (the trainers'
    prune of a model initialised from 3DGS; after an opacity reset it would remove every row), densify every 10 steps,
    an opacity reset, then the K-NN rebuild and one regularised coarse step.  Every densify or prune is compared with
    the oracle fed the same state."""
    from sugar_b200 import densify, knn, scenes, steps
    sc = scenes.make_scene(20_000, 320, 240, seed=4)
    cam = steps.camera_from_scene(sc, DEV)
    ops = steps.ours_ops()
    gt = torch.rand(3, 240, 320, generator=torch.Generator().manual_seed(2)).to(DEV)
    leaf = lambda t: torch.nn.Parameter(t.to(DEV))
    raw = dict(points=leaf(torch.from_numpy(sc.means3D)), sh_dc=leaf(torch.from_numpy(sc.shs[:, :1].copy())),
               sh_rest=leaf(torch.from_numpy(sc.shs[:, 1:].copy())),
               densities=leaf(torch.logit(torch.from_numpy(sc.opacities).clamp(1e-4, 1 - 1e-4))),
               scales=leaf(torch.from_numpy(sc.scales).log()), quaternions=leaf(torch.from_numpy(sc.rotations)))
    opt = torch.optim.Adam([{"params": [raw[k]], "name": k, "lr": 1e-3} for k in KEYS], eps=1e-15)
    extent = float(np.linalg.norm(sc.means3D.max(0) - sc.means3D.min(0))) * 0.5
    d = densify.Densifier(raw, opt, max_grad=2e-5, scene_extent=extent)
    for it in range(1, 31):
        a = steps.activate(raw)
        image, radii, viewspace = steps.render(ops, a, cam, torch.zeros(3, device=DEV), 3)
        (image - gt).abs().mean().backward()
        d.update_densification_stats(viewspace, radii, radii > 0)
        opt.step()
        opt.zero_grad(set_to_none=True)
        if it == 5:
            params, mom, st = oracle_state(raw, opt, d)
            mask = (torch.sigmoid(raw["densities"].detach()) < 0.5).squeeze(1)
            p2, m2, s2 = do.prune_points(params, mom, st, mask)
            d.prune_points(mask)
            assert 0 < raw["points"].shape[0] < mask.shape[0]
            assert all(torch.equal(raw[k].detach(), p2[k]) for k in KEYS) and torch.equal(d.accum, s2["accum"])
        if it % 10 == 0:
            run_both(raw, opt, d, seed=it, max_screen_size=20 if it > 10 else None, extent=extent)
        if it == 20:
            params, mom, _ = oracle_state(raw, opt, d)
            p3, m3 = do.reset_opacity(params, mom)
            d.reset_opacity()
            assert torch.equal(raw["densities"].detach(), p3["densities"])
    knn_idx = knn.reset_neighbors(raw["points"].detach(), 16)[1]
    loss, _ = steps.coarse_sdf_step(raw, cam, gt, knn_idx, ops, n_samples=20_000,
                                    generator=torch.Generator(device=DEV).manual_seed(1))
    assert torch.isfinite(loss)
    opt.step()


def test_two_ranks_stay_identical(tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    import subprocess
    code = ("import os, sys, torch, torch.distributed as dist; sys.path.insert(0, %r)\n"
            "sys.path.insert(0, os.path.join(%r, 'tests')); from test_gpu_densify import make_model, KEYS\n"
            "from sugar_b200 import densify\n"
            "dist.init_process_group('nccl'); r = dist.get_rank(); torch.cuda.set_device(r); dev = f'cuda:{r}'\n"
            "raw0, st = make_model(50000, seed=1)\n"
            "raw = {k: torch.nn.Parameter(v.to(dev)) for k, v in raw0.items()}\n"
            "opt = torch.optim.Adam([{'params': [raw[k]], 'name': k} for k in KEYS])\n"
            "d = densify.Densifier(raw, opt, scene_extent=1.0, group=dist.group.WORLD)\n"
            "d.accum.copy_(st['accum'] * (r + 1)); d.denom.copy_(st['denom'])\n"
            "d.densify_and_prune(max_screen_size=20, generator=torch.Generator(device=dev).manual_seed(r))\n"
            "for k in KEYS:\n"
            "    x = raw[k].detach().clone(); y = x.clone(); dist.broadcast(y, 0)\n"
            "    assert torch.equal(x, y), k\n"
            "dist.destroy_process_group()\n") % (ROOT, ROOT)
    script = tmp_path / "two_ranks.py"
    script.write_text(code)
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nproc_per_node=2", str(script)],
                         capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-3000:]
