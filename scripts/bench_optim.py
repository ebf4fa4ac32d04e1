#!/usr/bin/env python
"""Time the trainers' optimizer step (sugar_b200/optim.py) and one train_coarse iteration per phase.

    python scripts/bench_optim.py [--iters 20] [--rounds 5] [--no-train] [--out FILE]

Optimizer step over SuGaR's six groups (59 float32 per Gaussian), gradients of 1e-3 scale, state already created:
    unbound 1M        P = 1M Gaussians, steps.activate's keys
    unbound 3M        P = 3M
    bound 500k x 6    500k faces x 6 = 3M Gaussians on 250k vertices (scales / quaternions [P,2]: 57 floats per
                      Gaussian plus 3 per vertex)
Arms, CUDA events around `iters` steps, `rounds` rounds alternating the arms in one process, medians:
    ours          sugar_b200.optim.Adam: one sgr_adam_step launch
    foreach       torch.optim.Adam(foreach=True): the reference's update (seven elementwise passes per tensor list)
    fused         torch.optim.Adam(fused=True): torch's one-kernel Adam, a different arithmetic (not bit-identical)
Byte models: 28 B per element for one pass (param, grad, exp_avg, exp_avg_sq read; three written) and 72 B for the
foreach sequence (lerp 12, mul 8, addcmul 12, sqrt 8, div 8, add 8, addcdiv 16).  GB/s are model bytes over time,
HBM shares against the H100 SXM data sheet's 3.35 TB/s.  Peak memory: max_memory_allocated over one step minus the
allocation before it.
train_coarse: the time of one iteration in each phase (photometric, entropy, SDF, both coarse modes) at 1M Gaussians,
1920x1080, 1M samples, from CUDA events between consecutive on_iteration calls, median over the timed iterations.
Every result carries the card's name, power limit and max SM clock, read in the same run.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_meshloss import card, median  # noqa: E402
from sugar_b200 import knn, mcubes, optim, scenes, steps, train  # noqa: E402

DEV = "cuda:0"
PEAK_GBS = 3350.0
UNBOUND = {"points": (3,), "sh_dc": (1, 3), "sh_rest": (15, 3), "densities": (1,), "scales": (3,), "quaternions": (4,)}
BOUND = {"sh_dc": (1, 3), "sh_rest": (15, 3), "densities": (1,), "scales": (2,), "quaternions": (2,)}


def make_params(P, bound=False, V=0):
    g = torch.Generator(device=DEV).manual_seed(0)
    shapes = BOUND if bound else UNBOUND
    raw = {k: torch.nn.Parameter(torch.randn((P,) + s, generator=g, device=DEV)) for k, s in shapes.items()}
    if bound:
        raw["verts"] = torch.nn.Parameter(torch.randn(V, 3, generator=g, device=DEV))
    for v in raw.values():
        v.grad = torch.randn(v.shape, generator=g, device=DEV) * 1e-3
    return raw


def event_ms(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def peak_bytes(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def bench_step(label, raw, iters, rounds, bound):
    n = sum(v.numel() for v in raw.values())
    table = optim.group_table(1.0, bound)
    groups = [{"params": [raw[k]], "lr": lr, "name": name} for name, k, lr in table]
    arms = {"ours": optim.Adam(groups, lr=0.0, eps=1e-15),
            "foreach": torch.optim.Adam([dict(g) for g in groups], lr=0.0, eps=1e-15, foreach=True),
            "fused": torch.optim.Adam([dict(g) for g in groups], lr=0.0, eps=1e-15, fused=True)}
    for opt in arms.values():   # state, modules and allocator warm
        for _ in range(3):
            opt.step()
    times = {k: [] for k in arms}
    for _ in range(rounds):
        for k, opt in arms.items():
            times[k].append(event_ms(opt.step, iters))
    res = {"case": label, "elements": n}
    for k, opt in arms.items():
        ms = median(times[k])
        model = 72 if k == "foreach" else 28
        gbs = n * model / ms / 1e6
        res[k] = {"ms": round(ms, 4), "model_bytes_per_element": model, "gb_s": round(gbs, 1),
                  "hbm_share": round(gbs / PEAK_GBS, 3), "peak_extra_mb": round(peak_bytes(opt.step) / 2 ** 20, 1),
                  "rounds_ms": [round(t, 4) for t in times[k]]}
    res["foreach_over_ours"] = round(res["foreach"]["ms"] / res["ours"]["ms"], 2)
    res["fused_over_ours"] = round(res["fused"]["ms"] / res["ours"]["ms"], 2)
    print(json.dumps(res))
    return res


def bench_train(P=1_000_000, W=1920, H=1080, samples=1_000_000, iters=8, warm=3):
    sc = scenes.make_scene(P, W, H, seed=0)
    g = torch.Generator().manual_seed(0)
    views = []
    for yaw, shift in ((0.0, (0, 0, 0)), (0.05, (0.2, 0, 0)), (-0.05, (-0.2, 0.1, 0))):
        v = scenes.with_camera_offset(sc, yaw, shift)
        views.append((steps.camera_from_scene(v, DEV), torch.rand(3, H, W, generator=g).to(DEV)))
    extent = mcubes.camera_spatial_extent(torch.stack([c.campos.cpu() for c, _ in views]))
    big = 10 ** 9
    phases = {"photometric": dict(regularize_from=big, entropy_window=(big, big + 1), sdf_from=big),
              "entropy": dict(regularize_from=big, entropy_window=(0, big), sdf_from=big),
              "sdf": dict(regularize_from=0, entropy_window=(0, 1), sdf_from=0)}
    out = []
    for mode in ("sdf", "density"):
        for phase, sched in phases.items():
            if mode == "density" and phase != "sdf":
                continue   # the two modes share the unregularised phases
            raw = dict(points=torch.from_numpy(sc.means3D), sh_dc=torch.from_numpy(sc.shs[:, :1].copy()),
                       sh_rest=torch.from_numpy(sc.shs[:, 1:].copy()),
                       densities=torch.logit(torch.from_numpy(sc.opacities).clamp(1e-4, 1 - 1e-4)),
                       scales=torch.from_numpy(sc.scales).log(), quaternions=torch.from_numpy(sc.rotations) * 1.3)
            raw = {k: v.to(DEV).requires_grad_(True) for k, v in raw.items()}
            knn_idx = knn.reset_neighbors(raw["points"].detach(), 16)[1]
            marks = []

            def hook(it, loss, ev):
                e = torch.cuda.Event(enable_timing=True)
                e.record()
                marks.append(e)
            train.train_coarse(raw, views, knn_idx, mode=mode, spatial_extent=extent, num_iterations=warm + iters,
                               prune_at=(), reset_neighbors_every=big, n_samples=samples, on_iteration=hook, **sched)
            torch.cuda.synchronize()
            dts = [marks[i].elapsed_time(marks[i + 1]) for i in range(warm, len(marks) - 1)]
            r = {"train_coarse": mode, "phase": phase, "P": P, "image": f"{W}x{H}", "samples": samples,
                 "iteration_ms": round(median(dts), 2), "all_ms": [round(t, 2) for t in dts]}
            print(json.dumps(r))
            out.append(r)
            del raw, knn_idx
            torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--no-train", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_optim.py needs a CUDA device")
    info = {"card": card()}
    print(json.dumps(info))
    res = []
    for label, P, bound, V in (("unbound 1M", 1_000_000, False, 0), ("unbound 3M", 3_000_000, False, 0),
                               ("bound 500k x 6", 3_000_000, True, 250_000)):
        raw = make_params(P, bound, V)
        res.append(bench_step(label, raw, a.iters, a.rounds, bound))
        del raw
        torch.cuda.empty_cache()
    info["step"] = res
    if not a.no_train:
        info["train"] = bench_train()
    info["card_after"] = card()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(info, f, indent=1)


if __name__ == "__main__":
    main()
