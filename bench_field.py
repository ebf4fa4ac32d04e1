#!/usr/bin/env python
"""Secondary benchmark: SuGaR density/SDF field (get_field_values) forward+backward.

    python bench_field.py [--gaussians 1000000] [--samples 1000000] [--k 16] [--steps 20]

BASELINE.md section 2 "B-cpu-density" / config 1 and 3: fused sugar_b200 kernels vs the reference's op chain
(restated in oracle/field_oracle.py) run with PyTorch on the same GPU and on the host cores (bounded sample).
Prints one JSON line.  The headline benchmark is bench.py.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gaussians", type=int, default=1_000_000)
    ap.add_argument("--samples", type=int, default=1_000_000)
    ap.add_argument("--k", type=int, default=16)
    ap.add_argument("--steps", type=int, default=20)
    a = ap.parse_args()
    import torch
    from oracle import field_oracle as fo
    from sugar_b200 import field, _lib
    dev = torch.device("cuda")
    P, N, K = a.gaussians, a.samples, a.k
    g = torch.Generator(device="cpu").manual_seed(0)
    points = torch.randn(P, 3, generator=g).to(dev)
    scaling = torch.exp(torch.randn(P, 3, generator=g) * 0.5 - 4.0).to(dev)
    quats = torch.nn.functional.normalize(torch.randn(P, 4, generator=g), dim=-1).to(dev)
    strengths = torch.sigmoid(torch.randn(P, generator=g) * 2).to(dev)
    # neighbours as the trainer has them (sugar_model.py:1013-1030, coarse_sdf.py:631): the exact K-NN table of the
    # cloud against itself (self is neighbour 0), looked up at the Gaussian each sample was drawn in -- the gather
    # locality of the field kernels is the trainer's, not that of random "nearby" indices
    from sugar_b200 import knn
    _, knn_idx = knn.reset_neighbors(points, K)
    gi = torch.randint(0, P, (N,), generator=g).to(dev)
    nbr = knn_idx[gi].contiguous()
    x = points[gi] + fo.quaternion_apply(quats[gi], 1.5 * scaling[gi] * torch.randn(N, 3, generator=g).to(dev))
    leaves = [t.clone().requires_grad_(True) for t in (x, points, scaling, quats, strengths)]
    w = torch.randn(N, device=dev)

    def ours():
        f = field.field_values(leaves[0], nbr, *leaves[1:], density_factor=1.0 / K, return_sdf=True,
                               return_closest_gaussian_opacities=True, return_beta=True)
        (f["sdf"] * w).sum().backward()
        for t in leaves:
            t.grad = None

    def torch_ref():
        f = fo.field_values_torch(leaves[0], nbr, *leaves[1:], density_factor=1.0 / K)
        (f["sdf"] * w).sum().backward()
        for t in leaves:
            t.grad = None

    def timeit(fn, steps):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / steps

    _lib.profile(True)
    ours(); torch.cuda.synchronize(); _lib.profile_read()
    ms = timeit(ours, a.steps)
    prof = _lib.profile_read()
    _lib.profile(False)
    ms_ref = timeit(torch_ref, max(3, a.steps // 4))
    # CPU: the same op chain on the host cores, bounded sample
    ns = min(N, 100_000)
    cl = [t.detach().cpu()[:ns].clone().requires_grad_(True) if i == 0 else t.detach().cpu().clone().requires_grad_(True)
          for i, t in enumerate(leaves)]
    nbr_c, w_c = nbr[:ns].cpu(), w[:ns].cpu()
    torch.set_num_threads(os.cpu_count())
    t0 = time.perf_counter()
    f = fo.field_values_torch(cl[0], nbr_c, *cl[1:], density_factor=1.0 / K)
    (f["sdf"] * w_c).sum().backward()
    cpu_s = time.perf_counter() - t0
    # K-NN table build (reset_neighbors): cloud against itself
    from sugar_b200 import knn
    for _ in range(2):
        knn.reset_neighbors(points, K)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(5):
        kd, ki = knn.reset_neighbors(points, K)
    e1.record()
    torch.cuda.synchronize()
    knn_ms = e0.elapsed_time(e1) / 5
    # "better normal" loss (coarse_sdf.py:688-716): fused kernels vs the reference's op chain on the same GPU
    with torch.no_grad():
        opac = field.field_values(x, nbr, points, scaling, quats, strengths, density_factor=1.0 / K,
                                  return_closest_gaussian_opacities=True)["closest_gaussian_opacities"]
    ql = quats.clone().requires_grad_(True)

    def normal_ours():
        field.better_normal_loss(x, gi, nbr, points, scaling, ql, opac).mean().backward()
        ql.grad = None

    def normal_ref():
        fo.better_normal_loss_torch(x, gi, nbr, points, scaling, ql, opac).mean().backward()
        ql.grad = None
    nl_ms, nl_ref_ms = timeit(normal_ours, a.steps), timeit(normal_ref, max(3, a.steps // 4))
    # level-set ray sampling (sugar_model.py:1970-2081): N rays x 21 samples, 3 levels + normals
    try:
        from sugar_b200 import levelset
        cam = torch.tensor([0.0, 0.0, -8.0], device=dev)

        def ls():
            return levelset.level_surface_points(x, cam, nbr, points, scaling, quats, strengths, density_factor=1.0,
                                                 return_normals=True)
        ls_ms = timeit(ls, max(3, a.steps // 4))
        ls_out = ls()
        levelset_res = {"ms": ls_ms, "rays": N, "samples_per_ray": 21, "rays_per_s": N / (ls_ms * 1e-3),
                        "valid_at_0.3": int(ls_out[0.3]["valid"].sum())}
    except Exception as e:  # keep the line printable
        levelset_res = {"error": repr(e)[:200]}
    fwd_bytes = N * (12 + 8 * K + 48 * K)
    stages = {k: {"ms": round(v[0] / v[1], 4)} for k, v in prof.items()}
    if "field_forward" in stages:
        stages["field_forward"]["gbs"] = round(fwd_bytes / (stages["field_forward"]["ms"] * 1e-3) / 1e9, 1)
    print(json.dumps({
        "metric": "density/SDF field samples/sec fwd+bwd", "value": N / (ms * 1e-3), "unit": "samples/s",
        "ms_per_step": ms, "config": {"workload": f"{P} Gaussians, {N} samples, K={K}"},
        "torch_same_gpu": {"value": N / (ms_ref * 1e-3), "ms_per_step": ms_ref},
        "cpu_baseline": {"value": ns / cpu_s, "unit": "samples/s", "cores": os.cpu_count(), "kind": "port",
                         "sample": f"{ns} samples of the workload, PyTorch op chain of sugar_model.py:1247-1316"},
        "knn_reset_neighbors": {"ms": knn_ms, "points_per_s": P / (knn_ms * 1e-3), "K": K,
                                "note": "exact K-NN of the cloud against itself (uniform grid), replaces pytorch3d.knn_points"},
        "level_set_sampling": levelset_res,
        "better_normal_loss": {"ms_fwd_bwd": nl_ms, "torch_same_gpu_ms": nl_ref_ms, "samples_per_s": N / (nl_ms * 1e-3)},
        "stages": stages}))


if __name__ == "__main__":
    main()
