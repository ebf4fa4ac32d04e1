"""Colour + depth in one rasterizer call (sugar_b200/depth.py) against the two calls it replaces, timed with CUDA events.

    python scripts/bench_depth.py [--out results.json] [--rounds 3] [--iters 20]

1. forward + backward of "RGB call + depth call" against one rasterize_with_depth call, at 3M Gaussians / 1080p
   SH 3 and 1M Gaussians / 1080p SH 3;
2. the blend kernels of each arm (libsugar_b200's per-kind event profile, one call's worth);
3. steps.coarse_sdf_step at 1M Gaussians / 1080p with fused_depth False against True.

The arms alternate inside each round; each number is reported as min-max over the rounds.  The card's name, power
limit and SM clock are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:   # the numbers stand without it, but say so
        return f"unknown ({e})"


def timed(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def raster_arms(P, W, H):
    from sugar_b200 import depth, diff_gaussian_rasterization as dgr, scenes
    sc = scenes.make_scene(P, W, H, seed=0)
    t = {k: torch.from_numpy(np.ascontiguousarray(getattr(sc, k))).cuda()
         for k in ("means3D", "scales", "rotations", "opacities", "shs", "viewmatrix", "projmatrix", "campos")}
    leaf = lambda x: x.clone().requires_grad_(True)
    L = {k: leaf(t[k]) for k in ("means3D", "scales", "rotations", "opacities", "shs")}
    dL = torch.from_numpy(scenes.upstream_grad(W, H, seed=1)).cuda()
    dD = torch.from_numpy(scenes.upstream_grad(W, H, seed=2)[0]).cuda()

    def st(bg, deg):
        return dgr.GaussianRasterizationSettings(
            image_height=H, image_width=W, tanfovx=sc.tanfovx, tanfovy=sc.tanfovy, bg=bg, scale_modifier=1.0,
            viewmatrix=t["viewmatrix"], projmatrix=t["projmatrix"], sh_degree=deg, campos=t["campos"],
            prefiltered=False, debug=False)

    def values():
        return (L["means3D"] @ t["viewmatrix"][:3, :3] + t["viewmatrix"][3, :3])[:, 2]
    zero3 = torch.zeros(3, device="cuda")

    def two():
        z = values()
        zmax = z.max().detach()
        m2a = torch.zeros_like(L["means3D"], requires_grad=True)
        img, _ = dgr.GaussianRasterizer(st(zero3, 3))(means3D=L["means3D"], means2D=m2a, opacities=L["opacities"],
                                                      shs=L["shs"], scales=L["scales"], rotations=L["rotations"])
        m2b = torch.zeros_like(L["means3D"], requires_grad=True)
        d = dgr.GaussianRasterizer(st(zmax + zero3, 0))(means3D=L["means3D"], means2D=m2b, opacities=L["opacities"],
                                                        colors_precomp=z[:, None].expand(-1, 3), scales=L["scales"],
                                                        rotations=L["rotations"])[0][0]
        ((img * dL).sum() + (d * dD).sum()).backward()

    def one():
        z = values()
        m2 = torch.zeros_like(L["means3D"], requires_grad=True)
        img, d, _ = depth.rasterize_with_depth(L["means3D"], m2, L["opacities"], z, st(zero3, 3), z.max().detach(),
                                               shs=L["shs"], scales=L["scales"], rotations=L["rotations"])
        ((img * dL).sum() + (d * dD).sum()).backward()
    return two, one


def kernel_profile(fn):
    from sugar_b200 import _lib
    torch.cuda.synchronize()
    _lib.profile(True)
    fn()
    torch.cuda.synchronize()
    prof = _lib.profile_read()
    _lib.profile(False)
    return {k: v for k, v in prof.items() if k in ("blend_forward", "blend_backward", "preprocess",
                                                      "preprocess_backward", "scatter", "tile_sort_smem",
                                                      "tile_sort_global", "tile_scan")}


def step_arms(P, W, H):
    from sugar_b200 import knn, scenes, steps
    sc = scenes.make_scene(P, W, H, seed=0)
    dev = torch.device("cuda")
    cam = steps.camera_from_scene(sc, dev)
    gt = torch.rand(3, H, W, generator=torch.Generator().manual_seed(0)).to(dev)
    leaf = lambda x: x.to(dev).requires_grad_(True)
    raw = dict(points=leaf(torch.from_numpy(sc.means3D)), sh_dc=leaf(torch.from_numpy(sc.shs[:, :1].copy())),
               sh_rest=leaf(torch.from_numpy(sc.shs[:, 1:].copy())),
               densities=leaf(torch.logit(torch.from_numpy(sc.opacities).clamp(1e-4, 1 - 1e-4))),
               scales=leaf(torch.from_numpy(sc.scales).log()), quaternions=leaf(torch.from_numpy(sc.rotations) * 1.3))
    knn_idx = knn.reset_neighbors(raw["points"].detach(), 16)[1]
    ops = steps.ours_ops()
    g = torch.Generator(device=dev)

    def arm(fused):
        def run():
            g.manual_seed(1)
            steps.coarse_sdf_step(raw, cam, gt, knn_idx, ops, n_samples=1_000_000, generator=g, fused_depth=fused)
            for v in raw.values():
                v.grad = None
        return run
    return arm(False), arm(True)


def compare(arms, rounds, iters, warmup=3):
    for fn in arms.values():
        for _ in range(warmup):
            fn()
    torch.cuda.synchronize()
    res = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():   # alternate the arms inside each round
            res[k].append(timed(fn, iters))
    return {k: [round(min(v), 4), round(max(v), 4)] for k, v in res.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_depth.py measures on the GPU; there is no CPU path"
    out = {"card (name, power limit, max SM clock, SM clock)": card(), "unit": "ms per call, min-max over rounds"}
    for name, (P, W, H) in (("3M_1080p_sh3", (3_000_000, 1920, 1080)), ("1M_1080p_sh3", (1_000_000, 1920, 1080))):
        two, one = raster_arms(P, W, H)
        out[f"fwd+bwd {name}"] = compare({"rgb call + depth call": two, "fused call": one}, args.rounds, args.iters)
        out[f"kernels {name} (ms, launches)"] = {"rgb call + depth call": kernel_profile(two),
                                                 "fused call": kernel_profile(one)}
        del two, one
        torch.cuda.empty_cache()
        print(json.dumps(out, indent=1), flush=True)
    plain, fused = step_arms(1_000_000, 1920, 1080)
    out["coarse_sdf_step 1M_1080p"] = compare({"fused_depth=False": plain, "fused_depth=True": fused}, args.rounds,
                                              max(args.iters // 4, 3))
    out["card after"] = card()
    print(json.dumps(out, indent=1))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
