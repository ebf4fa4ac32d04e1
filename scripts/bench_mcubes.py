#!/usr/bin/env python
"""Time the marching-cubes extraction (sugar_b200/mcubes.py): the density grid, marching cubes and the whole driver.

    python scripts/bench_mcubes.py [--P 1000000 3000000] [--R 256 512] [--repeats 3] [--composed-512]

Workloads: scenes.make_scene(P) clouds (z in [2, 10], about 17% outside a 60-degree frustum laterally, 2% near the
camera), camera extent e = 10, the reference's grids: foreground torch.linspace(-1, 1, R) * e, background * 4 e with
the foreground box zeroed, surface level 0.3.  Arms, CUDA events around one call after one warm-up call, `repeats`
rounds, the median printed:
    density_fg / density_bg   mcubes.density_grid on the foreground / background grid
    marching_cubes            mcubes.marching_cubes of the foreground volume (includes its one host read)
    driver                    mcubes.extract_mesh_marching_cubes at resolution R (both grids, colours, normals)
    composed                  this package's knn.knn_points + field.compute_density over the foreground grid's points
                              in the reference's 2M-point passes (R = 256; R = 512 with --composed-512)
Rates are voxels per second.  Every line carries the card's name, power limit and max SM clock, read in the same run.
Prints only; writes nothing.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_meshloss import card, median  # noqa: E402

EXTENT, LEVEL = 10.0, 0.3


def time_ms(torch, fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def composed(torch, pts, sc, q, st, X):
    from sugar_b200 import field, knn
    xx, yy, zz = torch.meshgrid(X, X, X, indexing="ij")
    grid = torch.cat([xx.reshape(-1, 1), yy.reshape(-1, 1), zz.reshape(-1, 1)], dim=-1)
    out = []
    for i in range(0, grid.shape[0], 2_000_000):
        g = grid[i:i + 2_000_000].cuda()
        out.append(field.compute_density(g, knn.knn_points(g, pts, 16)[1], pts, sc, q, st))
    return torch.cat(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--P", type=int, nargs="+", default=[1_000_000, 3_000_000])
    ap.add_argument("--R", type=int, nargs="+", default=[256, 512])
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--composed-512", action="store_true")
    args = ap.parse_args()
    import torch
    from sugar_b200 import mcubes, scenes
    info = card()
    for P in args.P:
        sc_ = scenes.make_scene(P, 1920, 1080, seed=0)
        t = lambda a: torch.from_numpy(a).cuda()
        pts, sc, q, st, sh = t(sc_.means3D), t(sc_.scales), t(sc_.rotations), t(sc_.opacities), t(sc_.shs[:, 0])
        for R in args.R:
            Xf = torch.linspace(-1, 1, R) * EXTENT
            Xb = torch.linspace(-1, 1, R) * 4 * EXTENT
            arms = {
                "density_fg": lambda: mcubes.density_grid(pts, sc, q, st, Xf, Xf, Xf),
                "density_bg": lambda: mcubes.density_grid(pts, sc, q, st, Xb, Xb, Xb, exclude_box=EXTENT),
                "driver": lambda: mcubes.extract_mesh_marching_cubes(pts, sc, q, st, sh, EXTENT, resolution=R,
                                                                     surface_level=LEVEL),
            }
            vol = mcubes.density_grid(pts, sc, q, st, Xf, Xf, Xf)
            arms["marching_cubes"] = lambda: mcubes.marching_cubes(vol, LEVEL)
            if R == 256 or args.composed_512:
                arms["composed"] = lambda: composed(torch, pts, sc, q, st, Xf)
            ms = {k: [] for k in arms}
            for k, fn in arms.items():
                fn()
                torch.cuda.synchronize()
            for _ in range(args.repeats):
                for k, fn in arms.items():
                    ms[k].append(time_ms(torch, fn))
                    print(f"P={P} R={R} {k}: {ms[k][-1]:.2f} ms", file=sys.stderr, flush=True)   # long arms: progress
            nvox = R ** 3
            if "composed" in arms:
                want = composed(torch, pts, sc, q, st, Xf)
                same = float((want == vol.reshape(-1)).float().mean())
            else:
                same = None
            v, f = mcubes.marching_cubes(vol, LEVEL)
            bgv = mcubes.density_grid(pts, sc, q, st, Xb, Xb, Xb, exclude_box=EXTENT)
            print(json.dumps({
                "P": P, "R": R, "ms": {k: round(median(x), 2) for k, x in ms.items()},
                "ms_all": {k: [round(y, 2) for y in x] for k, x in ms.items()},
                "gvoxels_per_s": {k: round(nvox / median(x) / 1e6, 3) for k, x in ms.items() if k != "driver"},
                "fg_mesh": [int(v.shape[0]), int(f.shape[0])], "bg_nonzero_voxels": int((bgv > 0).sum()),
                "composed_bit_identical_fraction": same, "card": info}), flush=True)
            del vol, bgv, v, f
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
