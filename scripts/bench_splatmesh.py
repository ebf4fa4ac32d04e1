#!/usr/bin/env python
"""Time the level-set extraction's mesh depth source (sugar_b200/splatmesh.py) and the whole per-view level-set call on
both depth sources.

    python scripts/bench_splatmesh.py [--sizes 1000000 3000000] [--iters 20] [--repeats 3] [--out DIR]

Scenes: scenes.make_scene(P, 1920, 1080, seed=0, camera='posed'), the knn_idx table (knn.reset_neighbors(points, 16))
built once outside the timed region.  Arms, CUDA events around `iters` calls, `repeats` rounds alternating the arms in
one process:
    splat_mesh      splatmesh.splat_mesh (the diamond vertices + the face table)
    rasterize_mesh  splatmesh.rasterize_mesh of that mesh (includes the one host read of the face-id check)
    levelset_mesh   levelset.level_surface_points_from_camera(use_gaussian_depth=False, knn_idx=...)
    levelset_gauss  the same with use_gaussian_depth=True (blended depth + per-point K-NN), the existing path
There is no reference arm: pytorch3d is not available.  Per-kernel times come from a separate torch.profiler run of one
call of each of the first three arms (a chrome trace per size is written under --out, default a temporary directory).
Byte model (per call): splat_mesh_kernel 88 B per Gaussian (40 in, 48 out); mesh_setup_kernel 128 B per face (24 B ids,
36 B vertex gathers, 64 B record, 4 B piece count); mesh_fragment_kernel 64 B per piece + 16 B per candidate pixel (the
key read and at most one 8-byte atomic); mesh_resolve_kernel 20 B per pixel (+ 8 B for the memset of the keys).  HBM
shares are against the H100 SXM data sheet's 3.35 TB/s.  Every line carries the card's name, power limit and max SM
clock, read in the same run.
"""
import argparse
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_meshloss import card, median  # noqa: E402

PEAK_GBS = 3350.0


def time_ms(torch, fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def candidate_stats(torch, verts, faces, cam):
    """Faces that reach the setup's box stage, their clipped pixel boxes and 8x8 pieces (the fragment kernel's work)."""
    W, H = cam.width, cam.height
    v = verts.double()
    z = v @ cam.viewmatrix[:3, 2].double() + cam.viewmatrix[3, 2].double()
    hom = v @ cam.projmatrix[:3].double() + cam.projmatrix[3].double()
    x = ((hom[:, 0] / (hom[:, 3] + 1e-7) + 1) * W - 1) / 2
    y = ((hom[:, 1] / (hom[:, 3] + 1e-7) + 1) * H - 1) / 2
    X, Y, Z = x[faces], y[faces], z[faces]
    ok = torch.isfinite(X).all(1) & torch.isfinite(Y).all(1) & (Z.max(1).values >= 0)
    x0 = X.min(1).values.clamp(0, W).ceil()
    x1 = X.max(1).values.clamp(-1, W - 1).floor()
    y0 = Y.min(1).values.clamp(0, H).ceil()
    y1 = Y.max(1).values.clamp(-1, H - 1).floor()
    bw, bh = (x1 - x0 + 1).clamp(min=0), (y1 - y0 + 1).clamp(min=0)
    ok &= (bw > 0) & (bh > 0)
    cand = torch.where(ok, bw * bh, 0.0)
    pieces = torch.where(ok, torch.ceil(bw / 8) * torch.ceil(bh / 8), 0.0)
    return int(ok.sum()), int(cand.sum()), int(pieces.sum()), int(cand.max())


def profile_kernels(torch, arms, out_dir, tag):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for fn in arms.values():
            fn()
        torch.cuda.synchronize()
    prof.export_chrome_trace(os.path.join(out_dir, f"splatmesh_{tag}.pt.trace.json"))
    kern = {}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
        if t > 0 and ("mesh" in ev.key or "splat" in ev.key):
            name = ev.key.split("(")[0].split("::")[-1].split("<")[0]
            kern[name] = round(kern.get(name, 0.0) + t / 1e3, 4)
    return kern


def size_line(args, P, info):
    import torch
    from sugar_b200 import knn, levelset, scenes, splatmesh, steps
    sc = scenes.make_scene(P, 1920, 1080, seed=0, camera="posed")
    c = lambda a: torch.from_numpy(a).cuda()
    pts, scaling, quats, strengths = c(sc.means3D), c(sc.scales), c(sc.rotations), c(sc.opacities[:, 0])
    cam = steps.camera_from_scene(sc, "cuda")
    knn_idx = knn.reset_neighbors(pts, 16)[1]
    verts, faces = splatmesh.splat_mesh(pts, scaling, quats, cam)
    lv = lambda gd: levelset.level_surface_points_from_camera(pts, scaling, quats, strengths, cam,
                                                              use_gaussian_depth=gd, knn_idx=knn_idx)
    arms = {"splat_mesh": lambda: splatmesh.splat_mesh(pts, scaling, quats, cam),
            "rasterize_mesh": lambda: splatmesh.rasterize_mesh(verts, faces, cam),
            "levelset_mesh": lambda: lv(False), "levelset_gauss": lambda: lv(True)}
    iters = {"splat_mesh": args.iters, "rasterize_mesh": args.iters, "levelset_mesh": args.lv_iters,
             "levelset_gauss": args.lv_iters}
    for fn in arms.values():
        for _ in range(2):
            fn()
    ms = {k: [] for k in arms}
    for _ in range(args.repeats):
        for k, fn in arms.items():
            ms[k].append(round(time_ms(torch, fn, iters[k]), 4))
    zbuf, p2f = splatmesh.rasterize_mesh(verts, faces, cam)
    z2, f2 = splatmesh.rasterize_mesh(verts, faces, cam)
    n_faces, cand, pieces, cand_max = candidate_stats(torch, verts, faces, cam)
    kern = profile_kernels(torch, {k: arms[k] for k in ("splat_mesh", "rasterize_mesh", "levelset_mesh")},
                           args.out, f"{P}")
    F, npix = faces.shape[0], 1920 * 1080
    model = {"splat_mesh_kernel": 88 * P, "mesh_setup_kernel": 128 * F, "mesh_fragment_kernel": 64 * pieces + 16 * cand,
             "mesh_resolve_kernel": 20 * npix}
    # the profiled run calls rasterize_mesh twice (once directly, once inside levelset_mesh) and splat_mesh twice
    per_call = {k: round(v / 2, 4) for k, v in kern.items()}
    gbs = {k: round(model[k] / (per_call[k] * 1e-3) / 1e9, 1) for k in model if per_call.get(k)}
    print(json.dumps({
        "what": "splatted diamond mesh + nearest-face z-buffer, level-set per view", "gaussians": P, "faces": F,
        "image": "1920x1080", "iters": iters, "repeats": args.repeats, "ms": ms,
        "median_ms": {k: median(v) for k, v in ms.items()},
        "faces_boxed": n_faces, "candidate_pixels": cand, "pieces": pieces, "largest_box_pixels": cand_max,
        "covered_pixels": int((p2f >= 0).sum()),
        "deterministic": bool(torch.equal(zbuf, z2) and torch.equal(p2f, f2)),
        "kernels_ms_per_call": per_call, "model_bytes": model, "achieved_gbs": gbs,
        "hbm_frac_of_3350_gbs": {k: round(g / PEAK_GBS, 3) for k, g in gbs.items()}, "card": info}), flush=True)
    del verts, faces, knn_idx
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[1_000_000, 3_000_000])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--lv-iters", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    args.out = args.out or tempfile.mkdtemp(prefix="bench_splatmesh_")
    os.makedirs(args.out, exist_ok=True)
    info = card()
    for P in args.sizes:
        size_line(args, P, info)
    return 0


if __name__ == "__main__":
    sys.exit(main())
