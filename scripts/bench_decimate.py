#!/usr/bin/env python
"""Time the quadric decimation (sugar_b200/decimate.py) on the meshes the coarse-mesh extraction hands it.

    python scripts/bench_decimate.py [--R 256 512] [--targets 1000000 200000] [--repeats 3] [--no-model]

Workloads: marching cubes (mcubes.marching_cubes) of analytic volumes on [-1, 1]^3 at R^3 -- a sphere (radius 0.7), a
torus (0.6 / 0.25), noisy blobs (six Gaussians plus 2% noise) and a
sphere of radius 0.8 with a cavity of radius 0.5 holding a torus (0.3 / 0.1) -- and the foreground mesh of
mcubes.extract_mesh_marching_cubes for a scenes.make_scene(1M) cloud (extent 10, surface level 0.3) at R = 256.  Each
mesh is decimated to each target below its face count: CUDA events around one whole simplify_quadric_decimation call
(host reads included) after one warm-up call, `repeats` calls, the median printed, with the number of rounds, the input
faces per second, the mean time per round and the clean_mesh time.  open3d's time is not measured: open3d is not
available on the machines this package is built for, and the Python greedy loop of oracle/decimate_oracle.py is not a
fair stand-in for it.  Every line carries the card's name, power limit and max SM clock, read in the same run.
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
from bench_mcubes import time_ms  # noqa: E402


def volume(torch, kind, R):
    g = torch.linspace(-1, 1, R, device="cuda")
    X, Y, Z = torch.meshgrid(g, g, g, indexing="ij")
    if kind == "sphere":
        return (0.7 - torch.sqrt(X ** 2 + Y ** 2 + Z ** 2)).contiguous()
    if kind == "shell_torus":       # the GPU test's mesh: spheres of radius 0.8 and 0.5 and a torus inside
        r = torch.sqrt(X ** 2 + Y ** 2 + Z ** 2)
        torus = 0.1 - torch.sqrt((torch.sqrt(X ** 2 + Y ** 2) - 0.3) ** 2 + Z ** 2)
        return torch.maximum(torch.minimum(0.8 - r, r - 0.5), torus).contiguous()
    if kind == "torus":
        return (0.25 - torch.sqrt((torch.sqrt(X ** 2 + Y ** 2) - 0.6) ** 2 + Z ** 2)).contiguous()
    gen = torch.Generator(device="cuda").manual_seed(0)
    c = torch.rand(6, 3, generator=gen, device="cuda") - 0.5
    f = torch.full_like(X, -0.5)
    for x, y, z in c.tolist():
        f += torch.exp(-((X - x) ** 2 + (Y - y) ** 2 + (Z - z) ** 2) / 0.06)
    return (f + 0.02 * torch.randn(f.shape, generator=gen, device="cuda")).contiguous()


def meshes(torch, args):
    from sugar_b200 import mcubes, scenes
    for R in args.R:
        for kind in ("sphere", "torus", "blobs", "shell_torus"):
            vol = volume(torch, kind, R)
            vi, faces = mcubes.marching_cubes(vol, 0.0)
            del vol
            yield f"{kind}_R{R}", vi * (2.0 / (R - 1)) - 1.0, faces, None, None
    if not args.no_model:
        sc = scenes.make_scene(1_000_000, 1920, 1080, seed=0)
        t = lambda a: torch.from_numpy(a).cuda()
        m = mcubes.extract_mesh_marching_cubes(t(sc.means3D), t(sc.scales), t(sc.rotations), t(sc.opacities),
                                               t(sc.shs[:, 0]), 10.0, resolution=256)["foreground"]
        yield "model_1M_R256_fg", m["verts"], m["faces"], m["colors"], m["normals"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--R", type=int, nargs="+", default=[256, 512])
    ap.add_argument("--targets", type=int, nargs="+", default=[1_000_000, 200_000])
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--no-model", action="store_true")
    args = ap.parse_args()
    import torch
    from sugar_b200 import decimate
    info = card()
    for name, verts, faces, colors, normals in meshes(torch, args):
        F = int(faces.shape[0])
        for target in args.targets:
            if target >= F:
                print(json.dumps({"mesh": name, "faces": F, "target": target, "skipped": "target >= faces",
                                  "card": info}), flush=True)
                continue
            call = lambda: decimate.simplify_quadric_decimation(verts, faces, target, colors, normals)
            m = call()
            torch.cuda.synchronize()
            ms = [time_ms(torch, call) for _ in range(args.repeats)]
            clean_ms = time_ms(torch, lambda: decimate.clean_mesh(m["verts"], m["faces"], m["colors"], m["normals"]))
            t = median(ms)
            print(json.dumps({
                "mesh": name, "verts": int(verts.shape[0]), "faces": F, "target": target,
                "faces_out": int(m["faces"].shape[0]), "rounds": m["rounds"], "ms": round(t, 2),
                "ms_all": [round(x, 2) for x in ms], "ms_per_round": round(t / max(m["rounds"], 1), 3),
                "mfaces_per_s": round(F / t / 1e3, 2), "clean_mesh_ms": round(clean_ms, 2), "card": info}), flush=True)
        del verts, faces, colors, normals
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
