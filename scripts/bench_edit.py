"""Edited binding and composited frames at the reference's two refinement presets: 400k faces x 6 Gaussians
(`--low_poly`) and 2M faces x 1 (`--high_poly`), bound to a height field posed by a per-vertex jitter, 1600x1200.

    python scripts/bench_edit.py [--reps 7] [--iters 20] [--json out.json]

Arms, alternated in one process, CUDA events around `--iters` calls, median over `--reps` rounds:
  fused         one sgr_meshbind_edited_forward launch into preallocated buffers
  fused_rows    the same through an out_rows map that renders every Gaussian (per-thread stores)
  torch         the oracle's float32 PyTorch chain (oracle/editmesh_oracle.py, the reference's ops) on the GPU
  colors        one sgr_sh_colors_rotated launch over all rows (SH degree 3, M = 16)
  render        Composition.render, one bound part, sh_rotations None (in-kernel SH)
  render_rot    Composition.render with an sh_rotation (precomputed colours)
Achieved GB/s against the least traffic: edited binding 96 B per face (three current and three reference vertices, the
face's ids) + 56 B per Gaussian (two raw pairs in; point, scaling and quaternion out), 72 B with out_rows; rotated
colours 12 + 12 M + 12 B per Gaussian.  The card's name, power limit and max SM clock are read in the same run.  Needs a
GPU.
"""
import argparse
import json
import math
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import editmesh_oracle as eo  # noqa: E402
from sugar_b200 import compose, meshbind, scenes  # noqa: E402

PRESETS = {"low_poly_400k_x6": (448, 6), "high_poly_2m_x1": (1001, 1)}   # grid side -> F = 2 (side - 1)^2
W, H, M = 1600, 1200, 16


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    return out[torch.cuda.current_device()] if out else torch.cuda.get_device_name()


def model(side, n_per, seed=0):
    ref, faces = scenes.height_field_mesh(side, side, seed=seed)
    cur = eo.deform("jitter", ref.astype(np.float64), faces, seed).astype(np.float32)
    F = faces.shape[0]
    P = F * n_per
    g = torch.Generator(device="cuda").manual_seed(seed)
    edge = 1.0 / (side - 1)
    return dict(verts=torch.from_numpy(ref).cuda(), posed=torch.from_numpy(cur).cuda(), faces=torch.from_numpy(faces).cuda(),
                bary=meshbind.bary_coords(n_per, "cuda"),
                scales_raw=torch.randn(P, 2, device="cuda", generator=g) * 0.3 + math.log(0.5 * edge / math.sqrt(n_per)),
                complex_raw=torch.randn(P, 2, device="cuda", generator=g), thickness=1e-5,
                densities=torch.randn(P, 1, device="cuda", generator=g) + 1.0,
                sh=0.3 * torch.randn(P, M, 3, device="cuda", generator=g))


def timed(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def bench(name, side, n_per, reps, iters):
    m = model(side, n_per)
    F, P = m["faces"].shape[0], m["scales_raw"].shape[0]
    a = meshbind.edited_args(m["posed"], m["verts"], m["faces"], m["bary"], m["scales_raw"], m["complex_raw"],
                             m["thickness"])
    pts, scl, qts = torch.empty(P, 3, device="cuda"), torch.empty(P, 3, device="cuda"), torch.empty(P, 4, device="cuda")
    rows = torch.arange(P, device="cuda")          # every Gaussian rendered, through the map
    comp = compose.Composition([{k: m[k] for k in ("verts", "faces", "bary", "scales_raw", "complex_raw", "thickness",
                                                   "densities", "sh")}])
    c2w = torch.eye(4)
    c2w[:3, 3] = torch.tensor([0.5, 0.5, 1.6])            # above the unit square, looking down -z
    fov_x = 2 * math.atan(0.36)
    fov_y = 2 * math.atan(0.36 * H / W)
    R = eo.rotation([0.2, 1.0, 0.1], 0.7)
    campos = torch.tensor([0.5, 0.5, 1.6], device="cuda")
    group_start = torch.tensor([0, P], device="cuda")
    group_rot = R.reshape(1, 9).cuda()
    colors = torch.empty(P, 3, device="cuda")
    arms = {
        "fused": lambda: meshbind.edited_launch(a, pts, scl, qts),
        "fused_rows": lambda: meshbind.edited_launch(a, pts, scl, qts, rows),
        "torch": lambda: eo.edited_bind_torch(m["posed"], m["verts"], m["faces"], m["bary"], m["scales_raw"],
                                              m["complex_raw"], m["thickness"]),
        "colors": lambda: compose._colors_launch(P, M, 3, pts, m["sh"], campos, 1, group_start, group_rot, colors),
        "render": lambda: comp.render(c2w, fov_x, fov_y, H, W, verts=[m["posed"]]),
        "render_rot": lambda: comp.render(c2w, fov_x, fov_y, H, W, verts=[m["posed"]], sh_rotations=[R]),
    }
    with torch.no_grad():
        for fn in arms.values():       # warm-up: module load, allocator, the rasterizer's capacity hint
            fn(), fn()
        torch.cuda.synchronize()
        ms = {k: [] for k in arms}
        for _ in range(reps):
            for k, fn in arms.items():
                ms[k].append(timed(fn, iters if not k.startswith("render") else max(iters // 4, 3)))
        # outputs of the timed arms: the fused kernel against the float32 chain it replaces
        meshbind.edited_launch(a, pts, scl, qts)
        p32, s32, q32 = eo.edited_bind_torch(m["posed"], m["verts"], m["faces"], m["bary"], m["scales_raw"],
                                             m["complex_raw"], m["thickness"])
        p64, s64, q64 = eo.edited_bind_torch(*(m[k].double() if m[k].is_floating_point() else m[k] for k in
                                               ("posed", "verts", "faces", "bary", "scales_raw", "complex_raw")),
                                             m["thickness"])
        diff = {}
        for name_, (x, y, z) in dict(points=(pts, p32, p64), scaling=(scl, s32, s64), quaternions=(qts, q32, q64)).items():
            def d(u, v):   # max |u - v| / max |v|; q and -q are one rotation
                e = (u.double() - v.double()).abs()
                if name_ == "quaternions":
                    e = torch.minimum(e.amax(-1), (u.double() + v.double()).abs().amax(-1))
                return float(e.max() / v.abs().max())
            diff[name_] = dict(fused_vs_torch32=d(x, y), fused_vs_fp64=d(x, z), torch32_vs_fp64=d(y, z))
        covered = float((comp.render(c2w, fov_x, fov_y, H, W, verts=[m["posed"]]).sum(-1) > 0).float().mean())
    med = {k: float(np.median(v)) for k, v in ms.items()}
    spread = {k: [float(min(v)), float(max(v))] for k, v in ms.items()}
    bytes_bind, bytes_rows, bytes_col = 96 * F + 56 * P, 96 * F + 72 * P, (12 + 12 * M + 12) * P
    res = dict(preset=name, faces=F, gaussians=P, ms=med, ms_min_max=spread,
               gbps=dict(fused=bytes_bind / med["fused"] / 1e6, fused_rows=bytes_rows / med["fused_rows"] / 1e6,
                         colors=bytes_col / med["colors"] / 1e6),
               speedup_vs_torch=med["torch"] / med["fused"], rel_diff=diff, image_coverage=covered)
    print(f"{name}: F={F} P={P}")
    for k in arms:
        print(f"  {k:11s} {med[k]:8.3f} ms  (min {spread[k][0]:.3f}, max {spread[k][1]:.3f})")
    print(f"  fused {res['gbps']['fused']:.0f} GB/s, with out_rows {res['gbps']['fused_rows']:.0f} GB/s, colours "
          f"{res['gbps']['colors']:.0f} GB/s (of 3350); {res['speedup_vs_torch']:.1f}x the float32 torch chain; "
          f"{100 * covered:.0f} % of pixels covered")
    for k, v in diff.items():
        print(f"  {k:11s} max rel diff: " + ", ".join(f"{a} {b:.2e}" for a, b in v.items()))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_edit.py needs a GPU"
    gpu = card()
    print("card (name, power limit, max SM clock):", gpu)
    out = dict(card=gpu, width=W, height=H, results=[bench(k, side, n, args.reps, args.iters)
                                                     for k, (side, n) in PRESETS.items()])
    line = json.dumps(out)
    print(line)
    if args.json:
        with open(args.json, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
