"""Screened-Poisson reconstruction at the reference's point budget: 10M oriented samples on a synthetic surface (a
sphere with a torus through it, normals out) at depths 8, 9 and 10.

    python scripts/bench_poisson.py [--n 10000000] [--depths 8 9 10] [--json out.json]

Per depth: the time of each stage from CUDA events (binning, splat, coarse-q pyramid and |b|, each V-cycle, iso-value,
marching cubes, the density grid of depth - 2, the nearest sample of every vertex, colour, trim), the cycle count and final residual ratio, the peak
torch.cuda.max_memory_allocated, and the card's name and power limit read in the same run.  A second, profiled solve
gives the splat and red-black smoother kernels' times (torch.profiler); their bytes per pass are computed from the
shapes (the least traffic: each grid value read or written once, each sample record read once) and reported as a share
of the H100 SXM's 3.35 TB/s.  Needs a GPU.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from sugar_b200 import poisson  # noqa: E402

HBM = 3.35e12


def surface(n, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    m = n // 2
    d = torch.nn.functional.normalize(torch.randn(m, 3, device="cuda", generator=g), dim=-1)
    a = torch.rand(n - m, device="cuda", generator=g) * 2 * np.pi
    b = torch.rand(n - m, device="cuda", generator=g) * 2 * np.pi
    c = torch.stack([torch.cos(a), torch.zeros_like(a), torch.sin(a)], 1)
    tn = torch.cos(b)[:, None] * c + torch.sin(b)[:, None] * torch.tensor([0.0, 1.0, 0.0], device="cuda")
    pts = torch.cat([0.8 * d, c * 0.9 + 0.15 * tn + torch.tensor([0.5, 0.0, 0.0], device="cuda")])
    nrm = torch.cat([d, tn])
    col = torch.rand(n, 3, device="cuda", generator=g)
    return pts.contiguous(), nrm.contiguous(), col


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    return out[torch.cuda.current_device()] if out else torch.cuda.get_device_name()


def kernel_ms(depth, pts, nrm):
    """-> {kernel: [ms of each finest-level launch]} of one profiled solve: the system splat, and the smoother's
    finest-level launches (4 sweeps x 2 colours per V-cycle, the longest of its launches)."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        s = poisson.solve(pts, nrm, depth)
        torch.cuda.synchronize()
    cycles = s["cycles"]
    del s
    times = {"poi_splat_kernel": [], "poi_smooth_kernel": []}
    for e in prof.events():
        if "poi_splat_kernel<0>" in e.name:
            times["poi_splat_kernel"].append(e.time_range.elapsed_us() / 1000.0)
        elif "poi_smooth_kernel" in e.name:
            times["poi_smooth_kernel"].append(e.time_range.elapsed_us() / 1000.0)
    times["poi_smooth_kernel"] = sorted(times["poi_smooth_kernel"], reverse=True)[:8 * cycles]
    return times


def run(depth, pts, nrm, col):
    N, n = 1 << depth, pts.shape[0]
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    t = poisson._Timer(True)
    m = poisson.poisson_reconstruction(pts, nrm, depth=depth, colors=col, _timer=t)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    thr = poisson.quantile(m["densities"], 0.1)
    trimmed = poisson.remove_vertices_by_mask(m["verts"], m["faces"], m["densities"].double() < thr, m["colors"])
    e1.record()
    stages = t.stages() + [("trim", e0.elapsed_time(e1))]
    peak = torch.cuda.max_memory_allocated()
    res = {"depth": depth, "n": n, "stages_ms": stages, "cycles": m["cycles"], "residual": m["residual"],
           "verts": int(m["verts"].shape[0]), "faces": int(m["faces"].shape[0]),
           "verts_after_trim": int(trimmed["verts"].shape[0]), "peak_bytes": peak}
    del m, trimmed
    ms = kernel_ms(depth, pts, nrm)
    splat_bytes = N ** 3 * (4 + 8) + n * (16 + 12)           # ends read, b and q written; records and normals read
    smooth_bytes = N ** 3 // 2 * (4 + 4 + 4 + 4) + N ** 3 // 2 * 4   # one colour: u, b, q read, u written; other u read
    res["kernels"] = []
    for key, nbytes in (("poi_splat_kernel", splat_bytes), ("poi_smooth_kernel", smooth_bytes)):
        if ms[key]:
            per = float(np.median(ms[key]))
            res["kernels"].append({"kernel": key, "calls": len(ms[key]), "median_ms": per, "bytes_per_call": nbytes,
                                   "share_of_3.35TBps": nbytes / (per * 1e-3) / HBM})
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--depths", type=int, nargs="+", default=[8, 9, 10])
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_poisson.py needs a GPU")
    pts, nrm, col = surface(a.n)
    run(min(a.depths), pts, nrm, col)                          # warm-up: module loads, allocator
    out = {"card": card(), "runs": [run(d, pts, nrm, col) for d in a.depths]}
    print(json.dumps(out, indent=1))
    if a.json:
        with open(a.json, "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
