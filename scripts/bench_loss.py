#!/usr/bin/env python
"""Time the fused L1 + D-SSIM loss (sugar_b200/loss.py) against the reference's PyTorch chain on the same tensors.

    python scripts/bench_loss.py [--iters 200] [--repeats 3] [--no-step]

One JSON line per image size (3 x 1920x1080, 3 x 1600x1200, 3 x 3840x2160): forward + backward of
0.8 L1 + 0.2 (1 - SSIM) per iteration, CUDA events, warm-up first, the two arms alternated in one process
(`repeats` rounds of `iters` iterations each), the fused op's per-kernel times from the library's event profiler, and
its achieved GB/s against the byte model:
    forward  reads img1, img2 (8 B) and writes the three partial-derivative maps (12 B) per element
    backward reads the maps (12 B) and img1, img2 (8 B) and writes dL/dimg1 (4 B) per element
    = 44 B per element, as a fraction of the HBM peak (MEASURED_PEAKS.json when present, else the H100 SXM data
    sheet's 3.35 TB/s, named as such).
Then one line for bench.py's coarse_sdf_step workload (1M Gaussians, 1920x1080) with dssim_factor 0.0 and 0.2 over
this package's ops, and with 0.2 over the reference's building blocks (oracle/_ref + the PyTorch chain) when
oracle/_ref is present; each arm runs in its own process.  Every line carries the card's name, power limit and max
SM clock, read in the same run.  Prints only; writes nothing.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
BYTES_PER_ELEMENT = 44
SIZES = [(1920, 1080), (1600, 1200), (3840, 2160)]


def card(index=0):
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i", str(index)],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return {"name": out[0].strip(), "power_limit_w": float(out[1]), "sm_max_mhz": float(out[2])}
    except Exception as ex:
        return {"error": repr(ex)}


def time_ms(torch, fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def loss_lines(args, info):
    import torch
    import bench
    from oracle import ssim_oracle as so
    from sugar_b200 import _lib, loss
    peak, peak_src = bench.load_peaks()
    dev = torch.device("cuda", 0)
    for W, H in SIZES:
        gen = torch.Generator(device=dev).manual_seed(W)
        coarse = torch.rand(1, 3, H // 16 + 2, W // 16 + 2, device=dev, generator=gen)
        gt = torch.nn.functional.interpolate(coarse, size=(H, W), mode="bilinear", align_corners=False)[0].contiguous()
        pred = (gt + 0.01 * (2 * torch.rand(gt.shape, device=dev, generator=gen) - 1)).requires_grad_(True)

        def step(fn):
            def run():
                fn(pred, gt, 0.2).backward()
                pred.grad = None
            return run
        arms = {"fused": step(loss.l1_dssim_loss), "reference_chain": step(so.l1_dssim_torch)}
        for fn in arms.values():
            for _ in range(20):
                fn()
        torch.cuda.synchronize()
        ms = {k: [] for k in arms}
        for _ in range(args.repeats):
            for k, fn in arms.items():
                ms[k].append(time_ms(torch, fn, args.iters))
        _lib.profile(True)
        time_ms(torch, arms["fused"], args.iters)
        prof = _lib.profile_read()
        _lib.profile(False)
        kern = {k: round(t / args.iters, 5) for k, (t, c) in prof.items()}
        n = 3 * W * H
        kms = sum(kern.values())
        gbs = BYTES_PER_ELEMENT * n / (kms * 1e-3) / 1e9 if kms else None
        print(json.dumps({
            "what": "L1 + D-SSIM forward+backward", "size": f"3x{H}x{W}", "iters": args.iters, "repeats": args.repeats,
            "fused_ms": [round(v, 4) for v in ms["fused"]], "reference_chain_ms": [round(v, 4) for v in ms["reference_chain"]],
            "speedup_median": round(sorted(ms["reference_chain"])[len(ms["reference_chain"]) // 2] /
                                    sorted(ms["fused"])[len(ms["fused"]) // 2], 2),
            "fused_kernels_ms": kern, "model_bytes": BYTES_PER_ELEMENT * n,
            "achieved_gbs": round(gbs, 1) if gbs else None, "hbm_frac": round(gbs / peak, 3) if gbs else None,
            "peak_gbs": peak, "peak_source": peak_src, "card": info}), flush=True)


def step_arm(impl, factors, repeats, n_steps):
    """One process per arm: coarse_sdf_step at bench.py's workload size, the factors alternated."""
    import numpy as np
    import torch
    import bench
    import bench_workloads as bw
    cfg = bw.WORKLOADS["coarse_sdf_step"]
    dev = torch.device("cuda", 0)
    P, W, H = cfg["P"], cfg["W"], cfg["H"]
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    scenes = bench.load_scenes()
    if impl == "reference":
        import helpers as h
        if not h.have_ref():
            return {"impl": impl, "unavailable": "oracle/_ref (reference CUDA build) is not present"}
        ops = bw.reference_ops(torch, h.load_ref_module())
        steps = bw._load_steps_without_package()
    else:
        from sugar_b200 import steps
        ops = steps.ours_ops()
    g = torch.Generator().manual_seed(0)
    sc = scenes.make_scene(P, W, H, seed=0)
    cam = steps.camera_from_scene(sc, dev)
    gt = torch.rand(3, H, W, generator=g).to(dev)
    leaf = lambda t: t.to(dev).requires_grad_(True)
    raw = dict(points=leaf(torch.from_numpy(sc.means3D)), sh_dc=leaf(torch.from_numpy(sc.shs[:, :1].copy())),
               sh_rest=leaf(torch.from_numpy(sc.shs[:, 1:].copy())),
               densities=leaf(torch.logit(torch.from_numpy(sc.opacities).clamp(1e-4, 1 - 1e-4))),
               scales=leaf(torch.from_numpy(sc.scales).log()), quaternions=leaf(torch.from_numpy(sc.rotations) * 1.3))
    if impl == "reference":
        from scipy.spatial import cKDTree
        knn_idx = torch.from_numpy(cKDTree(sc.means3D).query(sc.means3D, k=cfg["K"], workers=-1)[1].astype(np.int64)).to(dev)
    else:
        from sugar_b200 import knn
        knn_idx = knn.reset_neighbors(raw["points"].detach(), cfg["K"])[1]
    sgen = torch.Generator(device=dev)

    def make(f):
        def run():
            sgen.manual_seed(1)
            steps.coarse_sdf_step(raw, cam, gt, knn_idx, ops, n_samples=cfg["samples"], generator=sgen, dssim_factor=f)
            for t in raw.values():
                t.grad = None
        return run
    runs = {f: make(f) for f in factors}
    for fn in runs.values():
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    ms = {f: [] for f in factors}
    for _ in range(repeats):
        for f, fn in runs.items():
            ms[f].append(round(time_ms(torch, fn, n_steps), 3))
    return {"impl": impl, "ms_per_step": {str(f): v for f, v in ms.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--no-step", action="store_true")
    ap.add_argument("--step-arm", choices=["ours", "reference"])
    args = ap.parse_args()
    if args.step_arm:
        factors = (0.0, 0.2) if args.step_arm == "ours" else (0.2,)
        print(json.dumps(step_arm(args.step_arm, factors, args.repeats, args.steps)), flush=True)
        return 0
    info = card()
    loss_lines(args, info)
    if args.no_step:
        return 0
    out = {"what": "coarse_sdf_step, 1M Gaussians 1920x1080, fwd+bwd", "steps": args.steps, "repeats": args.repeats,
           "card": info}
    for arm in ("ours", "reference"):
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--step-arm", arm, "--repeats",
                            str(args.repeats), "--steps", str(args.steps)], capture_output=True, text=True, cwd=ROOT)
        lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
        out[arm] = json.loads(lines[-1]) if lines else {"error": (r.stderr or r.stdout)[-2000:]}
    print(json.dumps(out), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
