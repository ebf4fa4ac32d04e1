"""Time the coarse_density trainer's density estimation loss (field.density_estimation_loss) and its composed step
(steps.coarse_density_step).  Arms alternate within the call; every number is the median over rounds.

    python scripts/bench_density_step.py [--rounds 5] [--reps 5] [--no-step]

Op level, N = 1M samples, K = 16, P = 1M Gaussians, forward + backward of the mean loss:
    fused      field.density_estimation_loss (two kernels and the pack / unpack passes)
    field+     field_values(return_beta, return_closest_gaussian_opacities) and the trainer's lines as torch
    reference  the trainer's op chain as torch (oracle/densest_oracle.py on the GPU)
Step level: coarse_density_step at 1M Gaussians, 1920x1080, 1M samples, this package's ops against bench_workloads'
reference_ops with the reference rasterizer (oracle/_ref, when built), at dssim_factor 0 and 0.2.
Prints the card and its power limit, and a byte model of the fused kernels.
"""
import argparse
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import densest_oracle as deo  # noqa: E402
from oracle import field_oracle as fo  # noqa: E402
from sugar_b200 import field, knn, scenes, steps  # noqa: E402

DEV = "cuda:0"


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def timed(fn, reps):
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def field_epilogue(x, gi, nbr, points, scaling, quats, strengths):
    """field_values' density / beta / opacities, then coarse_density.py:654-656, 684-691 as torch."""
    f = field.field_values(x, nbr, points, scaling, quats, strengths, density_factor=1.0, return_sdf=False,
                           return_beta=True, return_closest_gaussian_opacities=True)
    e = ((x - points[gi]) * fo.smallest_axis(scaling, quats)[gi]).sum(dim=-1)
    return (f["density"] - torch.exp(-0.5 * e.pow(2) / f["beta"].pow(2))).abs(), f["closest_gaussian_opacities"]


def byte_model(N, K, P):
    """Bytes the fused passes move from HBM / L2 at the model's granularity (each gathered record counted once per
    use: an upper bound on HBM traffic, which L2 reuse of neighbouring samples' records lowers)."""
    rec, idx = 48, 8
    pack = P * (12 + 12 + 16 + 4 + rec)                                   # read the parameters, write the records
    fwd = N * (12 + 8 + K * (idx + rec) + 32 + 12 + 4 + 4 * K)            # x, own id, K gathers, own axis, loss, opac
    bwd = N * (12 + 8 + 2 * K * (idx + rec) + 2 * (32 + 12) + 4 + 12)     # two passes, own axis twice, g_loss, g_x
    scatter = N * (K * 3 + 2) * 16                                        # red.v4 into the 48-byte gradient records
    unpack = P * (48 + 48) + P * 48                                       # memset, read the records, write 4 grads
    return dict(forward=pack + fwd, backward=pack + bwd + scatter + unpack, scatter=scatter)


def bench_op(rounds, reps, N=1_000_000, K=16, P=1_000_000):
    sc = scenes.make_scene(P, 1920, 1080, seed=0)
    points = torch.from_numpy(sc.means3D).to(DEV)
    scaling = torch.from_numpy(sc.scales).to(DEV)
    quats = torch.nn.functional.normalize(torch.from_numpy(sc.rotations).to(DEV), dim=-1)
    strengths = torch.from_numpy(sc.opacities).to(DEV).view(-1, 1)
    knn_idx = knn.reset_neighbors(points, K)[1]
    g = torch.Generator(device=DEV).manual_seed(0)
    x, gi = field.sample_points_in_gaussians(points, scaling, quats, strengths, N, sampling_scale_factor=1.5,
                                             probabilities_proportional_to_volume=False, generator=g)
    nbr = knn_idx[gi]
    leaves = [t.clone().requires_grad_(True) for t in (x, points, scaling, quats, strengths)]

    def arm(fn):
        def run():
            for t in leaves:
                t.grad = None
            xx, pp, ss, qq, st = leaves
            loss, _ = fn(xx, gi, nbr, pp, ss, qq, st)
            loss.mean().backward()
        return run
    arms = {"fused": arm(lambda *a: field.density_estimation_loss(*a, return_closest_gaussian_opacities=True)),
            "field+torch": arm(field_epilogue),
            "reference": arm(lambda *a: deo.density_estimation_loss_torch(*a, 1.0, True))}
    fused_fwd = lambda: field.density_estimation_loss(x, gi, nbr, points, scaling, quats, strengths,
                                                      return_closest_gaussian_opacities=True)
    for fn in arms.values():
        fn()
    t = {k: [] for k in list(arms) + ["fused forward"]}
    for _ in range(rounds):
        for k, fn in arms.items():
            t[k].append(timed(fn, reps))
        with torch.no_grad():
            t["fused forward"].append(timed(fused_fwd, reps))
    med = {k: float(np.median(v)) for k, v in t.items()}
    print(f"op, N={N} K={K} P={P}, forward + backward (median of {rounds} rounds x {reps}):")
    for k in arms:
        print(f"  {k:12s} {med[k]:8.3f} ms   ({med[k] / med['fused']:.2f}x fused)")
    bm = byte_model(N, K, P)
    fwd, bwd = med["fused forward"], med["fused"] - med["fused forward"]
    print(f"  fused forward {fwd:.3f} ms: model {bm['forward'] / 1e9:.3f} GB -> {bm['forward'] / fwd / 1e6:.0f} GB/s; "
          f"backward {bwd:.3f} ms: model {bm['backward'] / 1e9:.3f} GB ({bm['scatter'] / 1e9:.3f} GB of it red.v4) "
          f"-> {bm['backward'] / bwd / 1e6:.0f} GB/s")


def bench_step(rounds, P=1_000_000, W=1920, H=1080, samples=1_000_000):
    import bench_workloads as bw
    import helpers as h
    sc = scenes.make_scene(P, W, H, seed=0)
    cam = steps.camera_from_scene(sc, DEV)
    gt = torch.rand(3, H, W, generator=torch.Generator().manual_seed(0)).to(DEV)
    leaf = lambda t: t.to(DEV).requires_grad_(True)
    raw = dict(points=leaf(torch.from_numpy(sc.means3D)), sh_dc=leaf(torch.from_numpy(sc.shs[:, :1].copy())),
               sh_rest=leaf(torch.from_numpy(sc.shs[:, 1:].copy())),
               densities=leaf(torch.logit(torch.from_numpy(sc.opacities).clamp(1e-4, 1 - 1e-4))),
               scales=leaf(torch.from_numpy(sc.scales).log()), quaternions=leaf(torch.from_numpy(sc.rotations) * 1.3))
    knn_idx = knn.reset_neighbors(raw["points"].detach(), 16)[1]
    arms = {"ours": steps.ours_ops()}
    if h.have_ref():
        arms["reference"] = bw.reference_ops(torch, h.load_ref_module())
    else:
        print("step: oracle/_ref is not built, timing this package's ops alone")
    sgen = torch.Generator(device=DEV)
    for dssim in (0.0, 0.2):
        def step(ops):
            sgen.manual_seed(1)
            steps.coarse_density_step(raw, cam, gt, knn_idx, ops, n_samples=samples, generator=sgen,
                                      dssim_factor=dssim)
            for v in raw.values():
                v.grad = None
        for ops in arms.values():
            step(ops)
        t = {k: [] for k in arms}
        for _ in range(rounds):
            for k, ops in arms.items():
                t[k].append(timed(lambda: step(ops), 3))
        med = {k: float(np.median(v)) for k, v in t.items()}
        line = ", ".join(f"{k} {m:.2f} ms ({1e3 / m:.1f} steps/s)" for k, m in med.items())
        ratio = f", {med['reference'] / med['ours']:.2f}x" if "reference" in med else ""
        print(f"coarse_density_step P={P} {W}x{H} {samples} samples dssim_factor={dssim}: {line}{ratio}")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--no-step", action="store_true")
    a = ap.parse_args()
    print("card:", card())
    bench_op(a.rounds, a.reps)
    if not a.no_step:
        bench_step(a.rounds)


if __name__ == "__main__":
    main()
