#!/usr/bin/env python
"""Time the fused mesh normal-consistency loss (sugar_b200/meshloss.py) against the PyTorch restatement of pytorch3d's
op (oracle/meshloss_oracle.py, with its Python pair loop) on the same meshes.

    python scripts/bench_meshloss.py [--iters 50] [--repeats 3] [--oracle-iters 2] [--no-step]

Meshes (sugar_b200/scenes.height_field_mesh): 1001x1001 vertices = 2M faces (the default 1M-vertex refinement mesh)
and 501x501 = 500k faces (BASELINE config 4), each in grid order and with vertex ids and face order permuted.
One JSON line per mesh, forward + backward per iteration, host clock around a synchronise:
    fused_cached    mesh_normal_consistency(verts, topology=topo), the topology built once
    fused_rebuild   mesh_normal_consistency(verts, faces): mesh_topology on every call
    oracle_chain    mesh_normal_consistency_torch(verts, faces): edges rebuilt and pairs listed by the Python
                    comprehension every call, as pytorch3d does (fewer iterations: it takes seconds)
the two fused arms alternated over `repeats` rounds, the fused op's per-kernel times from the library's event
profiler, and its achieved GB/s against the byte model
    forward   per pair 16 B of indices + 4 x 12 B of vertex gathers                               = 64 Q
    backward  the same gathers + 48 B of per-pair vertex gradients written and read back, the CSR
              (4 (V + 1) B of offsets + 4 x 4 B of entries per pair) + 12 B per vertex written = 176 Q + 16 V + 4
as a fraction of the HBM peak (MEASURED_PEAKS.json when present, else the H100 SXM data sheet's 3.35 TB/s, named as
such).  Then one line for refine_step at BASELINE config 4's size (500k faces x 6 = 3M Gaussians, 1600x1200) on the
connected 500k-face mesh with normal_consistency_factor 0 and 0.1, alternated in one process.  Every line carries the
card's name, power limit and max SM clock, read in the same run.  Prints only; writes nothing.
"""
import argparse
import json
import os
import subprocess
import sys
import time
from types import SimpleNamespace

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
MESHES = [(1001, False), (1001, True), (501, False), (501, True)]


def card(index=0):
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i", str(index)],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return {"name": out[0].strip(), "power_limit_w": float(out[1]), "sm_max_mhz": float(out[2])}
    except Exception as ex:
        return {"error": repr(ex)}


def time_ms(torch, fn, iters):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(iters):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / iters


def median(v):
    return sorted(v)[len(v) // 2]


def loss_lines(args, info):
    import torch
    import bench
    from oracle import meshloss_oracle as mlo
    from sugar_b200 import _lib, meshloss, scenes
    peak, peak_src = bench.load_peaks()
    dev = torch.device("cuda", 0)
    for n, permute in MESHES:
        v_np, f_np = scenes.height_field_mesh(n, n, seed=n, permute=permute)
        verts = torch.from_numpy(v_np).to(dev).requires_grad_(True)
        faces = torch.from_numpy(f_np).to(dev)
        t0 = time.perf_counter()
        topo = meshloss.mesh_topology(faces, verts.shape[0])
        torch.cuda.synchronize()
        first_build_ms = (time.perf_counter() - t0) * 1e3
        Q, V, F = topo.num_pairs, verts.shape[0], faces.shape[0]

        def arm(fn):
            def run():
                fn().backward()
                verts.grad = None
            return run
        arms = {"fused_cached": arm(lambda: meshloss.mesh_normal_consistency(verts, topology=topo)),
                "fused_rebuild": arm(lambda: meshloss.mesh_normal_consistency(verts, faces))}
        for fn in arms.values():
            for _ in range(5):
                fn()
        ms = {k: [] for k in arms}
        for _ in range(args.repeats):
            for k, fn in arms.items():
                ms[k].append(round(time_ms(torch, fn, args.iters), 4))
        build_ms = round(time_ms(torch, lambda: meshloss.mesh_topology(faces, V), args.iters), 4)
        _lib.profile(True)
        time_ms(torch, arms["fused_cached"], args.iters)
        prof = _lib.profile_read()
        _lib.profile(False)
        kern = {k: round(t / args.iters, 5) for k, (t, c) in prof.items()}
        oracle = arm(lambda: mlo.mesh_normal_consistency_torch(verts, faces))
        oracle()
        oracle_ms = [round(time_ms(torch, oracle, args.oracle_iters), 1) for _ in range(args.repeats)]
        model = {"mesh_nc_forward": 64 * Q, "mesh_nc_backward": 176 * Q + 16 * V + 4}
        gbs = {k: round(model[k] / (kern[k] * 1e-3) / 1e9, 1) for k in model if kern.get(k)}
        print(json.dumps({
            "what": "mesh normal consistency forward+backward", "mesh": f"{n}x{n} grid{' permuted' if permute else ''}",
            "faces": F, "verts": V, "pairs": Q, "iters": args.iters, "repeats": args.repeats,
            "fused_cached_ms": ms["fused_cached"], "fused_rebuild_ms": ms["fused_rebuild"],
            "topology_build_ms": build_ms, "first_topology_build_ms": round(first_build_ms, 2),
            "oracle_chain_ms": oracle_ms, "oracle_iters": args.oracle_iters,
            "speedup_cached_vs_oracle": round(median(oracle_ms) / median(ms["fused_cached"]), 1),
            "fused_kernels_ms": kern, "model_bytes": model, "achieved_gbs": gbs,
            "hbm_frac": {k: round(g / peak, 3) for k, g in gbs.items()}, "peak_gbs": peak, "peak_source": peak_src,
            "card": info}), flush=True)
        del topo, verts, faces
        torch.cuda.empty_cache()


def step_line(args, info):
    """refine_step at BASELINE config 4's size on a connected mesh, normal_consistency_factor 0 vs 0.1."""
    import torch
    import bench_workloads as bw
    from sugar_b200 import meshbind, meshloss, scenes, steps
    cfg = bw.WORKLOADS["refine_step"]
    dev = torch.device("cuda", 0)
    W, H, n_per = cfg["W"], cfg["H"], cfg["n_per"]
    v_np, f_np = scenes.height_field_mesh(501, 501, seed=3, permute=True)
    sc = scenes.make_scene(1000, W, H, seed=0)
    cam = steps.camera_from_scene(sc, dev)
    g = torch.Generator().manual_seed(0)
    v = torch.from_numpy(v_np).clone()
    v[:, 0] = (v[:, 0] - 0.5) * 2 * 5 * sc.tanfovx          # fills the view at depth ~5
    v[:, 1] = (v[:, 1] - 0.5) * 2 * 5 * sc.tanfovy
    v[:, 2] = 5.0 + 5.0 * v[:, 2]
    F, P = f_np.shape[0], f_np.shape[0] * n_per
    faces = torch.from_numpy(f_np).to(dev)
    mesh = SimpleNamespace(faces=faces, bary=meshbind.bary_coords(n_per, dev), thickness=1e-5,
                           topology=meshloss.mesh_topology(faces, v.shape[0]))
    leaf = lambda t: t.to(dev).requires_grad_(True)
    raw = dict(verts=leaf(v), sh_dc=leaf(0.5 * torch.randn(P, 1, 3, generator=g)),
               sh_rest=leaf(0.1 * torch.randn(P, 15, 3, generator=g)), densities=leaf(torch.randn(P, 1, generator=g) * 2),
               scales=leaf(torch.randn(P, 2, generator=g) * 0.4 - 4.6), quaternions=leaf(torch.randn(P, 2, generator=g)))
    gt = torch.rand(3, H, W, generator=g).to(dev)
    ops = steps.ours_ops()

    def make(fac):
        def run():
            steps.refine_step(raw, mesh, cam, gt, ops, normal_consistency_factor=fac)
            for t in raw.values():
                t.grad = None
        return run
    runs = {f: make(f) for f in (0.0, 0.1)}
    for fn in runs.values():
        for _ in range(3):
            fn()
    ms = {f: [] for f in runs}
    for _ in range(args.repeats):
        for f, fn in runs.items():
            ms[f].append(round(time_ms(torch, fn, args.steps), 3))
    print(json.dumps({"what": f"refine_step, {P} Gaussians bound to a connected {F}-face mesh, {W}x{H}, fwd+bwd",
                      "steps": args.steps, "repeats": args.repeats,
                      "ms_per_step": {str(f): v for f, v in ms.items()},
                      "added_ms_median": round(median(ms[0.1]) - median(ms[0.0]), 3), "card": info}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--oracle-iters", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--no-step", action="store_true")
    args = ap.parse_args()
    info = card()
    loss_lines(args, info)
    if not args.no_step:
        step_line(args, info)
    return 0


if __name__ == "__main__":
    sys.exit(main())
