#!/usr/bin/env python
"""Time the fused mesh Laplacian smoothing loss (sugar_b200/meshloss.py) against the PyTorch restatement of pytorch3d's
op (oracle/meshlap_oracle.py, its sparse Laplacian rebuilt every call) on the same mesh.

    python scripts/bench_meshlap.py [--iters 50] [--repeats 3] [--steps 10] [--no-step]

Mesh: sugar_b200/scenes.height_field_mesh(501, 501, permute=True), a connected 500k-face mesh (BASELINE config 4's
face count) with vertex ids and face order shuffled.  One JSON line per method, forward + backward per iteration, host
clock around a synchronise, the three arms alternated over `repeats` rounds in one process:
    fused_cached    mesh_laplacian_smoothing(verts, method=m, topology=lap), the topology built once
    fused_rebuild   mesh_laplacian_smoothing(verts, faces, m): laplacian_topology on every call
    oracle_chain    mesh_laplacian_smoothing_torch(verts, faces, m): pytorch3d's sparse chain, L rebuilt every call
plus the fused op's kernel time from the library's event profiler (its launches are counted as "misc") and the
achieved GB/s against the byte model of what the kernels request (the vertex gathers mostly hit L2; E unique edges):
    uniform  forward   4 (V + 1) offsets + 2E x (4 B entry + 12 B vertex) + 12 B own vertex + 16 B row written per
                       vertex                                                                  = 4 (V + 1) + 32 E + 28 V
             backward  4 (V + 1) + 2E x (4 B entry + 16 B row) + 16 B own row + 12 B gradient per vertex + 4
                                                                                               = 4 (V + 1) + 40 E + 28 V + 4
    cot(curv) forward  face pass 12 B ids + 36 B vertices + 16 B written per face, then 4 (V + 1) + per corner (3F) 4 B
                       entry + 12 B face + 16 B face values + 24 B two vertices, + 28 B per vertex
                                                                                               = 4 (V + 1) + 232 F + 28 V
             backward  4 (V + 1) + per corner 4 + 12 + 16 + 32 B (two rows) + 28 B per vertex + 4
                                                                                               = 4 (V + 1) + 192 F + 28 V + 4
as a fraction of the HBM peak (MEASURED_PEAKS.json when present, else the H100 SXM data sheet's 3.35 TB/s, named as
such).  Then one line for refine_step at BASELINE config 4's size (500k faces x 6 = 3M Gaussians, 1600x1200) on the
same kind of mesh with laplacian_smoothing_factor 0 and 5 for each method, alternated in one process.  Every line
carries the card's name, power limit and max SM clock, read in the same run.  Prints only; writes nothing.
"""
import argparse
import json
import os
import sys
from types import SimpleNamespace

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from bench_meshloss import card, median, time_ms  # noqa: E402

METHODS = ("uniform", "cot", "cotcurv")


def byte_model(method, V, F, E):
    if method == "uniform":
        return {"forward": 4 * (V + 1) + 32 * E + 28 * V, "backward": 4 * (V + 1) + 40 * E + 28 * V + 4}
    return {"forward": 4 * (V + 1) + 232 * F + 28 * V, "backward": 4 * (V + 1) + 192 * F + 28 * V + 4}


def loss_lines(args, info):
    import torch
    import bench
    from oracle import meshlap_oracle as lo
    from sugar_b200 import _lib, meshloss, scenes
    peak, peak_src = bench.load_peaks()
    dev = torch.device("cuda", 0)
    v_np, f_np = scenes.height_field_mesh(501, 501, seed=501, permute=True)
    verts = torch.from_numpy(v_np).to(dev).requires_grad_(True)
    faces = torch.from_numpy(f_np).to(dev)
    V, F = verts.shape[0], faces.shape[0]
    lap = meshloss.laplacian_topology(faces, V)
    E = int(lap.nbr_ptr[-1]) // 2
    for method in METHODS:
        def arm(fn):
            def run():
                fn().backward()
                verts.grad = None
            return run
        arms = {"fused_cached": arm(lambda: meshloss.mesh_laplacian_smoothing(verts, method=method, topology=lap)),
                "fused_rebuild": arm(lambda: meshloss.mesh_laplacian_smoothing(verts, faces, method)),
                "oracle_chain": arm(lambda: lo.mesh_laplacian_smoothing_torch(verts, faces, method))}
        for fn in arms.values():
            for _ in range(3):
                fn()
        ms = {k: [] for k in arms}
        for _ in range(args.repeats):
            for k, fn in arms.items():
                ms[k].append(round(time_ms(torch, fn, args.iters), 4))
        build_ms = round(time_ms(torch, lambda: meshloss.laplacian_topology(faces, V), args.iters), 4)
        # kernel time from the event profiler: the forward alone, then forward + backward (the backward is the rest)
        kern = {}
        for part in ("forward", "both"):
            torch.cuda.synchronize()
            _lib.profile(True)
            for _ in range(args.iters):
                out = meshloss.mesh_laplacian_smoothing(verts, method=method, topology=lap)
                if part == "both":
                    out.backward()
                    verts.grad = None
            torch.cuda.synchronize()
            prof = _lib.profile_read()
            _lib.profile(False)
            kern[part] = round(sum(t for t, _ in prof.values()) / args.iters, 5)
        kern["backward"] = round(kern.pop("both") - kern["forward"], 5)
        model = byte_model(method, V, F, E)
        gbs = {k: round(model[k] / (kern[k] * 1e-3) / 1e9, 1) for k in model if kern.get(k)}
        print(json.dumps({
            "what": f"mesh Laplacian smoothing ({method}) forward+backward", "mesh": "501x501 grid permuted",
            "faces": F, "verts": V, "unique_edges": E, "iters": args.iters, "repeats": args.repeats,
            "fused_cached_ms": ms["fused_cached"], "fused_rebuild_ms": ms["fused_rebuild"],
            "oracle_chain_ms": ms["oracle_chain"], "topology_build_ms": build_ms,
            "speedup_cached_vs_oracle": round(median(ms["oracle_chain"]) / median(ms["fused_cached"]), 1),
            "fused_kernels_ms": kern, "model_bytes": model, "achieved_gbs": gbs,
            "hbm_frac": {k: round(g / peak, 3) for k, g in gbs.items()}, "peak_gbs": peak, "peak_source": peak_src,
            "card": info}), flush=True)


def step_line(args, info):
    """refine_step at BASELINE config 4's size on a connected mesh, laplacian_smoothing_factor 0 vs 5 per method."""
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
                           laplacian_topology=meshloss.laplacian_topology(faces, v.shape[0]))
    leaf = lambda t: t.to(dev).requires_grad_(True)
    raw = dict(verts=leaf(v), sh_dc=leaf(0.5 * torch.randn(P, 1, 3, generator=g)),
               sh_rest=leaf(0.1 * torch.randn(P, 15, 3, generator=g)), densities=leaf(torch.randn(P, 1, generator=g) * 2),
               scales=leaf(torch.randn(P, 2, generator=g) * 0.4 - 4.6), quaternions=leaf(torch.randn(P, 2, generator=g)))
    gt = torch.rand(3, H, W, generator=g).to(dev)
    ops = steps.ours_ops()

    def make(fac, method):
        def run():
            steps.refine_step(raw, mesh, cam, gt, ops, laplacian_smoothing_factor=fac, laplacian_smoothing_method=method)
            for t in raw.values():
                t.grad = None
        return run
    runs = {"0": make(0.0, "uniform"), **{f"5 {m}": make(5.0, m) for m in METHODS}}
    for fn in runs.values():
        for _ in range(3):
            fn()
    ms = {k: [] for k in runs}
    for _ in range(args.repeats):
        for k, fn in runs.items():
            ms[k].append(round(time_ms(torch, fn, args.steps), 3))
    print(json.dumps({"what": f"refine_step, {P} Gaussians bound to a connected {F}-face mesh, {W}x{H}, fwd+bwd",
                      "steps": args.steps, "repeats": args.repeats, "ms_per_step": ms,
                      "added_ms_median": {k: round(median(v) - median(ms["0"]), 3) for k, v in ms.items() if k != "0"},
                      "card": info}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
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
