"""bench.py's secondary workloads: the trainers' steps around the rasterizer (SURVEY 8f / BASELINE configs 3, 4).

    python bench.py --workload coarse_sdf_step   1M Gaussians, 1920x1080, SH 3: RGB render + depth render + 1M-sample
                                                 density/SDF regularisation + better-normal loss, fwd+bwd
    python bench.py --workload refine_step       3M mesh-bound Gaussians (500k faces x 6), 1600x1200, SH 3: binding
                                                 prologue + render, fwd+bwd

Both arms run the SAME recipe (sugar_b200/steps.py, following sugar_trainers/coarse_sdf.py:506-716 and
refine.py); `--impl ours` plugs in this package's fused operators, `--impl reference` the reference's own building
blocks: its unmodified CUDA rasterizer build (oracle/_ref), its python SH colour path and its PyTorch op chains
for the field, the normal loss and the mesh binding (restated in oracle/, which only this arm may execute).
One JSON line, same keys as the headline line.
"""
import json
import math
import os
import sys
import time
from types import SimpleNamespace

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))

WORKLOADS = {
    "coarse_sdf_step": dict(P=1_000_000, W=1920, H=1080, metric="coarse_sdf train steps/sec @1M Gaussians 1920x1080",
                            samples=1_000_000, K=16),
    "refine_step": dict(P=3_000_000, W=1600, H=1200, metric="refine train steps/sec @3M mesh-bound Gaussians 1600x1200",
                        faces=500_000, n_per=6),
}


def reference_ops(torch, ref_mod):
    """The reference's building blocks behind the `ops` interface of sugar_b200/steps.py."""
    from oracle import densest_oracle as deo
    from oracle import field_oracle as fo
    from oracle import meshbind_oracle as mo
    from oracle import meshlap_oracle as lo
    from oracle import meshloss_oracle as mlo
    from oracle import ssim_oracle as so

    def bind(verts, faces, bary, scales_raw, complex_raw, thickness):
        p, s, q = mo.bind_to_mesh_torch(verts, faces, bary, scales_raw, complex_raw, thickness)
        return SimpleNamespace(points=p, scaling=s, quaternions=q)
    return SimpleNamespace(
        rasterizer=ref_mod,
        colors=lambda points, sh, campos, deg: fo.points_rgb_torch(points, sh, campos, deg + 1),
        field_values=lambda x, nbr, points, scaling, quats, strengths, density_factor=1.0, density_threshold=1.0, **_:
            fo.field_values_torch(x, nbr, points, scaling, quats, strengths, density_factor, density_threshold),
        better_normal_loss=fo.better_normal_loss_torch, bind_to_mesh=bind, l1_dssim=so.l1_dssim_torch,
        density_estimation_loss=deo.density_estimation_loss_torch,
        # pytorch3d's cost: a new Meshes every call (edges rebuilt) and its Python pair loop; no cached topology
        mesh_normal_consistency=lambda verts, faces, topology=None: mlo.mesh_normal_consistency_torch(verts, faces),
        # a new Meshes every call: the sparse Laplacian rebuilt from the faces (and the moving vertices for cot)
        mesh_laplacian_smoothing=lambda verts, faces, method, topology=None:
            lo.mesh_laplacian_smoothing_torch(verts, faces, method))


def run(args, scenes, load_peaks, ClockSampler, cpu_density_baseline):
    import torch
    name = args.workload
    cfg = WORKLOADS[name]
    dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", "0")))
    torch.cuda.set_device(dev)
    P, W, H = (args.gaussians or cfg["P"]), (args.width or cfg["W"]), (args.height or cfg["H"])
    use_ref = args.impl == "reference"
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    if use_ref:
        import helpers as h
        if not h.have_ref():
            print(json.dumps({"impl": "reference", "unavailable": "oracle/_ref (reference CUDA build) is not present"}))
            return 0
        ops = reference_ops(torch, h.load_ref_module())
        steps = _load_steps_without_package()
        _lib = None
    else:
        from sugar_b200 import _lib, steps
        ops = steps.ours_ops()
    g = torch.Generator().manual_seed(0)
    sc = scenes.make_scene(P if name == "coarse_sdf_step" else 1000, W, H, seed=0)
    cam = steps.camera_from_scene(sc, dev)
    gt = torch.rand(3, H, W, generator=g).to(dev)
    leaf = lambda t: t.to(dev).requires_grad_(True)
    if name == "coarse_sdf_step":
        raw = dict(points=leaf(torch.from_numpy(sc.means3D)), sh_dc=leaf(torch.from_numpy(sc.shs[:, :1].copy())),
                   sh_rest=leaf(torch.from_numpy(sc.shs[:, 1:].copy())),
                   densities=leaf(torch.logit(torch.from_numpy(sc.opacities).clamp(1e-4, 1 - 1e-4))),
                   scales=leaf(torch.from_numpy(sc.scales).log()), quaternions=leaf(torch.from_numpy(sc.rotations) * 1.3))
        # the K-NN table the trainer rebuilds every 500 iterations (sugar_model.py:1013-1030): a real one
        if use_ref:
            from scipy.spatial import cKDTree  # pytorch3d is not in the image; exact K-NN on the host, untimed
            pts = sc.means3D
            knn_idx = torch.from_numpy(cKDTree(pts).query(pts, k=cfg["K"], workers=-1)[1].astype(np.int64)).to(dev)
        else:
            from sugar_b200 import knn
            knn_idx = knn.reset_neighbors(raw["points"].detach(), cfg["K"])[1]
        sgen = torch.Generator(device=dev)

        def step():
            sgen.manual_seed(1)
            loss, stats = steps.coarse_sdf_step(raw, cam, gt, knn_idx, ops, n_samples=cfg["samples"], generator=sgen)
            for t in raw.values():
                t.grad = None
            return loss, stats
        desc = (f"{P} Gaussians (SH deg 3) {W}x{H}: RGB render + depth render + {cfg['samples']} samples x K={cfg['K']} "
                "density/SDF + better-normal loss, fwd+bwd (coarse_sdf.py:506-716)")
    else:
        from types import SimpleNamespace as NS
        F, n = (P // cfg["n_per"]), cfg["n_per"]
        centers = torch.stack([(torch.rand(F, generator=g) - 0.5) * 2 * 6 * sc.tanfovx, (torch.rand(F, generator=g) - 0.5) * 2 * 6 * sc.tanfovy,
                               2 + 8 * torch.rand(F, generator=g)], 1)
        centers[:, :2] *= (centers[:, 2:3] / 6.0)
        tri = centers[:, None] + 0.02 * torch.randn(F, 3, 3, generator=g)
        bary_tab = {6: [[2 / 3, 1 / 6, 1 / 6], [1 / 6, 2 / 3, 1 / 6], [1 / 6, 1 / 6, 2 / 3], [1 / 6, 5 / 12, 5 / 12],
                        [5 / 12, 1 / 6, 5 / 12], [5 / 12, 5 / 12, 1 / 6]]}
        mesh = NS(faces=torch.arange(3 * F).view(F, 3).to(dev), bary=torch.tensor(bary_tab[n]).to(dev), thickness=1e-5)
        Pn = F * n
        raw = dict(verts=leaf(tri.reshape(-1, 3)), sh_dc=leaf(0.5 * torch.randn(Pn, 1, 3, generator=g)),
                   sh_rest=leaf(0.1 * torch.randn(Pn, 15, 3, generator=g)), densities=leaf(torch.randn(Pn, 1, generator=g) * 2),
                   scales=leaf(torch.randn(Pn, 2, generator=g) * 0.4 - 4.6), quaternions=leaf(torch.randn(Pn, 2, generator=g)))

        def step():
            loss, stats = steps.refine_step(raw, mesh, cam, gt, ops)
            for t in raw.values():
                t.grad = None
            return loss, stats
        desc = (f"{Pn} Gaussians bound to {F} faces x {n} (SH deg 3) {W}x{H}: mesh-binding prologue + render, fwd+bwd "
                "(sugar_model.py:384-479, refine.py)")

    for _ in range(max(args.warmup, 3)):
        loss, stats = step()
    torch.cuda.synchronize()
    clocks = ClockSampler(dev.index or 0)
    t_load0 = time.perf_counter()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    probe = max(3, args.steps // 2)
    for _ in range(probe):
        step()
    if _lib is not None:
        _lib.profile(True)
        step()
        torch.cuda.synchronize()
        _lib.profile_read()
    launches0 = _lib.lib.sgr_launch_count() if _lib is not None else 0
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    e0.record()
    for _ in range(args.steps):
        loss, stats = step()
    e1.record()
    torch.cuda.synchronize()
    t1 = time.perf_counter()
    ms = e0.elapsed_time(e1) / args.steps
    prof = _lib.profile_read() if _lib is not None else {}
    if _lib is not None:
        _lib.profile(False)
    launches = int(_lib.lib.sgr_launch_count() - launches0) if _lib is not None else 0
    for _ in range(3):
        step()
    torch.cuda.synchronize()
    clk = clocks.stop(load=(t_load0, time.perf_counter()), timed=(t0, t1))
    peak, peak_src = load_peaks()
    out = {"metric": cfg["metric"], "value": 1e3 / ms, "unit": "steps/s", "n_gpus": 1, "steps": args.steps,
           "warmup": max(args.warmup, 3), "ms_per_step": ms, "higher_is_better": True, "scaling": "weak",
           "vs_baseline": None, "dtype": "f32", "data": "synthetic",
           "config": {"workload": desc, "l2_policy": "inputs larger than L2; no flush"},
           "workload_stats": dict(stats, loss=float(loss)), "clocks": clk, "gpu_launches": launches,
           "e2e": {"value": 1e3 / ms, "unit": "steps/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 8,
                   "note": "the step is already the trainer-level call (parameters, K-NN table and ground-truth image "
                           "device-resident as in the reference's loop); the visibility / sample counts are read back "
                           "by the recipe itself every step (int(mask.sum()), as the reference's `if n_gaussians_in_sampling > 0`)"}}
    if use_ref:
        out["impl"] = "reference"
        out["impl_note"] = ("reference building blocks: unmodified CUDA rasterizer build (oracle/_ref), python SH colours, "
                            "PyTorch op chains for field / normal loss / mesh binding, all on the same GPU")
        out["gpu_launches"] = 0
        out["cpu_baseline"] = {"value": out["value"], "unit": "steps/s", "cores": 0, "kind": "reference",
                               "sample": "full workload on the GPU"}
    else:
        total = sum(t for t, _ in prof.values())
        out["stages"] = {k: {"ms": round(t / args.steps, 4), "launches_per_step": c / args.steps} for k, (t, c) in prof.items()}
        out["kernel_ms_per_step"] = round(total / args.steps, 4)
        dom = max(out["stages"], key=lambda k: out["stages"][k]["ms"]) if out["stages"] else None
        if dom:
            out["roofline"] = {"kernel": dom, "bound": "see stages", "achieved": None, "peak": peak, "unit": "GB/s",
                               "frac": None, "traffic": None, "peak_source": peak_src,
                               "note": "per-kernel rooflines are reported on the headline workload (python bench.py)"}
        if not args.no_cpu_baseline and name == "coarse_sdf_step":
            try:
                out["cpu_baseline"] = cpu_density_baseline(args)
            except Exception as ex:
                out["cpu_baseline"] = {"error": repr(ex)}
    print(json.dumps(out))
    return 0


def _load_steps_without_package():
    """sugar_b200/steps.py + field.sample_points_in_gaussians for the reference arm, without importing the package
    (which would map libsugar_b200.so): steps.py only needs torch at module level."""
    import importlib.util
    import types
    pkg = types.ModuleType("sgr_ref_steps_pkg")
    pkg.__path__ = []
    sys.modules["sgr_ref_steps_pkg"] = pkg
    fld = types.ModuleType("sgr_ref_steps_pkg.field")
    src = open(os.path.join(ROOT, "sugar_b200", "field.py")).read()
    # the two pure-PyTorch helpers of field.py (sampling keeps the reference's RNG semantics); nothing CUDA-specific
    start = src.index("def quaternion_apply(")
    exec(compile("import torch\n" + src[start:], "field_helpers", "exec"), fld.__dict__)
    sys.modules["sgr_ref_steps_pkg.field"] = fld
    spec = importlib.util.spec_from_file_location("sgr_ref_steps_pkg.steps", os.path.join(ROOT, "sugar_b200", "steps.py"))
    mod = importlib.util.module_from_spec(spec)
    sys.modules["sgr_ref_steps_pkg.steps"] = mod
    spec.loader.exec_module(mod)
    return mod
