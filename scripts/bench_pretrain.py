"""Time the vanilla 3DGS pre-training pieces on one GPU.

    python scripts/bench_pretrain.py [--sizes 100000 1000000 3000000] [--gaussians 1000000] [--reps 20]

1. knn.dist_cuda2 at each size, and the reference build's distCUDA2 (oracle/_ref/simple_knn, oracle/build_ref_knn.py)
   when it is there, on the same uniform cloud: median of --reps CUDA-event timings after a warm-up, alternating the
   two, with a check that the results are bit-identical.
2. One train_3dgs iteration at --gaussians Gaussians and 1920x1080 (sh degree 3): without a densification, and with one
   (densify_from_iter=0, every iteration), each the median of --reps iterations timed with CUDA events through
   on_iteration.
Prints one JSON line per measurement.
"""
import argparse
import json
import os
import random
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from sugar_b200 import knn, mcubes, scenes, steps, train  # noqa: E402


def reference_dist_cuda2():
    d = os.path.join(ROOT, "oracle", "_ref", "simple_knn")
    if not os.path.exists(os.path.join(d, "simple_knn_C.so")):
        return None
    sys.path.insert(0, d)
    import simple_knn_C
    return simple_knn_C.distCUDA2


def time_ms(fn, reps):
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b))
    return statistics.median(out)


def bench_dist(sizes, reps):
    ref = reference_dist_cuda2()
    for P in sizes:
        pts = (torch.rand(P, 3, generator=torch.Generator().manual_seed(P)) * 10.0).cuda()
        ours = lambda: knn.dist_cuda2(pts)
        same = None
        if ref is not None:
            same = bool(torch.equal(ours().view(torch.int32), ref(pts).view(torch.int32)))
        ours(), ref and ref(pts)
        t_ours, t_ref = [], []
        for _ in range(3):   # alternate: clock and thermal drift hit both sides
            t_ours.append(time_ms(ours, reps))
            if ref is not None:
                t_ref.append(time_ms(lambda: ref(pts), reps))
        print(json.dumps({"bench": "dist_cuda2", "P": P, "ours_ms": round(statistics.median(t_ours), 4),
                          "reference_ms": round(statistics.median(t_ref), 4) if t_ref else None,
                          "bit_identical": same}), flush=True)


def bench_iteration(G, reps, W=1920, H=1080):
    sc = scenes.make_scene(G, W, H, seed=3, camera="posed")
    views = []
    for i in range(4):
        v = scenes.with_camera_offset(sc, 0.05 * i, (0.1 * i, 0.0, 0.0))
        views.append((steps.camera_from_scene(v, "cuda"), torch.rand(3, H, W, device="cuda")))
    extent = mcubes.nerfpp_radius(torch.stack([c.campos.cpu() for c, _ in views]))
    for label, sched in (("no_densify", dict(densify_from_iter=10 ** 9)),
                         ("densify", dict(densify_from_iter=0, densification_interval=1, densify_grad_threshold=1e9))):
        raw = train.init_from_points(torch.from_numpy(sc.means3D).cuda(), torch.rand(G, 3).double().numpy())
        marks = {}

        def hook(it, loss, ev):
            e = torch.cuda.Event(enable_timing=True)
            e.record()
            marks[it] = e
        n = reps + 5
        train.train_3dgs(raw, views, extent, num_iterations=n + 1, sh_every=1, rng=random.Random(0),
                         on_iteration=hook, **sched)
        torch.cuda.synchronize()
        ms = [marks[i - 1].elapsed_time(marks[i]) for i in range(6, n + 1)]
        print(json.dumps({"bench": "train_3dgs_iteration", "mode": label, "gaussians": G, "resolution": f"{W}x{H}",
                          "median_ms": round(statistics.median(ms), 3), "min_ms": round(min(ms), 3),
                          "P_end": raw["points"].shape[0]}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[100_000, 1_000_000, 3_000_000])
    ap.add_argument("--gaussians", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    print(json.dumps({"gpu": torch.cuda.get_device_name(0)}), flush=True)
    bench_dist(a.sizes, a.reps)
    bench_iteration(a.gaussians, a.reps)


if __name__ == "__main__":
    main()
