#!/usr/bin/env python
"""Time the refined mesh's post-processing (sugar_b200/postprocess.py).

    python scripts/bench_postprocess.py [--cases 400k_n6 2m_n1] [--iters 20] [--repeats 5] [--rounds 5]

Workloads: permuted scenes.height_field_mesh of ~400k faces with 6 bound Gaussians per face (low poly) and ~2M faces
(a 1001 x 1001 grid) with 1 (high poly); strengths spread over (0.02, 0.3) around the default threshold 0.1.
Arms, CUDA events around `iters` calls, `repeats` rounds alternating the arms in one process, medians:
    peel            the erosion kernel alone, `rounds` launches (sgr_border_peel on a prebuilt edge-run table)
    erode           erode_border_faces: id check, table build (torch sort) and the peel
    peel_torch      the same rounds in PyTorch on the same table: per round a bincount of the live entries per run,
                    a gather per entry and an all over each face's three
    postprocess     the whole postprocess_mesh (erosion, re-admission over the eroded faces, compaction)
Byte model of one peel round: per face 1 B mask read + 12 B entry runs + 24 B run offsets + 24 B run members (two per
run on a manifold mesh) + 6 B member masks + 1 B written, before cache reuse.  HBM shares are against the H100 SXM data
sheet's 3.35 TB/s.  Every line carries the card's name, power limit and max SM clock, read in the same run.
"""
import argparse
import json
import math
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_meshloss import card, median  # noqa: E402

PEAK_GBS = 3350.0
CASES = {"400k_n6": (448, 448, 6), "2m_n1": (1001, 1001, 1)}
BYTES_PER_FACE_ROUND = 1 + 12 + 24 + 24 + 6 + 1


def time_ms(torch, fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def make_case(torch, nx, ny, n, dev):
    from sugar_b200 import scenes
    v, f = scenes.height_field_mesh(nx, ny, seed=nx, permute=True)
    g = torch.Generator().manual_seed(nx)
    F = f.shape[0]
    P = F * n
    lo, hi = math.log(0.02 / 0.98), math.log(0.3 / 0.7)
    h = 1.0 / (nx - 1)
    return dict(verts=torch.from_numpy(v).to(dev), faces=torch.from_numpy(f).to(dev), n=n,
                scales_raw=(torch.randn(P, 2, generator=g) * 0.2 + math.log(0.3 * h)).to(dev),
                complex_raw=torch.randn(P, 2, generator=g).to(dev),
                densities_raw=(lo + (hi - lo) * torch.rand(P, 1, generator=g)).to(dev),
                sh_dc=torch.randn(P, 1, 3, generator=g).to(dev), sh_rest=torch.randn(P, 15, 3, generator=g).to(dev),
                thickness=1e-3 * h)


def peel_torch(torch, entry_run, run_faces, live, rounds):
    m = live.clone()
    F = m.shape[0]
    for _ in range(rounds):
        per_run = torch.bincount(entry_run.long(), weights=m.repeat_interleave(3).float(), minlength=3 * F)
        m = m & (per_run[entry_run.long()].view(F, 3) >= 2).all(1)
    return m


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", nargs="*", default=list(CASES))
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    import torch
    from sugar_b200 import postprocess
    from sugar_b200._lib import check, lib, stream
    assert torch.cuda.is_available(), "bench_postprocess.py measures on the GPU only"
    dev = torch.device("cuda", 0)
    info = card(0)
    for name in args.cases:
        nx, ny, n = CASES[name]
        c = make_case(torch, nx, ny, n, dev)
        F, V = c["faces"].shape[0], c["verts"].shape[0]
        entry_run, run_ptr, run_faces = postprocess._edge_runs(c["faces"], V)
        live = torch.ones(F, dtype=torch.bool, device=dev)
        mask = torch.ones(F, dtype=torch.uint8, device=dev)
        tmp = torch.empty_like(mask)

        def peel():
            mask.fill_(1)
            check(lib.sgr_border_peel(F, args.rounds, entry_run.data_ptr(), run_ptr.data_ptr(), run_faces.data_ptr(),
                                      mask.data_ptr(), tmp.data_ptr(), stream(dev)))

        arms = {"peel": peel,
                "erode": lambda: postprocess.erode_border_faces(c["faces"], V, args.rounds),
                "peel_torch": lambda: peel_torch(torch, entry_run, run_faces, live, args.rounds),
                "postprocess": lambda: postprocess.postprocess_mesh(**c, iterations=args.rounds)}
        ref = peel_torch(torch, entry_run, run_faces, live, args.rounds)
        peel()
        assert torch.equal(mask.bool(), ref) and torch.equal(postprocess.erode_border_faces(c["faces"], V,
                                                                                            args.rounds), ref)
        out = postprocess.postprocess_mesh(**c, iterations=args.rounds)
        for fn in arms.values():            # warm-up of every shape
            fn()
        torch.cuda.synchronize()
        times = {k: [] for k in arms}
        for _ in range(args.repeats):
            for k, fn in arms.items():
                times[k].append(time_ms(torch, fn, args.iters))
        ms = {k: median(v) for k, v in times.items()}
        gbs = BYTES_PER_FACE_ROUND * F * args.rounds / (ms["peel"] * 1e-3) / 1e9
        print(json.dumps({"case": name, "faces": F, "n": n, "rounds": args.rounds, "eroded": int(out.eroded.numel()),
                          "kept": int(out.faces.shape[0]), **{f"{k}_ms": round(v, 4) for k, v in ms.items()},
                          **{f"{k}_ms_range": [round(min(v), 4), round(max(v), 4)] for k, v in times.items()},
                          "peel_gbs_model": round(gbs, 1), "peel_hbm_share": round(gbs / PEAK_GBS, 3), "card": info}))


if __name__ == "__main__":
    main()
