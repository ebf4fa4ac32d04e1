"""Time densification and pruning (sugar_b200/densify.py) against the reference's statements run as torch on the same
device (oracle/densify_oracle.py).  The two implementations alternate within the call.

    python scripts/bench_densify.py [--reps 5] [--sizes 1000000 3000000]

Prints the card and its power limit; update_densification_stats per call and the host synchronisations each side
makes; densify_and_prune at each P (M = 16, with Adam state, about 4% clone, 4% split and 1% prune) per call; and the
emit kernel's bytes (from the shapes) and bandwidth.
"""
import argparse
import os
import subprocess
import sys
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import densify_oracle as do  # noqa: E402
from sugar_b200 import _lib, densify  # noqa: E402

DEV = "cuda:0"


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def syncs(fn):
    """-> host synchronisations fn() makes (torch's sync debug mode, one warning each)."""
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode("default")
    return sum("called a synchronizing CUDA operation" in str(x.message) for x in w)


def timed(fn):
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def model(P, seed):
    """M = 16 raw parameters with about 4% clone, 4% split and 1% prune, and one Adam step's state."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    r = lambda *s: torch.rand(*s, generator=g, device=DEV)
    scale = torch.where(r(P, 1) < 0.5, 0.005, 0.02) * (0.8 + 0.4 * r(P, 3))
    raw = {"points": torch.randn(P, 3, generator=g, device=DEV), "densities": torch.where(r(P, 1) < 0.01, -9.0, 2.0),
           "scales": scale.log(), "quaternions": torch.randn(P, 4, generator=g, device=DEV),
           "sh_dc": torch.randn(P, 1, 3, generator=g, device=DEV),
           "sh_rest": torch.randn(P, 15, 3, generator=g, device=DEV)}
    raw = {k: torch.nn.Parameter(v) for k, v in raw.items()}
    opt = torch.optim.Adam([{"params": [raw[k]], "name": k} for k in densify.KEYS])
    for v in raw.values():
        v.grad = torch.randn_like(v) * 1e-3
    opt.step()
    opt.zero_grad(set_to_none=True)
    denom = torch.full((P, 1), 4.0, device=DEV)
    accum = denom * torch.where(r(P, 1) < 0.08, 4e-4, 1e-5)
    return raw, opt, accum, denom


def bench_stats(reps):
    P = 3_000_000
    raw, opt, _, _ = model(P, 1)
    d = densify.Densifier(raw, opt, scene_extent=1.0)
    ref = do.zero_stats(P, DEV)
    grad = torch.randn(P, 3, device=DEV)
    radii = torch.randint(0, 30, (P,), device=DEV, dtype=torch.int32)
    vis = radii > 0
    ours = lambda: d.update_densification_stats(grad, radii, vis)
    theirs = lambda: do.update_stats(ref, grad, radii, vis)
    ours(), theirs()
    t = {"ours": [], "torch": []}
    for _ in range(reps):
        t["ours"].append(timed(lambda: [ours() for _ in range(10)]) / 10)
        t["torch"].append(timed(lambda: [theirs() for _ in range(10)]) / 10)
    print(f"update_densification_stats P={P}: ours {np.median(t['ours']):.3f} ms ({syncs(ours)} host syncs), "
          f"reference statements {np.median(t['torch']):.3f} ms ({syncs(theirs)} host syncs)")


def emit_bytes(raw, opt, P, P_out):
    """Bytes the emit must move: each column's surviving rows read once (new rows read the parent's parameter, not
    its moments) and every output row written once.  Rows are counted at P_out for the reads: an upper bound that
    counts a child's parent once per child."""
    n = 0
    for k, v in raw.items():
        w = v[0].numel() * 4
        n += (P_out * w) * 2                              # parameter: read + write
        if v in opt.state:
            n += (P_out * w) * 2 * 2                      # two moments, read (or zero) + write
    return n


def bench_densify(P, reps):
    res = {"ours": [], "torch": [], "emit": []}
    for rep in range(reps):
        for side in ("ours", "torch"):
            raw, opt, accum, denom = model(P, 2 + rep)
            if side == "ours":
                d = densify.Densifier(raw, opt, scene_extent=1.0)
                d.accum.copy_(accum), d.denom.copy_(denom)
                _lib.profile(True)
                _lib.profile_read()
                ms = timed(lambda: d.densify_and_prune(max_screen_size=20,
                                                       generator=torch.Generator(device=DEV).manual_seed(rep)))
                tl = _lib.profile_timeline()
                _lib.profile(False)
                P_out = raw["points"].shape[0]
                emit_ms = tl[-1][2] - tl[-1][1]                 # the last launch is the emit
                res["emit"].append((emit_ms, emit_bytes(raw, opt, P, P_out)))
            else:
                params = {k: v.detach() for k, v in raw.items()}
                mom = {k: (opt.state[v]["exp_avg"], opt.state[v]["exp_avg_sq"]) for k, v in raw.items()}
                stats = {"accum": accum, "denom": denom, "max_radii": torch.zeros(P, device=DEV)}
                ms = timed(lambda: do.densify_and_prune(params, mom, stats, 2e-4, 0.005, 1.0, 20,
                                                        generator=torch.Generator(device=DEV).manual_seed(rep)))
            res[side].append(ms)
            del raw, opt
            torch.cuda.empty_cache()
    em = sorted(res["emit"])[len(res["emit"]) // 2]
    print(f"densify_and_prune P={P} M=16 with Adam state: ours {np.median(res['ours'][1:]):.2f} ms, reference "
          f"statements {np.median(res['torch'][1:]):.2f} ms (median of {reps - 1} after one warm-up pair); emit "
          f"{em[0]:.3f} ms for {em[1] / 1e9:.3f} GB = {em[1] / em[0] / 1e6:.0f} GB/s")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--sizes", type=int, nargs="+", default=[1_000_000, 3_000_000])
    a = ap.parse_args()
    print("card:", card())
    bench_stats(a.reps)
    for P in a.sizes:
        bench_densify(P, a.reps)


if __name__ == "__main__":
    main()
