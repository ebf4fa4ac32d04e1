#!/usr/bin/env python
"""Time LPIPS (sugar_b200/lpips.py) against torchvision's VGG16 plus the reference's LPIPS formula on cuDNN.

    python scripts/bench_lpips.py [--iters 20] [--repeats 3]

One JSON line per image size (1920x1080 and 800x800), one (render, ground truth) pair each: both arms use the same
seeded random weights (tests/lpips_cases.py) on the same card in the same process, warmed up, then alternated
(`repeats` rounds of `iters` calls each, CUDA events).  The cuDNN arm runs at torch's defaults
(torch.backends.cudnn.allow_tf32 True: TF32 convolutions), as the reference's metrics.py does on an H100.
Reported: ms per pair for each arm (every round, and the median), achieved TFLOP/s from the shape-derived conv count
(lpips.pair_flops, both images), its share of the H100 SXM data sheet's 495 TFLOP/s dense TF32 (a data-sheet figure,
not a measured peak), our kernels' per-launch times from the library's event profiler, the two arms' values, and
the card's name and power limit read in the same run.  Prints only; writes nothing.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
SIZES = [(1920, 1080), (800, 800)]
TF32_DATASHEET_TFLOPS = 495.0


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


def cudnn_lpips(torch, vgg_sd, lin_sd, dev):
    """torchvision's vgg16 features with the given weights and the reference's LPIPS formula, float32 on cuDNN."""
    import torchvision
    feats = torchvision.models.vgg16(weights=None).features
    feats.load_state_dict({k.split(".", 1)[1]: v for k, v in vgg_sd.items()})
    feats = feats.to(dev).eval()
    lins = [lin_sd[f"lin{i}.model.1.weight"].to(dev) for i in range(5)]
    mean = torch.tensor([-.030, -.088, -.188], device=dev).view(1, 3, 1, 1)
    std = torch.tensor([.458, .448, .450], device=dev).view(1, 3, 1, 1)
    taps = (3, 8, 15, 22, 29)   # the ReLUs after conv1_2, 2_2, 3_3, 4_3, 5_3

    def net(x):
        x, out = (x - mean) / std, []
        for i, layer in enumerate(feats):
            x = layer(x)
            if i in taps:
                out.append(x / (torch.sqrt((x ** 2).sum(1, keepdim=True)) + 1e-10))
                if len(out) == 5:
                    return out

    @torch.no_grad()
    def run(x, y):
        fx, fy = net(x), net(y)
        return sum(torch.nn.functional.conv2d((a - b) ** 2, w).mean((2, 3)) for a, b, w in zip(fx, fy, lins))[:, 0]
    return run


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    import torch
    import lpips_cases as lc
    from sugar_b200 import _lib, lpips
    info = card()
    dev = torch.device("cuda", 0)
    vgg_sd, lin_sd = lc.make_state_dicts()
    with tempfile.TemporaryDirectory() as d:
        ours = lpips.LPIPS(*lc.write_weight_files(d), device=dev)
    theirs = cudnn_lpips(torch, vgg_sd, lin_sd, dev)
    for W, H in SIZES:
        x, y = (t.to(dev) for t in lc.image_pair(1, H, W, 0.05, seed=W))
        arms = {"sugar_b200": lambda: ours(x, y), "torchvision_cudnn_tf32": lambda: theirs(x, y)}
        for fn in arms.values():
            for _ in range(3):
                fn()
        torch.cuda.synchronize()
        ms = {k: [] for k in arms}
        for _ in range(args.repeats):
            for k, fn in arms.items():
                ms[k].append(round(time_ms(torch, fn, args.iters), 3))
        _lib.profile(True)
        time_ms(torch, arms["sugar_b200"], 1)
        prof = _lib.profile_timeline()
        _lib.profile(False)
        _lib.profile_read()
        flops = lpips.pair_flops(H, W)
        med = {k: sorted(v)[len(v) // 2] for k, v in ms.items()}
        tflops = {k: round(flops / (v * 1e-3) / 1e12, 1) for k, v in med.items()}
        print(json.dumps({
            "what": "LPIPS vgg v0.1, one pair", "size": f"{W}x{H}", "iters": args.iters, "repeats": args.repeats,
            "ms": ms, "ms_median": med, "conv_tflop_per_pair": round(flops / 1e12, 4), "achieved_tflops": tflops,
            "share_of_tf32_datasheet_495": {k: round(v / TF32_DATASHEET_TFLOPS, 3) for k, v in tflops.items()},
            "our_launches_ms": [round(e - b, 4) for _, b, e in prof],
            "lpips": {"sugar_b200": float(ours(x, y)[0]), "torchvision_cudnn_tf32": float(theirs(x, y)[0])},
            "card": info}), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
