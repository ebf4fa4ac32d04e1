#!/usr/bin/env python
"""Time the ground-truth image preparation (sugar_b200/dataset.py: prepare_image, csrc/sgr_image.cu) at Mip-NeRF-360-
like sizes, with the host decode and Pillow's CPU resize of the same image beside it.

    python scripts/bench_dataset.py [--iters 50] [--repeats 3]

Cases (seeded noise images; noise is the worst case for nothing here, the kernels are data-independent):
    rgb_5187x3361_to_1600   an RGB frame to 3DGS's 1.6K width (-r -1)        both passes
    rgb_4946x3286_to_1920   an RGB frame to SuGaR's 1920 cap                 both passes
    rgba_5187x3361_to_1600  an RGBA PNG, premultiplied through RGBa          both passes
    nerf_800_white          an 800x800 NeRF-synthetic RGBA frame over white  composite only
    nerf_1600_white_to_800  a 1600x1600 RGBA frame over white, to 800        composite fused into the first pass
Per case one JSON line, each number the median of `repeats` rounds of `iters` images (tables uploaded once):
    kernel_ms_per_image  the sgr_image kernels alone: the library's event profiler brackets each launch (the image
                         passes are logged under its "misc" kind, and nothing else launches in the window)
    call_ms_per_image    CUDA events around whole prepare_image calls: the kernels plus the host work between them
                         (argument checks, two allocations, the ctypes call); on small frames this is the host's issue
                         rate, not the kernels
and the kernels' achieved bytes/s against the byte model
    source H_in W_in C + (both passes) intermediate written and read 2 H_in W_out C_mid + output 12 H_out W_out
(the resample tables are a few kB and omitted), as a fraction of the HBM peak (MEASURED_PEAKS.json when present, else
the H100 SXM data sheet's 3.35 TB/s, named as such); the host decode of the same image as a PNG (objfile.read_png,
labelled host); and Pillow's Image.resize of it on the CPU (labelled host; absent when Pillow is missing).  Every line
carries the card's name, power limit and max SM clock, read in the same run.  Prints only; writes nothing but a
temporary PNG, removed at the end.
"""
import argparse
import json
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from bench_meshloss import card, median  # noqa: E402

CASES = (   # name, (H, W, C), (w, h), background
    ("rgb_5187x3361_to_1600", (3361, 5187, 3), (1600, 1036), None),
    ("rgb_4946x3286_to_1920", (3286, 4946, 3), (1920, 1276), None),
    ("rgba_5187x3361_to_1600", (3361, 5187, 4), (1600, 1036), None),
    ("nerf_800_white", (800, 800, 4), (800, 800), "white"),
    ("nerf_1600_white_to_800", (1600, 1600, 4), (800, 800), "white"),
)


def byte_model(shape, w, h, bg):
    H, W, C = shape
    mid = 4 if C == 4 and bg is None else 3
    both = W != w and H != h
    return H * W * C + (2 * H * w * mid if both else 0) + 12 * h * w


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    import numpy as np
    import torch
    import bench
    import dataset_cases as dc
    from sugar_b200 import _lib, dataset, objfile
    if not torch.cuda.is_available():
        raise SystemExit("bench_dataset.py needs a GPU")
    info = card(0)
    peak, peak_src = bench.load_peaks()
    dev = torch.device("cuda", 0)
    try:
        from PIL import Image
    except ImportError:
        Image = None
    tmp = tempfile.mkdtemp()
    try:
        for name, shape, (w, h), bg in CASES:
            rng = np.random.Generator(np.random.PCG64(len(name)))
            img = rng.integers(0, 256, shape, dtype=np.uint8)
            src = torch.from_numpy(img).to(dev)
            dataset.prepare_image(src, w, h, background=bg, device=dev)   # tables uploaded, kernels loaded
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            kernel, call = [], []
            for _ in range(args.repeats):
                torch.cuda.synchronize()
                e0.record()
                for _ in range(args.iters):
                    dataset.prepare_image(src, w, h, background=bg, device=dev)
                e1.record()
                torch.cuda.synchronize()
                call.append(e0.elapsed_time(e1) / args.iters)
                _lib.profile_read()          # clears the log
                _lib.profile(True)
                for _ in range(args.iters):
                    dataset.prepare_image(src, w, h, background=bg, device=dev)
                torch.cuda.synchronize()
                log = _lib.profile_read()
                _lib.profile(False)
                assert set(log) == {"misc"}, log
                kernel.append(log["misc"][0] / args.iters)
            ms = median(kernel)
            launches = log["misc"][1] // args.iters
            nbytes = byte_model(shape, w, h, bg)
            png = os.path.join(tmp, "frame.png")
            dc.write_png(png, img)
            t0 = time.perf_counter()
            objfile.read_png(png, keep_alpha=True)
            decode_ms = (time.perf_counter() - t0) * 1e3
            line = dict(case=name, in_shape=list(shape), out_size=[w, h], background=bg,
                        kernel_ms_per_image=round(ms, 4), kernel_ms_rounds=[round(x, 4) for x in kernel],
                        launches_per_image=launches, call_ms_per_image=round(median(call), 4),
                        call_ms_rounds=[round(x, 4) for x in call],
                        model_bytes=nbytes, achieved_gbs=round(nbytes / ms / 1e6, 1),
                        fraction_of_hbm_peak=round(nbytes / ms / 1e6 / peak, 3), hbm_peak_gbs=peak,
                        hbm_peak_source=peak_src, host_png_decode_ms=round(decode_ms, 1))
            if Image is not None:
                im = Image.fromarray(img, "RGB" if shape[2] == 3 else "RGBA")
                t0 = time.perf_counter()
                im.resize((w, h))
                line["host_pil_resize_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
            line["card"] = info
            print(json.dumps(line), flush=True)
    finally:
        for f in os.listdir(tmp):
            os.remove(os.path.join(tmp, f))
        os.rmdir(tmp)


if __name__ == "__main__":
    main()
