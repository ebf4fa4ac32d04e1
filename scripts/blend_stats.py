"""What the blend loops do on the headline scene (needs the -DSGR_BLEND_STATS build):
    SGR_LIB_OUT=sugar_b200/lib/variants/lib_stats.so SGR_NVCC_EXTRA=-DSGR_BLEND_STATS python sugar_b200/build.py --force
    SGR_LIB_PATH=$PWD/sugar_b200/lib/variants/lib_stats.so python scripts/blend_stats.py [P W H]
Prints strip-splat visits / candidates / contributing visits and lane utilisation of both blend kernels, and the
instances of the forward's lists: all R of them (the reference's list) and the live ones the sorts and blend kernels
walk (scatter leaves out the instances whose footprint mask is empty)."""
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import torch
import helpers as h
from sugar_b200 import _lib, diff_gaussian_rasterization as ours, scenes

P, W, H = (int(a) for a in sys.argv[1:4]) if len(sys.argv) > 3 else (3_000_000, 1920, 1080)
fn = _lib.lib.sgr_debug_blend_stats
fn.restype = C.c_int
fn.argtypes = [C.c_void_p, C.c_int]
buf = (C.c_ulonglong * 16)()
sc = scenes.make_scene(P, W, H, seed=0)
dL = scenes.upstream_grad(W, H)
fn(buf, 1)
out = h.run_module(ours, sc, (0, 0, 0), dL, use_sh=True, sh_degree=3)
torch.cuda.synchronize()
fn(buf, 1)
v = [int(x) for x in buf]
# tile_start / tile_cursor of the image state (sgr_internal.cuh, ImageState): the live list of tile t ends at cursor[t]
T = ((W + 15) // 16) * ((H + 15) // 16)
align = lambda x: (x + 255) // 256 * 256
img = out["img"]
p = align(img.data_ptr()) - img.data_ptr() + 2 * align(W * H * 4) + align(T * 4)
start = img[p:p + 4 * T].view(torch.int32).long()
q = p + align((T + 1) * 4)
live = int((img[q:q + 4 * T].view(torch.int32).long() - start).sum())
names = ["visits", "visits_with_candidate", "visits_with_contributor", "candidate_lanes", "contributing_pairs",
         "live_lanes", "records_staged", "-"]
R = out["num_rendered"]
res = {"P": P, "W": W, "H": H, "R": R, "live": live, "dropped": round(1.0 - live / max(R, 1), 4),
       "forward": dict(zip(names, v[:8])), "backward": dict(zip(names, v[8:]))}
for k in ("forward", "backward"):
    d = res[k]
    d["contrib_visits_per_visit"] = round(d["visits_with_contributor"] / max(d["visits"], 1), 3)
    d["lanes_per_contrib_visit"] = round(d["contributing_pairs"] / max(d["visits_with_contributor"], 1), 2)
    d["visits_per_staged_record"] = round(d["visits"] / max(d["records_staged"], 1), 3)
print(json.dumps(res, indent=1))
