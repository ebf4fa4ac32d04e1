"""Generate golden vectors from the UNMODIFIED reference CUDA build (oracle/_ref).

Must run on a GPU box:   python tests/golden/make_golden.py gpurun_out/golden
Inputs are NOT stored: they are regenerated from the seed by sugar_b200.scenes.make_scene
(numpy PCG64, platform independent).  Outputs are what the reference's own kernels produced on
the GPU: every array of its GeometryState / BinningState / ImageState plus image and gradients.
The committed .npz files under tests/golden/ pin the CPU oracle (tests/test_oracle_golden.py).
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

# name -> (P, W, H, seed, camera, use_sh, sh_degree, bg, extra scene kwargs)
GOLDEN_CASES = {
    "sh3_posed": (1500, 160, 96, 11, "posed", True, 3, (0.0, 0.0, 0.0), {}),
    "colors_identity": (1500, 160, 96, 12, "identity", False, 0, (0.1, 0.2, 0.3), {}),
    "sh1_flat": (1200, 128, 80, 13, "posed", True, 1, (1.0, 1.0, 1.0), {"mesh_bound": True}),
}


def main(outdir):
    import torch
    import helpers as h
    from sugar_b200 import scenes
    ref = h.load_ref_module()
    os.makedirs(outdir, exist_ok=True)
    for name, (P, W, H, seed, camera, use_sh, deg, bg, extra) in GOLDEN_CASES.items():
        sc = scenes.make_scene(P, W, H, seed=seed, camera=camera, **extra)
        dL = scenes.upstream_grad(W, H, seed=seed + 100)
        out = h.run_module(ref, sc, bg, None, use_sh=use_sh, sh_degree=deg)
        st = h.decode_ref_state(out, P, W, H)
        arrays = {k: v.cpu().numpy() for k, v in st.items()}
        arrays["radii"] = out["radii"].cpu().numpy()
        arrays["color"] = out["color"].cpu().numpy()
        arrays["num_rendered"] = np.int64(out["num_rendered"])
        outb = h.run_module(ref, sc, bg, dL, use_sh=use_sh, sh_degree=deg)
        for k, g in outb["grads"].items():
            arrays["grad_" + k] = g.cpu().numpy()
        np.savez_compressed(os.path.join(outdir, name + ".npz"), **arrays)
        print(name, "R =", out["num_rendered"], "visible =", int((out["radii"] > 0).sum()))
    print("torch", torch.__version__, torch.cuda.get_device_name(0))


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "gpurun_out/golden")
