"""Golden results of the UNMODIFIED reference CUDA build (oracle/_ref) on the projection edge scenes.

    python tests/golden/make_projection_golden.py [OUT_DIR]     (needs a GPU and oracle/_ref, oracle/build_ref.py)

For every scene of tests/edge_scenes.CASES (the guard band, the near plane, far off-screen centres, scale_modifier)
it writes OUT_DIR (default tests/golden)/
  * refbuild_projection_<scene>.npz: digests of the forward outputs the GPU tests hold bit-exact, cov3D's included,
    and every gradient whole, with the reference's own run-to-run difference (make_refbuild_golden.parity_case's
    layout);
  * projection_<scene>.npz for the scenes in WHOLE_STATE: the reference's whole forward state, image and gradients
    (make_golden.py's layout), which tests/test_projection_edges_cpu.py holds the CPU oracle to.
Inputs are not stored: they are rebuilt from the seeds.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))
import edge_scenes as es  # noqa: E402
import helpers as h  # noqa: E402
import test_gpu_parity  # noqa: E402
from make_refbuild_golden import digests, grads, noise  # noqa: E402

WHOLE_STATE = ("guard_band_identity_colors", "guard_band_posed_sh3", "guard_edge", "near_plane", "offscreen_centres",
               "scale_mod_1.7_guard_band")


def projection_case(ref, name):
    c = es.CASES[name]
    sc, _ = c["build"]()
    P, W, H = sc.means3D.shape[0], sc.width, sc.height
    dL = es.upstream(name)
    opts = es.opts(name)
    b = h.run_module(ref, sc, c["bg"], None, **opts)
    rs = h.decode_ref_state(b, P, W, H)
    d = {"num_rendered": np.int64(b["num_rendered"])}
    d.update(digests(test_gpu_parity.forward_fields(b, rs, c["use_sh"])))
    # with precomputed colours the reference leaves rgb and the clamp bits unwritten
    whole = {k: v.cpu().numpy() for k, v in rs.items() if c["use_sh"] or k not in ("rgb", "clamped")}
    whole.update(radii=b["radii"].cpu().numpy(), color=b["color"].cpu().numpy(),
                 num_rendered=np.int64(b["num_rendered"]))
    for k in ("depths", "means2D", "cov3D", "conic_opacity", "rgb", "clamped"):   # unwritten for culled Gaussians
        if k in whole:
            whole[k][whole["radii"] <= 0] = 0
    b = h.run_module(ref, sc, c["bg"], dL, **opts)
    b2 = h.run_module(ref, sc, c["bg"], dL, **opts)
    d.update(grads(b))
    d.update(noise(b, b2))
    whole.update({"grad_" + k: g.cpu().numpy() for k, g in b["grads"].items()})
    return d, whole


def main():
    out_dir = sys.argv[1] if len(sys.argv) > 1 else HERE
    os.makedirs(out_dir, exist_ok=True)
    if not h.have_ref():
        raise SystemExit("oracle/_ref not built: python oracle/build_ref.py")
    ref = h.load_ref_module()
    for name in es.CASES:
        d, whole = projection_case(ref, name)
        np.savez_compressed(os.path.join(out_dir, f"refbuild_projection_{name}.npz"), **d)
        if name in WHOLE_STATE:
            np.savez_compressed(os.path.join(out_dir, f"projection_{name}.npz"), **whole)
        print("wrote", name, "R =", int(d["num_rendered"]), flush=True)


if __name__ == "__main__":
    main()
