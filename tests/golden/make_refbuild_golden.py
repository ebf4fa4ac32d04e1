"""Golden results of the UNMODIFIED reference CUDA build (oracle/_ref) for the GPU tests that compare with it.

    python tests/golden/make_refbuild_golden.py [OUT_DIR]      (needs a GPU and oracle/_ref, oracle/build_ref.py)

writes OUT_DIR (default tests/golden)/refbuild_*.npz, one file per test case, from the same seeded inputs the
tests build.  Outputs the tests hold to be bit-identical are kept as SHA-256 digests of their values
(helpers.digest); each gradient as its shape, |g|_inf, an evenly spaced sample and its largest entries, and
whole where a case's gradients hold at most helpers.WHOLE_MAX entries (helpers.grad_summary); plus the reference's
own run-to-run difference (fp32 atomics) where a test uses it.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))
import helpers as h  # noqa: E402
import test_gpu_configs  # noqa: E402
import test_gpu_parity  # noqa: E402


def grads(out):
    whole = sum(g.numel() for g in out["grads"].values()) <= h.WHOLE_MAX
    d = {}
    for k, g in out["grads"].items():
        d.update(h.grad_summary(f"grad_{k}", g, whole=whole))
    return d


def noise(b, b2):
    return {f"noise_{k}": np.float64(h.rel_err(b2["grads"][k].cpu().numpy(), b["grads"][k].cpu().numpy()))
            for k in b["grads"]}


def digests(fields):
    return {"digest_" + k: h.digest(v) for k, v in fields.items()}


def parity_case(ref, case):
    from sugar_b200 import scenes
    name, P, W, H, camera, use_sh, deg, covpre, bg = case
    sc = test_gpu_parity._scene(name, P, W, H, camera)
    dL = scenes.upstream_grad(W, H)
    cov3D = test_gpu_parity._cov_from_oracle(sc) if covpre else None
    opts = dict(use_sh=use_sh, sh_degree=deg, use_cov_precomp=covpre, cov3D=cov3D)
    b = h.run_module(ref, sc, bg, None, **opts)
    rs = h.decode_ref_state(b, P, W, H)
    d = {"num_rendered": np.int64(b["num_rendered"])}
    d.update(digests(test_gpu_parity.forward_fields(b, rs, use_sh)))
    b = h.run_module(ref, sc, bg, dL, **opts)
    b2 = h.run_module(ref, sc, bg, dL, **opts)
    d.update(grads(b))
    d.update(noise(b, b2))
    return d


def config_case(ref, cfg):
    from sugar_b200 import scenes
    name, P, W, H, deg, mesh = cfg
    sc = scenes.make_scene(P, W, H, seed=0, mesh_bound=mesh)
    dL = scenes.upstream_grad(W, H)
    b = h.run_module(ref, sc, (0.0, 0.0, 0.0), dL, use_sh=True, sh_degree=deg)
    rs = h.decode_ref_state(b, P, W, H)
    d = {"num_rendered": np.int64(b["num_rendered"])}
    d.update(digests(dict(radii=b["radii"], color=b["color"], n_contrib=rs["n_contrib"], final_T=rs["final_T"],
                          point_list=rs["point_list"], keys=rs["keys"], ranges=rs["ranges"])))
    del rs
    d.update(grads(b))
    if mesh:
        d.update(noise(b, h.run_module(ref, sc, (0.0, 0.0, 0.0), dL, use_sh=True, sh_degree=deg)))
    return d


def sh_layout_case(ref, M, deg):
    color, radii, g = test_gpu_parity.run_sh_layout(ref, M, deg)
    d = digests(dict(radii=radii, color=color))
    d.update(grads({"grads": g}))
    return d


def render_case(ref):
    import torch
    g = np.load(os.path.join(HERE, "render_wrapper.npz"))
    t = lambda k: torch.from_numpy(g[k]).cuda()
    H, W = (int(v) for v in g["hw"])
    st = ref.GaussianRasterizationSettings(
        image_height=H, image_width=W, tanfovx=float(g["tanfov"][0]), tanfovy=float(g["tanfov"][1]), bg=t("bg"),
        scale_modifier=1.0, viewmatrix=t("viewmatrix"), projmatrix=t("projmatrix"), sh_degree=int(g["sh_degree"]),
        campos=t("campos"), prefiltered=False, debug=False)
    m3 = t("means3D")
    img, radii = ref.GaussianRasterizer(st)(means3D=m3, means2D=torch.zeros_like(m3), opacities=t("opacities"),
                                            colors_precomp=t("colors_precomp"), scales=t("scales"),
                                            rotations=t("rotations"))
    return {"image": img.cpu().numpy().astype(np.float32), "radii": radii.cpu().numpy().astype(np.int32)}


def main():
    out_dir = sys.argv[1] if len(sys.argv) > 1 else HERE
    os.makedirs(out_dir, exist_ok=True)
    if not h.have_ref():
        raise SystemExit("oracle/_ref not built: python oracle/build_ref.py")
    ref = h.load_ref_module()

    def save(name, d):
        np.savez_compressed(os.path.join(out_dir, f"refbuild_{name}.npz"), **d)
        print("wrote", name, flush=True)
    for case in test_gpu_parity.CASES:
        save("parity_" + case[0], parity_case(ref, case))
    for M, deg in test_gpu_parity.SH_LAYOUTS:
        save(f"sh_layout_{M}_{deg}", sh_layout_case(ref, M, deg))
    for cfg in test_gpu_configs.CONFIGS:
        save("config_" + cfg[0], config_case(ref, cfg))
    save("render", render_case(ref))


if __name__ == "__main__":
    main()
