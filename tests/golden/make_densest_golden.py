"""Golden vectors for the coarse_density trainer's density estimation loss from the reference's OWN code.

Runs in the build container (needs /root/reference):  python tests/golden/make_densest_golden.py
The loss is not a function in the reference: it is a block inside the training loop.  This script reads exactly
sugar_trainers/coarse_density.py:642-649 (get_field_values), :654-656 (the projection-mode estimate) and :684-691
(the 'density' mode loss) from /root/reference at run time, dedents each and executes them unchanged in a namespace
holding what the loop has in scope there (`sugar`, `sdf_samples`, `sdf_gaussian_idx` and the trainer's flags,
coarse_density.py:121-156).  `sugar` is duck-typed: get_field_values / get_covariance / get_beta / get_normals /
get_smallest_axis are the reference's SuGaR methods called unbound (the stubs of make_field_golden.py).  Nothing of
the reference is copied into the repository; only the resulting numbers are stored.

Each case runs in float32 and in float64.  Outputs: tests/golden/densest_<case>.npz with, per dtype suffix
(none for float32, `_f64`): density, beta, estimate (e), target, loss (per sample), the scalar `total` the trainer adds
and the autograd gradients of sum(w * loss) for a seeded w [N]; closest_gaussian_opacities in float32 only.
"""
import os
import sys
import textwrap
from unittest import mock

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
from oracle import field_oracle as fo  # noqa: E402

CASES = {"c1_1k_2k": dict(P=1000, N=2000, K=16, seed=0),
         "k8": dict(P=400, N=600, K=8, seed=5),
         "k5_odd": dict(P=500, N=1001, K=5, seed=7),      # 32 samples per CTA at K = 5: N is not a multiple
         "degenerate": dict(P=600, N=1200, K=16, seed=11)}
BLOCKS = [("sugar_trainers/coarse_density.py", 642, 649), ("sugar_trainers/coarse_density.py", 654, 656),
          ("sugar_trainers/coarse_density.py", 684, 691)]
LEAVES = ("x", "points", "scaling", "quaternions", "strengths")


def make_densest_case(name):
    """fo.make_case at density_factor 1 (the trainer's, coarse_density.py:150-152).  'degenerate' also has
    - samples at their own Gaussian's centre (e = 0, target = 1),
    - samples far along their Gaussian's normal, away from every neighbour (rho = 0 and target = 0: |0 - 0|),
    - Gaussians whose two smallest scales are equal (the normal is the first of them, like torch.min).
    (Samples far inside their Gaussian's plane are left out on purpose: there e is the rounding noise of
    <x - mu, n> at |x - mu| = 100, and dL/dq = dL/de (x - mu) amplifies that noise past any fixed tolerance.)"""
    cfg = CASES[name]
    case = fo.make_case(density_factor=1.0, density_threshold=1.0, **cfg)
    if name != "degenerate":
        return case
    x, s, gi = case["x"].copy(), case["scaling"].copy(), case["gaussian_idx"]
    s[0::4, 1] = s[0::4, 0]                                   # first two equal ...
    s[0::4, 2] = 2.0 * np.maximum(s[0::4, 0], s[0::4, 2])     # ... and the smallest
    s[1::4, 2] = s[1::4, 1]                                   # last two equal ...
    s[1::4, 0] = 2.0 * np.maximum(s[1::4, 0], s[1::4, 1])     # ... and the smallest
    s[2::8] = s[2::8, :1]                                     # all three equal
    q = torch.from_numpy(case["quaternions"]).double()
    R = fo.quaternion_to_matrix(q).numpy()
    col = s.argmin(1)
    n = R[np.arange(len(s)), :, col]                           # the normal column of each Gaussian
    pts = case["points"].astype(np.float64)
    x[0::5] = case["points"][gi[0::5]]
    x[1::5] = (pts[gi[1::5]] + 100.0 * n[gi[1::5]]).astype(np.float32)
    case.update(x=np.ascontiguousarray(x), scaling=np.ascontiguousarray(s.astype(np.float32)))
    return case


def import_reference_sugar():
    from make_field_golden import import_reference_sugar as imp
    return imp()


def weights(N, seed=99):
    return torch.randn(N, generator=torch.Generator().manual_seed(seed)).numpy()


def main():
    torch.set_num_threads(1)   # index_put's accumulation order, and so the float32 gradients, then repeat exactly
    SuGaR = import_reference_sugar().SuGaR
    code = []
    for path, a, b in BLOCKS:
        lines = open(os.path.join("/root/reference", path)).read().splitlines()[a - 1:b]
        code.append(compile(textwrap.dedent("\n".join(lines)), f"{os.path.basename(path)}:{a}-{b}", "exec"))
    for name, cfg in CASES.items():
        case = make_densest_case(name)
        out = {}
        for dt, suffix in ((torch.float32, ""), (torch.float64, "_f64")):
            leaf = {k: torch.from_numpy(case[k]).to(dt).clone().requires_grad_(True) for k in LEAVES}

            class Fake:
                beta_mode = "average"
                device = "cpu"
                binded_to_surface_mesh = False
                points = leaf["points"]
                scaling = leaf["scaling"]
                quaternions = leaf["quaternions"]
                strengths = leaf["strengths"].view(-1, 1)
                knn_idx = fo.knn_idx(torch.from_numpy(case["points"]), cfg["K"])

                def get_covariance(self, **kw):
                    return SuGaR.get_covariance(self, **kw)

                def get_beta(self, *a, **kw):
                    return SuGaR.get_beta(self, *a, **kw)

                def get_field_values(self, *a, **kw):
                    return SuGaR.get_field_values(self, *a, **kw)

                def get_smallest_axis(self, **kw):
                    return SuGaR.get_smallest_axis(self, **kw)

                def get_normals(self, **kw):
                    return SuGaR.get_normals(self, **kw)
            sugar = Fake()
            gi = torch.from_numpy(case["gaussian_idx"])
            assert torch.equal(sugar.knn_idx[gi], torch.from_numpy(case["nbr_idx"]))
            ns = dict(torch=torch, sugar=sugar, sdf_samples=leaf["x"], sdf_gaussian_idx=gi,
                      use_sdf_estimation_loss=True, enforce_samples_to_be_on_surface=False,
                      sdf_estimation_mode="density", iteration=9001, start_sdf_estimation_from=9000,
                      use_sdf_better_normal_loss=True, start_sdf_better_normal_from=9000, density_threshold=1.0,
                      density_factor=1.0, squared_sdf_estimation_loss=False, sdf_estimation_factor=1.0, loss=0.0,
                      CONSOLE=mock.MagicMock())
            for c in code:
                exec(c, ns)
            w = torch.from_numpy(weights(case["x"].shape[0])).to(dt)
            (ns["sdf_estimation_loss"] * w).sum().backward()
            f = ns["fields"]
            vals = dict(density=f["density"], beta=f["beta"], closest_gaussian_opacities=f["closest_gaussian_opacities"],
                        estimate=ns["sdf_estimation"], target=ns["target_densities"], loss=ns["sdf_estimation_loss"],
                        total=ns["loss"])
            if suffix:
                vals.pop("closest_gaussian_opacities")   # the float32 run's is what the kernels are compared with
            out.update({k + suffix: v.detach().numpy() for k, v in vals.items()})
            out.update({"grad_" + k + suffix: v.grad.numpy() for k, v in leaf.items()})
        np.savez_compressed(os.path.join(HERE, f"densest_{name}.npz"), **out)
        print(name, float(out["total"]), {k: float(np.abs(v).max()) for k, v in out.items()
                                          if k.startswith("grad_") and not k.endswith("_f64")})


if __name__ == "__main__":
    main()
