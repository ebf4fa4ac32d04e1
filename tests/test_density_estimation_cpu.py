"""CPU: the coarse_density trainer's density estimation loss.  The oracle (oracle/densest_oracle.py) against golden
vectors from the trainer's own source lines (tests/golden/make_densest_golden.py), the op's argument checks, the C
entry points' checks, and coarse_density_step's recipe over the reference's op chains with a stand-in rasterizer."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

import helpers as h

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
from make_densest_golden import CASES, LEAVES, make_densest_case, weights  # noqa: E402
from oracle import densest_oracle as deo  # noqa: E402

VALUES = ("density", "beta", "estimate", "target", "loss")


def oracle_run(case, dtype):
    """-> (values incl. the oracle's own e / target, gradients of sum(w * loss)) in `dtype`."""
    from oracle import field_oracle as fo
    leaf = {k: torch.from_numpy(case[k]).to(dtype).clone().requires_grad_(True) for k in LEAVES}
    gi, nbr = torch.from_numpy(case["gaussian_idx"]), torch.from_numpy(case["nbr_idx"])
    loss, opac = deo.density_estimation_loss_torch(leaf["x"], gi, nbr, leaf["points"], leaf["scaling"],
                                                   leaf["quaternions"], leaf["strengths"], 1.0, True)
    (loss * torch.from_numpy(weights(len(loss))).to(dtype)).sum().backward()
    with torch.no_grad():
        f = fo.field_values_torch(leaf["x"], nbr, leaf["points"], leaf["scaling"], leaf["quaternions"],
                                  leaf["strengths"], 1.0)
        e = ((leaf["x"] - leaf["points"][gi]) * fo.smallest_axis(leaf["scaling"], leaf["quaternions"])[gi]).sum(-1)
    vals = dict(density=f["density"], beta=f["beta"], estimate=e, target=torch.exp(-0.5 * e.pow(2) / f["beta"].pow(2)),
                loss=loss.detach(), closest_gaussian_opacities=opac)
    return {k: v.numpy() for k, v in vals.items()}, {k: v.grad.numpy() for k, v in leaf.items()}


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_matches_the_trainer_lines(name):
    gold = np.load(os.path.join(HERE, "golden", f"densest_{name}.npz"))
    case = make_densest_case(name)
    v32, g32 = oracle_run(case, torch.float32)
    for k in VALUES + ("closest_gaussian_opacities",):
        assert h.rel_err(v32[k], gold[k]) < 2e-5, k
    assert abs(float(v32["loss"].mean()) - float(gold["total"])) <= 2e-5 * abs(float(gold["total"]))
    for k in LEAVES:
        assert h.rel_err(g32[k], gold["grad_" + k]) < 2e-5, k
    v64, g64 = oracle_run(case, torch.float64)
    for k in VALUES:
        assert h.rel_err(v64[k], gold[k + "_f64"]) < 1e-12, k
    for k in LEAVES:
        assert h.rel_err(g64[k], gold["grad_" + k + "_f64"]) < 1e-12, k


def test_degenerate_golden_covers_its_cases():
    """The degenerate case really has samples with e = 0 / target = 1, with rho = target = 0, and equal smallest
    scales; abs' gradient at rho == target is 0, so those samples move nothing."""
    gold = np.load(os.path.join(HERE, "golden", "densest_degenerate.npz"))
    case = make_densest_case("degenerate")
    assert (gold["target"] == 1.0).sum() >= 200 and ((gold["density"] == 0) & (gold["target"] == 0)).sum() >= 200
    s = np.sort(case["scaling"], 1)
    assert (s[:, 0] == s[:, 1]).sum() >= len(s) // 2
    still = (gold["density"] == gold["target"])
    gx = gold["grad_x"][still]
    assert still.sum() >= 200 and not gx.any()


def _args(P=8, N=5, K=4):
    g = torch.Generator().manual_seed(0)
    idx = torch.randint(0, P, (N, K), generator=g)
    return dict(x=torch.randn(N, 3, generator=g), gaussian_idx=idx[:, 0], closest_gaussians_idx=idx,
                points=torch.randn(P, 3, generator=g), scaling=torch.rand(P, 3, generator=g) + 0.1,
                quaternions=torch.nn.functional.normalize(torch.randn(P, 4, generator=g), dim=-1),
                strengths=torch.rand(P, 1, generator=g))


@pytest.mark.parametrize("arg,bad", [("x", lambda t: t[:, :2]), ("gaussian_idx", lambda t: t[1:]),
                                     ("closest_gaussians_idx", lambda t: t[1:]), ("points", lambda t: t[:, :2]),
                                     ("scaling", lambda t: t[1:]), ("quaternions", lambda t: t[:, :3]),
                                     ("strengths", lambda t: t[1:]), ("strengths", lambda t: t.expand(-1, 2))])
def test_op_checks_shapes(arg, bad):
    from sugar_b200 import field
    a = _args()
    a[arg] = bad(a[arg])
    with pytest.raises(ValueError, match=arg):
        field.density_estimation_loss(**a)


@pytest.mark.parametrize("arg,bad", [("x", lambda t: t.int()), ("points", lambda t: t.long()),
                                     ("gaussian_idx", lambda t: t.float()), ("closest_gaussians_idx", lambda t: t.double()),
                                     ("closest_gaussians_idx", lambda t: t > 2), ("quaternions", lambda t: t.int())])
def test_op_checks_dtypes(arg, bad):
    from sugar_b200 import field
    a = _args()
    a[arg] = bad(a[arg])
    with pytest.raises(ValueError, match=arg):
        field.density_estimation_loss(**a)


def test_valid_cpu_arguments_reach_the_cuda_requirement():
    from sugar_b200 import field
    a = _args()
    a["gaussian_idx"] = a["gaussian_idx"].int()       # int32 indices and float64 inputs are converted, not refused
    a["x"] = a["x"].double()
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        field.density_estimation_loss(**a)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        field.density_estimation_loss(**a, return_closest_gaussian_opacities=True)


def test_entry_points_validate_without_gpu():
    from sugar_b200 import _lib
    L = _lib.lib
    names = [L.sgr_kernel_name(k).decode() for k in range(L.sgr_num_kernel_kinds())]
    assert {"density_estimation_forward", "density_estimation_backward"} <= set(names)
    assert names[:20][-2:] == ["loss_forward", "loss_backward"] and names[-2:] == ["mesh_nc_forward", "mesh_nc_backward"]
    d = ctypes.c_void_p(256)

    def params(N=4, K=2, P=3, group=0):
        p = _lib.SgrFieldParams()
        p.N, p.K, p.P, p.samples_per_idx_row, p.density_factor = N, K, P, group, 1.0
        return ctypes.byref(p)
    fwd = lambda p, *ptrs: L.sgr_density_estimation_forward(p, *ptrs, None)
    bwd = lambda p, *ptrs: L.sgr_density_estimation_backward(p, *ptrs, None)
    for p in (None, params(N=-1), params(K=0), params(P=0), params(group=2)):
        assert fwd(p, *([d] * 8), d, d) == -1 and b"bad field sizes" in L.sgr_last_error()
        assert bwd(p, *([d] * 8), *([d] * 6)) == -1 and b"bad field sizes" in L.sgr_last_error()
    for i in range(8):                                  # x, own, nbr, points, scaling, quaternions, strengths, loss
        ptrs = [d] * 8
        ptrs[i if i < 7 else 7] = None
        args = ptrs[:7] + [ptrs[7], d, d]               # loss, nbr_opacity (may be NULL), scratch
        assert fwd(params(), *args) == -1 and b"null pointer" in L.sgr_last_error(), i
        bargs = ptrs[:7] + [ptrs[7]] + [d] * 6         # g_loss, g_x .. g_strengths, scratch
        assert bwd(params(), *bargs) == -1 and b"null pointer" in L.sgr_last_error(), i
    # N = 0: nothing to compute and nothing to check beyond the sizes; no CUDA call is made by the forward
    assert fwd(params(N=0), *([None] * 8), None, d) == 0


def test_coarse_density_step_recipe_runs_and_reaches_every_parameter():
    import bench
    import bench_workloads as bw
    from oracle import field_oracle as fo
    from test_steps_cpu import FakeRasterizerModule
    steps = bw._load_steps_without_package()
    scenes = bench.load_scenes()
    sc = scenes.make_scene(500, 64, 48, seed=0)
    cam = steps.camera_from_scene(sc, "cpu")
    ops = bw.reference_ops(torch, FakeRasterizerModule)
    leaf = lambda t: t.clone().requires_grad_(True)
    raw = dict(points=leaf(torch.from_numpy(sc.means3D)), sh_dc=leaf(torch.from_numpy(sc.shs[:, :1].copy())),
               sh_rest=leaf(torch.from_numpy(sc.shs[:, 1:].copy())),
               densities=leaf(torch.logit(torch.from_numpy(sc.opacities).clamp(1e-4, 1 - 1e-4))),
               scales=leaf(torch.from_numpy(sc.scales).log()), quaternions=leaf(torch.from_numpy(sc.rotations) * 1.3))
    knn = fo.knn_idx(raw["points"].detach(), 16)
    g = torch.Generator().manual_seed(1)
    loss, stats = steps.coarse_density_step(raw, cam, torch.rand(3, 48, 64), knn, ops, n_samples=2000, generator=g)
    assert np.isfinite(float(loss)) and stats == {"visible": 500, "sampled_gaussians": 500}
    for k, v in raw.items():
        assert v.grad is not None and bool(torch.isfinite(v.grad).all()), k
    for k in ("points", "scales", "quaternions", "densities"):
        assert float(raw[k].grad.abs().max()) > 0, k
