"""GPU: the fused density estimation loss (field.density_estimation_loss, csrc/sgr_field.cu densest_*_kernel) against
the golden vectors of the trainer's own lines, the oracle in float64, and the field op's own outputs; and
coarse_density_step through steps.ours_ops() against the same step over the oracle chain.

Tolerances: the field's, 2e-5 relative per tensor for values and 1e-4 for gradients (sums of atomically accumulated
terms) against the goldens.  Against float64, per sample and per Gaussian row, ours may be off by a small floor plus
a few times what the float32 oracle itself is off (e = <x - mu, n> cancels for samples near their Gaussian's plane)."""
import os
import sys

import numpy as np
import pytest
import torch

import helpers as h
from oracle import densest_oracle as deo
from oracle import field_oracle as fo

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
from make_densest_golden import CASES, LEAVES, make_densest_case, weights  # noqa: E402


def _ours(case, w, dev="cuda"):
    from sugar_b200 import field
    leaf = {k: torch.from_numpy(case[k]).to(dev).requires_grad_(True) for k in LEAVES}
    loss, nbr = field.density_estimation_loss(leaf["x"], torch.from_numpy(case["gaussian_idx"]).to(dev),
                                              torch.from_numpy(case["nbr_idx"]).to(dev), leaf["points"],
                                              leaf["scaling"], leaf["quaternions"], leaf["strengths"],
                                              density_factor=1.0, return_closest_gaussian_opacities=True)
    assert not nbr.requires_grad
    (loss * torch.from_numpy(w).to(dev)).sum().backward()
    return loss.detach().cpu().numpy(), nbr.cpu().numpy(), {k: v.grad.cpu().numpy() for k, v in leaf.items()}


def _oracle(case, w, dtype):
    leaf = {k: torch.from_numpy(case[k]).to(dtype).clone().requires_grad_(True) for k in LEAVES}
    loss = deo.density_estimation_loss_torch(leaf["x"], torch.from_numpy(case["gaussian_idx"]),
                                             torch.from_numpy(case["nbr_idx"]), leaf["points"], leaf["scaling"],
                                             leaf["quaternions"], leaf["strengths"], 1.0)
    (loss * torch.from_numpy(w).to(dtype)).sum().backward()
    with torch.no_grad():
        c = {k: v.detach() for k, v in leaf.items()}
        rho = fo.field_values_torch(c["x"], torch.from_numpy(case["nbr_idx"]), c["points"], c["scaling"],
                                    c["quaternions"], c["strengths"])["density"]
    return loss.detach().numpy(), rho.numpy(), {k: v.grad.numpy() for k, v in leaf.items()}


def _check_against_oracle(case):
    N = case["x"].shape[0]
    w = weights(N, seed=5)
    loss, _, grads = _ours(case, w)
    l32, _, g32 = _oracle(case, w, torch.float32)
    l64, rho64, g64 = _oracle(case, w, torch.float64)
    # per sample: |loss - loss64| <= 2e-5 (1 + rho) + 3 |loss32 - loss64|
    bound = 2e-5 * (1.0 + np.abs(rho64)) + 3.0 * np.abs(l32 - l64)
    bad = np.abs(loss - l64) > bound
    assert not bad.any(), (int(bad.sum()), float((np.abs(loss - l64) / bound).max()))
    # per Gaussian row (and per sample row for x)
    for k in LEAVES:
        want = g64[k].reshape(len(g64[k]), -1)
        bound = (1e-4 * np.abs(want).max(1, keepdims=True) + 4.0 * np.abs(g32[k].reshape(want.shape) - want) +
                 1e-5 * np.abs(want).max())
        r = h.row_errors(grads[k].reshape(want.shape), want, np.broadcast_to(bound, want.shape))
        assert r["n_over"] == 0, (k, r["ratio"], r["worst_row"])


@pytest.mark.parametrize("name", sorted(CASES))
def test_matches_reference_golden(name):
    gold = np.load(os.path.join(HERE, "golden", f"densest_{name}.npz"))
    case = make_densest_case(name)
    loss, nbr, grads = _ours(case, weights(case["x"].shape[0]))
    assert h.rel_err(loss, gold["loss"]) < 2e-5
    assert h.rel_err(nbr, gold["closest_gaussian_opacities"]) < 2e-5
    for k in LEAVES:
        assert h.rel_err(grads[k], gold["grad_" + k]) < 1e-4, k


# group widths G = 1, 2, 4, 8, 16, 32 and two pairs per lane at K = 33
@pytest.mark.parametrize("K", [1, 2, 3, 7, 16, 32, 33])
def test_matches_float64_oracle_at_every_group_width(K):
    case = fo.make_case(P=1500, N=3001, K=K, seed=40 + K, density_factor=1.0)
    _check_against_oracle(case)


def test_degenerate_samples_and_scales_match_float64_oracle():
    _check_against_oracle(make_densest_case("degenerate"))


@pytest.mark.parametrize("K", [5, 16, 32])
def test_rho_and_opacities_are_the_field_bits(K):
    """nbr_opacity equals field_values(density_factor=1)'s closest_gaussian_opacities bit for bit, and at samples on
    their own centre (e = 0, target = 1 exactly) loss equals |density - 1| of field_values bit for bit."""
    from sugar_b200 import field
    case = fo.make_case(P=2000, N=4000, K=K, seed=K, density_factor=1.0)
    case["x"][0::3] = case["points"][case["gaussian_idx"][0::3]]
    t = {k: torch.from_numpy(v).cuda() for k, v in case.items() if isinstance(v, np.ndarray)}
    args = (t["points"], t["scaling"], t["quaternions"], t["strengths"])
    loss, nbr = field.density_estimation_loss(t["x"], t["gaussian_idx"], t["nbr_idx"], *args,
                                              return_closest_gaussian_opacities=True)
    f = field.field_values(t["x"], t["nbr_idx"], *args, density_factor=1.0, return_sdf=False,
                           return_closest_gaussian_opacities=True)
    assert torch.equal(nbr, f["closest_gaussian_opacities"])
    assert torch.equal(loss[0::3], (f["density"][0::3] - 1.0).abs())
    assert torch.equal(field.density_estimation_loss(t["x"], t["gaussian_idx"], t["nbr_idx"], *args), loss)


def test_no_samples_gives_empty_loss_and_zero_gradients():
    from sugar_b200 import field
    case = fo.make_case(P=300, N=10, K=16, seed=1, density_factor=1.0)
    leaf = {k: torch.from_numpy(case[k]).cuda().requires_grad_(True) for k in LEAVES}
    loss = field.density_estimation_loss(leaf["x"][:0], torch.from_numpy(case["gaussian_idx"][:0]).cuda(),
                                         torch.from_numpy(case["nbr_idx"][:0]).cuda(), leaf["points"],
                                         leaf["scaling"], leaf["quaternions"], leaf["strengths"])
    assert loss.shape == (0,)
    loss.sum().backward()
    for k in ("points", "scaling", "quaternions", "strengths"):
        assert leaf[k].grad is not None and not leaf[k].grad.any(), k


def test_arguments_split_across_devices_are_refused():
    from sugar_b200 import field
    case = fo.make_case(P=50, N=20, K=4, seed=2, density_factor=1.0)
    t = {k: torch.from_numpy(v).cuda() for k, v in case.items() if isinstance(v, np.ndarray)}
    a = dict(x=t["x"], gaussian_idx=t["gaussian_idx"], closest_gaussians_idx=t["nbr_idx"], points=t["points"],
             scaling=t["scaling"], quaternions=t["quaternions"], strengths=t["strengths"])
    for k in a:
        if k == "x":
            continue
        b = dict(a, **{k: a[k].cpu()})
        with pytest.raises(ValueError, match=k):
            field.density_estimation_loss(**b)


@pytest.mark.parametrize("dssim_factor", [0.0, 0.2])
def test_coarse_density_step_matches_oracle_chain(dssim_factor):
    """coarse_density_step through steps.ours_ops() against the same step with the oracle as
    ops.density_estimation_loss (float32 and float64), by test_gpu_loss's rule for coarse_sdf_step."""
    from sugar_b200 import knn, scenes, steps
    P, W, H = 20_000, 320, 240
    sc = scenes.make_scene(P, W, H, seed=0)
    dev = torch.device("cuda")
    cam = steps.camera_from_scene(sc, dev)
    gt = torch.rand(3, H, W, generator=torch.Generator().manual_seed(0)).to(dev)
    leaf = lambda t: t.to(dev).requires_grad_(True)
    raw = dict(points=leaf(torch.from_numpy(sc.means3D)), sh_dc=leaf(torch.from_numpy(sc.shs[:, :1].copy())),
               sh_rest=leaf(torch.from_numpy(sc.shs[:, 1:].copy())),
               densities=leaf(torch.logit(torch.from_numpy(sc.opacities).clamp(1e-4, 1 - 1e-4))),
               scales=leaf(torch.from_numpy(sc.scales).log()), quaternions=leaf(torch.from_numpy(sc.rotations) * 1.3))
    knn_idx = knn.reset_neighbors(raw["points"].detach(), 16)[1]

    def oracle64(x, gi, nbr, points, scaling, quats, strengths, density_factor=1.0,
                 return_closest_gaussian_opacities=False):
        loss, opac = deo.density_estimation_loss_torch(x.double(), gi, nbr, points.double(), scaling.double(),
                                                       quats.double(), strengths.double(), density_factor, True)
        return loss.float(), opac.float()

    def run(est):
        ops = steps.ours_ops()
        if est is not None:
            ops.density_estimation_loss = est
        gen = torch.Generator(device=dev).manual_seed(1)
        loss, stats = steps.coarse_density_step(raw, cam, gt, knn_idx, ops, n_samples=20_000, generator=gen,
                                                dssim_factor=dssim_factor)
        assert stats["visible"] > 1000 and stats["sampled_gaussians"] == stats["visible"]
        grads = {k: v.grad.detach().cpu().numpy().copy() for k, v in raw.items()}
        for v in raw.values():
            v.grad = None
        return float(loss), grads
    a, a2 = run(None), run(None)
    r32 = run(deo.density_estimation_loss_torch)
    r64 = run(oracle64)
    assert abs(a[0] - r64[0]) <= max(2 * abs(r32[0] - r64[0]), 1e-6, 2 * abs(a[0] - a2[0]))
    for k in a[1]:
        err = h.rel_err(a[1][k], r64[1][k])
        allowed = max(2 * h.rel_err(r32[1][k], r64[1][k]), 1e-5, 2 * h.rel_err(a[1][k], a2[1][k]))
        assert err <= allowed, (k, err, allowed)
