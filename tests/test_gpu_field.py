"""GPU: fused density / SDF field kernels vs the CPU oracle (values and gradients) and vs the
golden vectors of the reference's own code.  fp32 tolerance: 2e-5 relative per tensor for values,
1e-4 for gradients (sums of N*K atomically accumulated terms)."""
import os
import sys

import numpy as np
import pytest
import torch

import helpers as h
from oracle import field_oracle as fo

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))


def _run_ours(case, weights, dev="cuda"):
    from sugar_b200 import field
    leaf = {k: torch.from_numpy(case[k]).to(dev).requires_grad_(True)
            for k in ("x", "points", "scaling", "quaternions", "strengths")}
    out = field.field_values(leaf["x"], torch.from_numpy(case["nbr_idx"]).to(dev), leaf["points"], leaf["scaling"],
                             leaf["quaternions"], leaf["strengths"], density_factor=case["density_factor"],
                             density_threshold=case["density_threshold"], return_sdf=True,
                             return_closest_gaussian_opacities=True, return_beta=True)
    loss = sum((out[k] * torch.from_numpy(weights[k]).to(dev)).sum() for k in weights)
    loss.backward()
    return out, {k: v.grad for k, v in leaf.items()}


@pytest.mark.parametrize("name", ["c1_1k_2k", "k8"])
def test_field_matches_reference_golden(name):
    from make_field_golden import CASES
    from oracle import field_oracle as fo
    gold = np.load(os.path.join(HERE, "golden", f"field_{name}.npz"))
    case = fo.make_case(density_threshold=1.0, **CASES[name])
    w = {k: gold["w_" + k] for k in ("density", "sdf", "beta", "closest_gaussian_opacities")}
    out, grads = _run_ours(case, w)
    for k in w:
        assert h.rel_err(out[k].detach().cpu().numpy(), gold[k]) < 2e-5, k
    for k, g in grads.items():
        assert h.rel_err(g.cpu().numpy(), gold["grad_" + k]) < 1e-4, k


@pytest.mark.parametrize("P,N,K", [(5000, 20000, 16), (3000, 7001, 5), (2000, 4000, 32)])
def test_field_matches_oracle(P, N, K):
    from oracle import field_oracle as fo
    case = fo.make_case(P=P, N=N, K=K, seed=P % 97, density_factor=1.0 / K)
    rng = np.random.default_rng(1)
    w = {"density": rng.normal(size=N).astype(np.float32), "sdf": rng.normal(size=N).astype(np.float32),
         "beta": rng.normal(size=N).astype(np.float32),
         "closest_gaussian_opacities": rng.normal(size=(N, K)).astype(np.float32)}
    out, grads = _run_ours(case, w)
    leaf = {k: torch.from_numpy(case[k]).clone().requires_grad_(True)
            for k in ("x", "points", "scaling", "quaternions", "strengths")}
    ref = fo.field_values_torch(leaf["x"], torch.from_numpy(case["nbr_idx"]), leaf["points"], leaf["scaling"],
                                leaf["quaternions"], leaf["strengths"], case["density_factor"], 1.0)
    sum((ref[k] * torch.from_numpy(w[k])).sum() for k in w).backward()
    for k in w:
        assert h.rel_err(out[k].detach().cpu().numpy(), ref[k].detach().numpy()) < 2e-5, k
    for k, g in grads.items():
        assert h.rel_err(g.cpu().numpy(), leaf[k].grad.numpy()) < 1e-4, k


FIELD_LEAVES = ("x", "points", "scaling", "quaternions", "strengths")


def _weights(N, K, seed=1):
    rng = np.random.default_rng(seed)
    return {"density": rng.normal(size=N).astype(np.float32), "sdf": rng.normal(size=N).astype(np.float32),
            "beta": rng.normal(size=N).astype(np.float32),
            "closest_gaussian_opacities": rng.normal(size=(N, K)).astype(np.float32)}


def _field_oracle64(case, w):
    """field_oracle.field_values_torch in float64: the weighted outputs and the gradients of the leaves."""
    leaf = {k: torch.from_numpy(case[k]).double().requires_grad_(True) for k in FIELD_LEAVES}
    ref = fo.field_values_torch(leaf["x"], torch.from_numpy(case["nbr_idx"]), leaf["points"], leaf["scaling"],
                                leaf["quaternions"], leaf["strengths"], case["density_factor"], 1.0)
    sum((ref[k] * torch.from_numpy(w[k]).double()).sum() for k in w).backward()
    return {k: ref[k].detach().numpy() for k in w}, {k: v.grad.numpy() for k, v in leaf.items()}


def _check_field(case, w=None):
    N, K = case["nbr_idx"].shape
    w = w or _weights(N, K)
    out, grads = _run_ours(case, w)
    ref, rgrads = _field_oracle64(case, w)
    for k in w:
        assert h.rel_err(out[k].detach().cpu().numpy(), ref[k]) < 2e-5, k
    for k, g in grads.items():
        assert h.rel_err(g.cpu().numpy(), rgrads[k]) < 1e-4, k


def _check_normal(case):
    opac = fo.field_values(**case)["closest_gaussian_opacities"]
    loss, gq = _normal_ours(case, opac)
    t = lambda k: torch.from_numpy(case[k])

    def oracle(dt):
        q = t("quaternions").to(dt).clone().requires_grad_(True)
        ref = fo.better_normal_loss_torch(t("x").to(dt), t("gaussian_idx"), t("nbr_idx"), t("points").to(dt),
                                          t("scaling").to(dt), q, torch.from_numpy(opac).to(dt))
        ref.mean().backward()
        return ref.detach().numpy(), q.grad.numpy()
    l32, g32 = oracle(torch.float32)
    l64, g64 = oracle(torch.float64)
    # the same allowance as test_normal_loss_matches_oracle: 3x the fp32 op chain's own distance from float64
    assert h.rel_err(loss, l64) < max(2e-5, 3 * h.rel_err(l32, l64))
    assert h.rel_err(gq, g64) < max(1e-4, 3 * h.rel_err(g32, g64))


# K = 1 and 2: one lane group per sample of width 1 / 2; K = 33, 64: a 32-lane group with two pairs per lane
@pytest.mark.parametrize("P,N,K", [(1500, 3001, 1), (1500, 3001, 2), (2000, 4000, 33), (1000, 2003, 64)])
def test_field_and_normal_loss_at_group_widths_the_trainers_do_not_use(P, N, K):
    case = fo.make_case(P=P, N=N, K=K, seed=P % 97 + K, density_factor=1.0 / K)
    _check_field(case)
    _check_normal(case)


def _edge_case(kind):
    """A K = 16 case with one kind of degenerate input on a third of the samples / Gaussians."""
    case = fo.make_case(P=1200, N=3000, K=16, seed=21, density_factor=1.0 / 16)
    rng = np.random.default_rng(3)
    N, P = case["nbr_idx"].shape[0], case["points"].shape[0]
    if kind == "repeated_ids":
        # the scatters of one row collide: pairs, a run of four, and rows that are one Gaussian K times
        idx = case["nbr_idx"].copy()
        idx[0::3, 1] = idx[0::3, 0]
        idx[1::3, 4:8] = idx[1::3, 9:10]
        idx[2::9, :] = idx[2::9, :1]
        case["nbr_idx"] = idx
    elif kind == "isotropic":
        # SuGaR initialises all three scales equal; the first smallest axis decides beta's column and the normal
        s = case["scaling"].copy()
        s[0::3, 1:] = s[0::3, :1]                       # all three equal
        s[1::3, 2] = s[1::3, 1] = np.minimum(s[1::3, 1], s[1::3, 2])   # the two last equal, possibly the minimum
        s[2::6, 0] = s[2::6, 2] = np.minimum(s[2::6, 0], s[2::6, 2])
        case["scaling"] = s
    elif kind == "tiny_scale":
        # below scaling.clamp(min=1e-8): 1/s is clamped, the clamped entry gets no gradient through it
        s = case["scaling"].copy()
        pick = rng.choice(P, P // 3, replace=False)
        s[pick, rng.integers(0, 3, pick.size)] = np.float32(3e-9)
        case["scaling"] = s
    return case


@pytest.mark.parametrize("kind", ["repeated_ids", "isotropic", "tiny_scale"])
def test_field_and_normal_loss_on_degenerate_inputs(kind):
    case = _edge_case(kind)
    _check_field(case)
    _check_normal(case)


def test_compute_density_with_samples_sharing_index_rows():
    """compute_density(samples_per_idx_row=4): row n // 4 of the index table serves sample n (ray samples sharing their
    pixel's neighbours) -- forward and backward against the oracle on the table with every row repeated four times.
    N is not a multiple of 4: the last row serves fewer samples."""
    from sugar_b200 import field
    case = fo.make_case(P=1500, N=1000, K=16, seed=8, density_factor=1.0 / 16)
    rng = np.random.default_rng(4)
    N = 4 * 1000 - 3
    x = np.repeat(case["x"], 4, axis=0)[:N] + rng.normal(0, 0.03, (N, 3)).astype(np.float32)
    rows = case["nbr_idx"]
    case4 = dict(case, x=np.ascontiguousarray(x, np.float32), nbr_idx=np.repeat(rows, 4, axis=0)[:N])
    wd, wn = rng.normal(size=N).astype(np.float32), rng.normal(size=(N, 16)).astype(np.float32)
    leaf = {k: torch.from_numpy(case4[k]).cuda().requires_grad_(True) for k in FIELD_LEAVES}
    d, nb = field.compute_density(leaf["x"], torch.from_numpy(rows).cuda(), leaf["points"], leaf["scaling"],
                                  leaf["quaternions"], leaf["strengths"], density_factor=1 / 16,
                                  return_closest_gaussian_opacities=True, samples_per_idx_row=4)
    ((d * torch.from_numpy(wd).cuda()).sum() + (nb * torch.from_numpy(wn).cuda()).sum()).backward()
    ref, rgrads = _field_oracle64(case4, {"density": wd, "closest_gaussian_opacities": wn})
    assert h.rel_err(d.detach().cpu().numpy(), ref["density"]) < 2e-5
    assert h.rel_err(nb.detach().cpu().numpy(), ref["closest_gaussian_opacities"]) < 2e-5
    for k in FIELD_LEAVES:
        assert h.rel_err(leaf[k].grad.cpu().numpy(), rgrads[k]) < 1e-4, k


def test_compute_density_and_empty():
    from oracle import field_oracle as fo
    from sugar_b200 import field
    case = fo.make_case(P=800, N=1500, K=16, seed=4, density_factor=1 / 16)
    t = {k: torch.from_numpy(v).cuda() for k, v in case.items() if isinstance(v, np.ndarray)}
    d, nb = field.compute_density(t["x"], t["nbr_idx"], t["points"], t["scaling"], t["quaternions"], t["strengths"],
                                  density_factor=1 / 16, return_closest_gaussian_opacities=True)
    ref = fo.field_values(**case)
    assert h.rel_err(d.cpu().numpy(), ref["density"]) < 2e-5
    assert h.rel_err(nb.cpu().numpy(), ref["closest_gaussian_opacities"]) < 2e-5
    e = field.field_values(t["x"][:0], t["nbr_idx"][:0], t["points"], t["scaling"], t["quaternions"], t["strengths"])
    assert e["density"].numel() == 0 and e["sdf"].numel() == 0


def _normal_ours(case, opac, dev="cuda"):
    from sugar_b200 import field
    t = lambda k: torch.from_numpy(case[k]).to(dev)
    q = t("quaternions").requires_grad_(True)
    loss = field.better_normal_loss(t("x"), t("gaussian_idx"), t("nbr_idx"), t("points"), t("scaling"), q,
                                    torch.from_numpy(opac).to(dev))
    loss.mean().backward()
    return loss.detach().cpu().numpy(), q.grad.cpu().numpy()


@pytest.mark.parametrize("name", ["c1_1k_2k", "k8"])
def test_normal_loss_matches_reference_golden(name):
    """fused better-normal loss vs the trainer's own source lines (tests/golden/make_normal_golden.py)."""
    from make_field_golden import CASES
    from oracle import field_oracle as fo
    gold = np.load(os.path.join(HERE, "golden", f"normal_{name}.npz"))
    case = fo.make_case(density_threshold=1.0, **CASES[name])
    loss, gq = _normal_ours(case, gold["nbr_opacity"])
    assert h.rel_err(loss, gold["loss"]) < 2e-5
    assert h.rel_err(gq, gold["grad_quaternions"]) < 1e-4


@pytest.mark.parametrize("P,N,K", [(5000, 20000, 16), (3000, 7001, 5), (2000, 4000, 32)])
def test_normal_loss_matches_oracle(P, N, K):
    from oracle import field_oracle as fo
    case = fo.make_case(P=P, N=N, K=K, seed=P % 89, density_factor=1.0 / K)
    opac = fo.field_values(**case)["closest_gaussian_opacities"]
    loss, gq = _normal_ours(case, opac)
    t = lambda k: torch.from_numpy(case[k])

    def oracle(dt):
        c = lambda k: t(k).to(dt)
        q = c("quaternions").clone().requires_grad_(True)
        ref = fo.better_normal_loss_torch(c("x"), t("gaussian_idx"), t("nbr_idx"), c("points"), c("scaling"), q,
                                          torch.from_numpy(opac).to(dt))
        ref.mean().backward()
        return ref.detach().numpy(), q.grad.numpy()
    l32, g32 = oracle(torch.float32)
    l64, g64 = oracle(torch.float64)
    # <x - mu, n> cancels for samples close to their Gaussian's plane: the fp32 op chain of the
    # reference itself is only this close to the exact value, so allow 3x its own rounding noise
    assert h.rel_err(loss, l64) < max(2e-5, 3 * h.rel_err(l32, l64))
    assert h.rel_err(gq, g64) < max(1e-4, 3 * h.rel_err(g32, g64))


@pytest.mark.parametrize("name", ["c1_1k_2k", "k8"])
def test_sdf_grad_and_unsupported_modes(name):
    """fields['sdf_grad'] (sugar_model.py:1307-1314) from the fused backward kernel vs the reference's value;
    the beta modes no reference caller uses raise instead of silently returning 'average'."""
    from make_field_golden import CASES
    from oracle import field_oracle as fo
    from sugar_b200 import field
    gold = np.load(os.path.join(HERE, "golden", f"field_{name}.npz"))
    case = fo.make_case(density_threshold=1.0, **CASES[name])
    t = lambda k: torch.from_numpy(case[k]).cuda()
    args = (t("x"), t("nbr_idx"), t("points"), t("scaling"), t("quaternions"), t("strengths"))
    out = field.field_values(*args, density_factor=case["density_factor"], density_threshold=1.0, return_sdf_grad=True)
    assert not out["sdf_grad"].requires_grad
    assert h.rel_err(out["sdf_grad"].cpu().numpy(), gold["sdf_grad"]) < 1e-4
    assert h.rel_err(out["sdf"].cpu().numpy(), gold["sdf"]) < 2e-5
    for mode in ("learnable", "weighted_average"):
        with pytest.raises(NotImplementedError):
            field.field_values(*args, beta_mode=mode)
