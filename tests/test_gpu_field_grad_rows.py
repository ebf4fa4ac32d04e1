"""GPU: the gradients of field_values, density_estimation_loss, better_normal_loss and compute_density against
float64, row by row (per sample for dL/dx and sdf_grad, per Gaussian for the rest), on the surface-shaped clouds of
tests/field_cases.py, each edge group on its own.

The allowance is field_cases' gradient rule: 1e-4 of the row, 4x what the float32 oracle is off in two neighbour
orders plus twice what two of our runs differ by, twice the per-term rounding bound G (field_cases.grad_term_error,
which test_field_grad_rows_cpu.py shows bounds the float32 oracle in four orders and a float32 stand-in for these
kernels), and a floor of 1e-6 of the group's largest entry."""
import functools

import numpy as np
import pytest
import torch

import field_cases as fc

pytestmark = pytest.mark.gpu


@functools.lru_cache(maxsize=None)
def _case(name):
    return fc.surface(name)


@functools.lru_cache(maxsize=None)
def _field_ref(name):
    case = _case(name)
    return fc.probes(fc.field_oracle, case, fc.field_weights(case))


def _t(case, k):
    return torch.from_numpy(np.ascontiguousarray(case[k])).cuda()


def _assert_passes(kind, name, rep):
    print(f"{kind} {name}: worst ratio per tensor {fc.worst(rep)}; largest floor-dominated share "
          f"{max(v['floor_dominated'] for v in rep.values()):.3f}")
    bad = fc.failures(rep)
    assert not bad, (f"{kind} {name}: (group, tensor): (ratio, worst row, rows over, what dominates its allowance)",
                     bad)


def _ours_field(case, w):
    from sugar_b200 import field
    leaf = {k: _t(case, k).requires_grad_(True) for k in fc.LEAVES}
    out = field.field_values(leaf["x"], _t(case, "nbr_idx"), leaf["points"], leaf["scaling"], leaf["quaternions"],
                             leaf["strengths"], density_factor=case["density_factor"], return_sdf=True,
                             return_closest_gaussian_opacities=True, return_beta=True, return_sdf_grad=True)
    sum((out[k] * torch.from_numpy(w[k]).float().cuda()).sum() for k in w).backward()
    return ({"sdf_grad": out["sdf_grad"].double().cpu().numpy()},
            {k: v.grad.double().cpu().numpy() for k, v in leaf.items()})


@pytest.mark.parametrize("name", sorted(fc.SURFACE))
def test_field_gradients_per_row(name):
    """dL/dx, dL/dpoints, dL/dscaling, dL/dquaternions and dL/dstrengths of field_values per row, and sdf_grad per
    sample (its value floor, plus twice field_cases.sdf_grad_error)."""
    case = _case(name)
    w = fc.field_weights(case)
    got, got2 = _ours_field(case, w), _ours_field(case, w)
    rep = fc.check("field", case, got, _field_ref(name), got2, value_keys=("sdf_grad",),
                   model={"sdf_grad": fc.sdf_grad_error(case)}, gmodel=fc.grad_term_error(case, "field", w))
    _assert_passes("field", name, rep)


@pytest.mark.parametrize("name", sorted(fc.SURFACE))
def test_density_estimation_gradients_per_row(name):
    from sugar_b200 import field
    case = _case(name)
    N, K = case["nbr_idx"].shape
    w = fc.weights(N, K)["densest"]
    ref = fc.probes(fc.densest_oracle, case, w)

    def ours():
        leaf = {k: _t(case, k).requires_grad_(True) for k in fc.LEAVES}
        loss = field.density_estimation_loss(leaf["x"], _t(case, "gaussian_idx"), _t(case, "nbr_idx"), leaf["points"],
                                             leaf["scaling"], leaf["quaternions"], leaf["strengths"],
                                             density_factor=case["density_factor"])
        (loss * torch.from_numpy(w).float().cuda()).sum().backward()
        return {}, {k: v.grad.double().cpu().numpy() for k, v in leaf.items()}
    rep = fc.check("densest", case, ours(), ref, ours(), gmodel=fc.grad_term_error(case, "densest", w))
    _assert_passes("densest", name, rep)


@pytest.mark.parametrize("name", sorted(fc.SURFACE))
def test_better_normal_loss_and_gradients_per_row(name):
    """The per-sample loss (its value floor, 3 p and twice field_cases.normal_value_error: on flat Gaussians the
    weights' per-term rounding misses a p-only allowance by up to ~1e3 on CPU) and dL/dq per Gaussian; the oracle and
    the kernel get the same float32 neighbour opacities.  Samples whose sign is a float32 coin toss are excluded, and
    the groups whose dL/dq is zero in exact arithmetic are held on their values only."""
    from sugar_b200 import field
    case = _case(name)
    N, K = case["nbr_idx"].shape
    w = fc.weights(N, K)["normal"]
    opac = _field_ref(name)[1][0]["closest_gaussian_opacities"].astype(np.float32)
    exc = fc.normal_exclusions(case)
    assert exc.sum() <= fc.EXCLUDED_MAX * N
    ref = fc.probes(fc.normal_oracle, case, opac, w)

    def ours():
        q = _t(case, "quaternions").requires_grad_(True)
        loss = field.better_normal_loss(_t(case, "x"), _t(case, "gaussian_idx"), _t(case, "nbr_idx"),
                                        _t(case, "points"), _t(case, "scaling"), q,
                                        torch.from_numpy(opac).cuda())
        (loss * torch.from_numpy(w).float().cuda()).sum().backward()
        return {"normal": loss.detach().double().cpu().numpy()}, {"quaternions": q.grad.double().cpu().numpy()}
    rep = fc.check("normal", case, ours(), ref, ours(), excluded=exc,
                   model={"normal": fc.normal_value_error(case, opac)},
                   gmodel=fc.grad_term_error(case, "normal", w, opac))
    _assert_passes("normal", name, rep)


def test_compute_density_gradients_with_shared_index_rows():
    """compute_density(samples_per_idx_row=4) backward: the kernel reads index row n // 4 but the opacity gradient
    row n; against the oracle on the table with every row repeated four times.  N is not a multiple of 4."""
    from sugar_b200 import field
    base = fc.surface_case(P=3000, N=3000, K=16, seed=3, thin=1e-3)
    rng = np.random.default_rng(4)
    N = 4 * 3000 - 3
    s = base["scaling"][base["gaussian_idx"]].min(1, keepdims=True)
    x = np.repeat(base["x"], 4, axis=0)[:N] + (np.repeat(s, 4, axis=0)[:N] * rng.normal(size=(N, 3))).astype(np.float32)
    rows = base["nbr_idx"]
    case = dict(base, x=np.ascontiguousarray(x, np.float32), nbr_idx=np.repeat(rows, 4, axis=0)[:N],
                gaussian_idx=np.repeat(base["gaussian_idx"], 4)[:N])
    case["groups"] = {"surface": fc._all(case)}
    w = {k: v for k, v in fc.weights(N, 16, seed=5).items() if k in ("density", "closest_gaussian_opacities")}
    ref = fc.probes(fc.field_oracle, case, w)

    def ours():
        leaf = {k: _t(case, k).requires_grad_(True) for k in fc.LEAVES}
        d, nb = field.compute_density(leaf["x"], torch.from_numpy(rows).cuda(), leaf["points"], leaf["scaling"],
                                      leaf["quaternions"], leaf["strengths"], density_factor=case["density_factor"],
                                      return_closest_gaussian_opacities=True, samples_per_idx_row=4)
        ((d * torch.from_numpy(w["density"]).float().cuda()).sum() +
         (nb * torch.from_numpy(w["closest_gaussian_opacities"]).float().cuda()).sum()).backward()
        return {}, {k: v.grad.double().cpu().numpy() for k, v in leaf.items()}
    rep = fc.check("field", case, ours(), ref, ours(), gmodel=fc.grad_term_error(case, "field", w))
    _assert_passes("compute_density", "shared rows", rep)
