"""GPU: the forward values of the field (field_values, compute_density) and of the density-estimation loss against
float64, per sample and per entry, on the surface-shaped clouds of tests/field_cases.py, each edge group on its own.

The allowance is field_cases' value rule: a floor, 3x what the float32 oracle is off in two neighbour orders, twice
what two of our runs differ by, and twice the first-order bound of the per-term rounding (field_cases.term_error),
which dominates on flat Gaussians.  Gradients are not held to a per-row rule here (see field_cases.term_error)."""
import functools

import numpy as np
import pytest
import torch

import field_cases as fc
import helpers as h

pytestmark = pytest.mark.gpu


@functools.lru_cache(maxsize=None)
def _case(name):
    return fc.surface(name)


def _ours_field(case, w, outputs=fc.FIELD_OUTPUTS):
    from sugar_b200 import field
    leaf = {k: torch.from_numpy(case[k]).cuda().requires_grad_(True) for k in fc.LEAVES}
    out = field.field_values(leaf["x"], torch.from_numpy(case["nbr_idx"]).cuda(), leaf["points"], leaf["scaling"],
                             leaf["quaternions"], leaf["strengths"], density_factor=case["density_factor"],
                             return_sdf=True, return_closest_gaussian_opacities=True, return_beta=True,
                             return_sdf_grad=True)
    sum((out[k] * torch.from_numpy(w[k]).float().cuda()).sum() for k in w).backward()
    vals = {k: out[k].detach().double().cpu().numpy() for k in outputs + ("sdf_grad",)}
    return vals, {k: v.grad.double().cpu().numpy() for k, v in leaf.items()}


def test_field_gradients_finite_at_rho_ge_1_when_the_loss_skips_the_sdf():
    """At density factor 1, rho >= 1 on the dense_center group.  A loss on density, beta and the opacities alone has
    finite gradients, as the reference's are: the unused sdf's gradient must not reach the kernel as zeros, since
    its d/d rho is infinite there.  The sdf's values are 0 at rho >= 1 (beta (sqrt(-2 ln 1) - 0))."""
    case = _case("k16_df1")
    rows = case["groups"]["dense_center"][0]
    ref = fc.probes(fc.field_oracle, case, fc.field_weights(case))
    assert (ref[0][0]["density"][rows] >= 1.0).all()
    vals, grads = _ours_field(case, fc.field_weights(case))
    for k, g in grads.items():
        assert np.isfinite(g).all(), k
        assert np.isfinite(ref[0][1][k]).all(), k
    # the group's Gaussians are round (scales 0.03-0.05) and the samples near their centre, so the gradients are well
    # conditioned: every row within 1e-4 of itself plus 4x the float32 chain's own distance and 1e-6 of the group's max
    srows, grows = case["groups"]["dense_center"]
    for k, g in grads.items():
        r = grows if k != "x" else srows
        g64 = ref[0][1][k].reshape(len(g), -1)[r]
        p = np.maximum(*(np.abs(ref[i][1][k].reshape(len(g), -1)[r] - g64) for i in (1, 2)))
        bound = 1e-4 * np.abs(g64).max(1, keepdims=True) + 4 * p + 1e-6 * np.abs(g64).max()
        res = h.row_errors(g.reshape(len(g), -1)[r], g64, bound)
        assert res["n_over"] == 0 and np.abs(g64).max() > 0, (k, res["ratio"])
    assert (vals["sdf"][rows] == 0).all() and (np.abs(vals["sdf"][rows] - ref[0][0]["sdf"][rows]) < 1e-5).all()


@pytest.mark.parametrize("name", sorted(fc.SURFACE))
def test_field_values_per_sample(name):
    """density, beta, sdf and the neighbour opacities of field_values, K = 16, 8, 5, 33 at both density factors."""
    case = _case(name)
    w = fc.field_weights(case)
    ref = fc.probes(fc.field_oracle, case, w)
    got, got2 = _ours_field(case, w), _ours_field(case, w)
    rep = fc.check("field", case, (got[0], {}), ref, (got2[0], {}), value_keys=fc.FIELD_OUTPUTS,
                   model=fc.term_error(case))
    print(f"field {name}: worst ratio per value {fc.worst(rep)}")
    assert not fc.failures(rep), fc.failures(rep)


@pytest.mark.parametrize("name", sorted(fc.SURFACE))
def test_density_estimation_values_per_sample(name):
    """density_estimation_loss's per-sample loss and its neighbour opacities."""
    from sugar_b200 import field
    case = _case(name)
    N, K = case["nbr_idx"].shape
    w = fc.weights(N, K)["densest"]
    ref = fc.probes(fc.densest_oracle, case, w)
    t = lambda k: torch.from_numpy(case[k]).cuda()

    def ours():
        loss, nbr = field.density_estimation_loss(t("x"), t("gaussian_idx"), t("nbr_idx"), t("points"), t("scaling"),
                                                  t("quaternions"), t("strengths"),
                                                  density_factor=case["density_factor"],
                                                  return_closest_gaussian_opacities=True)
        return {"densest": loss.double().cpu().numpy(), "closest_gaussian_opacities": nbr.double().cpu().numpy()}, {}
    rep = fc.check("densest", case, ours(), ref, ours(), model=fc.term_error(case))
    print(f"densest {name}: worst ratio per value {fc.worst(rep)}")
    assert not fc.failures(rep), fc.failures(rep)


def test_compute_density_per_sample_with_shared_index_rows():
    """compute_density(samples_per_idx_row=4): row n // 4 of the index table serves sample n; against the oracle on
    the table with every row repeated four times.  N is not a multiple of 4."""
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
    w = {"density": np.ones(N)}
    ref = fc.probes(fc.field_oracle, case, w)
    t = lambda k: torch.from_numpy(case[k]).cuda()

    def ours():
        d, nb = field.compute_density(t("x"), torch.from_numpy(rows).cuda(), t("points"), t("scaling"),
                                      t("quaternions"), t("strengths"), density_factor=case["density_factor"],
                                      return_closest_gaussian_opacities=True, samples_per_idx_row=4)
        return {"density": d.double().cpu().numpy(), "closest_gaussian_opacities": nb.double().cpu().numpy()}, {}
    rep = fc.check("field", case, ours(), ref, ours(), model=fc.term_error(case))
    assert not fc.failures(rep), fc.failures(rep)
