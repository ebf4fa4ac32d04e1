"""CPU: the surface-shaped cases and the per-row rule of tests/field_cases.py, without a GPU.

No false failures: a third float32 evaluation of the oracle, with each sample's neighbour columns in a random order,
must pass the rule on every case, group by group.  The report printed per case gives the worst error over allowance
per tensor, the rows that a per-tensor rel_err < 1e-4 bar cannot see (below 1e-4 of their tensor's largest entry) and
the normal-loss samples excluded."""
import numpy as np
import pytest
import torch

import field_cases as fc


@pytest.fixture(autouse=True)
def _one_thread():
    """index_put's accumulation order, and so the float32 oracle's gradients, repeat exactly on one thread."""
    n = torch.get_num_threads()
    torch.set_num_threads(1)
    yield
    torch.set_num_threads(n)


def _hidden(g):
    g = np.abs(g.reshape(len(g), -1)).max(1)
    return int(((g > 0) & (g < 1e-4 * g.max())).sum())


@pytest.mark.parametrize("name", sorted(fc.SURFACE))
def test_permuted_float32_oracle_passes_the_rule(name):
    case = fc.surface(name)
    N, K = case["nbr_idx"].shape
    w = fc.weights(N, K)
    fw = fc.field_weights(case)
    ref = fc.probes(fc.field_oracle, case, fw)
    rep = fc.check("field", case, fc.field_oracle(case, fw, torch.float32, 777), ref)
    opac = ref[1][0]["closest_gaussian_opacities"].astype(np.float32)
    exc = fc.normal_exclusions(case)
    nref = fc.probes(fc.normal_oracle, case, opac, w["normal"])
    nrep = fc.check("normal", case, fc.normal_oracle(case, opac, w["normal"], torch.float32, 777), nref, excluded=exc)
    dref = fc.probes(fc.densest_oracle, case, w["densest"])
    drep = fc.check("densest", case, fc.densest_oracle(case, w["densest"], torch.float32, 777), dref)
    hidden = {k: _hidden(v) for k, v in ref[0][1].items()}
    print(f"{name}: hidden field gradient rows {hidden}, normal dL/dq {_hidden(nref[0][1]['quaternions'])}; "
          f"excluded {int(exc.sum())} of {N}; worst field {fc.worst(rep)} normal {fc.worst(nrep)} "
          f"densest {fc.worst(drep)}")
    assert exc.sum() <= fc.EXCLUDED_MAX * N
    for kind, r in (("field", rep), ("normal", nrep), ("densest", drep)):
        assert not fc.failures(r), (kind, fc.failures(r))


def test_edge_groups_sit_on_their_boundaries():
    """Each named group exercises the branch it is named for."""
    case = fc.surface("thin1e-3")
    g = case["groups"]
    s, x = case["scaling"], case["x"]
    assert (s[g["inv_s_clamp"][1], 2] == np.array([fc.DOWN(1e-8), np.float32(1e-8), fc.UP(1e-8)])).all()
    assert sorted(s[g["min_scaling_clamp"][1]].min(1)) == sorted([fc.DOWN(1e-6), np.float32(1e-6), fc.UP(1e-6)])
    t = lambda k: torch.from_numpy(case[k]).double()
    n = fc.fo.smallest_axis(t("scaling"), t("quaternions")).numpy()
    rows = g["orthogonal_normals"][0]
    dots = np.einsum("nkc,nc->nk", n[case["nbr_idx"][rows]], n[case["gaussian_idx"][rows]])
    assert (dots == 0).any(1).all()
    own = case["gaussian_idx"][g["on_plane"][0]]
    assert (np.einsum("nc,nc->n", x[g["on_plane"][0]] - case["points"][own], n[own]) == 0).all()
    vals = fc.field_oracle(case, {"density": np.zeros(len(x))}, torch.float64)[0]
    assert (vals["density"][g["far_samples"][0]] < 1e-16).sum() >= 2
    assert (vals["density"][g["far_samples"][0]] > 1e-16).any()
    sg = np.abs(vals["sdf_grad"][g["sdf_grad_clip"][0]])
    assert (sg == 10).any() and ((sg > 0.1) & (sg < 10)).any()


@pytest.mark.parametrize("name", sorted(fc.SURFACE))
def test_term_error_bounds_the_float32_oracle_in_every_order(name):
    """field_cases.term_error must bound the float32 chain's own per-term rounding: the float32 oracle in four
    neighbour orders stays within floor + E of float64 for every value (the sdf where rho < 1: at rho >= 1 the
    straight-through clamp rounds to exactly 1 in float32, which p holds)."""
    case = fc.surface(name)
    N, K = case["nbr_idx"].shape
    E = fc.term_error(case)
    fw, wd = fc.field_weights(case), fc.weights(N, K)["densest"]
    v64, d64 = fc.field_oracle(case, fw, torch.float64)[0], fc.densest_oracle(case, wd, torch.float64)[0]
    v64["densest"] = d64["densest"]
    worst = {}
    for order in (None, "reversed", 777, 3):
        v32 = fc.field_oracle(case, fw, torch.float32, order)[0]
        v32["densest"] = fc.densest_oracle(case, wd, torch.float32, order)[0]["densest"]
        for k in ("closest_gaussian_opacities", "density", "beta", "sdf", "densest"):
            scale = fc.value_scale(k, case, dict(v64, closest_gaussian_opacities=v64["closest_gaussian_opacities"]))
            bound = fc.VALUE_FLOOR[k] * (np.abs(v64[k]) + scale) + E[k]
            err = np.abs(v32[k] - v64[k])
            if k == "sdf":
                err = np.where(v64["density"] < 1.0, err, 0.0)
            worst[k] = max(worst.get(k, 0.0), float(np.max(np.where(err == 0, 0.0, err / np.maximum(bound, 1e-300)))))
    print(f"{name}: float32 oracle error over floor + E, worst of four orders {worst}")
    assert max(worst.values()) <= 1.0, worst


# Share of planted defects the value rule catches, measured with the float32 oracle in a random neighbour order as
# "ours" (floors a little below the smallest share measured over thin1e-3, k5, k16_df1).  Every defect is
# planted only where rel_err < 1e-4 passes it.
#   zeroed: a density row between 1e-5 and 1e-4 of the largest set to 0                      measured 1.0 everywhere
#   rel1e-2: a 1e-2 relative error in such rows                                               measured 0.08-0.19
#   dropped: the last neighbour slot left out of the sum (K = 5: one partial lane group of 8) where the term lies
#            between 1e-5 of the sample's density and 1e-4 of the largest density              measured 0.12-0.18
# A 1e-3 relative error in those rows is caught in only 0-0.2 % of them, and that is the rounding, not the rule: these
# are samples far out on flat Gaussians (density 1e-5 to 1e-4 of the largest), where term_error shows float32 itself
# is only good to about 1e-3 (fewer than 3 such rows per case have an allowance under 1e-3 of their value).
CAUGHT_MIN = dict(zeroed=0.99, rel1e_2=0.05, dropped=0.1)


@pytest.mark.parametrize("name", ["thin1e-3", "k5", "k16_df1"])
def test_value_rule_catches_planted_defects(name):
    import helpers as h
    case = fc.surface(name)
    w = fc.field_weights(case)
    ref = fc.probes(fc.field_oracle, case, w)
    E = fc.term_error(case)
    ours = fc.field_oracle(case, w, torch.float32, 777)[0]
    v64 = ref[0][0]
    b = fc.value_bound("density", v64["density"], ref[1][0]["density"], ref[2][0]["density"],
                       fc.value_scale("density", case, v64), model=E["density"])[0]
    d, m = ours["density"], np.abs(v64["density"]).max()
    low = (np.abs(v64["density"]) > 1e-5 * m) & (np.abs(v64["density"]) < 1e-4 * m)
    band = np.where(low)[0]
    o = ours["closest_gaussian_opacities"][:, -1]
    drop = np.where((o < 0.9e-4 * m) & (o > 1e-5 * np.abs(v64["density"])))[0]
    shares = {}
    for kind, rows, f in (("zeroed", band, lambda v, r: 0.0 * v[r]), ("rel1e_2", band, lambda v, r: v[r] * (1 + 1e-2)),
                          ("dropped", drop, lambda v, r: v[r] - o[r])):
        planted = d.copy()
        planted[rows] = f(d, rows)
        assert h.rel_err(planted, v64["density"]) < 1e-4, kind
        shares[kind] = (float((np.abs(planted - v64["density"])[rows] > b[rows]).mean()), len(rows))
    print(f"{name}: caught share (rows) {shares}")
    for kind, (share, n) in shares.items():
        assert n >= 20 and share >= CAUGHT_MIN[kind], (kind, share, n)


def test_more_edge_groups_sit_on_their_boundaries():
    case = fc.surface("k16_df1")
    g = case["groups"]
    s, x, gi, nb = case["scaling"], case["x"], case["gaussian_idx"], case["nbr_idx"]
    t = lambda k: torch.from_numpy(case[k]).double()
    # Mahalanobis^2 of the flat Gaussian on both sides of 1e8
    rows = g["mahalanobis_clamp"][0]
    own = gi[rows]
    R = fc._rot(case["quaternions"][own].astype(np.float64))
    wv = np.einsum("nij,ni->nj", R, x[rows].astype(np.float64) - case["points"][own]) / s[own]
    d2 = (wv ** 2).sum(1)
    assert (d2 > 1e8).any() and (d2 < 1e8).any()
    # every neighbour of the zero_weights samples has e = 0 exactly: wsum = 0
    n = fc.fo.smallest_axis(t("scaling"), t("quaternions")).numpy()
    rows = g["zero_weights"][0]
    e = np.einsum("nkc,nkc->nk", x[rows][:, None].astype(np.float64) - case["points"][nb[rows]], n[nb[rows]])
    assert (e == 0).all()
    # tied smallest scales are exact ties, in every pattern
    ss = s[g["tied_scales"][1]]
    assert ((ss == ss.min(1, keepdims=True)).sum(1) >= 2).all() and ((ss == ss.min(1, keepdims=True)).sum(1) == 3).any()
    # the min_scaling_clamp samples' own smallest scale is the bound or one ulp either side
    rows = g["min_scaling_clamp"][0]
    assert set(s[gi[rows]].min(1)) == {fc.DOWN(1e-6), np.float32(1e-6), fc.UP(1e-6)}
    # rho >= 1 at density factor 1
    v = fc.field_oracle(case, {"density": np.zeros(len(x))}, torch.float64)[0]
    assert (v["density"][g["dense_center"][0]] >= 1.0).all()
