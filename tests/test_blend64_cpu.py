"""The float64 blend reference (tests/blend64.py) against the CPU oracle, Gaussian by Gaussian.

The oracle forms every pair's terms in fp32 in the reference's order and sums them in double, so its accumulators
must lie within E_pair (SAFETY x the pair part of the bound) of the float64 reference for every Gaussian and
component.  The bound must also be tight enough to matter: for the Gaussians whose rows the per-tensor bar of
test_gpu_parity (5e-4 of the tensor's largest entry) hides, E must be below 1e-4 of the row, so that a 1e-4 relative
error in one of them is caught; a perturbed or zeroed row of a mid-weight hidden Gaussian is caught while rel_err
passes it.  The GPU file test_gpu_grad_rows.py holds the kernels to the full bound on these scenes and more."""
import functools

import numpy as np
import pytest

import blend64 as b64
import helpers as h

# the test_gpu_parity scenes that run on the CPU in a few seconds each (the larger ones run in the GPU file)
CPU_CASES = ["sh3_posed", "sh2_identity", "sh0_posed", "colors_posed", "covpre_posed", "mesh_bound", "big_splats",
             "opacity_edge", "mid_tiles", "coplanar"]
ORACLE_GRAD_RTOL = 5e-4   # test_gpu_parity.test_matches_cpu_oracle's per-tensor bar
# Fraction of the hidden Gaussians (rows under ORACLE_GRAD_RTOL of their tensor's largest, in the geometric groups)
# whose bound is below 1e-4 of the row, measured per scene (floors 0.05 below).  The rest are rows whose terms cancel
# by more than ~1000x over their footprint, or pairs with hundreds of splats behind them (mid_tiles, coplanar), whose
# T recovered by division carries more rounding than a 1e-4 bar leaves room for.
TIGHT_MIN = dict(sh3_posed=0.72, sh2_identity=0.47, sh0_posed=0.41, colors_posed=0.67, covpre_posed=0.76,
                 mesh_bound=0.61, big_splats=0.82, mid_tiles=0.24, coplanar=0.63, opacity_edge=0.0)
# Share of the hidden rows whose geometric gradients, changed by 1e-4 relative, the row check catches (any component
# over its bound), measured per scene (floors 0.02 below): 0.89-1.0, except mid_tiles (0.43).
CAUGHT_MIN = dict(sh3_posed=0.96, sh2_identity=0.92, sh0_posed=0.87, colors_posed=0.96, covpre_posed=0.96,
                  mesh_bound=0.94, big_splats=0.98, mid_tiles=0.40, coplanar=0.87)
GEOMETRIC = ("means2D", "conic", "opacity")

@functools.lru_cache(maxsize=None)
def _run(name):
    import test_gpu_parity as tp
    from sugar_b200 import scenes
    case = next(c for c in tp.ORACLE_CASES if c[0] == name)
    _, P, W, H, camera, use_sh, deg, covpre, bg = case
    sc = tp._scene(name, P, W, H, camera)
    dL = scenes.upstream_grad(W, H)
    cov3D = tp._cov_from_oracle(sc) if covpre else None
    fw, bw = h.run_oracle(sc, np.asarray(bg, np.float32), dL, use_sh=use_sh, sh_degree=deg, use_cov_precomp=covpre,
                          cov3D=cov3D)
    r = b64.blend_backward64(fw, bg, dL, fw["colors"])
    return fw, b64.oracle_accumulators(bw, P), r


def _hidden(orc, r, group):
    cols = list(b64.GROUPS[group])
    rowmax = np.abs(orc[:, cols]).max(1)
    return r["touched"] & ~r["excluded"] & (rowmax > 0) & (rowmax < ORACLE_GRAD_RTOL * np.abs(orc[:, cols]).max())


@pytest.mark.parametrize("name", CPU_CASES)
def test_oracle_within_bound(name):
    fw, orc, r = _run(name)
    ok = r["touched"] & ~r["excluded"]
    nvis = int(ok.sum())
    assert nvis > 0
    assert int(r["excluded"].sum()) <= max(3, 0.01 * nvis), f"{int(r['excluded'].sum())} excluded of {nvis}"
    assert not orc[~r["touched"] & ~r["excluded"]].any(), "a Gaussian without a contributing pair has gradients"
    err = h.row_errors(orc, r["ref"], b64.SAFETY * r["e_pair"], rows=ok)
    med = {b64.NAMES[k]: float(np.median(r["bound"][ok, k] / np.maximum(np.abs(r["ref"][ok, k]), 1e-30)))
           for k in range(9)}
    print(f"\n[blend64] {name}: max |oracle - ref64| / E_pair {err['ratio']:.3f}, excluded {int(r['excluded'].sum())} "
          f"({r['n_ambiguous']} ambiguous pairs), median E / |ref| " + " ".join(f"{k} {v:.1e}" for k, v in med.items()))
    g, k = err["worst_row"], err["worst_col"]
    assert err["ratio"] <= 1.0, (f"Gaussian {g} {b64.NAMES[k]}: oracle {orc[g, k]:.9g} ref64 {r['ref'][g, k]:.9g} "
                                 f"ratio {err['ratio']:.3g}; {err['n_over']} rows over")


@pytest.mark.parametrize("name", CPU_CASES)
def test_bound_is_tight(name):
    _, orc, r = _run(name)
    rn = b64.row_norms(r["ref"])
    n_hidden = n_tight = 0
    for grp in GEOMETRIC:
        cols = list(b64.GROUPS[grp])
        hid = _hidden(orc, r, grp)
        n_hidden += int(hid.sum())
        n_tight += int((hid & (r["bound"][:, cols].max(1) < 1e-4 * rn[:, cols[0]])).sum())
    frac = n_tight / max(n_hidden, 1)
    print(f"\n[blend64] {name}: E < 1e-4 |row| for {n_tight} of {n_hidden} hidden rows ({frac:.3f})")
    assert n_hidden == 0 or frac >= TIGHT_MIN[name], frac


def _mid_weight_hidden(orc, r):
    """The Gaussian of median row norm among those hidden in every group (chosen without looking at the bound)."""
    rn = b64.row_norms(r["ref"])
    hid = np.logical_and.reduce([_hidden(orc, r, grp) for grp in ("means2D", "conic", "opacity", "colors")])
    cand = np.flatnonzero(hid)
    assert cand.size, "no Gaussian hidden in every group"
    return int(cand[np.argsort(rn[cand, 0])[cand.size // 2]])


@pytest.mark.parametrize("name", [n for n in CPU_CASES if n != "opacity_edge"])
def test_perturbed_and_zeroed_rows_are_caught(name):
    """A mid-weight hidden Gaussian's row, zeroed: rel_err passes it, the row check must not.  A 1e-4 relative change
    of the geometric gradients of every hidden row in turn (each passes rel_err): the share the row check catches is
    reported, and must reach the scene's floor."""
    _, orc, r = _run(name)
    ok = r["touched"] & ~r["excluded"]
    bound = r["bound"][:, :9]
    g = _mid_weight_hidden(orc, r)
    x = orc.copy()
    x[g] = 0.0
    for grp in ("means2D", "conic", "opacity", "colors"):
        cols = list(b64.GROUPS[grp])
        assert h.rel_err(x[:, cols], orc[:, cols]) <= ORACLE_GRAD_RTOL, grp
    err = h.row_errors(x, r["ref"], bound, rows=ok)
    assert err["n_over"] == 1 and err["worst_row"] == g, (g, err["worst_row"], err["ratio"])
    # the geometric components (dmean2D, dconic, dopacity) of every hidden row changed by 1e-4 relative, one row at
    # a time (rows are independent in row_errors); the colours are left alone, their bound is tight anyway
    hid = np.logical_or.reduce([_hidden(orc, r, grp) for grp in GEOMETRIC])
    geo = np.array([1 + 1e-4] * 6 + [1.0] * 3)
    pert = h.row_errors(orc * geo, r["ref"], bound, rows=hid)
    caught = float((pert["ratio_rows"][hid] > 1.0).mean())
    perturbed_g = h.row_errors(orc[g:g + 1] * geo, r["ref"][g:g + 1], bound[g:g + 1])["ratio"] > 1.0
    print(f"\n[blend64] {name}: 1e-4 change of a hidden row caught for {caught:.3f} of {int(hid.sum())}; "
          f"Gaussian {g} (median hidden row): {'caught' if perturbed_g else 'not caught'}")
    assert caught >= CAUGHT_MIN[name], caught


def test_row_errors_fails_on_non_finite_rows():
    """A NaN or inf in a compared row is reported as an infinite ratio, never skipped."""
    want = np.array([[0.5, 1.0], [2.0, 3.0], [1.0, 1.0]])
    bound = np.full_like(want, 1e-3)
    for bad in (np.nan, np.inf, -np.inf):
        got = want.copy()
        got[1, 0] = bad
        err = h.row_errors(got, want, bound)
        assert err["ratio"] == np.inf and err["worst_row"] == 1 and err["n_over"] == 1, (bad, err)
    got = want.copy()
    got[2, 1] = np.nan
    assert h.row_errors(got, want, bound, rows=np.array([True, True, False]))["n_over"] == 0   # row not compared
    assert h.row_errors(want, want, np.zeros_like(want))["ratio"] == 0.0
