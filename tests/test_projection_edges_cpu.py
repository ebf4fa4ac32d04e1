"""The projection's edges on the CPU: the edge scenes (tests/edge_scenes.py) keep rows in every class, the oracle
matches the reference build there, and the float64 chain (tests/project64.py) matches the oracle row by row and
sees the bugs it is meant to see.

* Scene classes: every class of every scene has at least MIN_ROWS rows that are visible (radius > 0) and contribute
  (a nonzero dL/dcolour under a random image gradient), so an edit cannot quietly hollow a scene out; guard_edge's
  txtz lands exactly where its class says in fp32; near_plane's classes are what the oracle's fp32 values make them.
* Oracle against the reference build's whole state (tests/golden/projection_<scene>.npz, make_projection_golden.py),
  under test_oracle_golden.py's rules: the guard band's clamp, the near-plane cull and the saturated radius.
* project64 against the oracle's per-Gaussian chain, row by row, on every scene, fed with the oracle's accumulators.
* Mutations: project64 with the gates set to 1 and t unclamped, with scale_modifier multiplied into dL/dscale, and
  with the denom2inv == 0 branch ignored must each miss the oracle by more than 10x the bar on at least MIN_ROWS
  rows of its scenes.
"""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import edge_scenes as es  # noqa: E402
import helpers as h  # noqa: E402
import project64 as p64  # noqa: E402
from make_projection_golden import WHOLE_STATE  # noqa: E402

MIN_ROWS = 3
_CACHE = {}


def run(name):
    """(scene, classes, oracle forward, oracle backward) of an edge scene, cached per module."""
    if name not in _CACHE:
        c = es.CASES[name]
        sc, cls = c["build"]()
        fw, bw = h.run_oracle(sc, np.asarray(c["bg"], np.float32), es.upstream(name), **es.opts(name))
        _CACHE[name] = sc, cls, fw, bw
    return _CACHE[name]


def _oracle_chain(bw):
    return dict(means3D=bw["dL_dmeans3D"], cov3D=bw["dL_dcov3D"], scales=bw["dL_dscales"],
                rotations=bw["dL_drotations"])


def _groups(name):
    return ["cov3D", "scales", "rotations"] + ([] if es.CASES[name]["use_sh"] else ["means3D"])


def chain_ratios(name, **mutation):
    """Per group: the per-row |oracle - project64| / bar ([P])."""
    sc, _, fw, bw = run(name)
    P = sc.means3D.shape[0]
    dm, dc = p64.accumulators_of(bw, P)
    ref, bar = p64.reference(sc, fw["cov3D"], fw["radii"], dm, dc, es.CASES[name]["scale_modifier"], **mutation)
    got = _oracle_chain(bw)
    return {k: h.row_errors(got[k], ref[k], bar[k])["ratio_rows"] for k in _groups(name)}


@pytest.mark.parametrize("name", list(es.CASES))
def test_scene_classes_are_visible_and_contributing(name):
    sc, cls, fw, bw = run(name)
    vis = fw["radii"] > 0
    contrib = np.abs(bw["dL_dcolors"]).max(1) > 0
    counts = {k: int((m & vis & contrib).sum()) for k, m in cls.items()}
    print(f"\n[edge scenes] {name}: visible, contributing rows per class {counts}")
    culled = {"at_plane", "behind"}
    for k, n in counts.items():
        if k in culled:
            assert not (cls[k] & vis).any(), f"{name}: class {k} has visible rows"
        else:
            assert n >= MIN_ROWS, f"{name}: class {k} has {n} visible, contributing rows"


@pytest.mark.parametrize("name", list(es.CASES))
def test_scene_has_few_ambiguous_pairs(name):
    """blend64 excludes the Gaussians in front of a pair whose fp32 alpha lies within a few ulps of 1/255; the GPU
    tests allow at most max(3, 1%) of the visible ones (test_gpu_grad_rows.MAX_EXCLUDED).  The oracle's forward
    state is the GPU's, bit for bit, so this holds the scene to that here."""
    import blend64 as b64
    c = es.CASES[name]
    sc, _, fw, _ = run(name)
    st = {k: fw[k] for k in ("means2D", "conic_opacity", "point_list", "ranges", "n_contrib", "final_T")}
    r = b64.blend_backward64(st, c["bg"], es.upstream(name), fw["rgb"] if c["use_sh"] else sc.colors_precomp)
    nvis, nex = int(r["touched"].sum()), int(r["excluded"].sum())
    assert nex <= max(3, 0.01 * nvis), f"{name}: {nex} of {nvis} Gaussians excluded ({r['n_ambiguous']} pairs)"


def test_guard_edge_lands_on_the_edge_in_fp32():
    """x / z with z = 2 is exact: txtz == limx at the edge rows, one and two ulps past (inside) it elsewhere; the
    gate is 1 at and inside the edge, 0 past it, for the axis each row probes."""
    sc, cls, _, _ = run("guard_edge")
    v = es.fp32_view(sc)
    gx, gy = es.gates(sc)
    for i, (axis, sign, k, _other) in enumerate(es.guard_edge_rows()):
        t, lim, g = (v["txtz"], v["limx"], gx) if axis == "x" else (v["tytz"], v["limy"], gy)
        e = lim
        for _ in range(abs(k)):
            e = np.nextafter(e, np.float32(np.inf) if k > 0 else np.float32(0))
        assert t[i] == np.float32(sign) * e, (i, axis, sign, k, t[i], e)
        assert g[i] == (k <= 0), (i, axis, sign, k)
    assert np.all(gx | gy)                               # no row leaves both axes


def test_near_plane_classes():
    """depth == 0.2f is culled, one ulp past it is kept (identity camera: depth == z exactly); the huge rows are
    what the oracle's fp32 values make them: denom^2 overflows (denom2inv == 0), and the radius saturates."""
    sc, cls, fw, _ = run("near_plane")
    v = es.fp32_view(sc)
    assert np.array_equal(v["tz"], sc.means3D[:, 2])
    assert np.all(v["tz"][cls["at_plane"]] == es.NEAR) and np.all(fw["radii"][cls["at_plane"]] == 0)
    assert np.all(v["tz"][cls["ulp1"]] == np.nextafter(es.NEAR, np.float32(1)))
    assert np.all(fw["radii"][cls["ulp1"] | cls["ulp2"] | cls["kept"]] > 0)
    over = p64.denom_overflows(sc, fw["cov3D"], fw["radii"] > 0)
    assert np.all(over[cls["overflow"]]) and np.all(over[cls["saturated"]])
    assert not over[cls["ulp1"] | cls["ulp2"] | cls["kept"]].any()
    assert np.all(fw["radii"][cls["saturated"]] == es.INT32_MAX)
    assert np.all(fw["radii"][cls["overflow"]] < es.INT32_MAX)
    assert np.array_equal(fw["tiles_touched"][cls["saturated"]],
                          np.full(int(cls["saturated"].sum()), ((es.W + 15) // 16) * ((es.H + 15) // 16)))


def test_offscreen_centres_reach_the_e_all_path():
    """The e_all rows' ellipse half-extent sqrt(k c / det) (conic, k = -2 tau) exceeds 1e6 px; the others are
    1 to 50 image sizes outside the image."""
    sc, cls, fw, _ = run("offscreen_centres")
    co = fw["conic_opacity"].astype(np.float64)
    k = 2.0 * (np.log(255.0 * co[:, 3]) + 1e-4)
    det = co[:, 0] * co[:, 2] - co[:, 1] ** 2
    ex = np.sqrt(k * co[:, 2] / det)
    assert np.all(ex[cls["e_all"]] > 2e6), ex[cls["e_all"]]
    m = fw["means2D"][cls["far"]]
    out = np.maximum(np.maximum(-m[:, 0], m[:, 0] - es.W) / es.W, np.maximum(-m[:, 1], m[:, 1] - es.H) / es.H)
    assert out.max() > 20 and out.min() > 4, out


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


WHOLE = sorted(n for n in es.CASES if os.path.exists(os.path.join(HERE, "golden", f"projection_{n}.npz")))


def test_whole_state_goldens_exist():
    assert WHOLE == sorted(WHOLE_STATE)


@pytest.mark.parametrize("name", WHOLE)
def test_oracle_matches_reference_golden(name):
    """test_oracle_golden.py's rules: integer / index outputs and every pre-blend float bit for bit, the blend
    within glibc expf's tolerance, gradients per tensor within 2e-4."""
    sc, _, fw, bw = run(name)
    use_sh = es.CASES[name]["use_sh"]
    gold = np.load(os.path.join(HERE, "golden", f"projection_{name}.npz"))
    assert fw["num_rendered"] == int(gold["num_rendered"])
    assert np.array_equal(fw["radii"], gold["radii"])
    vis = gold["radii"] > 0
    assert np.array_equal(fw["tiles_touched"][vis], gold["tiles_touched"][vis].astype(np.uint32))
    for k in ("depths", "means2D", "conic_opacity", "cov3D"):
        assert np.array_equal(_bits(fw[k][vis]), _bits(gold[k][vis])), k
    if use_sh:
        assert np.array_equal(fw["clamped"][vis].astype(bool), gold["clamped"][vis].astype(bool))
        assert np.array_equal(_bits(fw["rgb"][vis]), _bits(gold["rgb"][vis]))
    assert np.array_equal(fw["keys"], gold["keys"].view(np.uint64))
    assert np.array_equal(fw["point_list"], gold["point_list"].view(np.uint32))
    assert np.array_equal(fw["ranges"], gold["ranges"].view(np.uint32))
    assert int((fw["n_contrib"] != gold["n_contrib"].view(np.uint32)).sum()) <= 2
    d = np.abs(fw["color"] - gold["color"])
    assert np.quantile(d, 0.999) < 2e-6 and d.max() < 5e-3
    assert np.abs(fw["final_T"] - gold["final_T"]).max() < 5e-3
    names = dict(means3D="dL_dmeans3D", means2D="dL_dmeans2D", opacities="dL_dopacity", shs="dL_dsh",
                 colors_precomp="dL_dcolors", scales="dL_dscales", rotations="dL_drotations")
    for k, v in names.items():
        if "grad_" + k in gold.files:
            g = gold["grad_" + k]
            err = h.rel_err(bw[v].reshape(g.shape), g)
            assert err <= 2e-4, f"{k}: rel err {err:.2e}"


@pytest.mark.parametrize("name", list(es.CASES))
def test_project64_matches_oracle_chain(name):
    r = chain_ratios(name)
    rep = {k: float(v.max()) for k, v in r.items()}
    print(f"\n[project64] {name}: largest |oracle - ref64| / bar {rep}")
    bad = {k: (int(np.argmax(v)), float(v.max())) for k, v in r.items() if v.max() > 1.0}
    assert not bad, f"{name}: rows over the bar (row, ratio): {bad}"


MUTATIONS = {
    "ungated_unclamped": (dict(gate_clamp=False), ("guard_band_posed_colors", "guard_band_identity_colors",
                                                   "guard_band_posed_sh3", "guard_edge")),
    "mod_in_dscale": (dict(mod_in_dscale=True), ("scale_mod_0.5_posed_sh3", "scale_mod_1.7_posed_sh3",
                                                 "scale_mod_0.5_guard_band", "scale_mod_1.7_guard_band")),
    "overflow_ignored": (dict(honour_overflow=False), ("near_plane",)),
}


@pytest.mark.parametrize("mutation", list(MUTATIONS))
def test_mutations_are_seen(mutation):
    """Each wrong variant of the chain misses the oracle by > 10x the bar on >= MIN_ROWS rows of each of its
    scenes (on guard_edge: on its past-edge rows)."""
    kw, names = MUTATIONS[mutation]
    for name in names:
        r = chain_ratios(name, **kw)
        worst = np.max(np.stack(list(r.values())), axis=0)
        if name == "guard_edge":
            worst = np.where(run(name)[1]["past_edge"], worst, 0.0)
        n = int((worst > 10.0).sum())
        print(f"\n[mutation] {mutation} on {name}: {n} rows over 10x the bar")
        assert n >= MIN_ROWS, f"{mutation} on {name}: only {n} rows miss the oracle by > 10x the bar"
