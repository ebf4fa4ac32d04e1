"""The rasterizer at the projection's edges, Gaussian by Gaussian: the guard-band clamp and its gradient gates, the
near-plane cull, denom2inv == 0, the saturated radius, centres far off screen and scale_modifier != 1
(tests/edge_scenes.py).  Every scene runs with packed ids and with plain ids (P padded to 2^24 with culled Gaussians,
helpers.pad_culled).

* Forward: bit-exact to the CPU oracle and to the reference build's digests (tests/golden/
  refbuild_projection_<scene>.npz): radii, tiles_touched, depths, means2D, conic_opacity, rgb and clamp bits, keys,
  point_list and ranges; n_contrib, the image and final_T under test_gpu_parity's rules (bit-exact to the reference
  build).  The public gradients, through GaussianRasterizer with the scene's scale_modifier in its settings, against
  the reference build's within test_gpu_parity's GRAD_RTOL.  markVisible on near_plane against the oracle's.
* Footprint masks: no instance's mask clears a block that holds a pixel passing the alpha test, and every
  contributing pair of the walk lies in a block its mask sets; the looseness (set bits / needed bits) is reported and
  bounded as in test_gpu_configs.
* Backward: the blend accumulators against tests/blend64.py, and the per-Gaussian chain from the GPU's own
  accumulators against the oracle (test_gpu_grad_rows.check_chain) and against tests/project64.py, row by row.
  Culled rows (z = 0.2f among them) have exactly zero gradients, denom2inv == 0 rows exactly zero dL/dcov3D, scales
  and rotations, and on guard_edge the gate the GPU took is the fp32 one: its dL/dmeans3D is far (> 10x the bar)
  from the chain with that row's gate decided the other way.
* Raw-parameter mode (sugar_b200/fused.py) on a guard-band scene, as test_gpu_grad_rows.test_raw_parameter_mode.

Measured on an H100 80GB HBM3 (700 W limit), every scene and both id formats: the largest |gpu - ref64| / E of the
accumulators is 0.29, |gpu - oracle chain| / bar 0.08 and |gpu - project64| / bar 0.18 (dL/drotations of
scale_mod_1.7_posed_sh3); the masks set at most 1.15x the blocks the alpha test needs (near_plane, whose needle
splats take the masks' `all` path), 1.003x elsewhere.
"""
import numpy as np
import pytest

import blend64 as b64
import edge_scenes as es
import helpers as h
import project64 as p64
import test_gpu_grad_rows as tgr
import test_gpu_parity as tp

pytestmark = pytest.mark.gpu

IDS = dict(argnames="unpacked", argvalues=[False, True], ids=["packed_ids", "unpacked_ids"])
_ORACLE = {}


def _oracle(name):
    if name not in _ORACLE:
        c = es.CASES[name]
        sc, cls = c["build"]()
        fw, bw = h.run_oracle(sc, np.asarray(c["bg"], np.float32), es.upstream(name), **es.opts(name))
        _ORACLE[name] = sc, cls, fw, bw
    return _ORACLE[name]


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.mark.parametrize(**IDS)
@pytest.mark.parametrize("name", list(es.CASES))
def test_forward_matches_oracle_and_reference_build(name, unpacked):
    c = es.CASES[name]
    sc, _, fw, _ = _oracle(name)
    W, H = sc.width, sc.height
    o = h.run_state(sc, c["bg"], es.upstream(name), plain_ids=unpacked, **es.opts(name))
    assert int(o["num_rendered"]) == fw["num_rendered"]
    assert np.array_equal(o["radii"], fw["radii"])
    vis = fw["radii"] > 0
    assert np.array_equal(o["tiles_touched"][vis].astype(np.uint32), fw["tiles_touched"][vis])
    for k in ("depths", "means2D", "conic_opacity") + (("rgb",) if c["use_sh"] else ()):
        assert np.array_equal(_bits(o[k][vis]), _bits(fw[k][vis])), k
    if c["use_sh"]:
        assert np.array_equal(o["clamped"][vis].astype(bool), fw["clamped"][vis].astype(bool))
    assert np.array_equal(o["keys"].view(np.uint64), fw["keys"])
    assert np.array_equal(o["point_list"].view(np.uint32), fw["point_list"])
    assert np.array_equal(o["ranges"].view(np.uint32), fw["ranges"])
    flips = int((o["n_contrib"].view(np.uint32) != fw["n_contrib"]).sum())
    assert flips <= max(2, W * H // 5000), f"{flips} n_contrib mismatches"
    for img in (o["color"], o["color_bw"]):
        d = np.abs(img - fw["color"])
        assert np.quantile(d, 0.999) < 2e-6 and d.max() < 5e-3, (float(np.quantile(d, 0.999)), float(d.max()))
    assert np.abs(o["final_T"] - fw["final_T"]).max() < 5e-3

    gold = h.load_golden("projection_" + name)
    assert int(o["num_rendered"]) == int(gold["num_rendered"])
    fields = dict(radii=o["radii"], tiles_touched=o["tiles_touched"][vis], depths=o["depths"][vis],
                  means2D=o["means2D"][vis], conic_opacity=o["conic_opacity"][vis], keys=o["keys"],
                  point_list=o["point_list"], ranges=o["ranges"], n_contrib=o["n_contrib"], final_T=o["final_T"],
                  color=o["color"])
    if c["use_sh"]:
        fields.update(clamped=o["clamped"][vis].astype(bool), rgb=o["rgb"][vis])
    h.assert_digests(gold, fields)
    grads = {k[len("grad_"):]: v for k, v in o.items() if k.startswith("grad_")}
    assert {k[len("grad_"):-len("_inf")] for k in gold if k.startswith("grad_") and k.endswith("_inf")} == set(grads)
    for k, g in grads.items():
        err, noise = h.golden_rel_err(g, gold, "grad_" + k), float(gold["noise_" + k])
        assert err <= max(tp.GRAD_RTOL, 5.0 * noise), f"grad {k}: rel err vs the reference build {err:.3e}"


def test_mark_visible_at_the_near_plane():
    import torch
    from oracle import raster_oracle as ro
    from sugar_b200 import diff_gaussian_rasterization as ours
    sc, cls, _, _ = _oracle("near_plane")
    t = h.to_torch(sc)
    st = ours.GaussianRasterizationSettings(sc.height, sc.width, sc.tanfovx, sc.tanfovy, torch.zeros(3, device="cuda"),
                                            1.0, t["viewmatrix"], t["projmatrix"], 0, t["campos"], False, False)
    got = ours.GaussianRasterizer(st).markVisible(t["means3D"]).cpu().numpy()
    want = ro.mark_visible(sc.means3D, sc.viewmatrix, sc.projmatrix)
    assert np.array_equal(got, want)
    assert not want[cls["at_plane"] | cls["behind"]].any() and want[cls["ulp1"]].all()


@pytest.mark.parametrize("name", list(es.CASES))
def test_footprint_masks(name):
    """Packed ids carry each instance's mask: it must hold every block with a pixel passing the alpha test (power <= 0,
    alpha >= 1/255, over the whole 16x16 tile) and every block of a contributing pair of the walk."""
    c = es.CASES[name]
    sc, _, _, _ = _oracle(name)
    W = sc.width
    o = h.run_state(sc, c["bg"], None, **es.opts(name))
    gx = (W + 15) // 16
    tile = (o["keys"].view(np.uint64) >> np.uint64(32)).astype(np.int64)
    ids = o["point_list"].view(np.uint32).astype(np.int64)
    fp = o["footprint"].astype(np.int64)
    m2 = o["means2D"][ids].astype(np.float64)
    co = o["conic_opacity"][ids].astype(np.float64)
    ty, tx = tile // gx, tile % gx
    px = (tx[:, None, None] * 16 + np.arange(16)[None, None, :]).astype(np.float64)
    py = (ty[:, None, None] * 16 + np.arange(16)[None, :, None]).astype(np.float64)
    dx, dy = m2[:, 0, None, None] - px, m2[:, 1, None, None] - py
    power = -0.5 * (co[:, 0, None, None] * dx * dx + co[:, 2, None, None] * dy * dy) - co[:, 1, None, None] * dx * dy
    alpha = np.minimum(co[:, 3, None, None] * np.exp(np.minimum(power, 0.0)), 0.99)
    hit = (power <= 0) & (alpha >= 1.0 / 255.0)
    blocks = hit.reshape(-1, 4, 4, 2, 8).any(axis=4).any(axis=2)               # [R, band, half]
    truth = (blocks * (1 << (np.arange(4)[:, None] * 2 + np.arange(2)[None, :]))).sum((1, 2))
    missed = truth & ~fp
    bad = np.flatnonzero(missed)
    assert bad.size == 0, (f"{name}: {bad.size} masks clear a block with a pixel passing the alpha test, e.g. "
                           f"instance {bad[0]} (Gaussian {ids[bad[0]]}, tile {tile[bad[0]]}, mask {fp[bad[0]]:#x}, "
                           f"needed {truth[bad[0]]:#x}, centre {m2[bad[0]]})")
    # every contributing pair of the walk (the fp32 decisions of blend64) lies in a block its mask sets
    lo_of = np.asarray(o["ranges"]).view(np.uint32)[:, 0].astype(np.int64)
    blk_of = (b64.LY // 4) * 2 + b64.LX // 8
    n_pairs = 0
    for t in np.unique(tile):
        tpairs = b64.tile_pairs(o, t)
        if tpairs is None:
            continue
        V = tpairs["V"]                                                        # [256, n]
        n = V.shape[1]
        bits = (fp[lo_of[t]:lo_of[t] + n][None, :] >> blk_of[:, None]) & 1
        assert not (V & (bits == 0)).any(), f"{name}: a contributing pair of tile {t} lies in a block its mask clears"
        n_pairs += int(V.sum())
    pop = lambda v: int(sum(((v >> b) & 1).sum() for b in range(8)))
    print(f"\n[masks] {name}: set bits {pop(fp)}, needed {pop(truth)} (looseness {pop(fp) / max(pop(truth), 1):.3f}), "
          f"{n_pairs} contributing pairs, {int((fp == 0).sum())} dead instances of {len(fp)}")
    assert pop(fp) <= 1.25 * pop(truth) + 64, (pop(fp), pop(truth))


def _forward(sc, c, pad_to):
    """test_gpu_grad_rows._forward with the scene's scale_modifier."""
    from sugar_b200 import _C
    opts = dict(use_sh=c["use_sh"], sh_degree=c["sh_degree"])
    f = tgr._forward(sc, c["bg"], pad_to=pad_to, **opts)
    if c["scale_modifier"] != 1.0:
        args = f["args"][:6] + (c["scale_modifier"],) + f["args"][7:]
        R, _color, radii, geom, binning, img = _C.rasterize_gaussians(*args)[:6]
        st = _C.inspect_state(f["Pt"], sc.width, sc.height, R, geom, binning, img)
        f.update(args=args, R=R, radii=radii, geom=geom, binning=binning, img=img,
                 st={k: v.cpu().numpy() for k, v in st.items()})
    return f


@pytest.mark.parametrize(**IDS)
@pytest.mark.parametrize("name", list(es.CASES))
def test_backward_rows(name, unpacked):
    c = es.CASES[name]
    sc, cls, fw, _ = _oracle(name)
    P = sc.means3D.shape[0]
    label = f"{name}/{'plain' if unpacked else 'packed'}"
    dL = es.upstream(name)
    f = _forward(sc, c, h.PACKED_MAX_P if unpacked else None)
    grads, gacc = tgr._backward(f, dL)
    radii = f["radii"][:P].cpu().numpy()
    assert np.array_equal(radii, fw["radii"])
    if unpacked:
        assert not f["radii"][P:].any() and not gacc[P:].any() and not grads["colors"][P:].any()
    st = dict(f["st"])
    for k in h.PER_GAUSSIAN:
        if k in st:
            st[k] = st[k][:P]
    colors = st["rgb"] if c["use_sh"] else sc.colors_precomp
    r = b64.blend_backward64(st, c["bg"], dL, colors, clamped=st["clamped"] if c["use_sh"] else None)
    rep = tgr.check_accumulators(label, st, b64.gpu_accumulators(gacc[:P], grads["colors"][:P]), r)
    rep["chain_oracle"] = tgr.check_chain(label, fw, gacc, grads, c["use_sh"], False)

    # the chain against the float64 restatement, fed with the GPU's accumulators
    dm2d, dconic = gacc[:P, :2], gacc[:P, 2:5]
    ref, bar = p64.reference(sc, fw["cov3D"], radii, dm2d, dconic, c["scale_modifier"])
    groups = [k for k in p64.GROUPS if not (c["use_sh"] and k == "means3D")]
    ratios, bad = {}, []
    for k in groups:
        err = h.row_errors(grads[k][:P], ref[k], bar[k])
        ratios[k] = round(err["ratio"], 4)
        if err["ratio"] > 1.0:
            g = err["worst_row"]
            bad.append(f"{k}: Gaussian {g} gpu {grads[k][g]} ref64 {ref[k][g]} bar {bar[k][g, 0]:.3g} "
                       f"({err['n_over']} rows over)")
    rep["project64"] = ratios
    assert not bad, f"{label} against project64: " + "; ".join(bad)

    # explicit checks
    culled = radii == 0
    for k in ("means3D", "means2D", "cov3D", "scales", "rotations", "colors", "opacity") + (("sh",) if c["use_sh"]
                                                                                            else ()):
        assert not grads[k][:P][culled].any(), f"{label}: a culled Gaussian has a nonzero dL/d{k}"
    if name == "near_plane":
        assert culled[cls["at_plane"]].all()
        over = p64.denom_overflows(sc, fw["cov3D"], ~culled)
        assert over.sum() >= 7
        for k in ("cov3D", "scales", "rotations"):
            assert not grads[k][:P][over].any(), f"{label}: a denom2inv == 0 row has a nonzero dL/d{k}"
        assert np.abs(grads["means3D"][:P][over]).max() > 0          # the projection term remains
    if name == "guard_edge":
        rows = es.guard_edge_rows()
        fx = np.array([a == "x" for a, *_ in rows])
        probe = cls["at_edge"] | cls["past_edge"]
        flip = p64.chain64(sc, fw["cov3D"], radii, dm2d, dconic, flip_gates=(fx & probe, ~fx & probe))
        d = np.abs(grads["means3D"][:P].astype(np.float64) - flip["means3D"]).max(1) / bar["means3D"][:, 0]
        seen = probe & (d > 10.0)
        rep["gate_rows_told_apart"] = f"{int(seen.sum())} of {int(probe.sum())}"
        assert seen.sum() >= probe.sum() - 2, (f"{label}: the gate decision shows in dL/dmeans3D on only "
                                               f"{int(seen.sum())} of {int(probe.sum())} edge rows: {d[probe]}")
    print(f"\n[projection_edges] {label}: {rep}")


def test_raw_parameter_mode_in_the_guard_band():
    sc, _, _, _ = _oracle("guard_band_posed_sh3")
    tgr.run_raw_mode("raw/guard_band", sc, es.CASES["guard_band_posed_sh3"]["bg"], es.upstream("guard_band_posed_sh3"))
