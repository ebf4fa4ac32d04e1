"""CPU: size-independent properties of the rasterizer restated in the oracle -- the same invariants the GPU
tests use at sizes where no element-wise reference is affordable.

 * background:   image(bg) = image(0) + final_T * bg, and final_T / n_contrib / radii do not depend on bg
                 (forward.cu:361-367);
 * permutation:  with pairwise distinct depths the image does not depend on the order of the Gaussians in memory
                 (sort key = tile | depth, rasterizer_impl.cu:70-111), bit for bit;
 * linearity:    the backward is linear in the upstream image gradient (backward.cu is a chain of products with
                 dL_dpixel), up to fp32 rounding;
 * culling:      Gaussians behind the near plane (z <= 0.2) get radius 0 and exactly zero gradients."""
import numpy as np

import helpers as h


def _scene(P=1500, W=96, H=64, seed=5):
    from sugar_b200 import scenes
    return scenes.make_scene(P, W, H, seed=seed, camera="posed")


def test_background_enters_linearly_through_final_T():
    sc = _scene()
    fw0, _ = h.run_oracle(sc, np.zeros(3, np.float32))
    bg = np.array([0.25, 0.5, 1.0], np.float32)
    fw1, _ = h.run_oracle(sc, bg)
    assert np.array_equal(fw0["final_T"], fw1["final_T"]) and np.array_equal(fw0["n_contrib"], fw1["n_contrib"])
    assert np.array_equal(fw0["radii"], fw1["radii"])
    want = fw0["color"] + fw0["final_T"][None] * bg[:, None, None]
    assert np.abs(fw1["color"] - want).max() <= 1e-6


def test_image_is_invariant_under_permutation_of_the_gaussians():
    sc = _scene(seed=8)
    fw0, _ = h.run_oracle(sc, np.zeros(3, np.float32))
    vis = fw0["radii"] > 0
    assert len(np.unique(fw0["depths"][vis])) == int(vis.sum()), "test scene must have distinct depths"
    perm = np.random.default_rng(0).permutation(sc.means3D.shape[0])
    sc2 = sc._replace(means3D=sc.means3D[perm], scales=sc.scales[perm], rotations=sc.rotations[perm],
                      opacities=sc.opacities[perm], shs=sc.shs[perm], colors_precomp=sc.colors_precomp[perm])
    fw1, _ = h.run_oracle(sc2, np.zeros(3, np.float32))
    assert fw1["num_rendered"] == fw0["num_rendered"]
    assert np.array_equal(fw1["radii"], fw0["radii"][perm])
    assert np.array_equal(fw1["color"].view(np.uint32), fw0["color"].view(np.uint32))
    assert np.array_equal(fw1["n_contrib"], fw0["n_contrib"])


def test_backward_is_linear_in_the_upstream_gradient():
    from sugar_b200 import scenes
    sc = _scene(seed=11)
    W, H = sc.width, sc.height
    d1, d2 = scenes.upstream_grad(W, H, seed=1), scenes.upstream_grad(W, H, seed=2)
    a, b = 0.75, -1.5
    _, g1 = h.run_oracle(sc, np.zeros(3, np.float32), d1)
    _, g2 = h.run_oracle(sc, np.zeros(3, np.float32), d2)
    _, g12 = h.run_oracle(sc, np.zeros(3, np.float32), (a * d1 + b * d2).astype(np.float32))
    for k in ("dL_dmeans2D", "dL_dopacity", "dL_dmeans3D", "dL_dsh", "dL_dscales", "dL_drotations", "dL_dcov3D"):
        assert h.rel_err(g12[k], a * g1[k] + b * g2[k]) <= 2e-5, k


def test_culled_gaussians_have_zero_radius_and_zero_gradients():
    from sugar_b200 import scenes
    sc = _scene(seed=13)
    fw, bw = h.run_oracle(sc, np.zeros(3, np.float32), scenes.upstream_grad(sc.width, sc.height))
    V = sc.viewmatrix.astype(np.float64).T
    z = (sc.means3D.astype(np.float64) @ V[:3, :3].T + V[:3, 3])[:, 2]
    behind = z <= 0.2 - 1e-4
    assert behind.any() and (fw["radii"][behind] == 0).all()
    culled = fw["radii"] == 0
    for k in ("dL_dmeans2D", "dL_dopacity", "dL_dmeans3D", "dL_dsh", "dL_dscales", "dL_drotations"):
        assert not np.any(bw[k][culled]), k


def test_a_splat_of_opacity_one_255th_is_drawn_where_power_is_zero():
    """alpha = min(0.99, o exp(power)) is skipped when alpha < 1/255 (forward.cu:344).  At the pixel a mean projects
    to exactly, power == 0 and alpha == o, so o == 1/255 is drawn and the next float below it is not.  Restated here:
    the centre pixel's n_contrib, final_T and colour follow from the opacities alone, blended in fp32 front to back."""
    from sugar_b200 import scenes
    sc = h.opacity_edge_scene()
    P, W, H = sc.means3D.shape[0], sc.width, sc.height
    bg = np.array([0.25, 0.5, 1.0], np.float32)
    fw, _ = h.run_oracle(sc, bg, scenes.upstream_grad(W, H), use_sh=False)
    c = (W - 1) // 2
    assert np.all(fw["means2D"] == np.float32(c)) and np.all(fw["radii"] > 0)
    o = sc.opacities.reshape(-1)
    drawn = o >= h.ALPHA_MIN
    assert drawn.sum() == P - 2 and drawn[-1]
    T, C = np.float32(1), np.zeros(3, np.float32)
    for i in np.flatnonzero(drawn):      # means sorted by depth == index order
        a = np.float32(min(np.float32(0.99), o[i]))
        C = (C + T * (a * sc.colors_precomp[i])).astype(np.float32)
        T = np.float32(T * (np.float32(1) - a))
    assert int(fw["n_contrib"][c, c]) == P        # the farthest splat (1/255) is the last contributor
    assert abs(float(fw["final_T"][c, c]) - float(T)) <= 1e-7
    assert np.abs(fw["color"][:, c, c] - (C + T * bg)).max() <= 1e-6
    # the splats one ulp below 1/255 add nothing anywhere: the image equals the one with their opacity at zero
    fw1, _ = h.run_oracle(sc._replace(opacities=np.where(drawn[:, None], sc.opacities, 0).astype(np.float32)), bg,
                          use_sh=False)
    assert np.array_equal(fw1["n_contrib"], fw["n_contrib"]) and np.array_equal(fw1["color"], fw["color"])


def test_linear_properties_checker_on_the_oracle():
    """helpers.check_linear_properties (the checker the GPU suite runs at the headline size) on the CPU oracle."""
    sc = _scene(P=1200, W=80, H=48, seed=17)

    def run(bg, dL):
        fw, bw = h.run_oracle(sc, np.asarray(bg, np.float32), dL)
        grads = None if bw is None else {k: bw[k] for k in ("dL_dmeans3D", "dL_dmeans2D", "dL_dopacity", "dL_dsh",
                                                            "dL_dscales", "dL_drotations")}
        return fw["color"], fw["radii"], grads
    h.check_linear_properties(run, sc.width, sc.height, tol_img=1e-6, tol_grad=2e-5)


def test_a_views_sh_gradient_is_a_rank_one_product_of_its_colour_gradient():
    """What the multi-GPU exchange rests on (sugar_b200/parallel.py): per view, dL_dsh[i] = basis(normalize(mean_i -
    campos)) (x) (dL_dcolor_i masked where the forward clamped the colour) -- so 12 bytes per Gaussian and view describe
    its 192 bytes of SH gradient, and the sum over views can be rebuilt from the views' factors.  Checked on the restated
    reference backward (backward.cu:20-139) for two views and every SH degree."""
    from sugar_b200 import scenes
    P, W, H = 1200, 96, 64
    base = scenes.make_scene(P, W, H, seed=11, camera="posed")
    views = [base, scenes.with_camera_offset(base, 0.2, (0.3, -0.1, 0.2))]
    for deg in (0, 1, 2, 3):
        total, rebuilt = 0.0, 0.0
        for v, sc in enumerate(views):
            dL = scenes.upstream_grad(W, H, seed=3 + v)
            fw, bw = h.run_oracle(sc, np.zeros(3, np.float32), dL, use_sh=True, sh_degree=deg)
            vis = fw["radii"] > 0
            factor = bw["dL_dcolors"].astype(np.float64) * (1.0 - fw["clamped"].astype(np.float64))
            factor[~vis] = 0.0
            d = sc.means3D.astype(np.float64) - np.asarray(sc.campos, np.float64).reshape(1, 3)
            d /= np.linalg.norm(d, axis=1, keepdims=True)
            want = h.sh_basis(d, deg)[:, :, None] * factor[:, None, :]
            got = bw["dL_dsh"].astype(np.float64)
            assert vis.sum() > 100
            assert np.abs(got - want).max() <= 2e-6 * max(np.abs(want).max(), 1e-30), deg
            assert np.all(got[:, (deg + 1) ** 2:] == 0.0)
            total, rebuilt = total + got, rebuilt + want
        assert np.abs(total - rebuilt).max() <= 2e-6 * np.abs(total).max()
