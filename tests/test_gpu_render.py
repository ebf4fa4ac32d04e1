"""SuGaR.render_image_gaussian_rasterizer as the trainers call it (SURVEY a12): the mirror in sugar_b200/render.py
against the arguments the reference's own wrapper produced (tests/golden/render_wrapper.npz, made by running
sugar_model.py:2085-2294 with a recording rasterizer) rasterized by the UNMODIFIED reference CUDA build (its image and
radii: tests/golden/refbuild_render.npz, tests/golden/make_refbuild_golden.py)."""
import os

import numpy as np
import pytest

import helpers as h

pytestmark = pytest.mark.gpu


def test_render_wrapper_matches_reference_wrapper_plus_reference_rasterizer():
    import torch
    from sugar_b200 import render
    g = np.load(os.path.join(h.ROOT, "tests", "golden", "render_wrapper.npz"))
    t = lambda k: torch.from_numpy(g[k]).cuda()
    H, W = (int(v) for v in g["hw"])
    kw = dict(points=t("points"), scaling=t("scaling"), quaternions=t("quaternions"), opacities=t("strengths"),
              sh_coordinates=t("sh"), c2w=t("c2w"), fov_x=float(g["fov"][0]), fov_y=float(g["fov"][1]), image_height=H,
              image_width=W, bg_color=t("bg"), sh_deg=int(g["sh_degree"]),
              principal_point=(float(g["pp"][0]), float(g["pp"][1])))
    img_py = render.render_image_gaussian_rasterizer(compute_color_in_rasterizer=False, **kw)
    out = render.render_image_gaussian_rasterizer(compute_color_in_rasterizer=True, return_2d_radii=True, **kw)
    assert img_py.shape == (H, W, 3) and out["radii"].shape == (g["points"].shape[0],)
    assert float((out["radii"] > 0).float().mean()) > 0.5
    # in-kernel SH vs the python colour path: same polynomial, different evaluation order
    assert float((out["image"] - img_py).abs().max()) <= 1e-5
    ref = h.load_golden("render")
    img_ref = torch.from_numpy(ref["image"]).cuda()
    radii_ref = torch.from_numpy(ref["radii"]).cuda()
    assert float((img_py - img_ref.permute(1, 2, 0)).abs().max()) <= 2e-5
    assert float((radii_ref == out["radii"]).float().mean()) > 0.995
