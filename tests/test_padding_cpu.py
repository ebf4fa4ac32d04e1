"""The culled padding (helpers.pad_culled) on the CPU oracle.

The GPU tests reach the plain-id instance lists, which the library uses for clouds of 2^24 Gaussians or more, by
appending culled Gaussians to a small scene (helpers.run_state with plain_ids=True).  That checks the plain-id path
only if the padding changes nothing else.  Here the oracle renders scenes with and without a few thousand padded
rows: the padded rows must be culled (radius 0, no tiles, zero gradients), and the image, n_contrib, final_T, sort
keys, point list, ranges and the scene's own gradients must be bit-identical."""
import numpy as np
import pytest

import helpers as h

PAD = 3000
BG = np.asarray((0.25, 0.5, 1.0), np.float32)
CASES = [  # id, camera, use_sh, sh_degree
    ("identity_sh3", "identity", True, 3),
    ("posed_sh3", "posed", True, 3),
    ("identity_colors", "identity", False, 0),
    ("posed_colors", "posed", False, 0),
]


@pytest.mark.parametrize("camera,use_sh,deg", [c[1:] for c in CASES], ids=[c[0] for c in CASES])
def test_culled_padding_changes_no_output(camera, use_sh, deg):
    from sugar_b200 import scenes
    P, W, H = 1500, 96, 64
    sc = scenes.make_scene(P, W, H, seed=7, camera=camera)
    names = ["means3D", "opacities", "shs" if use_sh else "colors_precomp", "scales", "rotations"]
    padded = sc._replace(**{k: v.numpy() for k, v in h.pad_culled(h.to_torch(sc, "cpu"), names, P + PAD).items()})
    dL = scenes.upstream_grad(W, H)
    fw, bw = h.run_oracle(sc, BG, dL, use_sh=use_sh, sh_degree=deg)
    pw, pbw = h.run_oracle(padded, BG, dL, use_sh=use_sh, sh_degree=deg)
    assert pw["P"] == P + PAD and (fw["radii"] > 0).sum() > P // 2
    assert not pw["radii"][P:].any() and not pw["tiles_touched"][P:].any()
    assert np.array_equal(pw["radii"][:P], fw["radii"])
    for k in ("color", "n_contrib", "final_T", "keys", "point_list", "ranges"):
        assert np.array_equal(h.digest(pw[k]), h.digest(fw[k])), k
    for k, g in pbw.items():
        assert not g[P:].any(), k
        assert np.array_equal(h.digest(g[:P]), h.digest(bw[k])), k
