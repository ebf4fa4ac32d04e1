"""The forward blend's splat visit at its edges.

blend_forward_kernel stages the records of a tile's list in batches of 256 and lets each warp (one 8x4 pixel block)
walk the splats whose footprint mask has its block.  In a warp with a candidate lane (one that passes the power
window), every lane evaluates the splat's tail and keeps it only where it contributes: a lane that fails the alpha
test, or whose T would fall below 1e-4, keeps its T, colour and n_contrib, and the second case ends the pixel for good
while the warp's other lanes go on.  Each scene below puts one edge of that tail on block 0 of one tile:

  * done_mid_warp: one pixel of the block is finished by its second opaque splat, its neighbours keep blending;
  * done_on_batch_end / done_on_batch_start: the same pixel ends on list position 255 (the last record of the first
    batch) or 256 (the first record of the second);
  * alpha_threshold: on the optical axis, a splat of alpha exactly 1/255 behind one clamped at 0.99;
  * candidate_fails_alpha: a splat whose power window admits block pixels where its alpha is just under 1/255, while
    the pixels nearer its centre contribute in the same visit;
  * tile_256 / tile_257: a tile of exactly 256 and 257 list entries;
  * partial_edge_tiles: a 40x27 image, whose right and bottom tiles have lanes outside the image.

The test checks that each list has that shape (from the forward state and the footprint masks), then compares
n_contrib exactly and final_T and the image with the CPU oracle at the tolerance of tests/test_gpu_parity.py, for both
instance-list formats (packed ids with masks, and plain ids with the masks computed in the blend; the plain-id run
appends culled Gaussians up to P = 2^24, helpers.run_state)."""
import math

import numpy as np
import pytest

import helpers as h
from test_gpu_blend_backward_overlap import _scene

pytestmark = pytest.mark.gpu

FWD_B = 256                            # records per batch of the forward blend (sgr_forward.cu, BLEND_T)
BG = (0.25, 0.5, 1.0)
DONE_PIXEL = (1, 2)                    # (row, column) in block 0 of tile 0
OPAQUE = (2.0, 1.0, 0.3, 0.3, 1.0)     # (u, v, sigma x, sigma y, opacity): alpha clamped to 0.99 at DONE_PIXEL
WIDE = (3.5, 1.5, 4.0, 4.0, 0.5)       # covers block 0


def _fillers(n, seed):
    """n small splats in the bottom-right block of a 16x16 tile, all in front of z = 2: they fill list positions
    0..n-1 and none of them reaches block 0."""
    rng = np.random.Generator(np.random.PCG64(seed))
    return [(11.5 + rng.uniform(-1, 1), 13.5 + rng.uniform(-0.5, 0.5), 1.0 + 0.9 * i / n, 0.6, 0.6, 0.3)
            for i in range(n)]


def _done_scene(n_fill):
    """n_fill fillers, two opaque splats on DONE_PIXEL (the second finishes it), then a wide one behind."""
    u, v, sx, sy, op = OPAQUE
    return _fillers(n_fill, n_fill) + [(u, v, 2.0, sx, sy, op), (u, v, 2.1, sx, sy, op), (WIDE[0], WIDE[1], 3.0) + WIDE[2:]]


def _random(n, W, H, seed):
    rng = np.random.Generator(np.random.PCG64(seed))
    return [(rng.uniform(1, W - 1), rng.uniform(1, H - 1), 2.0 + 4.0 * i / n, rng.uniform(0.5, 1.5), rng.uniform(0.5, 1.5),
             rng.uniform(0.02, 0.2)) for i in range(n)]


def _candidate_fails_alpha():
    """A splat centred on pixel (2, 1) whose opacity puts the alpha at pixel (4, 2) 5e-5 (relative) under 1/255:
    the power window (tau carries a 1e-4 margin) admits that pixel, the alpha test rejects it, and the pixels near the
    centre contribute.  The opacity comes from the splat's projected conic (which does not depend on it)."""
    probe = [(2.0, 1.0, 2.0, 1.0, 1.0, 0.5)]
    fw, _ = h.run_oracle(_scene(16, 16, probe, seed=0), np.zeros(3, np.float32), use_sh=False)
    power = _power(fw, 0, 4, 2)
    op = math.exp(-power) / 255.0 * (1.0 - 5e-5)
    return [(2.0, 1.0, 2.0, 1.0, 1.0, op), (WIDE[0], WIDE[1], 3.0) + WIDE[2:]]


SCENES = {   # name: (W, H, splats)
    "done_mid_warp": (16, 16, _done_scene(0)),
    "done_on_batch_end": (16, 16, _done_scene(FWD_B - 2)),
    "done_on_batch_start": (16, 16, _done_scene(FWD_B - 1)),
    # pixel (16, 16) of a 33x33 image is on the optical axis: power == 0 there, alpha == min(0.99, opacity)
    "alpha_threshold": (33, 33, [(16.0, 16.0, 2.0, 0.6, 0.6, 1.0), (16.0, 16.0, 3.0, 0.6, 1.5, float(h.ALPHA_MIN)),
                                 (16.0, 16.0, 4.0, 1.5, 0.6, 0.5)]),
    "candidate_fails_alpha": (16, 16, None),
    "tile_256": (16, 16, _random(FWD_B, 16, 16, 256)),
    "tile_257": (16, 16, _random(FWD_B + 1, 16, 16, 257)),
    "partial_edge_tiles": (40, 27, _random(150, 40, 27, 4027)),
}


def _make(name):
    W, H, splats = SCENES[name]
    if splats is None:
        splats = _candidate_fails_alpha()
    return _scene(W, H, splats, seed=len(name))


def _power(o, g, px, py):
    """power of Gaussian g at pixel (px, py) from the forward state (float64)."""
    mx, my = (float(x) for x in o["means2D"][g])
    a, b, c, _ = (float(x) for x in o["conic_opacity"][g])
    dx, dy = mx - px, my - py
    return -0.5 * (a * dx * dx + c * dy * dy) - b * dx * dy


def _check_shape(name, o, masks):
    """The list has the shape the scene is built for (o: the forward state; masks: whether o holds footprint masks)."""
    W, H, _ = SCENES[name]
    nc = o["n_contrib"].astype(np.int64)
    lo, hi = (int(x) for x in o["ranges"][0])
    if name.startswith("done_"):
        n_fill = {"done_mid_warp": 0, "done_on_batch_end": FWD_B - 2, "done_on_batch_start": FWD_B - 1}[name]
        r, c = DONE_PIXEL
        assert hi - lo == n_fill + 3
        # the first opaque splat (list position n_fill) is the pixel's last contributor: the second one, at
        # position n_fill + 1, would take T below 1e-4 and ends the pixel there
        assert int(nc[r, c]) == n_fill + 1, int(nc[r, c])
        T = np.float32(o["final_T"][r, c])
        assert T >= np.float32(1e-4) and T * (np.float32(1) - np.float32(0.99)) < np.float32(1e-4), T
        # the rest of the block goes on to the wide splat behind
        assert int(nc[0:4, 0:8].max()) == n_fill + 3
        if masks:
            fp = o["footprint"][lo:hi].astype(np.int64)
            assert not (fp[:n_fill] & 1).any()          # no filler is a member of block 0
            assert (fp[n_fill:] & 1).all()
    elif name == "alpha_threshold":
        g = int(o["point_list"][lo + 1])
        assert np.float32(o["conic_opacity"][g][3]) == h.ALPHA_MIN
        assert np.array_equal(o["means2D"][g], np.float32([16.0, 16.0]))
        assert float(o["conic_opacity"][int(o["point_list"][lo])][3]) > 0.99   # alpha clamped to 0.99
        assert int(nc[16, 16]) == 3                      # drawn: alpha == 1/255 passes `alpha < 1/255`
    elif name == "candidate_fails_alpha":
        g = int(o["point_list"][lo])
        op = float(o["conic_opacity"][g][3])
        tau = -math.log(op * 255.0) - 1e-4               # the record's tau: lanes at power >= tau are candidates
        power = np.array([[_power(o, g, x, y) for x in range(8)] for y in range(4)])
        alpha = np.minimum(0.99, op * np.exp(power))
        assert ((power >= tau + 1e-5) & (alpha < (1.0 - 1e-5) / 255.0)).any(), (power, tau)
        assert (alpha >= 1.0 / 255.0).any()
        if masks:
            assert int(o["footprint"][lo]) & 1
    elif name.startswith("tile_"):
        assert hi - lo == int(name[5:])
    elif name == "partial_edge_tiles":
        gx, gy = (W + 15) // 16, (H + 15) // 16
        assert W % 16 and H % 16
        corner = o["ranges"][gx * gy - 1]
        assert int(corner[1]) > int(corner[0])           # the corner tile, with lanes outside the image, has splats


@pytest.mark.parametrize("unpacked", [False, True], ids=["packed_ids", "unpacked_ids"])
@pytest.mark.parametrize("name", list(SCENES))
def test_forward_visit_edges_match_cpu_oracle(name, unpacked):
    sc = _make(name)
    W, H = sc.width, sc.height
    fw, _ = h.run_oracle(sc, np.asarray(BG, np.float32), use_sh=False)
    o = h.run_state(sc, BG, plain_ids=unpacked, use_sh=False)
    _check_shape(name, o, masks=not unpacked)
    assert np.array_equal(o["point_list"].view(np.uint32), fw["point_list"])
    assert np.array_equal(o["ranges"].view(np.uint32), fw["ranges"])
    nc = o["n_contrib"].view(np.uint32)
    if name == "alpha_threshold":
        # as test_gpu_parity's opacity-edge test: bit-identical where power == 0 (exp(0) == 1 on both sides), and
        # elsewhere glibc expf vs MUFU.EX2 may flip a pair sitting on a threshold
        assert int(nc[16, 16]) == int(fw["n_contrib"][16, 16])
        assert o["final_T"][16, 16].view(np.uint32) == fw["final_T"][16, 16].view(np.uint32)
        assert np.array_equal(o["color"][:, 16, 16].view(np.uint32), fw["color"][:, 16, 16].view(np.uint32))
        assert int((nc != fw["n_contrib"]).sum()) <= 2
    else:
        assert np.array_equal(nc, fw["n_contrib"]), np.argwhere(nc != fw["n_contrib"])
    for got, want in ((o["final_T"], fw["final_T"]), (o["color"], fw["color"])):
        d = np.abs(got - want)
        assert np.quantile(d, 0.999) < 2e-6 and d.max() < 5e-3, (float(np.quantile(d, 0.999)), float(d.max()))
