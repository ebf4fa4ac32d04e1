"""The backward blend's splat walk at its boundaries.

blend_backward_kernel walks each 8x4 block's member splats back to front, one 64-record batch (one record stage) at a
time, reading 32-slot membership words.  A contributing visit parks the pixel's (S, alpha*T) pair and the splat's batch
slot; the splat's metadata is copied out of the record stage when its chunk of 16 is flushed or before the warp
releases the stage, so a chunk can hold splats of two stages.  Each scene below puts one boundary case on the first
8x4 block of one tile: a list of exactly 1, 2 or 3 members, a pair of members in two membership words, a pair in two
batches (with a chunk that straddles them), a member without a valid lane followed by a contributing one, and a second
member whose alpha is exactly 1/255.  The test checks that the list has that shape (from the forward state and the
footprint masks) and holds the gradients to the CPU oracle at the tolerance of tests/test_gpu_parity.py, for both
instance-list formats (packed ids with masks, and plain ids with the masks computed in the blend; the plain-id run
appends culled Gaussians up to P = 2^24, helpers.run_state)."""
import math

import numpy as np
import pytest

import helpers as h

pytestmark = pytest.mark.gpu

ORACLE_GRAD_RTOL = 5e-4   # test_gpu_parity.test_matches_cpu_oracle
GRAD_NAMES = dict(means3D="dL_dmeans3D", means2D="dL_dmeans2D", opacities="dL_dopacity",
                  colors_precomp="dL_dcolors", scales="dL_dscales", rotations="dL_drotations")
BWD_B = 64                # records per batch of the backward blend (sgr_backward.cu)


def _place(W, H, u, v, z, tanfovx, tanfovy):
    """World point (identity camera) whose mean projects to pixel (u, v)."""
    return [z * tanfovx * ((2.0 * u + 1.0) / W - 1.0), z * tanfovy * ((2.0 * v + 1.0) / H - 1.0), z]


def _scene(W, H, splats, seed):
    """splats: (u, v, z, pixel sigma x, pixel sigma y, opacity); identity camera, axis-aligned Gaussians."""
    from sugar_b200 import scenes
    P = len(splats)
    sc = scenes.make_scene(P, W, H, seed=seed, camera="identity", frac_behind=0.0)
    focal = W / (2.0 * sc.tanfovx)
    m = np.array([_place(W, H, u, v, z, sc.tanfovx, sc.tanfovy) for u, v, z, *_ in splats], np.float32)
    # pixel sigma s at depth z: world scale s * z / focal (the 0.3 px^2 low-pass filter comes on top)
    s = np.array([[sx * z / focal, sy * z / focal, 1e-4] for _, _, z, sx, sy, _ in splats], np.float32)
    q = np.tile(np.array([1.0, 0.0, 0.0, 0.0], np.float32), (P, 1))
    o = np.array([[op] for *_, op in splats], np.float32)
    return sc._replace(means3D=m, scales=s, rotations=q, opacities=o)


def _one_block(n, seed, z0=2.0, dz=0.05, op=0.5):
    """n small splats around the centre of block 0 of tile 0 (pixels 0-7 x 0-3), front to back."""
    rng = np.random.Generator(np.random.PCG64(seed))
    return [(3.5 + rng.uniform(-1.5, 1.5), 1.5 + rng.uniform(-0.5, 0.5), z0 + dz * i, 0.6, 0.6, op) for i in range(n)]


def _scenes():
    W = H = 16
    out = {
        "1_member": (W, H, _one_block(1, 1), 0),
        "2_members": (W, H, _one_block(2, 2), 0),
        "3_members": (W, H, _one_block(3, 3), 0),
        # 40 members: the walk's slots 31 and 32 are a pair in two membership words
        "word_straddle": (W, H, _one_block(40, 4, op=0.08), 0),
        # 90 members among 100 splats: slots 63 and 64 are a pair in two batches, so in two record stages, and the
        # 57 members of the first batch leave a chunk of 16 open across the stage boundary
        "batch_straddle": (W, H, [(12.0, 13.5) + sp[2:] if i % 10 == 7 else sp
                                  for i, sp in enumerate(_one_block(100, 5, op=0.04, dz=0.02))], 0),
        # the middle splat: wide in x, centred right of block 0 between rows 1 and 2.  Its footprint band reaches
        # block 0 at y = 1.5, but at the pixel rows 1 and 2 its alpha stays below 1/255 in columns 0-8, so it is a
        # member of the block without a valid lane, between two contributing members (the farther one keeps it
        # inside the warp's walk)
        "dead_first": (W, H, [(3.5, 1.5, 3.0, 0.6, 0.6, 0.5), (16.5, 1.5, 5.0, 8.0, 1e-3, 0.01),
                              (4.0, 2.0, 6.0, 0.6, 0.6, 0.5)], 0),
        # two splats on the optical axis of a 33x33 image (pixel (16, 16): block 0 of tile (1, 1), power == 0):
        # the walk's second member has opacity 1/255 there, so its alpha is exactly the threshold
        # (elliptical, so that the rotation gradients are not zero by symmetry)
        "threshold_second": (33, 33, [(16.0, 16.0, 3.0, 0.6, 1.5, float(h.ALPHA_MIN)),
                                      (16.0, 16.0, 4.0, 1.5, 0.6, 0.5)], 1),
    }
    return out


SCENES = _scenes()


def _make(name):
    W, H, splats, _ = SCENES[name]
    return _scene(W, H, splats, seed=len(name))


def _walk(o, tile, W, wid):
    """(instance ids, walk slots) of warp `wid`'s members in tile `tile`, in walk order (back to front), from the
    forward state and the packed lists' footprint masks."""
    lo, hi = (int(x) for x in o["ranges"][tile])
    gx = (W + 15) // 16
    ty, tx = divmod(tile, gx)
    nc = o["n_contrib"].astype(np.int64)
    ys, xs = slice(16 * ty, 16 * ty + 16), slice(16 * tx, 16 * tx + 16)
    n = int(nc[ys, xs].max())                       # the tile walks list positions [0, n)
    by, bx = 16 * ty + 4 * (wid >> 1), 16 * tx + 8 * (wid & 1)
    warp_last = int(nc[by:by + 4, bx:bx + 8].max())
    ids, slots = [], []
    for j in range(n):                              # walk slot j = list position n - 1 - j
        pos = n - 1 - j
        if pos < warp_last and (int(o["footprint"][lo + pos]) >> wid) & 1:
            ids.append(int(o["point_list"][lo + pos]))
            slots.append(j)
    return ids, slots


def _block_alpha_power(o, g, tile, W, wid):
    """power and the exact alpha of Gaussian g at the 32 pixels of warp `wid`'s block (float64)."""
    gx = (W + 15) // 16
    ty, tx = divmod(tile, gx)
    by, bx = 16 * ty + 4 * (wid >> 1), 16 * tx + 8 * (wid & 1)
    py, px = np.meshgrid(np.arange(by, by + 4), np.arange(bx, bx + 8), indexing="ij")
    m = o["means2D"][g].astype(np.float64)
    a, b, c, op = (float(v) for v in o["conic_opacity"][g])
    dx, dy = m[0] - px, m[1] - py
    power = -0.5 * (a * dx * dx + c * dy * dy) - b * dx * dy
    return power, np.minimum(0.99, op * np.exp(power)), op


def _check_shape(name, o):
    """The member list of block 0 of the scene's tile has the shape the scene is built for."""
    W = SCENES[name][0]
    tile = SCENES[name][3] * (((W + 15) // 16) + 1)  # tile (t, t)
    ids, slots = _walk(o, tile, W, 0)
    if name.endswith("member") or name.endswith("members"):
        assert len(ids) == int(name[0]), (name, ids)
    elif name == "word_straddle":
        assert 31 in slots and 32 in slots, slots
    elif name == "batch_straddle":
        assert BWD_B - 1 in slots and BWD_B in slots, slots
        assert sum(j < BWD_B for j in slots) % 16 != 0, slots
    elif name == "dead_first":
        assert len(ids) == 3, ids
        power, alpha, op = _block_alpha_power(o, ids[1], tile, W, 0)
        tau = -math.log(op * 255.0) - 1e-4         # the record's tau: no lane is a candidate below it
        assert power.max() < tau - 1e-3, (power.max(), tau)
        for g in (ids[0], ids[2]):
            assert _block_alpha_power(o, g, tile, W, 0)[1].max() >= 1.0 / 255.0
    elif name == "threshold_second":
        assert len(ids) == 2, ids
        g = ids[1]
        assert np.float32(o["conic_opacity"][g][3]) == h.ALPHA_MIN
        assert np.array_equal(o["means2D"][g], np.float32([16.0, 16.0]))
        assert int(o["n_contrib"][16, 16]) == 2     # drawn: alpha == 1/255 passes `alpha < 1/255`


@pytest.mark.parametrize("unpacked", [False, True], ids=["packed_ids", "unpacked_ids"])
@pytest.mark.parametrize("name", list(SCENES))
def test_backward_walk_boundaries_match_cpu_oracle(name, unpacked):
    from sugar_b200 import scenes
    sc = _make(name)
    P, W, H = sc.means3D.shape[0], sc.width, sc.height
    fw, bw = h.run_oracle(sc, np.asarray((0.25, 0.5, 1.0), np.float32), scenes.upstream_grad(W, H), use_sh=False)
    o = h.run_state(sc, (0.25, 0.5, 1.0), scenes.upstream_grad(W, H), plain_ids=unpacked, use_sh=False)
    if not unpacked:
        _check_shape(name, o)   # the plain-id lists carry no masks; the packed run checks the scene
    assert np.array_equal(o["point_list"].view(np.uint32), fw["point_list"])
    assert np.array_equal(o["ranges"].view(np.uint32), fw["ranges"])
    # glibc expf vs MUFU.EX2 in the forward: as in test_gpu_parity, a pair sitting on a threshold may flip
    assert int((o["n_contrib"].view(np.uint32) != fw["n_contrib"]).sum()) <= 2
    assert np.abs(bw["dL_dopacity"]).max() > 0 and np.abs(bw["dL_dcolors"]).max() > 0
    d = np.abs(o["color"] - fw["color"])
    assert np.quantile(d, 0.999) < 2e-6 and d.max() < 5e-3, (float(np.quantile(d, 0.999)), float(d.max()))
    for k, name_bw in GRAD_NAMES.items():
        want = bw[name_bw]
        got = o["grad_" + k].reshape(want.shape)
        err = h.rel_err(got, want)
        assert err <= ORACLE_GRAD_RTOL, f"grad {k}: rel err vs oracle {err:.3e}"
