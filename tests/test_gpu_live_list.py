"""The live instance list: scatter_kernel writes a word only for instances whose footprint mask is not empty, at the
front of the tile's segment, and the sorts and both blend kernels walk [tile_start[t], tile_cursor[t]) alone.

The reference's state is unchanged: sgr_inspect_state rebuilds the full list (dead instances included) and maps each
pixel's n_contrib, a position in the live list, back to the reference's count over the full list.  These tests read
both lists: the live one straight from the forward's opaque buffers (the layout of sgr_internal.cuh), the full one
through _C.inspect_state, and check

  * per tile, the live list is the full list with its mask-0 words removed, in the same order, and it ends at
    tile_cursor (classes scene: live counts at the sort classes' edges 512/513, 2048/2049 and 8192/8193, each tile
    padded with dead instances so that its full count falls in another class);
  * a pixel whose last contributor has dead instances in front of it gets the reference's n_contrib, and the
    backward bounded by the live n_contrib gives the oracle's gradients (behind_dead scene);
  * a forward whose optimistic capacity overflows re-runs into the same state;
  * the plain-id format (P padded to 2^24 with culled Gaussians, tests/helpers.py) gives the same lists and results.

Dead instances are made two ways: splats of opacity below 1/255 (dead in every tile of their rect) and a faint wide
splat whose 3-sigma rect reaches tiles its alpha >= 1/255 ellipse does not."""
import numpy as np
import pytest

import helpers as h

BG = (0.25, 0.5, 1.0)
ORACLE_GRAD_RTOL = 5e-4   # test_gpu_parity.test_matches_cpu_oracle
GRAD_NAMES = dict(means3D="dL_dmeans3D", means2D="dL_dmeans2D", opacities="dL_dopacity",
                  colors_precomp="dL_dcolors", scales="dL_dscales", rotations="dL_drotations")
# (live, dead) instances per tile of the classes scene: live counts at the edges of the sort classes, full counts in
# another class (merge <= 512 < bucket <= 2048 < merge <= 8192 < global radix)
CLASS_TILES = [(512, 200), (513, 1600), (2048, 100), (2049, 6200), (8192, 100), (8193, 300)]
DEAD_OPACITY = 0.003      # below 1/255: the splat reaches no pixel anywhere


def _scene(W, H, d, seed):
    """Splats placed in pixels under an identity camera (depth == z bit for bit).  d: arrays u, v (pixel of the mean),
    z, sx, sy (pixel sigmas), th (rotation in the image plane), op."""
    from sugar_b200 import scenes
    base = scenes.make_scene(1, W, H, seed=seed, camera="identity", frac_behind=0.0)
    rng = np.random.Generator(np.random.PCG64(seed))
    u, v = np.asarray(d["u"], np.float64), np.asarray(d["v"], np.float64)
    z = np.asarray(d["z"], np.float32)
    P = z.shape[0]
    focal = W / (2.0 * base.tanfovx)
    zz = z.astype(np.float64)
    m = np.stack([zz * base.tanfovx * ((2.0 * u + 1.0) / W - 1.0), zz * base.tanfovy * ((2.0 * v + 1.0) / H - 1.0),
                  zz], 1).astype(np.float32)
    m[:, 2] = z
    s = np.stack([np.asarray(d["sx"]) * zz / focal, np.asarray(d["sy"]) * zz / focal, np.full(P, 1e-4)],
                 1).astype(np.float32)
    th = np.asarray(d["th"], np.float64)
    q = np.stack([np.cos(th / 2), np.zeros(P), np.zeros(P), np.sin(th / 2)], 1).astype(np.float32)
    o = np.asarray(d["op"], np.float32).reshape(P, 1)
    col = rng.uniform(0, 1, (P, 3)).astype(np.float32)
    return base._replace(means3D=m, scales=s, rotations=q, opacities=o, colors_precomp=col,
                         shs=np.zeros((1, 16, 3), np.float32))


def _classes_scene():
    """One row of tiles; tile k holds CLASS_TILES[k]: splats centred 7.5-8.5 px into the tile with sigmas of 1.2-2 px
    (radius <= 7: exactly one tile), the live ones of opacity 0.05-0.2, the dead ones of DEAD_OPACITY; ids shuffled,
    random depths."""
    rng = np.random.Generator(np.random.PCG64(31))
    parts = []
    for t, (live, dead) in enumerate(CLASS_TILES):
        n = live + dead
        parts.append(dict(u=16 * t + rng.uniform(7.5, 8.5, n), v=rng.uniform(7.5, 8.5, n),
                          sx=rng.uniform(1.2, 2.0, n), sy=rng.uniform(1.2, 2.0, n), th=rng.uniform(0, np.pi, n),
                          op=np.concatenate([rng.uniform(0.05, 0.2, live), np.full(dead, DEAD_OPACITY)])))
    d = {k: np.concatenate([p[k] for p in parts]) for k in parts[0]}
    perm = rng.permutation(len(d["u"]))
    d = {k: v[perm] for k, v in d.items()}
    d["z"] = rng.uniform(2.0, 10.0, len(d["u"])).astype(np.float32)
    return _scene(16 * len(CLASS_TILES), 16, d, seed=31)


CENTRE = 8   # the pixel (CENTRE, CENTRE) of the behind_dead scene


def _behind_dead_scene():
    """A 32 x 32 image.  At pixel (8, 8), front to back: A (drawn), D1 (opacity below 1/255), D2 (a faint wide splat
    centred in tile 1: its rect covers tile 0, its alpha >= 1/255 ellipse does not), B (drawn, the last contributor).
    The tile-0 list is A, D1, D2, B: the reference's n_contrib there is 4, the live list's 2."""
    d = dict(u=np.array([8.2, 8.1, 24.0, 7.9]), v=np.array([8.1, 7.9, 8.0, 8.2]),
             z=np.array([2.0, 3.0, 3.5, 5.0], np.float32), sx=np.array([2.0, 2.0, 10.0, 2.5]),
             sy=np.array([1.5, 2.0, 10.0, 2.0]), th=np.array([0.3, 0.0, 0.0, 1.1]),
             op=np.array([0.3, DEAD_OPACITY, 0.0045, 0.4]))
    return _scene(32, 32, d, seed=32)


SCENES = dict(classes=_classes_scene, behind_dead=_behind_dead_scene)
_MADE = {}


def _make(name):
    if name not in _MADE:
        _MADE[name] = SCENES[name]()
    return _MADE[name]


def _reachable(o, W, H):
    """Per list position of the oracle's full list: whether its splat passes the alpha test at some pixel of its tile
    (float64 enumeration).  Such an instance has a non-empty footprint mask (the masks are conservative)."""
    plist = o["point_list"].astype(np.int64)
    n = o["ranges"][:, 1].astype(np.int64) - o["ranges"][:, 0]
    tile = np.repeat(np.arange(len(n)), n)
    gx = (W + 15) // 16
    m2, co = o["means2D"].astype(np.float64)[plist], o["conic_opacity"].astype(np.float64)[plist]
    px = ((tile % gx) * 16)[:, None, None] + np.arange(16)[None, None, :]
    py = ((tile // gx) * 16)[:, None, None] + np.arange(16)[None, :, None]
    dx, dy = m2[:, 0, None, None] - px, m2[:, 1, None, None] - py
    power = -0.5 * (co[:, 0, None, None] * dx * dx + co[:, 2, None, None] * dy * dy) - co[:, 1, None, None] * dx * dy
    alpha = np.minimum(co[:, 3, None, None] * np.exp(power), 0.99)
    return ((power <= 0) & (alpha >= 1.0 / 255.0)).any(axis=(1, 2)), tile


def _check_design(name, o, W, H):
    """The scene has the shape it is built for (o: a forward state in the reference's form, oracle or GPU)."""
    reach, tile = _reachable(o, W, H)
    dead_op = o["conic_opacity"][o["point_list"].astype(np.int64), 3] < 1.0 / 255.0
    assert not (reach & dead_op).any()
    n = o["ranges"][:, 1].astype(np.int64) - o["ranges"][:, 0]
    live = np.bincount(tile[reach], minlength=len(n))
    if name == "classes":
        assert [(int(a), int(b - a)) for a, b in zip(live, n)] == CLASS_TILES
        assert np.array_equal(reach, ~dead_op)
    else:
        lo = int(o["ranges"][0, 0])
        ids = o["point_list"][lo:int(o["ranges"][0, 1])].astype(np.int64)
        assert list(ids) == [0, 1, 2, 3] and list(reach[lo:lo + 4]) == [True, False, False, True]
        assert int(o["n_contrib"][CENTRE, CENTRE]) == 4


@pytest.mark.parametrize("name", list(SCENES))
def test_live_list_scene_shapes_on_cpu_oracle(name):
    sc = _make(name)
    fw, _ = h.run_oracle(sc, np.asarray(BG, np.float32), use_sh=False)
    _check_design(name, fw, sc.width, sc.height)


# ------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------
def _align(x, a=256):
    return (x + a - 1) // a * a


def _raw(a, W, H):
    """What the forward left in its opaque buffers (sgr_internal.cuh: ImageState / BinState): tile_start [T+1],
    tile_cursor [T] (the live ends), n_contrib [H, W] (live positions) and the sorted list words plist [R]."""
    import torch
    T = ((W + 15) // 16) * ((H + 15) // 16)
    img, binning = a["img"], a["binning"]
    p = _align(img.data_ptr()) - img.data_ptr()
    u32 = lambda buf, off, n: buf[off:off + 4 * n].view(torch.int32).cpu().numpy().view(np.uint32)
    n_contrib = u32(img, p + _align(W * H * 4), W * H).reshape(H, W)
    p += 2 * _align(W * H * 4) + _align(T * 4)                      # final_T, n_contrib, tile_count
    tile_start = u32(img, p, T + 1)
    tile_cursor = u32(img, p + _align((T + 1) * 4), T)
    q = _align(binning.data_ptr()) - binning.data_ptr()
    plist = u32(binning, q, a["num_rendered"])
    return dict(tile_start=tile_start, tile_cursor=tile_cursor, n_contrib=n_contrib, plist=plist)


def _run(sc, plain, dL=None, ctx=None):
    """Forward (+ backward with dL) of `sc` in one id format: (run_module's dict, the reference-form state, the raw
    live state)."""
    import contextlib
    from sugar_b200 import _C, diff_gaussian_rasterization as ours
    P, W, H = sc.means3D.shape[0], sc.width, sc.height
    pad = h.PACKED_MAX_P if plain else None
    with _C.use_context(ctx) if ctx is not None else contextlib.nullcontext():
        a = h.run_module(ours, sc, BG, dL, use_sh=False, pad_to=pad)
    st = _C.inspect_state(pad or P, W, H, a["num_rendered"], a["geom"], a["binning"], a["img"])
    st = {k: (v[:P] if k in h.PER_GAUSSIAN else v).cpu().numpy() for k, v in st.items()}
    return a, st, _raw(a, W, H)


def _live_of_full(st, raw, plain, footprint=None):
    """Check that every tile's live list is its full list without the mask-0 words, in order; return the live ids.
    footprint: the masks of the full list (the packed format's; the plain one carries none)."""
    T = len(raw["tile_cursor"])
    start, cursor, plist = raw["tile_start"].astype(np.int64), raw["tile_cursor"].astype(np.int64), raw["plist"]
    fp = st["footprint"] if footprint is None else footprint
    full_ids = st["point_list"].astype(np.int64)
    assert np.array_equal(start[:-1][start[1:] > start[:-1]], st["ranges"][:, 0][start[1:] > start[:-1]])
    assert int(start[-1]) == len(full_ids)
    live = []
    for t in range(T):
        keep = fp[start[t]:start[t + 1]] != 0
        want = full_ids[start[t]:start[t + 1]][keep]
        assert start[t] <= cursor[t] <= start[t + 1] and cursor[t] - start[t] == len(want), t
        words = plist[start[t]:cursor[t]].astype(np.int64)
        ids = words if plain else words >> 8
        assert np.array_equal(ids, want), f"tile {t}: live list is not the full list without its dead instances"
        if not plain:
            assert np.array_equal(words & 0xff, fp[start[t]:start[t + 1]][keep]), t
        live.append(ids)
    return live


@pytest.mark.gpu
@pytest.mark.parametrize("plain", [False, True], ids=["packed_ids", "plain_ids"])
def test_live_list_is_full_list_without_dead(plain):
    """Classes scene: the live lists, their class-edge counts, and the reference-form state against the oracle."""
    sc = _make("classes")
    W, H = sc.width, sc.height
    a, st, raw = _run(sc, False)
    _check_design("classes", st, W, H)
    live = _live_of_full(st, raw, False)
    assert [len(x) for x in live] == [n for n, _ in CLASS_TILES]
    if plain:
        import torch
        pa, pst, praw = _run(sc, True)
        torch.cuda.empty_cache()
        plive = _live_of_full(pst, praw, True, footprint=st["footprint"])
        assert all(np.array_equal(x, y) for x, y in zip(live, plive))
        for k in ("keys", "point_list", "ranges", "n_contrib", "final_T"):
            assert np.array_equal(pst[k], st[k]), k
        assert np.array_equal(praw["n_contrib"], raw["n_contrib"])
        assert torch.equal(pa["color"], a["color"])
        a, st = pa, pst
    fw, _ = h.run_oracle(sc, np.asarray(BG, np.float32), use_sh=False)
    assert np.array_equal(st["keys"].view(np.uint64), fw["keys"])
    assert np.array_equal(st["point_list"].astype(np.uint32), fw["point_list"])
    assert np.array_equal(st["ranges"].view(np.uint32), fw["ranges"])
    # glibc expf vs MUFU.EX2: as in test_gpu_parity, a pair sitting on a threshold may flip
    assert int((st["n_contrib"].view(np.uint32) != fw["n_contrib"]).sum()) <= max(2, W * H // 5000)
    for got, want in ((st["final_T"], fw["final_T"]), (a["color"].cpu().numpy(), fw["color"])):
        d = np.abs(got - want)
        assert np.quantile(d, 0.999) < 2e-6 and d.max() < 5e-3, (float(np.quantile(d, 0.999)), float(d.max()))


@pytest.mark.gpu
@pytest.mark.parametrize("plain", [False, True], ids=["packed_ids", "plain_ids"])
def test_n_contrib_behind_dead_instances(plain):
    """Behind_dead scene: the live n_contrib at the centre is 2, the reported one the reference's 4; the whole state
    and the gradients (the backward walks the live list up to the live n_contrib) match the oracle."""
    import torch
    from sugar_b200 import scenes
    sc = _make("behind_dead")
    W, H = sc.width, sc.height
    dL = scenes.upstream_grad(W, H)
    a, st, raw = _run(sc, plain, dL)
    fp = None
    if plain:
        fp = _run(sc, False)[1]["footprint"]
    _check_design("behind_dead", st, W, H)
    _live_of_full(st, raw, plain, footprint=fp)
    assert int(raw["n_contrib"][CENTRE, CENTRE]) == 2
    assert list(raw["plist"][:raw["tile_cursor"][0]] >> (0 if plain else 8)) == [0, 3]
    fw, bw = h.run_oracle(sc, np.asarray(BG, np.float32), dL, use_sh=False)
    nc = st["n_contrib"].view(np.uint32)
    assert int(nc[CENTRE, CENTRE]) == 4 and int((nc != fw["n_contrib"]).sum()) <= 2
    assert np.array_equal(st["keys"].view(np.uint64), fw["keys"])
    assert np.array_equal(st["point_list"].astype(np.uint32), fw["point_list"])
    for got, want in ((st["final_T"], fw["final_T"]), (a["color"].cpu().numpy(), fw["color"])):
        assert np.abs(got - want).max() < 2e-6
    for k, name_bw in GRAD_NAMES.items():
        want = bw[name_bw]
        got = a["grads"][k][:want.shape[0]].cpu().numpy()
        assert h.rel_err(got.reshape(want.shape), want) <= ORACLE_GRAD_RTOL, k
    if plain:
        torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("plain", [False, True], ids=["packed_ids", "plain_ids"])
def test_capacity_overflow_rerun_keeps_live_state(plain):
    """A capacity hint far below the instance count: the guarded attempt is a no-op and the re-run leaves the same
    live lists, live n_contrib, reference-form state, image and gradients as a run without a hint."""
    import torch
    from sugar_b200 import _C, scenes
    sc = _make("classes")
    W, H = sc.width, sc.height
    dL = scenes.upstream_grad(W, H)
    a, sa, ra = _run(sc, plain, dL, ctx=_C.Context())
    R = a["num_rendered"]
    tiny = _C.Context()
    tiny.capacity_hint[(torch.cuda.current_device(), H, W)] = 1 << 10
    assert R > (1 << 10)
    b, sb, rb = _run(sc, plain, dL, ctx=tiny)
    assert b["num_rendered"] == R
    for k in ("tile_start", "tile_cursor", "n_contrib", "plist"):
        assert np.array_equal(ra[k], rb[k]), k
    for k in ("keys", "point_list", "ranges", "n_contrib", "final_T", "footprint"):
        assert np.array_equal(sa[k], sb[k]), k
    assert torch.equal(a["color"], b["color"]) and torch.equal(a["radii"], b["radii"])
    for k in a["grads"]:
        assert h.rel_err(b["grads"][k].cpu().numpy(), a["grads"][k].cpu().numpy()) <= 1e-5, k
    if plain:
        torch.cuda.empty_cache()
