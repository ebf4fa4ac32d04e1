"""Tile binning and the per-tile sorts at their size-class, bucket, radix, scatter, scan and id-format edges.

The forward bins instances in four steps (sugar_b200/csrc/sgr_forward.cu): preprocess counts the tiles of each splat's
rect, tile_scan_kernel turns the counts into segments (in chunks of 4096 tiles), scatter_kernel writes one
(depth bits | id [| footprint mask]) word per instance into its tile's segment (a splat's own thread for rects of at
most SMALL tiles, the whole warp above), and one launch per size class sorts each tile: a merge sort up to 512
instances, a bucket sort with a merge fallback up to BK_CAP, a merge sort up to SORT_CAP, and an LSD radix sort through
global memory above.  Each scene below is built for a set of those edges, and asserts its own shape from the forward
state before anything is compared:

  * size_classes: one image whose tiles hold 0, 1, 7, 8, 9, 65, 511, 512, 513, 1024, 2047, 2048, 2049, 8191, 8192,
    8193 and 70 000 instances, each count with random, reversed and tied depths, and a tile above SORT_CAP whose
    depths differ only in their lowest byte (radix passes of both parities in both id formats);
  * bucket_edges: tiles of the bucket class whose fullest bucket holds exactly BUCKET_MAX and BUCKET_MAX + 1 words, and
    tiles whose depth-bit range is 0, 2^BK_LOG2NB - 1 and 2^BK_LOG2NB (the bucket shift changes between the two);
  * radix_many / merge_many: more than 2 * SMs tiles above SORT_CAP (whole-image splats of tied depth: only the id
    bytes vary, the mask byte is 0xff) and in the class below it, so every grid-stride CTA sorts several tiles;
  * scatter_paths: rects of exactly SMALL and SMALL + 1 tiles, rects of more than 32 tiles, warps in which several
    lanes have large rects, and thin rotated ellipses, with every footprint mask checked against a float64 per-pixel
    enumeration;
  * tile_scan_chunks: more than 4096 tiles with T % 4 == 1, sparse splats on both sides of the chunk boundary and on
    the last tile.

Depths never follow ids, so a sort that leaves a tile in scatter order fails.  Opacities are 0.01-0.05, so hundreds
of list positions reach the image and the gradients.  Every scene is compared with the CPU oracle in both instance-list
formats (keys, point_list and ranges bit-identical, n_contrib, final_T, image and every gradient at the oracle bars of
tests/test_gpu_parity.py; the plain-id run appends culled Gaussians up to P = 2^24, helpers.run_state), and its
lists are also checked without the oracle: (depth bits, id) strictly increasing in every tile and each tile's ids
exactly those the means and radii imply.  test_id_format_boundary runs P = 2^24 - 1
(packed ids, whose largest word 0xfffffeff sits one below the "no record" word) and P = 2^24 (plain ids, chosen by P)
against the same visible splats compacted into a five-Gaussian scene.  test_binning_scene_shapes_on_cpu_oracle builds
the scenes and asserts their designed shape on the CPU oracle alone."""
import math
import os
import re

import numpy as np
import pytest

import helpers as h

ORACLE_GRAD_RTOL = 5e-4   # test_gpu_parity.test_matches_cpu_oracle
GRAD_NAMES = dict(means3D="dL_dmeans3D", means2D="dL_dmeans2D", opacities="dL_dopacity",
                  colors_precomp="dL_dcolors", scales="dL_dscales", rotations="dL_drotations")
BG = (0.25, 0.5, 1.0)


def _constants():
    """The class bounds of the binning kernels, read from their source so that the scenes follow them."""
    with open(os.path.join(h.ROOT, "sugar_b200", "csrc", "sgr_forward.cu")) as f:
        src = f.read()
    one = lambda pat: int(re.search(pat, src).group(1))
    c = dict(SORT_CAP=one(r"constexpr int SORT_CAP = (\d+);"), BK_CAP=one(r"\bBK_CAP = (\d+)"),
             BUCKET_MAX=one(r"\bBUCKET_MAX = (\d+)"), BK_LOG2NB=one(r"\bBK_LOG2NB = (\d+)"),
             MERGE_SMALL=one(r"tile_sort_merge_kernel<(\d+), 0><<<"),
             SMALL=one(r"constexpr int SMALL = (\d+);"))
    assert one(r"tile_sort_bucket_kernel<<<[^;]*, (\d+)\);") == c["MERGE_SMALL"]   # the bucket class starts above it
    assert re.search(r"tile_sort_merge_kernel<%d, %d><<<" % (c["SORT_CAP"], c["BK_CAP"]), src)
    assert len(set(re.findall(r"constexpr int SMALL = (\d+);", src))) == 1           # preprocess and scatter agree
    return c


K = _constants()


# ------------------------------------------------------------------------------------------------------------------
# scene construction: splats placed in pixels, identity camera (depth == z bit for bit)
# ------------------------------------------------------------------------------------------------------------------
def _f32bits(bits):
    return np.asarray(bits, np.uint32).view(np.float32)


def _scene(W, H, d, seed):
    """d: arrays u, v (pixel of the mean), z, sx, sy (pixel sigmas), th (rotation in the image plane), op."""
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
    m[:, 2] = z                                         # depth bits exactly as designed
    s = np.stack([d["sx"] * zz / focal, d["sy"] * zz / focal, np.full(P, 1e-4)], 1).astype(np.float32)
    th = np.asarray(d["th"], np.float64)
    q = np.stack([np.cos(th / 2), np.zeros(P), np.zeros(P), np.sin(th / 2)], 1).astype(np.float32)
    o = np.asarray(d["op"], np.float32).reshape(P, 1)
    col = rng.uniform(0, 1, (P, 3)).astype(np.float32)
    return base._replace(means3D=m, scales=s, rotations=q, opacities=o, colors_precomp=col,
                         shs=np.zeros((1, 16, 3), np.float32))


def _cat(parts):
    return {k: np.concatenate([p[k] for p in parts]) for k in parts[0]}


def _in_tile(rng, tx, ty, n):
    """n small splats centred inside tile (tx, ty): radius <= 5 px around a centre 5.5-10.5 px into the tile, so each
    touches exactly that tile."""
    return dict(u=16 * tx + rng.uniform(5.5, 10.5, n), v=16 * ty + rng.uniform(5.5, 10.5, n), z=np.zeros(n, np.float32),
                sx=rng.uniform(0.5, 1.2, n), sy=rng.uniform(0.5, 1.2, n), th=rng.uniform(0, np.pi, n),
                op=rng.uniform(0.01, 0.05, n))


def _whole_image(rng, W, H, n):
    """n splats that reach every pixel of a W x H image with alpha >= 1/255: footprint mask 0xff in every tile."""
    return dict(u=W / 2 + rng.uniform(-10, 10, n), v=H / 2 + rng.uniform(-10, 10, n), z=np.zeros(n, np.float32),
                sx=rng.uniform(380, 420, n), sy=rng.uniform(380, 420, n), th=rng.uniform(0, np.pi, n),
                op=rng.uniform(0.01, 0.03, n))


def _depths(rng, mode, n):
    """Depths of a group's splats in increasing id order."""
    if isinstance(mode, np.ndarray):                     # explicit depth-bit offsets above 4.0
        return _f32bits(0x40800000 + rng.permutation(mode))
    if mode == "random":
        return rng.uniform(2.0, 10.0, n).astype(np.float32)
    if mode == "reversed":                               # strictly decreasing in id
        return np.linspace(9.0, 3.0, n, dtype=np.float32)
    if mode == "tied":
        return np.full(n, 4.0, np.float32)
    if mode == "lowbyte":                                # only the lowest byte of the depth bits varies
        return _f32bits(0x40a00000 + rng.integers(0, 256, n))
    raise ValueError(mode)


def _assemble(W, H, groups, seed):
    """groups: list of (splats dict, depth mode).  The splats get shuffled ids; each group's depths are then assigned
    in its id order, so "reversed" means reversed against the ids."""
    rng = np.random.Generator(np.random.PCG64(seed))
    d = _cat([g for g, _ in groups])
    gid = np.concatenate([np.full(len(g["u"]), i) for i, (g, _) in enumerate(groups)])
    perm = rng.permutation(len(gid))
    d = {k: v[perm] for k, v in d.items()}
    gid = gid[perm]
    z = np.zeros(len(gid), np.float32)
    for i, (_, mode) in enumerate(groups):
        ids = np.flatnonzero(gid == i)
        z[ids] = _depths(rng, mode, len(ids))
    d["z"] = z
    return _scene(W, H, d, seed), gid


def _size_classes():
    M, BK, SC = K["MERGE_SMALL"], K["BK_CAP"], K["SORT_CAP"]
    counts = [0, 1, 7, 8, 9, 65, M - 1, M, M + 1, 1024, BK - 1, BK, BK + 1, SC - 1, SC, SC + 1]
    rng = np.random.Generator(np.random.PCG64(1))
    gx, gy = 13, 4
    groups, tiles = [], {}
    t = 0
    for n in counts:
        for mode in ("random", "reversed", "tied"):
            tiles[(n, mode)] = t
            groups.append((_in_tile(rng, t % gx, t // gx, n), mode))
            t += 1
    tiles[(70_000, "random")] = t
    groups.append((_in_tile(rng, t % gx, t // gx, 70_000), "random"))
    tiles[(SC + 808, "lowbyte")] = t + 1
    groups.append((_in_tile(rng, (t + 1) % gx, (t + 1) // gx, SC + 808), "lowbyte"))
    sc, _ = _assemble(16 * gx, 16 * gy, groups, seed=11)
    return sc, dict(tiles=tiles)


def _bucket_edges():
    """Depth-bit offsets (above the bits of 4.0) of the bucket class's edge tiles."""
    rng = np.random.Generator(np.random.PCG64(2))
    NB, BM = 1 << K["BK_LOG2NB"], K["BUCKET_MAX"]

    def fullest(n, cnt):                                   # range NB - 1 (shift 0): one offset holds cnt words
        others = rng.choice(np.delete(np.arange(1, NB - 1), NB // 2 - 1), n - cnt - 2, replace=False)
        return np.concatenate([[0, NB - 1], np.full(cnt, NB // 2), others])

    def fullest_shifted(n, cnt):                           # range 2^20 - 1 (shift 20 - log2 NB): bucket 5 holds cnt
        sh = 20 - K["BK_LOG2NB"]
        per = np.concatenate([np.full(cnt, 5), np.resize(np.delete(np.arange(NB), 5), n - cnt)])
        off = (per << sh) + rng.integers(0, 1 << sh, n)
        off[-2], off[-1] = 0, (1 << 20) - 1                 # into bucket 0 and the last bucket
        return off
    M = K["MERGE_SMALL"]
    offs = {"fullest_max": fullest(1000, BM), "fullest_over": fullest(1000, BM + 1),
            "fullest_max_shifted": fullest_shifted(K["BK_CAP"], BM),
            "range_0": np.zeros(M + 88, np.int64), "range_nb_minus_1": np.arange(NB), "range_nb": np.arange(NB + 1)}
    groups, tiles = [], {}
    for t, (name, off) in enumerate(offs.items()):
        tiles[name] = t
        groups.append((_in_tile(rng, t % 3, t // 3, len(off)), np.asarray(off, np.int64)))
    sc, _ = _assemble(48, 32, groups, seed=12)
    return sc, dict(tiles=tiles)


def _radix_many():
    W, H = 320, 240                                      # 300 tiles
    rng = np.random.Generator(np.random.PCG64(3))
    sc, _ = _assemble(W, H, [(_whole_image(rng, W, H, K["SORT_CAP"] + 108), "tied")], seed=13)
    return sc, {}


def _merge_many():
    W, H = 320, 240
    rng = np.random.Generator(np.random.PCG64(4))
    sc, _ = _assemble(W, H, [(_whole_image(rng, W, H, (K["BK_CAP"] + K["SORT_CAP"]) // 2), "random")], seed=14)
    return sc, {}


def _scatter_paths():
    """Splats of every size on a 32 x 4 tile image, a third of them thin and rotated, a fifth centred above or below
    the image (their rects are clipped to one or two tile rows: rects of 6 and 7 tiles in one row)."""
    W, H = 512, 64
    rng = np.random.Generator(np.random.PCG64(5))
    n = 1024
    sx = np.exp(rng.uniform(math.log(0.7), math.log(60.0), n))
    thin = rng.uniform(0, 1, n) < 0.35
    sy = np.where(thin, sx / rng.uniform(8, 30, n), sx * rng.uniform(0.5, 1.0, n))
    u = rng.uniform(-30, W + 30, n)
    v = rng.uniform(-10, H + 10, n)
    off = rng.uniform(0, 1, n) < 0.2
    v[off] = np.where(rng.uniform(0, 1, off.sum()) < 0.5, rng.uniform(-60, -4, off.sum()), rng.uniform(H + 4, H + 60, off.sum()))
    sx[off] = rng.uniform(8, 30, off.sum())
    sy[off] = sx[off]
    d = dict(u=u, v=v, z=np.zeros(n, np.float32), sx=sx, sy=sy, th=rng.uniform(0, np.pi, n),
             op=rng.uniform(0.02, 0.9, n))
    sc, _ = _assemble(W, H, [(d, "random")], seed=15)
    return sc, {}


def _tile_scan_chunks():
    W, H = 1067, 1007                                    # 67 x 63 = 4221 tiles: T > 4096, T % 4 == 1
    gx, gy = (W + 15) // 16, (H + 15) // 16
    T = gx * gy
    rng = np.random.Generator(np.random.PCG64(6))
    want = {0: 2, 4093: 3, 4094: 5, 4095: 7, 4096: 4, 4097: 6, 4098: 1, T - 2: 2, T - 1: 9}
    for t in rng.choice(np.arange(1, T - 2), 20, replace=False):
        want.setdefault(int(t), int(rng.integers(1, 6)))
    groups = [(_in_tile(rng, t % gx, t // gx, n), "random") for t, n in want.items()]
    # three splats of two tiles each, across the boundary between tiles 4095 and 4096 (horizontal neighbours)
    ty, tx = divmod(4096, gx)
    two = dict(u=16.0 * tx + rng.uniform(-0.5, 0.5, 3), v=16 * ty + rng.uniform(6, 10, 3), z=np.zeros(3, np.float32),
               sx=np.full(3, 0.8), sy=np.full(3, 0.8), th=np.zeros(3), op=np.full(3, 0.05))
    groups.append((two, "random"))
    want[4095] += 3
    want[4096] += 3
    if T - 1 in want:                                   # the last tile is a partial one on both axes
        assert W % 16 and H % 16
    sc, _ = _assemble(W, H, groups, seed=16)
    return sc, dict(counts=want)


BUILDERS = dict(size_classes=_size_classes, bucket_edges=_bucket_edges, radix_many=_radix_many,
                merge_many=_merge_many, scatter_paths=_scatter_paths, tile_scan_chunks=_tile_scan_chunks)
_SCENES = {}


def _make(name):
    if name not in _SCENES:
        _SCENES[name] = BUILDERS[name]()
    return _SCENES[name]


# ------------------------------------------------------------------------------------------------------------------
# checks shared by the CPU oracle and the GPU forward state
# ------------------------------------------------------------------------------------------------------------------
def _rects(means2D, radii, W, H):
    """tile_rect (sgr_internal.cuh / getRect) in fp32, as the kernels round it."""
    gx, gy = (W + 15) // 16, (H + 15) // 16
    px, py = means2D[:, 0].astype(np.float32), means2D[:, 1].astype(np.float32)
    r = radii.astype(np.float32)
    q = np.float32(0.0625)
    cut = lambda x, g: np.clip(np.trunc(x).astype(np.int64), 0, g)
    x0, y0 = cut((px - r) * q, gx), cut((py - r) * q, gy)
    x1 = cut((((px + r) + np.float32(16)) + np.float32(-1)) * q, gx)
    y1 = cut((((py + r) + np.float32(16)) + np.float32(-1)) * q, gy)
    vis = radii > 0
    return np.where(vis, x0, 0), np.where(vis, y0, 0), np.where(vis, x1, 0), np.where(vis, y1, 0)


def _tile_of_position(ranges):
    n = ranges[:, 1].astype(np.int64) - ranges[:, 0]
    return np.repeat(np.arange(len(n)), n), n


def _check_lists(o, W, H):
    """Without the oracle: each tile's list is strictly increasing in (depth bits, id), and holds exactly the ids whose
    rect (from the means and radii) covers the tile."""
    plist = o["point_list"].astype(np.int64)
    tile, n = _tile_of_position(o["ranges"])
    assert len(tile) == len(plist) and np.array_equal(np.cumsum(n)[n > 0] - n[n > 0], o["ranges"][n > 0, 0])
    word = (o["depths"].view(np.uint32)[plist].astype(np.uint64) << np.uint64(32)) | plist.astype(np.uint64)
    same = tile[1:] == tile[:-1]
    bad = np.flatnonzero(same & (word[1:] <= word[:-1]))
    assert bad.size == 0, f"tile {tile[bad[0]]} not in (depth bits, id) order at list position {bad[0]}"
    x0, y0, x1, y1 = _rects(o["means2D"], o["radii"], W, H)
    gx = (W + 15) // 16
    cnt = (x1 - x0) * (y1 - y0)
    ids = np.repeat(np.arange(len(cnt)), cnt)
    k = np.arange(len(ids)) - np.repeat(np.cumsum(cnt) - cnt, cnt)
    w = np.repeat(x1 - x0, cnt)
    want_tile = (np.repeat(y0, cnt) + k // np.maximum(w, 1)) * gx + np.repeat(x0, cnt) + k % np.maximum(w, 1)
    want = np.lexsort((ids, want_tile))
    got = np.lexsort((plist, tile))
    assert np.array_equal(want_tile[want], tile[got]) and np.array_equal(ids[want], plist[got]), \
        "a tile's ids are not those its splats' rects imply"


def _words(o, packed):
    """The sort words of the list, (depth bits << 32) | id [<< 8 | footprint mask], in list order."""
    plist = o["point_list"].astype(np.uint64)
    low = (plist << np.uint64(8)) | o["footprint"].astype(np.uint64) if packed else plist
    return (o["depths"].view(np.uint32)[o["point_list"]].astype(np.uint64) << np.uint64(32)) | low


def _varying_bytes(words):
    x = int(np.bitwise_or.reduce(words ^ words[0]))
    return sum(((x >> (8 * b)) & 0xff) != 0 for b in range(8))


def _tile_slice(o, t):
    lo, hi = (int(x) for x in o["ranges"][t])
    return slice(lo, hi)


def _bucket_stats(depth_bits):
    """(shift, fullest bucket, range) of tile_sort_bucket_kernel for one tile's depth bits."""
    d = depth_bits.astype(np.int64)
    rng_ = int(d.max() - d.min())
    sh = max(0, rng_.bit_length() - K["BK_LOG2NB"])
    return sh, int(np.bincount((d - d.min()) >> sh).max()), rng_


def _check_shape(name, o, W, H, formats):
    """The forward state `o` (oracle or GPU) has the shape scene `name` is built for.  `formats`: the id formats whose
    words can be rebuilt from `o` (the packed one needs the footprint masks of a packed GPU run)."""
    _, meta = _make(name)
    tile, n = _tile_of_position(o["ranges"])
    T = len(n)
    dbits = o["depths"].view(np.uint32)
    SC, BK = K["SORT_CAP"], K["BK_CAP"]
    if name == "size_classes":
        for (cnt, mode), t in meta["tiles"].items():
            assert int(n[t]) == cnt, (cnt, mode, int(n[t]))
            ids = o["point_list"][_tile_slice(o, t)].astype(np.int64)
            zs = dbits[np.sort(ids)].astype(np.int64)
            if cnt > 1 and mode == "tied":
                assert np.all(zs == zs[0])
            elif cnt > 1 and mode == "reversed":
                assert np.all(np.diff(zs) < 0)
            elif cnt > 1 and mode == "random":      # the sorted list is far from id order
                assert not np.array_equal(np.sort(ids), ids)
        big = np.flatnonzero(n > SC)
        assert len(big) == 5
        lowbyte = meta["tiles"][(SC + 808, "lowbyte")]
        assert _varying_bytes(dbits[o["point_list"][_tile_slice(o, lowbyte)]].astype(np.uint64)) == 1
        for packed in formats:
            w = _words(o, packed)
            par = {_varying_bytes(w[_tile_slice(o, t)]) % 2 for t in big}
            assert par == {0, 1}, (packed, [_varying_bytes(w[_tile_slice(o, t)]) for t in big])
    elif name == "bucket_edges":
        NB, BM = 1 << K["BK_LOG2NB"], K["BUCKET_MAX"]
        want = {"fullest_max": (BM, None), "fullest_over": (BM + 1, None), "fullest_max_shifted": (BM, None),
                "range_0": (None, 0), "range_nb_minus_1": (1, NB - 1), "range_nb": (2, NB)}
        for nm, t in meta["tiles"].items():
            assert K["MERGE_SMALL"] < int(n[t]) <= BK, (nm, int(n[t]))
            sh, full, rng_ = _bucket_stats(dbits[o["point_list"][_tile_slice(o, t)]])
            wf, wr = want[nm]
            if wf is not None:
                assert full == wf, (nm, full)
            if wr is not None:
                assert rng_ == wr, (nm, rng_)
            if nm == "fullest_max_shifted":
                assert sh > 0, sh
        assert _bucket_stats(dbits[o["point_list"][_tile_slice(o, meta["tiles"]["range_nb"])]])[0] == 1
        assert _bucket_stats(dbits[o["point_list"][_tile_slice(o, meta["tiles"]["range_nb_minus_1"])]])[0] == 0
    elif name in ("radix_many", "merge_many"):
        lo_, hi_ = (SC, np.inf) if name == "radix_many" else (BK, SC)
        assert np.all((n > lo_) & (n <= hi_)) and T >= 300, (n.min(), n.max(), T)
        if name == "radix_many":
            assert np.all(dbits[o["point_list"]] == dbits[o["point_list"][0]])     # tied depths
            for packed in formats:
                w = _words(o, packed)
                if packed:
                    assert np.all(o["footprint"] == 0xff)
                for t in range(T):
                    assert _varying_bytes(w[_tile_slice(o, t)]) == 2       # the two id bytes of ids < 2^16
    elif name == "scatter_paths":
        x0, y0, x1, y1 = _rects(o["means2D"], o["radii"], W, H)
        cnt = (x1 - x0) * (y1 - y0)
        small = K["SMALL"]
        assert (cnt == small).sum() >= 3 and (cnt == small + 1).sum() >= 3 and (cnt > 32).sum() >= 20, \
            np.bincount(cnt)[:12]
        lanes = (cnt.reshape(-1, 32) > small).sum(1)   # a warp of scatter_kernel = 32 consecutive ids
        assert (lanes >= 3).sum() >= 5, lanes
        co = o["conic_opacity"].astype(np.float64)
        ev = np.linalg.eigvalsh(np.stack([np.stack([co[:, 0], co[:, 1]], 1), np.stack([co[:, 1], co[:, 2]], 1)], 1))
        slanted = (np.abs(co[:, 1]) > 0.2 * np.sqrt(co[:, 0] * co[:, 2])) & (ev[:, 1] > 25 * ev[:, 0]) & (cnt > 0)
        assert slanted.sum() >= 20, slanted.sum()   # thin ellipses off the axes
    elif name == "tile_scan_chunks":
        assert T > 4096 and T % 4 == 1
        assert {t: int(n[t]) for t in np.flatnonzero(n)} == meta["counts"]


# ------------------------------------------------------------------------------------------------------------------
# CPU: the scenes have their designed shape
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(BUILDERS))
def test_binning_scene_shapes_on_cpu_oracle(name):
    sc, _ = _make(name)
    fw, _ = h.run_oracle(sc, np.asarray(BG, np.float32), use_sh=False)
    o = dict(fw, point_list=fw["point_list"].astype(np.int64))
    _check_shape(name, o, sc.width, sc.height, formats=(False,))
    _check_lists(o, sc.width, sc.height)


# ------------------------------------------------------------------------------------------------------------------
# GPU: both id formats against the oracle
# ------------------------------------------------------------------------------------------------------------------
_ORACLE = {}


def _oracle(name):
    if name not in _ORACLE:
        from sugar_b200 import scenes
        sc, _ = _make(name)
        _ORACLE.clear()                                  # one scene's oracle state at a time
        _ORACLE[name] = h.run_oracle(sc, np.asarray(BG, np.float32), scenes.upstream_grad(sc.width, sc.height),
                                     use_sh=False)
    return _ORACLE[name]


def _check_masks(o, W, H):
    """Every footprint mask is conservative against a float64 per-pixel enumeration (no cleared block holds a pixel
    whose power reaches ln(1/(255 o)) with a margin for fp32 rounding), and not much looser than the truth, separately
    for the instances of the per-thread and the warp-shared scatter path."""
    import torch
    gx = (W + 15) // 16
    tile, _ = _tile_of_position(o["ranges"])
    ids = o["point_list"].astype(np.int64)
    x0, y0, x1, y1 = _rects(o["means2D"], o["radii"], W, H)
    warp_path = ((x1 - x0) * (y1 - y0) > K["SMALL"])[ids]
    dev = "cuda"
    t = torch.from_numpy(tile).to(dev)
    m2 = torch.from_numpy(o["means2D"].astype(np.float64)).to(dev)[torch.from_numpy(ids).to(dev)]
    co = torch.from_numpy(o["conic_opacity"].astype(np.float64)).to(dev)[torch.from_numpy(ids).to(dev)]
    fp = torch.from_numpy(o["footprint"].astype(np.int64)).to(dev)
    ar = torch.arange(16, device=dev, dtype=torch.float64)
    px = ((t % gx) * 16).double()[:, None, None] + ar[None, None, :]
    py = ((t // gx) * 16).double()[:, None, None] + ar[None, :, None]
    dx, dy = m2[:, 0, None, None] - px, m2[:, 1, None, None] - py
    power = -0.5 * (co[:, 0, None, None] * dx * dx + co[:, 2, None, None] * dy * dy) - co[:, 1, None, None] * dx * dy
    thr = -torch.log(255.0 * co[:, 3])[:, None, None]
    reach = (power >= thr + 1e-5 * (1.0 + thr.abs())) & (power <= 0)
    alpha = torch.clamp(co[:, 3, None, None] * torch.exp(power), max=0.99)
    truth_px = (power <= 0) & (alpha >= 1.0 / 255.0)
    bit = (1 << (torch.arange(4, device=dev)[:, None] * 2 + torch.arange(2, device=dev)[None, :]))
    blocks = lambda m: (m.view(-1, 4, 4, 2, 8).any(dim=4).any(dim=2).long() * bit).sum((1, 2))
    missed = blocks(reach) & ~fp
    assert int((missed != 0).sum()) == 0, "a footprint mask clears a block that holds a reachable pixel"
    truth = blocks(truth_px)
    pop = lambda v: sum(((v >> b) & 1) for b in range(8)).sum().item()
    wp = torch.from_numpy(warp_path).to(dev)
    for path in (False, True):
        sel = wp == path
        assert sel.sum().item() > 100, path
        assert pop(fp[sel]) <= 1.25 * pop(truth[sel]) + 64, (path, pop(fp[sel]), pop(truth[sel]))


@pytest.mark.gpu
@pytest.mark.parametrize("unpacked", [False, True], ids=["packed_ids", "unpacked_ids"])
@pytest.mark.parametrize("name", list(BUILDERS))
def test_binning_edges_match_cpu_oracle(name, unpacked):
    import torch
    from sugar_b200 import scenes
    sc, _ = _make(name)
    W, H = sc.width, sc.height
    o = h.run_state(sc, BG, scenes.upstream_grad(W, H), plain_ids=unpacked, use_sh=False)
    o = dict(o, point_list=o["point_list"].astype(np.int64))
    _check_shape(name, o, W, H, formats=(False,) if unpacked else (False, True))
    if name in ("radix_many", "merge_many"):
        n = o["ranges"][:, 1].astype(np.int64) - o["ranges"][:, 0]
        assert len(n) > 2 * torch.cuda.get_device_properties(0).multi_processor_count   # several tiles per CTA
    if name == "scatter_paths" and not unpacked:
        _check_masks(o, W, H)
    _check_lists(o, W, H)
    fw, bw = _oracle(name)
    assert np.array_equal(o["radii"], fw["radii"])
    assert np.array_equal(o["keys"].view(np.uint64), fw["keys"])
    assert np.array_equal(o["point_list"].astype(np.uint32), fw["point_list"])
    assert np.array_equal(o["ranges"].view(np.uint32), fw["ranges"])
    # glibc expf vs MUFU.EX2: as in test_gpu_parity, a pair sitting on a threshold may flip
    nc = o["n_contrib"].view(np.uint32)
    assert int((nc != fw["n_contrib"]).sum()) <= max(2, W * H // 5000)
    for got, want in ((o["final_T"], fw["final_T"]), (o["color"], fw["color"]), (o["color_bw"], fw["color"])):
        d = np.abs(got - want)
        assert np.quantile(d, 0.999) < 2e-6 and d.max() < 5e-3, (float(np.quantile(d, 0.999)), float(d.max()))
    assert np.abs(bw["dL_dopacity"]).max() > 0
    for k, name_bw in GRAD_NAMES.items():
        want = bw[name_bw]
        err = h.rel_err(o["grad_" + k].reshape(want.shape), want)
        assert err <= ORACLE_GRAD_RTOL, f"grad {k}: rel err vs oracle {err:.3e}"


# ------------------------------------------------------------------------------------------------------------------
# GPU: the id-format boundary at P = 2^24
# ------------------------------------------------------------------------------------------------------------------
def _boundary_scene(P):
    """P Gaussians, all behind the near plane except five at ids 0, 1, 2^23, P - 2 and P - 1 on a 64 x 48 image; ids 0
    and P - 1 reach every pixel (footprint mask 0xff)."""
    W, H = 64, 48
    vis = np.array([0, 1, 1 << 23, P - 2, P - 1], np.int64)
    d = dict(u=np.array([30.0, 12.0, 40.5, 52.0, 33.0]), v=np.array([20.0, 10.0, 30.0, 8.5, 25.0]),
             z=np.array([6.0, 3.0, 4.0, 3.0, 2.5], np.float32), sx=np.array([300.0, 2.0, 6.0, 1.5, 250.0]),
             sy=np.array([280.0, 0.5, 3.0, 4.0, 260.0]), th=np.array([0.3, 0.7, 2.0, 1.1, 0.0]),
             op=np.array([0.05, 0.6, 0.3, 0.9, 0.04]))
    small = _scene(W, H, d, seed=24)
    big = lambda a, fill: np.broadcast_to(np.asarray(fill, a.dtype), (P,) + a.shape[1:]).copy()
    means = big(small.means3D, [0.0, 0.0, -1.0])
    scales = big(small.scales, [0.01, 0.01, 0.01])
    rots = big(small.rotations, [1.0, 0.0, 0.0, 0.0])
    opac = big(small.opacities, [0.5])
    cols = big(small.colors_precomp, [0.5, 0.5, 0.5])
    for a, s in ((means, small.means3D), (scales, small.scales), (rots, small.rotations), (opac, small.opacities),
                 (cols, small.colors_precomp)):
        a[vis] = s
    return small._replace(means3D=means, scales=scales, rotations=rots, opacities=opac, colors_precomp=cols), small, vis


@pytest.mark.gpu
@pytest.mark.parametrize("P", [h.PACKED_MAX_P - 1, h.PACKED_MAX_P], ids=["packed_2^24-1", "plain_2^24"])
def test_id_format_boundary(P):
    """P = 2^24 - 1 keeps packed ids (the last id with a full mask is the word 0xfffffeff, one below the "no record"
    word); P = 2^24 switches to plain ids by P alone.  Both must give what the five visible splats give alone."""
    import torch
    from sugar_b200 import scenes
    big, small, vis = _boundary_scene(P)
    W, H = small.width, small.height
    dL = scenes.upstream_grad(W, H)
    want = h.run_state(small, BG, dL, use_sh=False)
    got = h.run_state(big, BG, dL, use_sh=False)
    torch.cuda.empty_cache()
    others = np.ones(P, bool)
    others[vis] = False
    assert np.array_equal(got["radii"][vis], want["radii"]) and not got["radii"][others].any()
    assert np.all(want["radii"] > 0)
    for k in ("color", "final_T", "n_contrib"):
        assert np.array_equal(got[k].view(np.uint32), want[k].view(np.uint32)), k
    assert np.array_equal(got["ranges"], want["ranges"])
    assert np.array_equal(got["point_list"].astype(np.int64), vis[want["point_list"].astype(np.int64)])
    last = got["point_list"].astype(np.int64) == P - 1
    assert last.sum() == (W // 16) * (H // 16)
    if P < h.PACKED_MAX_P:                               # the largest packed word, id 2^24 - 2 with mask 0xff
        assert np.all(got["footprint"][last] == 0xff)
        assert ((P - 1) << 8 | 0xff) == 0xfffffeff
    for k in GRAD_NAMES:
        g, w = got["grad_" + k].reshape(P, -1), want["grad_" + k].reshape(len(vis), -1)
        assert h.rel_err(g[vis], w) <= 1e-4, k
        assert not g[others].any(), k
