"""GPU: the grid K-NN (sugar_b200/knn.py, csrc/sgr_knn.cu) row for row against a float32 brute force
(oracle/knn_oracle.py) that rounds each distance as the kernel does and orders equal distances by index, so indices and
distances must be equal, not close.  A float64 check keeps the brute force honest.  Cases: random, surface-like,
degenerate and duplicated clouds, K at its edges, floaters beyond the grid's 4-sigma clip, a cloud far from the origin,
points rounded into the neighbouring cell at cell faces, and a grid larger than the cell scan's first chunk."""
import math

import numpy as np
import pytest
import torch

from oracle import knn_oracle as ko

pytestmark = pytest.mark.gpu


def _check(points, queries, K, rows=None, got=None):
    """knn_points(queries, points, K) (or `got`, its (d2, idx)) equals the brute force on `rows` (default: all)."""
    from sugar_b200 import knn
    p, q = points.float().cuda(), queries.float().cuda()
    d2, idx = got if got is not None else knn.knn_points(q, p, K)
    assert d2.shape == idx.shape == (q.shape[0], K)
    if rows is not None:
        rows = torch.as_tensor(rows, device="cuda").unique()
        q, d2, idx = q[rows], d2[rows], idx[rows]
    want_d2, want_idx = ko.knn_f32(q, p, K)
    bad = ((idx != want_idx) | (d2.view(torch.int32) != want_d2.view(torch.int32))).any(1).nonzero()[:, 0]
    if bad.numel():
        r = int(bad[0])
        pytest.fail(f"{bad.numel()} of {q.shape[0]} rows differ; row {r}: idx {idx[r].tolist()} d2 {d2[r].tolist()}, "
                    f"brute force idx {want_idx[r].tolist()} d2 {want_d2[r].tolist()}")
    # the float32 distance is within a few roundings of the float64 squared distance of the returned index
    exact = ((p.double()[idx] - q.double()[:, None]) ** 2).sum(-1)
    assert bool(((d2.double() - exact).abs() <= 2.0 ** -21 * exact + 1e-37).all())
    return d2, idx


def _dup_groups(pts):
    """per point, the smallest index among its exact copies."""
    uniq, inv = torch.unique(pts, dim=0, return_inverse=True)
    first = torch.full((uniq.shape[0],), pts.shape[0], dtype=torch.int64, device=pts.device)
    first.scatter_reduce_(0, inv, torch.arange(pts.shape[0], device=pts.device), "amin")
    return first[inv]


@pytest.mark.parametrize("P,Q,K", [(5000, 0, 16), (20000, 3000, 16), (777, 500, 5), (3000, 1000, 64), (40, 30, 16)])
def test_knn_matches_exact(P, Q, K):
    g = torch.Generator().manual_seed(P)
    pts = torch.randn(P, 3, generator=g)
    if Q == 0:   # reset_neighbors: cloud against itself, self must be neighbour 0 at distance 0
        from sugar_b200 import knn
        d2, idx = knn.reset_neighbors(pts.cuda(), K)
        assert bool((idx[:, 0].cpu() == torch.arange(P)).all()) and float(d2[:, 0].abs().max()) == 0.0
        _check(pts, pts, K, got=(d2, idx))
    else:
        qs = torch.randn(Q, 3, generator=g) * 1.5   # some queries outside the cloud's bounding box
        _check(pts, qs, K)


def test_knn_surface_like_and_degenerate_clouds():
    g = torch.Generator().manual_seed(3)
    # points on a thin sheet (most grid cells empty), plus a flat (zero-extent axis) cloud
    sheet = torch.randn(15000, 3, generator=g) * torch.tensor([1.0, 1.0, 1e-3])
    _check(sheet, sheet[:2000] + 0.01 * torch.randn(2000, 3, generator=g), 16)
    flat = torch.randn(4000, 3, generator=g); flat[:, 2] = 0.5
    _check(flat, flat[:1000], 8)
    # heavy duplicates
    dup = torch.randn(50, 3, generator=g).repeat(40, 1)
    _check(dup, dup[:300], 16)


def test_knn_planar_and_elongated_clouds_stay_fast():
    """Cubic cells with per-axis counts: a coplanar cloud (what SuGaR's surface-aligned Gaussians look like) or a
    cloud stretched along one axis by an outlier must not degrade to a linear scan per query (the shell bound was
    r * the smallest cell edge, i.e. ~0 on a degenerate axis)."""
    import time
    from sugar_b200 import knn
    g = torch.Generator().manual_seed(9)
    P = 400_000
    planar = torch.rand(P, 3, generator=g); planar[:, 2] = 0.25
    line = torch.rand(P, 3, generator=g) * torch.tensor([1.0, 1e-4, 1e-4])
    outlier = torch.randn(P, 3, generator=g); outlier[0] = torch.tensor([1e4, 0.0, 0.0])
    for name, pts in (("planar", planar), ("line", line), ("outlier", outlier)):
        pts = pts.cuda()
        knn.reset_neighbors(pts[:1000], 4)      # warm-up (context, allocator)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        d2, idx = knn.reset_neighbors(pts, 16)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        assert dt < 2.0, f"{name}: reset_neighbors took {dt:.2f} s for {P} points"
        assert bool((idx[:, 0] == torch.arange(P, device="cuda")).all()) or float(d2[:, 0].max()) == 0.0
        rows = torch.randperm(P, generator=g)[:2000].cuda()
        if name == "outlier":   # every row with the outlier in it
            rows = torch.cat([rows, (idx == 0).any(1).nonzero()[:, 0]])
        _check(pts, pts, 16, rows=rows, got=(d2, idx))


@pytest.mark.parametrize("K", [1, 2, 63, 64])
def test_knn_k_edges(K):
    g = torch.Generator().manual_seed(11 + K)
    pts = torch.randn(3000, 3, generator=g)
    _check(pts, torch.randn(700, 3, generator=g) * 1.5, K)
    from sugar_b200 import knn
    _check(pts, pts, K, got=knn.reset_neighbors(pts.cuda(), K))


@pytest.mark.parametrize("P", [1, 2, 7, 64])
def test_knn_k_equals_p(P):
    """K = P: every point in every row, a grid of one or two cells per axis."""
    g = torch.Generator().manual_seed(30 + P)
    pts = torch.randn(P, 3, generator=g)
    d2, idx = _check(pts, torch.randn(50, 3, generator=g) * 2.0, P)
    assert bool((idx.sort(1).values == torch.arange(P, device="cuda")).all())
    _check(pts, pts, P)


def _floater_cloud(seed, P=50_000, frac=0.01):
    """a Gaussian bulk plus `frac` floaters 6 sigma to 1e4 sigma out, on both sides of every axis (the grid clips its
    box to mean +- 4 sigma and clamps them into the border cells)."""
    g = torch.Generator().manual_seed(seed)
    pts = torch.randn(P, 3, generator=g)
    F = int(P * frac)
    ax = torch.arange(F) % 3
    sign = torch.where((torch.arange(F) // 3) % 2 == 0, 1.0, -1.0)
    mag = 6.0 * torch.exp(torch.rand(F, generator=g) * math.log(1e4 / 6.0))
    fl = torch.randn(F, 3, generator=g) * 2.0
    fl[torch.arange(F), ax] = sign * mag
    pts[:F] = fl
    return pts[torch.randperm(P, generator=g)].contiguous(), F


def test_knn_floaters_beyond_the_clip():
    pts, F = _floater_cloud(21)
    g = torch.Generator().manual_seed(22)
    floaters = pts[(pts.abs() > 5.5).any(1)]
    assert floaters.shape[0] >= F // 2
    between = torch.randn(600, 3, generator=g)
    between = between / between.norm(dim=1, keepdim=True) * (4.5 + 20 * torch.rand(600, 1, generator=g))
    qs = torch.cat([floaters, pts[torch.randperm(pts.shape[0], generator=g)[:1500]], between])
    d2, idx = _check(pts, qs, 16)
    # a floater's 16 mix floaters and bulk points somewhere
    far = (pts.cuda()[idx].abs() > 5.5).any(-1)
    assert bool((far[: floaters.shape[0]].any(1) & ~far[: floaters.shape[0]].all(1)).any())
    from sugar_b200 import knn
    _check(pts, pts, 16, rows=torch.cat([(pts.abs() > 5.5).any(1).nonzero()[:, 0], torch.arange(0, pts.shape[0], 97)]),
           got=knn.reset_neighbors(pts.cuda(), 16))


def test_knn_cloud_far_from_the_origin():
    """extent ~1 centred at (3e3, -2e3, 1e3): the double moments of the sigma clip cancel, and coordinates are
    quantised at 2^-13 or 2^-14, so many distances tie."""
    g = torch.Generator().manual_seed(41)
    pts = (torch.rand(30_000, 3, generator=g) - 0.5 + torch.tensor([3e3, -2e3, 1e3])).float()
    qs = pts[:2000] + 1e-3 * torch.randn(2000, 3, generator=g)
    _check(pts, qs, 16)
    from sugar_b200 import knn
    _check(pts, pts, 16, rows=torch.arange(0, 30_000, 7), got=knn.reset_neighbors(pts.cuda(), 16))


@pytest.mark.parametrize("K", [4, 16])
def test_knn_exact_duplicates_come_in_index_order(K):
    """clusters of 1, K - 1, K, K + 1 and 3K exact copies, shuffled so that copies land far apart in index (and in
    different CTAs): every row is the brute force's, neighbour 0 is the smallest index among the copies, and two runs
    give the same tables to the bit."""
    from sugar_b200 import knn
    g = torch.Generator().manual_seed(50 + K)
    base = torch.randn(8000, 3, generator=g)
    parts = [base]
    for c in (1, K - 1, K, K + 1, 3 * K):
        centres = torch.randn(12, 3, generator=g)
        parts.append(centres.repeat_interleave(c, 0))
    pts = torch.cat(parts)
    pts = pts[torch.randperm(pts.shape[0], generator=g)].contiguous().cuda()
    d2, idx = _check(pts, pts, K, got=knn.reset_neighbors(pts, K))
    assert torch.equal(idx[:, 0], _dup_groups(pts)) and float(d2[:, 0].max()) == 0.0
    d2b, idxb = knn.reset_neighbors(pts, K)
    assert torch.equal(idx, idxb) and torch.equal(d2.view(torch.int32), d2b.view(torch.int32))
    qs = pts[:3000] + 1e-4 * torch.randn(3000, 3, generator=g).cuda()
    _check(pts, qs, K)


def _grid_replica(P, ext=1.0):
    """knn_grid_setup_kernel's float32 bisection for a cloud whose clipped box is [0, ext]^3:
    (cells per axis, h, inv_h)."""
    f = np.float32
    n = max(1, min(256, int(math.ceil(np.cbrt(P / 4.0)))))
    e = f(ext)

    def cells(h):
        return int(min(np.floor(f(e / h)) + f(1.0), f(1e6)))

    h_hi, h_lo = f(e * f(1.0001)), f(e / f(f(8.0) * f(n)))
    for _ in range(40):
        mid = f(f(0.5) * f(h_lo + h_hi))
        if float(cells(mid)) ** 3 <= float(n) ** 3:
            h_hi = mid
        else:
            h_lo = mid
    return cells(h_hi), h_hi, f(f(1.0) / h_hi)


def _d2(p, q):
    """knn_dist2 of two float32 3-vectors."""
    f = np.float32
    d = (p - q).astype(np.float32)
    return f(f(f(d[0] * d[0]) + f(d[1] * d[1])) + f(d[2] * d[2]))


def test_knn_points_rounded_into_the_neighbouring_cell():
    """A uniform cloud in [0, 1]^3 with its eight corners, so that the 4-sigma clip does not bind, the box is [0, 1]^3
    and the grid is the float32 replica's.  cell_coord's rounding files a point near a face one cell over.  Traps, one
    per axis: p the largest float filed below face k1, q the smallest filed at or above face k2 = k1 + r, closer than
    r cell edges (as float32 distances) though the walk from q meets p only in shell r + 1, and p2 at a distance from q
    between |q - p| and r h along another axis, met in shell r.  A walk that stops on (r h)^2 after shell r returns p2
    for K = 1; the nearest is p.  The bulk is cleared around each trap.  Queries also sit one ulp either side of every
    face, with K = 1 and 16.  The device grid cannot be read back: should the replica differ from it, this is still an
    exactness check, only a less pointed one."""
    f = np.float32
    P = 52_000
    n, h, inv_h = _grid_replica(P)
    filed = lambda v: int(np.floor(f(f(v) * inv_h)))

    def below(k):   # the largest float filed below face k
        v = f(k * float(h))
        for _ in range(64):
            v = np.nextafter(v, f(2))
        while filed(v) >= k:
            v = np.nextafter(v, f(0))
        return v

    def above(k):   # the smallest float filed at or above face k
        v = f(k * float(h))
        for _ in range(64):
            v = np.nextafter(v, f(0))
        while filed(v) < k:
            v = np.nextafter(v, f(2))
        return v

    sq = lambda a, b: f(f(a - b) * f(a - b))
    traps = []   # (r, p, q, the old stop bound) along one axis
    for r in range(1, 6):
        for k1 in range(1, n - r):
            p, q = below(k1), above(k1 + r)
            bound = f(f(f(r) * h) * f(f(r) * h))
            if sq(q, p) < bound and len(traps) < 3:
                traps.append((r, p, q, bound))
    rng = np.random.default_rng(61)
    pts_sp, q_sp, want = [], [], []
    for ax, (r, p, q, bound) in enumerate(traps):
        # q and p on axis ax; p2 off q in the plane of the two other axes, at a float32 squared distance in
        # (|q - p|^2, bound], and within r cells of q on both of them
        lo = np.full(3, f(0.35), np.float32)
        lo[ax] = q
        dp = _d2(np.insert(np.delete(lo, ax), ax, p), lo)
        for _ in range(4000):
            t = rng.uniform(0.2, 1.3)
            p2 = lo.copy()
            p2[(ax + 1) % 3] = f(lo[(ax + 1) % 3] + r * float(h) * math.cos(t))
            p2[(ax + 2) % 3] = f(lo[(ax + 2) % 3] + r * float(h) * math.sin(t))
            for _ in range(8):
                p2[(ax + 2) % 3] = np.nextafter(p2[(ax + 2) % 3], f(0) if _d2(p2, lo) > bound else f(2))
                if dp < _d2(p2, lo) <= bound:
                    break
            if dp < _d2(p2, lo) <= bound and all(filed(p2[a]) - filed(lo[a]) <= r for a in range(3)):
                break
        assert dp < _d2(p2, lo) <= bound
        near = lo.copy()
        near[ax] = p
        pts_sp += [near, p2]
        q_sp.append(lo)
        want.append(near)
    pts_sp, q_sp = np.array(pts_sp, np.float32).reshape(-1, 3), np.array(q_sp, np.float32).reshape(-1, 3)
    corners = np.array([[i, j, k] for i in (0, 1) for j in (0, 1) for k in (0, 1)], np.float32)
    bulk = rng.random((2 * P, 3)).astype(np.float32)
    for (r, *_), qv in zip(traps, q_sp):
        bulk = bulk[np.linalg.norm(bulk - qv, axis=1) > (r + 0.5) * float(h)]
    pts = np.concatenate([corners, pts_sp, bulk[: P - 8 - len(pts_sp)]])
    assert pts.shape == (P, 3) and pts.min() == 0 and pts.max() == 1
    pts = torch.from_numpy(pts[rng.permutation(P)].copy())
    if traps:
        d2, idx = _check(pts, torch.from_numpy(q_sp), 1)
        assert torch.equal(pts[idx[:, 0].cpu()], torch.from_numpy(np.array(want)))
    # queries one ulp either side of each face, on one axis at a time
    qs = rng.random((6 * (n - 1), 3)).astype(np.float32)
    for k in range(1, n):
        face = f(k * float(h))
        for s, v in enumerate((np.nextafter(face, f(0)), np.nextafter(face, f(2)))):
            for ax in range(3):
                qs[6 * (k - 1) + 3 * s + ax, ax] = v
    for K in (1, 16):
        _check(pts, torch.from_numpy(qs), K)
    assert len(traps) == 3, "the float32 replica of the grid found fewer traps than axes"


def test_knn_grid_past_the_scans_first_chunk():
    """P = 2^24: 162 cells per axis, 4.25M cells and 1038 scan blocks, more than the block-sum scan's first chunk of
    1024.  4096 queries against the brute force, and sampled reset_neighbors rows."""
    from sugar_b200 import knn
    g = torch.Generator(device="cuda").manual_seed(71)
    P = 1 << 24
    pts = torch.rand(P, 3, generator=g, device="cuda")
    qs = torch.rand(4096, 3, generator=g, device="cuda") * 1.02 - 0.01
    _check(pts, qs, 16)
    d2, idx = knn.reset_neighbors(pts, 16)
    rows = torch.randint(0, P, (512,), generator=g, device="cuda")
    _check(pts, pts, 16, rows=rows, got=(d2, idx))
