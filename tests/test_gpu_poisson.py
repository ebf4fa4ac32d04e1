"""The screened-Poisson reconstruction on the GPU (sugar_b200/poisson.py, csrc/sgr_poisson.cu): grids node by node
and the solution against the float64 oracle (oracle/poisson_oracle.py), the multigrid's stopping rule, the geometry of
analytic surfaces, the density trim, outlier removal, determinism, and the extraction from a Gaussian shell."""
import math
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import mcubes_oracle as mo  # noqa: E402
from oracle import poisson_oracle as po  # noqa: E402

pytestmark = pytest.mark.gpu
EPS32 = 2.0 ** -24


def _unit(v):
    return v / np.linalg.norm(v, axis=1, keepdims=True)


def _cloud(kind, n, seed):
    """Oriented samples (float32 points, normals) on an analytic surface, normals pointing out."""
    rng = np.random.default_rng(seed)
    if kind == "sphere":
        d = _unit(rng.normal(size=(n, 3)))
        p, nr = 0.8 * d + np.array([0.1, -0.05, 0.02]), d
    elif kind == "torus":
        a, b = rng.uniform(0, 2 * np.pi, n), rng.uniform(0, 2 * np.pi, n)
        R, r = 0.6, 0.2
        c = np.stack([np.cos(a), np.sin(a), np.zeros(n)], 1)
        nr = np.cos(b)[:, None] * c + np.sin(b)[:, None] * np.array([0, 0, 1.0])
        p = R * c + r * nr
    elif kind == "nested":
        m = n * 4 // 5
        d = _unit(rng.normal(size=(n, 3)))
        p = np.concatenate([0.8 * d[:m], 0.4 * d[m:]])
        nr = np.concatenate([d[:m], -d[m:]])                    # the inner sphere's normals point inwards
    elif kind == "clusters":
        centres = rng.uniform(-1, 1, size=(6, 3))
        k = rng.integers(0, 6, n)
        d = _unit(rng.normal(size=(n, 3)))
        p, nr = centres[k] + rng.uniform(0.05, 0.3, (n, 1)) * d, d
    elif kind == "cap":                                     # an open hemisphere
        d = _unit(rng.normal(size=(n, 3)))
        d[:, 2] = np.abs(d[:, 2])
        p, nr = 0.8 * d, d
    return p.astype(np.float32), nr.astype(np.float32)


def _with_edges(p, nr, depth):
    """Add samples exactly on node planes (cell faces of the hat supports) and in the corner cells nearest the
    domain's boundary, keeping the bounding box (hence the domain)."""
    o, h, o32, ih = po.domain(p, depth)
    N = 1 << depth
    lo, hi = p.min(0), p.max(0)
    extra = [lo, hi, np.array([lo[0], hi[1], lo[2]], np.float32)]
    g = po.grid_coords(p[:200], o32, ih)
    on_plane = p[:200].copy()
    for a in range(3):                                     # find a float32 position whose g is an integer
        for s in range(200):
            target = np.float32(np.round(g[s, a]))
            x = np.float32(o32[a] + (target + np.float32(0.5)) / ih)
            for _ in range(8):
                gx = (np.float32(x - o32[a]) * ih) - np.float32(0.5)
                if gx == target:
                    break
                x = np.nextafter(x, np.float32(np.inf) if gx < target else np.float32(-np.inf))
            if lo[a] <= x <= hi[a]:
                on_plane[s, a] = x
    pts = np.concatenate([p, np.asarray(extra, np.float32), on_plane]).astype(np.float32)
    nrm = np.concatenate([nr, _unit(np.ones((3, 3))), nr[:200]]).astype(np.float32)
    gg = po.grid_coords(pts, o32, ih)
    assert (gg == np.round(gg)).sum() > 100, "no sample landed on a node plane"
    assert np.array_equal(pts.min(0), lo) and np.array_equal(pts.max(0), hi) and N > 0
    return pts, nrm


def _bound(points, depth, o32, ih, values=None, grad_normals=None):
    """Per node: the float32 accumulation bound (terms + 4) eps sum |term| of a splat, and its oracle value."""
    N = 1 << depth
    g = po.grid_coords(points, o32, ih)
    _, ids, ws, gr = po.hats(g, N)
    if grad_normals is not None:
        terms = np.einsum("sc,skc->sk", grad_normals.astype(np.float64), gr)
        abs_terms = np.einsum("sc,skc->sk", np.abs(grad_normals.astype(np.float64)), np.abs(gr))
    else:
        terms = ws if values is None else ws * values.astype(np.float64)[:, None]
        abs_terms = np.abs(terms)
    val, mag, cnt = np.zeros(N ** 3), np.zeros(N ** 3), np.zeros(N ** 3)
    np.add.at(val, ids.reshape(-1), terms.reshape(-1))
    np.add.at(mag, ids.reshape(-1), abs_terms.reshape(-1))
    np.add.at(cnt, ids.reshape(-1), 1.0)
    return val.reshape((N,) * 3), ((cnt + 8) * EPS32 * mag + 1e-30).reshape((N,) * 3)


@pytest.mark.parametrize("depth", [5, 6])
@pytest.mark.parametrize("kind", ["sphere", "torus", "clusters"])
def test_grids_match_the_oracle_node_by_node(kind, depth):
    from sugar_b200 import poisson
    p, nr = _with_edges(*_cloud(kind, 6000, seed=depth), depth)
    colors = np.random.default_rng(1).random(p.shape).astype(np.float32)
    tp, tn = torch.from_numpy(p).cuda(), torch.from_numpy(nr).cuda()
    s = poisson.solve(tp, tn, depth)
    ref = po.system(p, nr, depth)
    assert s["area"] == ref["area"]
    assert np.array_equal(s["o32"], ref["o32"]) and s["inv_h32"] == ref["inv_h32"]
    o32, ih = ref["o32"], ref["inv_h32"]
    a = ref["area"]
    val, tol = _bound(p, depth, o32, ih, grad_normals=nr)
    # b = -a * acc, q = (alpha a) * acc: two more roundings of the accumulated value
    assert np.all(np.abs(s["b"].cpu().numpy() - ref["b"]) <= a * tol + 3 * EPS32 * np.abs(ref["b"]))
    val, tol = _bound(p, depth, o32, ih)
    assert np.all(np.abs(s["q"].cpu().numpy() - ref["q"]) <= 4 * a * tol + 4 * EPS32 * np.abs(ref["q"]))
    # density grid of depth - 2 and the colour grids at full depth
    o, h = ref["o"], ref["h"]
    ih2 = np.float32((1 << (depth - 2)) / ((1 << depth) * h))
    ends, binned, _ = poisson._bin(tp, depth - 2, o32, ih2)
    got = poisson._splat(1 << (depth - 2), ends, binned, poisson.WEIGHT).cpu().numpy()
    want, tol = _bound(p, depth - 2, o32, ih2)
    assert np.all(np.abs(got - want) <= tol) and np.allclose(want, po.splat(p, depth - 2, o32, ih2))
    tc = torch.from_numpy(colors).cuda()
    for ch in range(3):
        got = poisson._splat(1 << depth, s["starts"], s["binned"], poisson.ATTRIBUTE, tc, ch).cpu().numpy()
        want, tol = _bound(p, depth, o32, ih, values=colors[:, ch])
        assert np.all(np.abs(got - want) <= tol), ch


@pytest.mark.parametrize("depth", [5, 6])
@pytest.mark.parametrize("kind", ["sphere", "torus", "clusters"])
def test_solution_and_iso_value_match_the_oracle(kind, depth):
    from sugar_b200 import poisson
    p, nr = _cloud(kind, 20000, seed=10 + depth)
    s = poisson.solve(torch.from_numpy(p).cuda(), torch.from_numpy(nr).cuda(), depth)
    ref = po.system(p, nr, depth)
    u = po.solve(ref["A"], ref["b"])
    scale = np.abs(u).max()
    assert np.abs(s["u"].cpu().numpy() - u).max() <= 1e-3 * scale
    iso = po.interpolate(u, po.grid_coords(p, ref["o32"], ref["inv_h32"])).mean()
    assert abs(s["iso"] - iso) <= 1e-3 * scale
    assert s["residual"] <= 1e-5 and s["cycles"] <= 30


@pytest.mark.parametrize("depth", [5, 6, 7, 8, 9])
def test_multigrid_meets_the_stopping_rule(depth):
    from sugar_b200 import poisson
    for kind in ("sphere", "clusters"):
        p, nr = _cloud(kind, 200_000, seed=depth)
        s = poisson.solve(torch.from_numpy(p).cuda(), torch.from_numpy(nr).cuda(), depth)
        assert s["residual"] <= 1e-5 and 1 <= s["cycles"] <= 30, (kind, s["cycles"], s["residual"])
        # the reported ratio is the true one
        dev = s["u"].device
        part = torch.empty(poisson.RED_BLOCKS, dtype=torch.float64, device=dev)
        import ctypes
        from sugar_b200._lib import lib, stream
        rn, bn = ctypes.c_double(), ctypes.c_double()
        N = 1 << depth
        lib.sgr_poisson_residual_norm(N, 1.0, s["u"].data_ptr(), s["b"].data_ptr(), s["q"].data_ptr(),
                                      part.data_ptr(), ctypes.byref(rn), stream(dev))
        lib.sgr_poisson_residual_norm(N, 1.0, None, s["b"].data_ptr(), None, part.data_ptr(), ctypes.byref(bn),
                                      stream(dev))
        assert rn.value / bn.value == s["residual"]


def _surface_distance(kind, v):
    if kind == "sphere":
        return np.abs(np.linalg.norm(v - np.array([0.1, -0.05, 0.02]), axis=1) - 0.8)
    if kind == "torus":
        rho = np.linalg.norm(v[:, :2], axis=1)
        return np.abs(np.sqrt((rho - 0.6) ** 2 + v[:, 2] ** 2) - 0.2)
    r = np.linalg.norm(v, axis=1)
    return np.minimum(np.abs(r - 0.8), np.abs(r - 0.4))


@pytest.mark.parametrize("kind,chi", [("sphere", 2), ("torus", 0), ("nested", 4)])
def test_geometry_of_analytic_surfaces_at_depth_8(kind, chi):
    from sugar_b200 import poisson
    p, nr = _cloud(kind, 1_000_000, seed=3)
    m = poisson.poisson_reconstruction(torch.from_numpy(p).cuda(), torch.from_numpy(nr).cuda(), depth=8)
    v = m["verts"].cpu().numpy().astype(np.float64)
    f = m["faces"].cpu().numpy()
    h = po.domain(p, 8)[1]
    d = _surface_distance(kind, v)
    assert d.max() <= 1.5 * h and d.mean() < 0.5 * h, (d.max() / h, d.mean() / h)
    uc, directed_once = mo.directed_edge_counts(f)
    assert (uc == 2).all() and directed_once                       # watertight, edge-manifold, consistently wound
    assert mo.euler_characteristic(len(v), f) == chi
    vol = np.einsum("ij,ij->i", v[f[:, 0]], np.cross(v[f[:, 1]], v[f[:, 2]])).sum() / 6
    assert vol > 0


def test_density_trim_on_an_open_hemisphere_cap():
    """On an open cap Poisson closes the surface away from the samples.  The density stays positive and falls with
    the distance there, so the 0.1 quantile trim removes the farthest tenth of the vertices; the dense grid meshes the
    closing surface at full resolution, so more than a tenth lies beyond 2h.  A quantile equal to that share leaves the
    vertices within 2h of a sample, but for a band just past the cap's rim (splat-ordered, not distance-ordered) that
    stays within 3h."""
    from sugar_b200 import knn, poisson
    p, nr = _cloud("cap", 300_000, seed=4)
    tp = torch.from_numpy(p).cuda()
    m = poisson.poisson_reconstruction(tp, torch.from_numpy(nr).cuda(), depth=7)
    h = po.domain(p, 7)[1]
    dens = m["densities"]
    V = dens.shape[0]
    d = knn.knn_points(m["verts"], tp, 1)[0][:, 0].sqrt()
    assert float(dens.min()) > 0
    beyond = d > 2 * h
    share = float(beyond.double().mean())
    assert share > 0.1                                          # the closing surface (see the docstring)
    trim = lambda q: dens.double() < poisson.quantile(dens, q)
    removed = trim(0.1)
    assert 0.09 * V <= int(removed.sum()) <= 0.1 * V + 1
    assert float(d[removed].min()) > 2 * h
    assert float(d[removed].min()) >= float(d[~removed].max()) - 1e-6    # the farthest first
    removed = trim(share)
    kept = d[~removed]
    assert float(kept.max()) <= 3 * h, (float(kept.max()) / h, share, V)
    assert int((kept > 2 * h).sum()) <= 0.005 * V
    t0 = poisson.remove_vertices_by_mask(m["verts"], m["faces"], trim(0.0))
    assert torch.equal(t0["verts"], m["verts"]) and torch.equal(t0["faces"], m["faces"])


@pytest.mark.parametrize("depth", [3, 5, 8])
def test_binning_is_a_stable_sort_by_bin_even_in_crowded_bins(depth):
    """Half the samples crowd into one bin: the records come out sorted by bin and, within a bin, by sample id, in a
    time that does not grow with the bin's size squared."""
    import time
    from sugar_b200 import poisson
    rng = np.random.default_rng(depth)
    n = 2_000_000
    p = rng.uniform(-1, 1, size=(n, 3)).astype(np.float32)
    crowd = rng.random(n) < 0.5
    p[crowd] = (0.3 + 1e-4 * rng.random((int(crowd.sum()), 3))).astype(np.float32)
    tp = torch.from_numpy(p).cuda()
    o, h, o32, ih = po.domain(p, depth)
    poisson._bin(tp, depth, o32, ih)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    starts, binned, occupied = poisson._bin(tp, depth, o32, ih)
    torch.cuda.synchronize()
    elapsed = time.perf_counter() - t0
    N = 1 << depth
    g = po.grid_coords(p, o32, ih)
    L = np.clip(np.floor(g).astype(np.int64), 0, N - 2)
    key = (L[:, 0] * N + L[:, 1]) * N + L[:, 2]
    order = np.argsort(key, kind="stable")
    got = binned.cpu().numpy()
    assert np.array_equal(got[:, 3].view(np.int32), order)
    assert np.array_equal(got[:, :3], g[order].astype(np.float32))
    assert occupied == len(np.unique(key))
    want_starts = np.searchsorted(key[order], np.arange(N ** 3))
    assert np.array_equal(starts.cpu().numpy(), want_starts)
    assert elapsed < 0.5, elapsed


def test_outlier_removal_equals_the_oracle():
    from sugar_b200 import poisson
    rng = np.random.default_rng(7)
    for n, ratio in ((3000, 20.0), (3000, 2.0), (2000, 1.0)):
        p, _ = _cloud("sphere", n, seed=n)
        fl = rng.uniform(-3, 3, size=(15, 3)).astype(np.float32)
        p = np.concatenate([p, fl]).astype(np.float32)
        got = poisson.remove_statistical_outlier(torch.from_numpy(p).cuda(), 20, ratio).cpu().numpy()
        want = po.outlier_kept(p, 20, ratio)
        # away from exact ties: no point's value sits within float32 rounding of the bound
        d = np.sort(np.linalg.norm(p[:, None] - p[None], axis=-1), 1)[:, :20].mean(1)
        bound = d.mean() + ratio * d.std(ddof=1)
        assert np.abs(d - bound).min() > 1e-5 * bound
        assert np.array_equal(got, want)
        if ratio <= 2.0:
            assert len(want) < len(p)


def test_reconstruction_is_bit_identical_from_run_to_run():
    from sugar_b200 import poisson
    p, nr = _cloud("clusters", 300_000, seed=8)
    c = np.random.default_rng(2).random(p.shape).astype(np.float32)
    args = [torch.from_numpy(x).cuda() for x in (p, nr, c)]
    s1 = poisson.solve(args[0], args[1], 7)
    s2 = poisson.solve(args[0], args[1], 7)
    assert torch.equal(s1["u"], s2["u"]) and s1["iso"] == s2["iso"]
    m1 = poisson.poisson_reconstruction(args[0], args[1], depth=7, colors=args[2])
    m2 = poisson.poisson_reconstruction(args[0], args[1], depth=7, colors=args[2])
    for k in ("verts", "faces", "colors", "densities"):
        assert torch.equal(m1[k], m2[k]), k
    assert m1["colors"].shape == m1["verts"].shape and bool(torch.isfinite(m1["colors"]).all())


def _look_at(eye, fov):
    from types import SimpleNamespace
    from sugar_b200 import render
    eye = np.asarray(eye, np.float64)
    z = eye / np.linalg.norm(eye)                                 # OpenGL: the camera looks along -z
    x = np.cross([0.0, 0.0, 1.0] if abs(z[2]) < 0.9 else [0.0, 1.0, 0.0], z)
    x /= np.linalg.norm(x)
    y = np.cross(z, x)
    c2w = torch.tensor(np.stack([x, y, z, eye], 1), dtype=torch.float32, device="cuda")
    wv, fp, cc = render.camera_matrices(c2w, fov, fov)
    return SimpleNamespace(viewmatrix=wv, projmatrix=fp, campos=cc, width=256, height=256,
                           tanfovx=math.tan(fov / 2), tanfovy=math.tan(fov / 2))


def test_gaussian_shell_to_poisson_mesh_to_ply(tmp_path):
    from sugar_b200 import mcubes, poisson
    gen = torch.Generator().manual_seed(6)
    P = 60_000
    d = torch.nn.functional.normalize(torch.randn(P, 3, generator=gen), dim=-1)
    pts = (1.2 * d + 0.005 * torch.randn(P, 3, generator=gen)).cuda()
    # flat Gaussians tangent to the shell: their smallest axis along the normal
    up = torch.tensor([0.0, 0.0, 1.0]).expand(P, 3)
    axis = torch.nn.functional.normalize(torch.linalg.cross(up, d), dim=-1)
    ang = torch.acos(d[:, 2].clamp(-1, 1))
    q = torch.cat([torch.cos(ang / 2)[:, None], axis * torch.sin(ang / 2)[:, None]], 1)    # rotates z to d
    sc = torch.tensor([0.03, 0.03, 0.002]).expand(P, 3).clone()
    st = torch.full((P, 1), 0.9)
    sh = torch.rand(P, 1, 3, generator=gen)
    pts, sc, q, st, sh = (t.float().cuda().contiguous() for t in (pts, sc, q, st, sh))
    eyes = [(3.5, 0, 0.5), (-3.5, 0.3, 0), (0, 3.5, -0.5), (0, -3.5, 0.4), (0.3, 0.2, 3.5), (0.2, -0.3, -3.5)]
    cams = [_look_at(e, math.radians(50)) for e in eyes]
    g = torch.Generator(device="cuda").manual_seed(0)
    cloud = poisson.surface_point_cloud(pts, sc, q, st, sh, cams, n_total_points=200_000, generator=g)
    n = cloud["points"].shape[0]
    assert 50_000 < n <= 200_000 + len(cams)
    r = cloud["points"].norm(dim=-1)
    assert float((r - 1.2).abs().quantile(0.99)) < 0.05
    # the level-set normals point up the density gradient (the reference's sign), here into the shell's layer of
    # Gaussians as the outside cameras see it
    assert float((cloud["normals"] * cloud["points"] / r[:, None]).sum(-1).median()) < -0.9
    assert float(cloud["colors"].min()) >= 0 and float(cloud["colors"].max()) <= 1
    centers = torch.tensor(eyes)
    e = mcubes.camera_spatial_extent(centers)
    out = poisson.extract_mesh_poisson(cloud["points"], cloud["colors"], cloud["normals"], e, poisson_depth=9,
                                       decimation_target=20_000)
    fg = out["foreground"]
    assert 0 < fg["faces"].shape[0] <= 20_000
    # the mesh follows the level-set points: the same median radius to within the grid's spacing h, and a 1 % tail
    # (after the trim and the decimation) a few h beyond the points' own
    h = poisson.domain(cloud["points"], 9)[1]
    rv = fg["verts"].norm(dim=-1)
    q99 = lambda x: float((x - 1.2).abs().quantile(0.99))
    assert abs(float(rv.median()) - float(r.median())) <= h
    assert q99(rv) <= q99(r) + 6 * h, (q99(rv), q99(r), h)
    assert out["background"]["verts"].shape[0] == 0
    comb = out["combined"]
    path = str(tmp_path / "mesh.ply")
    mcubes.write_ply(path, comb["verts"], comb["faces"], comb["colors"], comb["normals"])
    with open(path, "rb") as fh:
        data = fh.read()
    head, body = data.split(b"end_header\n", 1)
    V, F = comb["verts"].shape[0], comb["faces"].shape[0]
    assert f"element vertex {V}".encode() in head and f"element face {F}".encode() in head
    rec = np.frombuffer(body[:V * 51], dtype=[("p", "<f8", 3), ("n", "<f8", 3), ("c", "u1", 3)])
    assert np.allclose(rec["p"], comb["verts"].cpu().double().numpy())
    fr = np.frombuffer(body[V * 51:], dtype=[("k", "u1"), ("i", "<i4", 3)])
    assert (fr["k"] == 3).all() and np.array_equal(fr["i"], comb["faces"].cpu().numpy())


def test_argument_checks():
    from sugar_b200 import poisson
    p, nr = _cloud("sphere", 1000, seed=9)
    tp, tn = torch.from_numpy(p).cuda(), torch.from_numpy(nr).cuda()
    for depth in (4, 11, 5.0):
        with pytest.raises(ValueError, match="depth"):
            poisson.poisson_reconstruction(tp, tn, depth=depth)
    with pytest.raises(ValueError, match="normals"):
        poisson.poisson_reconstruction(tp, tn[1:], depth=5)
    with pytest.raises(ValueError, match="colors"):
        poisson.poisson_reconstruction(tp, tn, depth=5, colors=tn[:, :2])
    zero = tn.clone()
    zero[5] = 0
    with pytest.raises(ValueError, match="non-zero"):
        poisson.poisson_reconstruction(tp, zero, depth=5)
    with pytest.raises(ValueError, match="empty"):
        poisson.poisson_reconstruction(tp[:0], tn[:0], depth=5)
    with pytest.raises(ValueError, match="bounding box"):
        poisson.poisson_reconstruction(tp[:1].expand(10, 3), tn[:10], depth=5)
    with pytest.raises(ValueError, match="Both"):
        poisson.extract_mesh_poisson(tp + 100.0, tn, tn, 1.0, poisson_depth=5)
