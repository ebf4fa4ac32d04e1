"""The marching-cubes extraction on the GPU (sugar_b200/mcubes.py, csrc/sgr_mcubes.cu): grid densities against goldens
made by the reference's own lines and against this package's K-NN + field composition; marching cubes against the numpy
oracle array for array; mesh properties at larger sizes; the extraction driver; and the whole coarse -> mesh -> refine
-> texture path."""
import glob
import os

import numpy as np
import pytest

import helpers as h

pytestmark = pytest.mark.gpu
GOLDEN = sorted(glob.glob(os.path.join(h.ROOT, "tests", "golden", "mcubes_*.npz")))


def _cloud(g):
    import torch
    return [torch.from_numpy(np.ascontiguousarray(g[k])).cuda() for k in ("points", "scaling", "quaternions", "strengths")]


@pytest.mark.parametrize("path", GOLDEN, ids=os.path.basename)
def test_grid_density_matches_reference_golden(path):
    import torch
    from sugar_b200 import mcubes
    g = np.load(path)
    e, R = float(g["extent"]), int(g["resolution"])
    pts, sc, q, st = _cloud(g)
    X = torch.linspace(-1, 1, R) * e
    fg = mcubes.density_grid(pts, sc, q, st, X, X, X).cpu().numpy()
    assert h.rel_err(fg, g["fg_volume"]) < 2e-5
    X = torch.linspace(-1, 1, R) * 4 * e
    bg = mcubes.density_grid(pts, sc, q, st, X, X, X, exclude_box=e).cpu().numpy()
    assert h.rel_err(bg, g["bg_volume"]) < 2e-5
    assert np.array_equal(bg == 0, g["bg_volume"] == 0)


def _far_cloud(P, seed):
    """A Gaussian blob with floaters beyond mean +- 4 sigma (the K-NN grid clamps them into its border cells)."""
    import torch
    gen = torch.Generator().manual_seed(seed)
    pts = torch.randn(P, 3, generator=gen) * torch.tensor([1.0, 0.6, 0.3])
    pts[:40] = torch.randn(40, 3, generator=gen) * 6.0                   # floaters around and far from the blob
    sc = torch.exp(torch.randn(P, 3, generator=gen) * 0.3 - 3.0)
    q = torch.nn.functional.normalize(torch.randn(P, 4, generator=gen), dim=-1)
    st = torch.sigmoid(torch.randn(P, generator=gen))
    return [t.float().cuda() for t in (pts, sc, q, st)]


def _far_grid():
    import torch
    R = 128
    X = torch.linspace(-1, 1, R) * 12.0
    Y = torch.linspace(-1, 1, R) * 9.0
    Z = torch.linspace(-1, 1, R) * 10.0 + 1.5
    xx, yy, zz = torch.meshgrid(X, Y, Z, indexing="ij")
    return (X, Y, Z), torch.stack([xx.reshape(-1), yy.reshape(-1), zz.reshape(-1)], -1).cuda()


def test_grid_density_equals_knn_plus_field_far_outside_the_cloud():
    """The density grid's walk and knn_points share the distance, the (distance, index) order and the stop radius, so
    every voxel, inside the grid's box or far outside it, equals compute_density over knn_points' neighbours to the
    bit."""
    import torch
    from sugar_b200 import field, knn, mcubes
    pts, sc, q, st = _far_cloud(200_000, 3)
    axes, grid = _far_grid()
    got = mcubes.density_grid(pts, sc, q, st, *axes).reshape(-1)
    want = field.compute_density(grid, knn.knn_points(grid, pts, 16)[1], pts, sc, q, st)
    diff = (got.view(torch.int32) != want.view(torch.int32)).nonzero()[:, 0]
    assert diff.numel() == 0, (diff.numel(), diff[:5].tolist())


def test_grid_density_equals_the_field_over_brute_force_neighbours():
    """The same grid against neighbours that come from no grid walk: the float32 brute force (oracle/knn_oracle.py) on
    voxels well inside the 4-sigma box, far outside it, and next to each floater."""
    import torch
    from oracle import knn_oracle as ko
    from sugar_b200 import field, mcubes
    pts, sc, q, st = _far_cloud(200_000, 3)
    axes, grid = _far_grid()
    got = mcubes.density_grid(pts, sc, q, st, *axes).reshape(-1)
    p64 = pts.double()
    mean, sd = p64.mean(0), p64.std(0)
    z = ((grid.double() - mean) / sd).abs()
    gen = torch.Generator(device="cuda").manual_seed(5)
    pick = lambda m, k: m.nonzero()[:, 0][torch.randperm(int(m.sum()), generator=gen, device="cuda")[:k]]
    inside, outside = pick((z < 3.5).all(1), 3000), pick((z > 5.0).any(1), 3000)
    floaters = ((pts.double() - mean) / sd).abs().gt(4.0).any(1).nonzero()[:, 0]
    near = ko.knn_f32(pts[floaters], grid, 8)[1].reshape(-1)      # the voxels around each floater
    assert inside.numel() == outside.numel() == 3000 and floaters.numel() >= 10
    sel = torch.cat([inside, outside, near]).unique()
    idx = ko.knn_f32(grid[sel], pts, 16)[1]
    want = field.compute_density(grid[sel], idx, pts, sc, q, st)
    bad = (got[sel].view(torch.int32) != want.view(torch.int32)).nonzero()[:, 0]
    assert bad.numel() == 0, (bad.numel(), sel[bad[:5]].tolist())


def test_exclusion_box_writes_exact_zeros():
    import torch
    from sugar_b200 import mcubes
    pts, sc, q, st = _far_cloud(20_000, 4)
    sc = sc * 20.0       # wide Gaussians: every voxel has a positive density
    X = torch.linspace(-1, 1, 40) * 4.0
    full = mcubes.density_grid(pts, sc, q, st, X, X, X)
    ex = mcubes.density_grid(pts, sc, q, st, X, X, X, exclude_box=1.0)
    inside = (X > -1.0) & (X < 1.0)
    m = (inside[:, None, None] & inside[None, :, None] & inside[None, None, :]).cuda()
    assert bool((full[m] > 0).all()) and bool((ex[m] == 0).all())
    assert torch.equal(ex[~m], full[~m])


def _blobs(R, seed):
    rng = np.random.default_rng(seed)
    x = np.arange(R, dtype=np.float64)
    X, Y, Z = np.meshgrid(x, x[: R - 3], x[: R - 5], indexing="ij")
    vol = np.zeros(X.shape)
    for _ in range(12):
        c = rng.uniform(0, R, 3)
        s = rng.uniform(0.05, 0.2) * R
        vol += np.exp(-((X - c[0]) ** 2 + (Y - c[1]) ** 2 + (Z - c[2]) ** 2) / (2 * s * s))
    return (vol + 0.05 * rng.normal(size=vol.shape)).astype(np.float32)


@pytest.mark.parametrize("R,level", [(20, 0.5), (48, 0.3), (96, 0.4)])
def test_marching_cubes_equals_the_oracle(R, level):
    import torch
    from oracle import mcubes_oracle as mo
    from sugar_b200 import mcubes
    vol = _blobs(R, R)
    v, f = mcubes.marching_cubes(torch.from_numpy(vol).cuda(), level)
    ov, of = mo.marching_cubes(vol, level)
    assert v.dtype == torch.float32 and f.dtype == torch.int64 and len(of) > 100
    assert np.array_equal(f.cpu().numpy(), of)
    assert np.array_equal(v.cpu().numpy(), ov.astype(np.float32))


@pytest.mark.parametrize("path", GOLDEN, ids=os.path.basename)
def test_marching_cubes_on_golden_volumes(path):
    import torch
    from oracle import mcubes_oracle as mo
    from sugar_b200 import mcubes
    g = np.load(path)
    for pre in ("fg", "bg"):
        v, f = mcubes.marching_cubes(torch.from_numpy(g[f"{pre}_volume"]).cuda(), float(g["level"]))
        assert np.array_equal(f.cpu().numpy(), g[f"{pre}_faces"])
        ov, _ = mo.marching_cubes(g[f"{pre}_volume"], float(g["level"]))
        assert np.array_equal(v.cpu().numpy(), ov.astype(np.float32))


def test_watertight_sphere_and_torus_at_256():
    import torch
    from sugar_b200 import mcubes
    R = 256
    x = torch.linspace(-1, 1, R, device="cuda")
    X, Y, Z = torch.meshgrid(x, x, x, indexing="ij")
    for vol, chi in (((0.7 ** 2 - (X * X + Y * Y + Z * Z)), 2),
                     ((0.2 ** 2 - ((X * X + Y * Y).sqrt() - 0.6) ** 2 - Z * Z), 0)):
        v, f = mcubes.marching_cubes(vol.contiguous(), 0.0)
        d = torch.cat([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
        und, cnt = torch.unique(d.sort(1).values, dim=0, return_counts=True)
        assert bool((cnt == 2).all())
        assert torch.unique(d, dim=0).shape[0] == d.shape[0]         # each directed edge once: consistent winding
        assert v.shape[0] - und.shape[0] + f.shape[0] == chi


def test_empty_results_and_bad_arguments():
    import torch
    from sugar_b200 import mcubes
    for val in (0.0, 1.0):
        v, f = mcubes.marching_cubes(torch.full((16, 17, 18), val, device="cuda"), 0.5)
        assert v.shape == (0, 3) and f.shape == (0, 3)
    v, f = mcubes.marching_cubes(torch.zeros(1, 1, 1, device="cuda"), 0.5)
    assert v.shape == (0, 3) and f.shape == (0, 3)
    pts, sc, q, st = _far_cloud(1000, 5)
    X = torch.linspace(-1, 1, 8)
    with pytest.raises(ValueError, match="K"):
        mcubes.density_grid(pts[:10], sc[:10], q[:10], st[:10], X, X, X, K=16)
    with pytest.raises(ValueError):
        mcubes.marching_cubes(torch.zeros(4, 4, device="cuda"), 0.5)
    # any K <= 64 (the general path) agrees with the composition too
    from sugar_b200 import field, knn
    d = mcubes.density_grid(pts, sc, q, st, X * 3, X * 3, X * 3, K=9).reshape(-1)
    xx, yy, zz = torch.meshgrid(X * 3, X * 3, X * 3, indexing="ij")
    grid = torch.stack([xx.reshape(-1), yy.reshape(-1), zz.reshape(-1)], -1).cuda()
    want = field.compute_density(grid, knn.knn_points(grid, pts, 9)[1], pts, sc, q, st)
    assert torch.equal(d, want)


def _shell_model(P, seed):
    import torch
    gen = torch.Generator().manual_seed(seed)
    d = torch.nn.functional.normalize(torch.randn(P, 3, generator=gen), dim=-1)
    pts = 1.2 * d + 0.01 * torch.randn(P, 3, generator=gen)
    pts[:20] = torch.randn(20, 3, generator=gen) * 3.0 + 4.0          # a few Gaussians in the background grid
    sc = torch.exp(torch.randn(P, 3, generator=gen) * 0.2 - 3.0)
    q = torch.nn.functional.normalize(torch.randn(P, 4, generator=gen), dim=-1)
    st = torch.sigmoid(torch.randn(P, 1, generator=gen) + 2.0)
    sh = torch.randn(P, 1, 3, generator=gen)
    return [t.float().cuda() for t in (pts, sc, q, st, sh)]


def test_extract_mesh_on_a_gaussian_shell():
    import torch
    from sugar_b200 import knn, mcubes
    pts, sc, q, st, sh = _shell_model(60_000, 6)
    e = mcubes.camera_spatial_extent(torch.tensor([[2.0, 0, 0], [-2.0, 0, 0], [0, 2.0, 0]]))
    out = mcubes.extract_mesh_marching_cubes(pts, sc, q, st, sh, e, resolution=96)
    again = mcubes.extract_mesh_marching_cubes(pts, sc, q, st, sh, e, resolution=96)
    fg, bg, comb = out["foreground"], out["background"], out["combined"]
    assert fg["faces"].shape[0] > 1000
    for m, ext in ((fg, e), (bg, 4 * e)):
        assert float(m["verts"].abs().max()) <= ext
        if m["verts"].shape[0]:
            nearest = knn.knn_points(m["verts"], pts, 1)[1][:, 0]
            assert torch.equal(m["colors"], sh[nearest, 0] * 0.28209479177387814 + 0.5)
            used = torch.zeros(m["verts"].shape[0], dtype=torch.bool, device="cuda")
            used[m["faces"].reshape(-1)] = True
            assert float((m["normals"][used].norm(dim=-1) - 1).abs().max()) < 1e-5
    assert comb["verts"].shape[0] == fg["verts"].shape[0] + bg["verts"].shape[0]
    assert torch.equal(comb["faces"][fg["faces"].shape[0]:], bg["faces"] + fg["verts"].shape[0])
    for part in out:
        for k in out[part]:
            assert torch.equal(out[part][k], again[part][k]), (part, k)


def test_coarse_model_to_mesh_to_refinement_to_texture():
    """One script: a coarse model (one regularised coarse step on a synthetic scene) -> marching-cubes mesh ->
    Gaussians bound to it -> one refinement step -> UV texture."""
    import torch
    from types import SimpleNamespace
    from sugar_b200 import knn, mcubes, meshbind, scenes, steps, texture
    W, H = 160, 96
    sc = scenes.make_scene(6000, W, H, seed=8, px_sigma=25.0, frac_behind=0.0, zrange=(3.0, 6.0))
    leaf = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda().requires_grad_(True)
    raw = dict(points=leaf(sc.means3D), sh_dc=leaf(sc.shs[:, :1]), sh_rest=leaf(sc.shs[:, 1:]),
               densities=leaf(np.log(sc.opacities / (1 - sc.opacities))), scales=leaf(np.log(sc.scales)),
               quaternions=leaf(sc.rotations))
    cam = steps.camera_from_scene(sc, "cuda")
    gt = torch.rand(3, H, W, device="cuda")
    knn_idx = knn.reset_neighbors(raw["points"].detach())[1]
    loss, _ = steps.coarse_sdf_step(raw, cam, gt, knn_idx, steps.ours_ops(), n_samples=20_000)
    assert torch.isfinite(loss)
    a = steps.activate({k: v.detach() for k, v in raw.items()})
    m = mcubes.extract_mesh_marching_cubes(a.points, a.scaling, a.quaternions, a.strengths, a.sh[:, :1], 8.0,
                                           resolution=48)["combined"]
    verts, faces = m["verts"], m["faces"]
    F = faces.shape[0]
    assert F > 100
    g = torch.Generator().manual_seed(0)
    n = 1
    P = F * n
    rr = dict(verts=verts.clone().requires_grad_(True),
              sh_dc=(0.5 * torch.randn(P, 1, 3, generator=g)).cuda().requires_grad_(True),
              sh_rest=(0.1 * torch.randn(P, 15, 3, generator=g)).cuda().requires_grad_(True),
              densities=torch.randn(P, 1, generator=g).cuda().requires_grad_(True),
              scales=(torch.randn(P, 2, generator=g) * 0.3 - 2.0).cuda().requires_grad_(True),
              quaternions=torch.randn(P, 2, generator=g).cuda().requires_grad_(True))
    mesh = SimpleNamespace(faces=faces, bary=meshbind.bary_coords(n, "cuda"), thickness=1e-5)
    loss, stats = steps.refine_step(rr, mesh, cam, gt, steps.ours_ops())
    assert torch.isfinite(loss) and stats["visible"] > 0 and rr["verts"].grad is not None
    b = meshbind.bind_to_mesh(rr["verts"].detach(), faces, mesh.bary, rr["scales"].detach(),
                              rr["quaternions"].detach(), mesh.thickness)
    verts_uv, faces_uv, tex = texture.extract_texture_image_and_uv_from_gaussians(
        rr["verts"].detach(), faces, b.points.detach(), b.scaling.detach(), b.quaternions.detach(),
        torch.sigmoid(rr["densities"].detach()), rr["sh_dc"].detach(), [cam], square_size=4)
    assert tex.shape[0] == tex.shape[1] == texture.texture_size(F, 4) and bool(torch.isfinite(tex).all())
    assert faces_uv.shape == (F, 3)
