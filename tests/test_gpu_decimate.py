"""The quadric decimation on the GPU (sugar_b200/decimate.py, csrc/sgr_decimate.cu): array for array against the numpy
round algorithm, quality against the sequential greedy loop, 512^3 marching-cubes meshes decimated to the refinement
presets' 1M and 200k faces, and the marching-cubes extraction with decimation feeding one refinement step and the
texture bake."""
import os
import sys

import numpy as np
import pytest

import helpers as h

sys.path.insert(0, h.ROOT)
from oracle import decimate_oracle as do  # noqa: E402
from oracle import mcubes_oracle as mo  # noqa: E402

pytestmark = pytest.mark.gpu


def _field(kind, R, seed=0):
    """Analytic volumes on [-1, 1]^3 (numpy, float32): positive inside."""
    g = np.linspace(-1, 1, R, dtype=np.float64)
    X, Y, Z = np.meshgrid(g, g, g, indexing="ij")
    if kind == "sphere":
        f = 0.7 - np.sqrt(X ** 2 + Y ** 2 + Z ** 2)
    elif kind == "torus":
        f = 0.25 - np.sqrt((np.sqrt(X ** 2 + Y ** 2) - 0.6) ** 2 + Z ** 2)
    elif kind == "cut":                              # a sphere cut open by the grid box
        f = 1.15 - np.sqrt(X ** 2 + Y ** 2 + Z ** 2)
    else:                                            # noisy blobs
        rng = np.random.default_rng(seed)
        c = rng.uniform(-0.5, 0.5, (6, 3))
        f = sum(np.exp(-((X - x) ** 2 + (Y - y) ** 2 + (Z - z) ** 2) / 0.06) for x, y, z in c) - 0.5
        f = f + 0.02 * rng.standard_normal(f.shape)
    return f.astype(np.float32)


def _mesh(kind, R, seed=0):
    v, f = mo.marching_cubes(_field(kind, R, seed), 0.0)
    rng = np.random.default_rng(seed + 1)
    return v.astype(np.float32), f, rng.random((len(v), 3)).astype(np.float32), \
        rng.standard_normal((len(v), 3)).astype(np.float32)


def _run(v, f, target, col=None, nrm=None):
    import torch
    from sugar_b200 import decimate
    t = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda()
    m = decimate.simplify_quadric_decimation(t(v), t(f), target, t(col), t(nrm))
    return {k: (x.cpu().numpy() if torch.is_tensor(x) else x) for k, x in m.items()}


CASES = [("sphere", 40), ("torus", 48), ("cut", 36), ("blobs", 56)]


@pytest.mark.parametrize("kind,R", CASES, ids=[f"{k}{r}" for k, r in CASES])
def test_kernels_equal_the_round_oracle(kind, R):
    v, f, col, nrm = _mesh(kind, R)
    F = len(f)
    assert 5_000 <= F <= 50_000, F
    for target in (F // 2, F // 10, F // 50, F, F + 10):
        want = do.decimate_rounds(v, f, target, col, nrm)
        got = _run(v, f, target, col, nrm)
        np.testing.assert_array_equal(got["faces"], want["faces"], err_msg=f"faces, target {target}")
        np.testing.assert_array_equal(got["verts"], want["verts"].astype(np.float32), err_msg=f"verts {target}")
        np.testing.assert_array_equal(got["colors"], want["colors"].astype(np.float32), err_msg=f"colors {target}")
        np.testing.assert_array_equal(got["normals"], want["normals"].astype(np.float32), err_msg=f"normals {target}")
        assert (got["rounds"], got["last_removed"]) == (want["rounds"], want["last_removed"]), target
        if target >= F:
            used = np.unique(f)
            assert got["rounds"] == 0 and np.array_equal(got["verts"], v[used])
            np.testing.assert_array_equal(got["faces"], np.searchsorted(used, f))
    got = _run(v, f, F // 10)                       # no colours or normals
    assert got["colors"] is None and got["normals"] is None
    np.testing.assert_array_equal(got["faces"], do.decimate_rounds(v, f, F // 10)["faces"])


def _point_to_mesh(points, verts, faces, k=24):
    """Distance from each point to the nearest of the k triangles whose centroids are nearest to it (numpy
    point-to-triangle distance, Ericson's closest-point regions)."""
    from scipy.spatial import cKDTree
    tri = verts[faces]
    _, idx = cKDTree(tri.mean(1)).query(points, k=min(k, len(faces)))
    idx = idx.reshape(len(points), -1)
    p = np.repeat(points[:, None], idx.shape[1], 1).reshape(-1, 3)
    a, b, c = (tri[idx.reshape(-1), i] for i in range(3))
    ab, ac, ap = b - a, c - a, p - a
    dot = lambda x, y: (x * y).sum(-1)
    d1, d2 = dot(ab, ap), dot(ac, ap)
    bp, cp = p - b, p - c
    d3, d4, d5, d6 = dot(ab, bp), dot(ac, bp), dot(ab, cp), dot(ac, cp)
    va, vb, vc = d3 * d6 - d5 * d4, d5 * d2 - d1 * d6, d1 * d4 - d3 * d2
    with np.errstate(all="ignore"):
        den = va + vb + vc
        v_, w_ = vb / den, vc / den
        q = a + ab * v_[:, None] + ac * w_[:, None]                              # inside the face
        r = d1 / (d1 - d3)
        q = np.where(((vc <= 0) & (d1 >= 0) & (d3 <= 0))[:, None], a + ab * r[:, None], q)
        r = d2 / (d2 - d6)
        q = np.where(((vb <= 0) & (d2 >= 0) & (d6 <= 0))[:, None], a + ac * r[:, None], q)
        r = (d4 - d3) / ((d4 - d3) + (d5 - d6))
        q = np.where(((va <= 0) & (d4 - d3 >= 0) & (d5 - d6 >= 0))[:, None], b + (c - b) * r[:, None], q)
    q = np.where(((d1 <= 0) & (d2 <= 0))[:, None], a, q)
    q = np.where(((d3 >= 0) & (d4 <= d3))[:, None], b, q)
    q = np.where(((d6 >= 0) & (d5 <= d6))[:, None], c, q)
    return np.linalg.norm(p - q, axis=1).reshape(len(points), -1).min(1)


@pytest.mark.parametrize("kind,R", [("torus", 52), ("blobs", 72)], ids=["torus52", "blobs72"])
@pytest.mark.parametrize("frac", [0.1, 0.02])
def test_quality_against_the_sequential_greedy(kind, R, frac):
    v, f, _, _ = _mesh(kind, R, seed=4)
    F = len(f)
    assert 10_000 <= F <= 50_000, F
    target = int(F * frac)
    got = _run(v, f, target)
    ref = do.decimate_greedy(v, f, target)
    assert len(got["faces"]) <= target
    e_gpu = _point_to_mesh(v.astype(np.float64), got["verts"].astype(np.float64), got["faces"])
    e_seq = _point_to_mesh(v.astype(np.float64), ref["verts"], ref["faces"])
    ratios = e_gpu.mean() / e_seq.mean(), e_gpu.max() / e_seq.max()
    print(f"{kind}{R} F={F} target={target} rounds={got['rounds']} mean {e_gpu.mean():.4g} vs {e_seq.mean():.4g} "
          f"max {e_gpu.max():.4g} vs {e_seq.max():.4g} ratios {ratios[0]:.3f} {ratios[1]:.3f}")
    assert ratios[0] <= 1.5 and ratios[1] <= 1.5, ratios


def _edge_counts(faces):
    import torch
    e = torch.sort(torch.stack([faces, faces.roll(-1, 1)], 2).reshape(-1, 2), dim=1)[0]
    return torch.unique(e, dim=0, return_counts=True)[1]


@pytest.mark.parametrize("target", [1_000_000, 200_000])
def test_512_marching_cubes_meshes_decimated_to_the_presets(target):
    import torch
    from sugar_b200 import decimate, mcubes
    g = torch.linspace(-1, 1, 512, device="cuda")
    X, Y, Z = torch.meshgrid(g, g, g, indexing="ij")
    r = torch.sqrt(X ** 2 + Y ** 2 + Z ** 2)
    shell = torch.minimum(0.8 - r, r - 0.5)                  # a sphere of radius 0.8 with a cavity of radius 0.5
    torus = 0.1 - torch.sqrt((torch.sqrt(X ** 2 + Y ** 2) - 0.3) ** 2 + Z ** 2)   # inside the cavity
    vol = torch.maximum(shell, torus).float().contiguous()
    del X, Y, Z, r, shell, torus
    vi, faces = mcubes.marching_cubes(vol, 0.0)
    del vol
    verts = vi * (2.0 / 511) - 1.0
    F = faces.shape[0]
    assert F > target
    m = decimate.simplify_quadric_decimation(verts, faces, target)
    nf = m["faces"].shape[0]
    print(f"512^3 spheres + torus: F={F} -> {nf} in {m['rounds']} rounds (last collapse removed {m['last_removed']})")
    assert nf <= target < nf + m["last_removed"]
    again = decimate.simplify_quadric_decimation(verts, faces, target)
    assert torch.equal(m["faces"], again["faces"]) and torch.equal(m["verts"], again["verts"])
    assert m["rounds"] == again["rounds"]
    c = decimate.clean_mesh(m["verts"], m["faces"])
    cf = c["faces"]
    cnt = _edge_counts(cf)
    assert int(cnt.min()) >= 1 and int(cnt.max()) <= 2
    assert bool(((cf[:, 0] != cf[:, 1]) & (cf[:, 1] != cf[:, 2]) & (cf[:, 0] != cf[:, 2])).all())
    rot = (cf.argmin(dim=1, keepdim=True) + torch.arange(3, device="cuda")) % 3
    assert torch.unique(cf.gather(1, rot), dim=0).shape[0] == cf.shape[0]


def test_extraction_with_decimation_to_refinement_and_texture():
    """Coarse model -> marching cubes at 96^3 decimated and cleaned per part -> one refinement step -> UV texture."""
    import torch
    from types import SimpleNamespace
    from sugar_b200 import mcubes, meshbind, scenes, steps, texture
    W, H = 160, 96
    sc = scenes.make_scene(6000, W, H, seed=8, px_sigma=25.0, frac_behind=0.0, zrange=(3.0, 6.0))
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    a = steps.activate(dict(points=t(sc.means3D), sh_dc=t(sc.shs[:, :1]), sh_rest=t(sc.shs[:, 1:]),
                            densities=t(np.log(sc.opacities / (1 - sc.opacities))), scales=t(np.log(sc.scales)),
                            quaternions=t(sc.rotations)))
    args = (a.points, a.scaling, a.quaternions, a.strengths, a.sh[:, :1], 8.0)
    full = mcubes.extract_mesh_marching_cubes(*args, resolution=96)
    T = full["foreground"]["faces"].shape[0] // 4
    assert T > 100
    out = mcubes.extract_mesh_marching_cubes(*args, resolution=96, decimation_target=T)
    for part in ("foreground", "background"):
        m = out[part]
        assert m["faces"].shape[0] <= T
        assert m["colors"].shape == m["verts"].shape == m["normals"].shape
        assert float(m["colors"].min()) >= 0.0 and float(m["colors"].max()) <= 1.0
    m = out["combined"]
    assert m["faces"].shape[0] == out["foreground"]["faces"].shape[0] + out["background"]["faces"].shape[0]
    verts, faces = m["verts"], m["faces"]
    F = faces.shape[0]
    cam = steps.camera_from_scene(sc, "cuda")
    gt = torch.rand(3, H, W, device="cuda")
    g = torch.Generator().manual_seed(0)
    rr = dict(verts=verts.clone().requires_grad_(True),
              sh_dc=(0.5 * torch.randn(F, 1, 3, generator=g)).cuda().requires_grad_(True),
              sh_rest=(0.1 * torch.randn(F, 15, 3, generator=g)).cuda().requires_grad_(True),
              densities=torch.randn(F, 1, generator=g).cuda().requires_grad_(True),
              scales=(torch.randn(F, 2, generator=g) * 0.3 - 2.0).cuda().requires_grad_(True),
              quaternions=torch.randn(F, 2, generator=g).cuda().requires_grad_(True))
    mesh = SimpleNamespace(faces=faces, bary=meshbind.bary_coords(1, "cuda"), thickness=1e-5)
    loss, stats = steps.refine_step(rr, mesh, cam, gt, steps.ours_ops())
    assert torch.isfinite(loss) and stats["visible"] > 0 and rr["verts"].grad is not None
    b = meshbind.bind_to_mesh(rr["verts"].detach(), faces, mesh.bary, rr["scales"].detach(),
                              rr["quaternions"].detach(), mesh.thickness)
    verts_uv, faces_uv, tex = texture.extract_texture_image_and_uv_from_gaussians(
        rr["verts"].detach(), faces, b.points.detach(), b.scaling.detach(), b.quaternions.detach(),
        torch.sigmoid(rr["densities"].detach()), rr["sh_dc"].detach(), [cam], square_size=4)
    assert tex.shape[0] == tex.shape[1] == texture.texture_size(F, 4) and bool(torch.isfinite(tex).all())
    assert faces_uv.shape == (F, 3)
