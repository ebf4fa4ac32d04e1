"""GPU: the splatted diamond mesh (sugar_b200/splatmesh.py, csrc/sgr_splatmesh.cu) against the reference's own vertex
lines (golden), the nearest-face z-buffer against its float64 oracle (oracle/splatmesh_oracle.py), and the level-set
call's mesh-depth branch (use_gaussian_depth=False)."""
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import splatmesh_oracle as smo  # noqa: E402


def cam_of(sc_or_npz, W=None, H=None):
    g = sc_or_npz
    get = (lambda k: g[k]) if isinstance(g, dict) or hasattr(g, "files") else (lambda k: getattr(g, k))
    t = lambda k: torch.from_numpy(np.asarray(get(k), np.float32)).cuda()
    return SimpleNamespace(viewmatrix=t("viewmatrix"), projmatrix=t("projmatrix"), campos=t("campos"),
                           width=int(W or get("width")), height=int(H or get("height")))


@pytest.mark.parametrize("name", ["posed_500", "flat_2000", "offaxis_2000"])
def test_splat_vertices_match_reference_golden(name):
    from sugar_b200 import splatmesh
    g = np.load(os.path.join(HERE, "golden", f"splatmesh_{name}.npz"))
    c = lambda k: torch.from_numpy(g[k]).cuda()
    verts, faces = splatmesh.splat_mesh(c("points"), c("scaling"), c("quaternions"), cam_of(g))
    ref = g["verts"]
    P = g["points"].shape[0]
    assert faces.tolist() == [[4 * p + a, 4 * p + b, 4 * p + e] for p in range(P) for a, b, e in ((0, 2, 1), (0, 3, 2))]
    # the reference divides by v.d: where that is tiny against |v| its own rounding is amplified without bound
    t = lambda k: torch.from_numpy(g[k]).double()
    q = torch.nn.functional.normalize(t("quaternions"), dim=-1)
    view = t("viewmatrix")
    tv = (smo.triangle_vertices(t("points"), t("scaling"), q) @ view[:3, :3] + view[3, :3]).numpy()
    cv = (t("points") @ view[:3, :3] + view[3, :3]).numpy()
    d = np.repeat(cv / np.linalg.norm(cv, axis=1, keepdims=True), 4, axis=0)
    keep = np.abs((tv * d).sum(1)) >= 1e-3 * np.linalg.norm(tv, axis=1)
    print(f"{name}: {int((~keep).sum())} of {len(keep)} vertices excluded (|v.d| < 1e-3 |v|)")
    assert keep.mean() > 0.99
    err = np.abs(verts.cpu().numpy().astype(np.float64) - ref).max(1)
    assert (err[keep] <= 1e-5 * np.maximum(1.0, np.abs(ref[keep]).max(1))).all(), err[keep].max()


def hand_made(W, H):
    """Seeded triangles of all sizes and tilts in front of an identity camera, some overlapping, some crossing the
    image border, a degenerate one and one behind the camera."""
    from sugar_b200 import scenes
    sc = scenes.make_scene(10, W, H, seed=0)
    rng = np.random.default_rng(7)
    v = []
    for _ in range(40):
        z = rng.uniform(1.0, 8.0, 3)
        px, py = rng.uniform(-10, W + 10, 3), rng.uniform(-10, H + 10, 3)
        v += [[((2 * x + 1) / W - 1) * sc.tanfovx * zz, ((2 * y + 1) / H - 1) * sc.tanfovy * zz, zz]
              for x, y, zz in zip(px, py, z)]
    v += [[0, 0, 2.0], [0.5, 0.5, 2.0], [1.0, 1.0, 2.0], [-1, -1, -2.0], [1, -1, -2.0], [0, 1, -3.0]]
    verts = np.asarray(v, np.float32)
    return sc, verts, np.arange(len(v)).reshape(-1, 3)


def splat_case(P, W, H, seed):
    from sugar_b200 import scenes, splatmesh
    sc = scenes.make_scene(P, W, H, seed=seed, camera="posed")
    c = lambda a: torch.from_numpy(a).cuda()
    verts, faces = splatmesh.splat_mesh(c(sc.means3D), c(sc.scales), c(sc.rotations), cam_of(sc))
    return sc, verts.cpu().numpy(), faces.cpu().numpy()


def compare_with_oracle(sc, verts, faces, label):
    from sugar_b200 import splatmesh
    cam = cam_of(sc)
    zbuf, p2f = splatmesh.rasterize_mesh(torch.from_numpy(verts).cuda(), torch.from_numpy(faces).cuda(), cam)
    zbuf, p2f = zbuf.cpu().numpy(), p2f.cpu().numpy()
    ref = smo.rasterize(verts.astype(np.float64), faces, sc.viewmatrix, sc.projmatrix, sc.width, sc.height)
    rz = ref["zbuf"]
    clean = (ref["bary_margin"] > 1e-4) & ~(ref["depth_gap"] <= 1e-5 * np.abs(rz))
    same = p2f == ref["pix_to_face"]
    print(f"{label}: {int(clean.sum())} clean of {clean.size} pixels, {int((~same).sum())} disagree, "
          f"{int((ref['pix_to_face'] >= 0).sum())} covered")
    assert (ref["pix_to_face"] >= 0).sum() > 0.05 * clean.size
    assert same[clean].all(), np.argwhere(clean & ~same)[:10]
    cov = clean & (p2f >= 0)
    assert (np.abs(zbuf[cov] - rz[cov]) <= 1e-5 * np.abs(rz[cov])).all()
    assert (zbuf[p2f < 0] == -1).all()
    assert same.mean() >= 0.999
    assert clean[(p2f >= 0) != (ref["pix_to_face"] >= 0)].sum() == 0      # coverage differs at margin pixels only
    return zbuf, p2f


def test_rasterizer_matches_oracle_hand_made_64x48():
    compare_with_oracle(*hand_made(64, 48), "hand-made 64x48")


def test_rasterizer_matches_oracle_splat_mesh_2k_320x240():
    compare_with_oracle(*splat_case(2000, 320, 240, seed=41), "2k Gaussians 320x240")


def test_rasterizer_matches_oracle_and_is_deterministic_120k_faces_640x480():
    from sugar_b200 import splatmesh
    sc, verts, faces = splat_case(60_000, 640, 480, seed=42)
    assert faces.shape[0] >= 100_000
    zbuf, p2f = compare_with_oracle(sc, verts, faces, "60k Gaussians 640x480")
    z2, f2 = splatmesh.rasterize_mesh(torch.from_numpy(verts).cuda(), torch.from_numpy(faces).cuda(), cam_of(sc))
    assert np.array_equal(zbuf.view(np.uint32), z2.cpu().numpy().view(np.uint32))
    assert np.array_equal(p2f, f2.cpu().numpy())


def test_edge_sizes():
    from sugar_b200 import splatmesh
    sc, verts, faces = splat_case(3000, 67, 41, seed=43)          # neither side a multiple of any block size
    compare_with_oracle(sc, verts, faces, "3k Gaussians 67x41")
    cam = cam_of(sc)
    e = torch.empty(0, 3, device="cuda")
    v0, f0 = splatmesh.splat_mesh(e, e, torch.empty(0, 4, device="cuda"), cam)
    assert v0.shape == (0, 3) and f0.shape == (0, 3) and f0.dtype == torch.int64
    z, f = splatmesh.rasterize_mesh(v0, f0, cam)
    assert z.shape == (41, 67) and (z == -1).all() and (f == -1).all()
    with pytest.raises(ValueError, match="outside"):
        splatmesh.rasterize_mesh(torch.from_numpy(verts).cuda(), torch.tensor([[0, 1, len(verts)]], device="cuda"), cam)


def sheet():
    from sugar_b200 import scenes, steps
    W, H, P = 160, 96, 60_000
    sc = scenes.make_scene(1000, W, H, seed=0)
    g = torch.Generator().manual_seed(0)
    xy = (torch.rand(P, 2, generator=g) - 0.5) * torch.tensor([2 * 5 * sc.tanfovx, 2 * 5 * sc.tanfovy]) * 1.1
    pts = torch.cat([xy, torch.full((P, 1), 5.0)], 1).cuda()
    scaling = torch.tensor([0.06, 0.06, 0.004]).repeat(P, 1).cuda()
    quats = torch.tensor([1.0, 0.0, 0.0, 0.0]).repeat(P, 1).cuda()
    strengths = torch.full((P,), 0.95).cuda()
    return pts, scaling, quats, strengths, steps.camera_from_scene(sc, "cuda"), W, H


def test_level_surface_points_mesh_depth_finds_the_sheet():
    from sugar_b200 import knn, levelset, splatmesh
    pts, scaling, quats, strengths, cam, W, H = sheet()
    knn_idx = knn.reset_neighbors(pts, 16)[1]
    out = levelset.level_surface_points_from_camera(pts, scaling, quats, strengths, cam, surface_levels=(0.3,),
                                                    return_normals=True, return_pixel_idx=True,
                                                    return_gaussian_idx=True, use_gaussian_depth=False,
                                                    knn_idx=knn_idx)[0.3]
    n_valid = int(out["valid"].sum())
    assert n_valid > 0.8 * W * H and out["pixel_idx"].numel() == n_valid == out["gaussian_idx"].numel()
    z = out["intersection_points"][:, 2]
    assert float((z - 5.0).abs().quantile(0.99)) < 0.02
    assert float(out["normals"][:, 2].abs().quantile(0.05)) > 0.95
    verts, faces = splatmesh.splat_mesh(pts, scaling, quats, cam)
    _, p2f = splatmesh.rasterize_mesh(verts, faces, cam)
    assert torch.equal(out["gaussian_idx"], p2f.view(-1)[out["pixel_idx"]] // 2)
    sub = levelset.level_surface_points_from_camera(pts, scaling, quats, strengths, cam, surface_levels=(0.3,),
                                                    n_surface_points=1000, use_gaussian_depth=False,
                                                    knn_idx=knn_idx)[0.3]
    assert sub["valid"].numel() == 1000


def random_scene():
    from sugar_b200 import knn, scenes, steps
    sc = scenes.make_scene(20_000, 320, 240, seed=44, camera="posed")
    c = lambda a: torch.from_numpy(a).cuda()
    pts, scaling, quats, strengths = c(sc.means3D), c(sc.scales), c(sc.rotations), c(sc.opacities[:, 0])
    return pts, scaling, quats, strengths, steps.camera_from_scene(sc, "cuda"), knn.reset_neighbors(pts, 16)[1]


def test_level_surface_points_mesh_depth_is_the_manual_composition():
    from sugar_b200 import levelset, splatmesh
    pts, scaling, quats, strengths, cam, knn_idx = random_scene()
    levels = (0.1, 0.3, 0.5)
    out = levelset.level_surface_points_from_camera(pts, scaling, quats, strengths, cam, surface_levels=levels,
                                                    return_normals=True, return_pixel_idx=True,
                                                    return_gaussian_idx=True, use_gaussian_depth=False,
                                                    knn_idx=knn_idx)
    W, H = cam.width, cam.height
    verts, faces = splatmesh.splat_mesh(pts, scaling, quats, cam)
    zbuf, p2f = splatmesh.rasterize_mesh(verts, faces, cam)
    keep = (zbuf >= 0).view(-1).nonzero()[:, 0]
    z = zbuf.view(-1)[keep]
    py, px = (keep // W).float(), (keep % W).float()
    xv = ((2.0 * px + 1.0) / W - 1.0) * cam.tanfovx * z
    yv = ((2.0 * py + 1.0) / H - 1.0) * cam.tanfovy * z
    world = (torch.stack([xv, yv, z], dim=1) - cam.viewmatrix[3, :3]) @ cam.viewmatrix[:3, :3].transpose(0, 1)
    gidx = p2f.view(-1)[keep] // 2
    ref = levelset.level_surface_points(world, cam.campos, knn_idx[gidx], pts, scaling, quats, strengths,
                                        surface_levels=levels, return_normals=True)
    assert keep.numel() > 0.2 * W * H
    for lv in levels:
        assert torch.equal(out[lv]["valid"], ref[lv]["valid"]) and out[lv]["valid"].any()
        assert torch.equal(out[lv]["intersection_points"], ref[lv]["intersection_points"])
        assert torch.equal(out[lv]["normals"], ref[lv]["normals"])
        assert torch.equal(out[lv]["pixel_idx"], keep[ref[lv]["valid"]])
        assert torch.equal(out[lv]["gaussian_idx"], gidx[ref[lv]["valid"]])


def test_level_surface_points_default_is_the_gaussian_depth_branch():
    from sugar_b200 import levelset
    pts, scaling, quats, strengths, cam, _ = random_scene()
    kw = dict(surface_levels=(0.3,), return_normals=True, return_pixel_idx=True)
    a = levelset.level_surface_points_from_camera(pts, scaling, quats, strengths, cam, **kw)[0.3]
    b = levelset.level_surface_points_from_camera(pts, scaling, quats, strengths, cam, use_gaussian_depth=True,
                                                  **kw)[0.3]
    assert set(a) == set(b) == {"intersection_points", "valid", "normals", "pixel_idx"}
    for k in a:
        assert torch.equal(a[k], b[k]), k
