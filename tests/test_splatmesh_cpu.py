"""CPU checks of the splatted mesh and the nearest-face z-buffer: the float64 restatement (oracle/splatmesh_oracle.py)
pinned by properties with known answers and against the reference's own vertex lines (tests/golden/splatmesh_*.npz),
the C entry points and prototypes without a GPU, and the Python entry points' argument validation."""
import ctypes
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import splatmesh_oracle as smo  # noqa: E402
from sugar_b200 import scenes  # noqa: E402

W, H = 64, 48
GOLDEN = ["posed_500", "flat_2000", "offaxis_2000"]


def camera(W=W, H=H, pose="identity", seed=0):
    sc = scenes.make_scene(10, W, H, seed=seed, camera=pose)
    return sc


def at_pixel(sc, px, py, z):
    """World point (identity camera) whose projection is the pixel coordinate (px, py) at view depth z."""
    ndc_x, ndc_y = (2.0 * px + 1.0) / sc.width - 1.0, (2.0 * py + 1.0) / sc.height - 1.0
    return [ndc_x * sc.tanfovx * (z + 1e-7), ndc_y * sc.tanfovy * (z + 1e-7), z]


def raster(sc, verts, faces):
    return smo.rasterize(np.asarray(verts, np.float64), np.asarray(faces), sc.viewmatrix, sc.projmatrix, sc.width,
                         sc.height)


def test_projection_convention():
    sc = camera()
    v = np.array([at_pixel(sc, 10.25, 7.5, 3.0), at_pixel(sc, 0.0, 47.0, 0.5)])
    x, y, z = smo.project(v, sc.viewmatrix, sc.projmatrix, W, H)
    assert np.allclose(x, [10.25, 0.0], atol=1e-5) and np.allclose(y, [7.5, 47.0], atol=1e-5) and np.allclose(z, [3, 0.5])


def test_axis_parallel_quad_covers_exactly_its_interior():
    sc = camera()
    x0, x1, y0, y1, z = 10.3, 30.7, 5.6, 20.2, 4.0
    verts = [at_pixel(sc, x0, y0, z), at_pixel(sc, x1, y0, z), at_pixel(sc, x1, y1, z), at_pixel(sc, x0, y1, z)]
    out = raster(sc, verts, [[0, 1, 2], [0, 2, 3]])
    jj, ii = np.mgrid[0:H, 0:W]
    inside = (ii > x0) & (ii < x1) & (jj > y0) & (jj < y1)
    # the shared diagonal passes through no sample point, so the two triangles tile the interior
    assert np.abs((jj - y0) * (x1 - x0) - (ii - x0) * (y1 - y0))[inside].min() > 1e-3
    assert np.array_equal(out["pix_to_face"] >= 0, inside)
    assert np.allclose(out["zbuf"][inside], z, rtol=1e-12) and (out["zbuf"][~inside] == -1).all()
    assert set(np.unique(out["pix_to_face"][inside])) == {0, 1}


def test_tilted_triangle_depth_is_the_ray_plane_intersection():
    sc = camera(pose="posed", seed=3)
    Vt = sc.viewmatrix.astype(np.float64)             # row-vector world -> view
    view_pts = np.array([[-1.5, -1.0, 3.0], [2.0, -0.5, 6.0], [0.0, 1.5, 4.5]])
    inv = np.linalg.inv(Vt)
    verts = view_pts @ inv[:3, :3] + inv[3, :3]
    out = raster(sc, verts, [[0, 1, 2]])
    n = np.cross(view_pts[1] - view_pts[0], view_pts[2] - view_pts[0])
    c = n @ view_pts[0]
    jj, ii = np.mgrid[0:H, 0:W]
    cov = out["pix_to_face"] == 0
    assert cov.sum() > 200
    d = np.stack([((2 * ii + 1) / W - 1) * sc.tanfovx, ((2 * jj + 1) / H - 1) * sc.tanfovy, np.ones_like(ii, float)], -1)
    t = c / (d @ n)
    assert np.allclose(out["zbuf"][cov], t[cov], rtol=1e-6)


@pytest.mark.parametrize("order", [(0, 1), (1, 0)])
def test_the_nearer_of_two_overlapping_faces_wins(order):
    sc = camera()
    tri = lambda z, s: [at_pixel(sc, 5 + s, 5, z), at_pixel(sc, 55 + s, 8, z), at_pixel(sc, 20 + s, 44, z)]
    near, far = tri(2.0, 0.0), tri(5.0, 3.0)
    faces_verts = [near, far]
    verts = faces_verts[order[0]] + faces_verts[order[1]]
    out = raster(sc, verts, [[0, 1, 2], [3, 4, 5]])
    near_id = order.index(0)
    alone = raster(sc, near, [[0, 1, 2]])["pix_to_face"] == 0
    assert alone.sum() > 300
    assert (out["pix_to_face"][alone] == near_id).all() and np.allclose(out["zbuf"][alone], 2.0)
    rest = (out["pix_to_face"] >= 0) & ~alone
    assert rest.sum() > 0 and (out["pix_to_face"][rest] == 1 - near_id).all()
    assert np.isfinite(out["depth_gap"][alone & (out["depth_gap"] < np.inf)]).all()


def test_faces_behind_the_camera_and_zero_area_faces_are_ignored():
    sc = camera()
    behind = [[-1.0, -1.0, -2.0], [1.0, -1.0, -2.0], [0.0, 1.0, -3.0]]        # all z < 0
    flat = [at_pixel(sc, 5, 5, 3.0), at_pixel(sc, 30, 20, 3.0), at_pixel(sc, 55, 35, 3.0)]   # collinear
    out = raster(sc, behind + flat, [[0, 1, 2], [3, 4, 5]])
    assert (out["pix_to_face"] == -1).all() and (out["zbuf"] == -1).all()
    # the same faces moved in front of the camera / opened up are drawn
    front = [[-1.0, -1.0, 2.0], [1.0, -1.0, 2.0], [0.0, 1.0, 3.0]]
    opened = [at_pixel(sc, 5, 5, 3.0), at_pixel(sc, 30, 25, 3.0), at_pixel(sc, 55, 35, 3.0)]
    out = raster(sc, front + opened, [[0, 1, 2], [3, 4, 5]])
    assert (out["pix_to_face"] == 0).any() and (out["pix_to_face"] == 1).any()


def test_the_two_triangles_of_a_diamond_tile_it_without_overlap():
    sc = camera(W=96, H=80)
    pts = torch.tensor([[0.1, -0.05, 3.0]], dtype=torch.float64)
    sca = torch.tensor([[0.01, 0.4, 0.3]], dtype=torch.float64)
    q = torch.nn.functional.normalize(torch.tensor([[0.9, 0.2, -0.3, 0.1]], dtype=torch.float64), dim=-1)
    verts, faces = smo.splat_mesh(pts, sca, q, torch.from_numpy(sc.viewmatrix))
    assert faces.tolist() == [[0, 2, 1], [0, 3, 2]]
    both = raster(sc, verts, faces)
    f0 = raster(sc, verts, faces[:1])["pix_to_face"] == 0
    f1 = raster(sc, verts, faces[1:])["pix_to_face"] == 0
    assert f0.sum() > 50 and f1.sum() > 50 and not (f0 & f1).any()
    assert np.array_equal(both["pix_to_face"] >= 0, f0 | f1)
    # the splatted diamond is planar, perpendicular to the centre's ray, and through the centre
    vv = verts.numpy() @ sc.viewmatrix[:3, :3].astype(np.float64) + sc.viewmatrix[3, :3]
    c = pts.numpy()[0] @ sc.viewmatrix[:3, :3].astype(np.float64) + sc.viewmatrix[3, :3]
    assert np.allclose((vv - c) @ (c / np.linalg.norm(c)), 0.0, atol=1e-12)


@pytest.mark.parametrize("name", GOLDEN)
def test_oracle_vertices_match_the_reference_golden(name):
    g = np.load(os.path.join(HERE, "golden", f"splatmesh_{name}.npz"))
    t = lambda k: torch.from_numpy(g[k]).double()
    q = torch.nn.functional.normalize(t("quaternions"), dim=-1)
    verts, faces = smo.splat_mesh(t("points"), t("scaling"), q, t("viewmatrix"))
    ref = g["verts"]
    assert verts.shape == ref.shape and faces.shape == (ref.shape[0] // 2, 3)
    err = np.abs(verts.numpy() - ref).max(1) / np.maximum(1.0, np.abs(ref).max(1))
    assert err.max() < 1e-9, err.max()


def test_library_lists_the_new_entry_points():
    from sugar_b200 import _lib
    L = _lib.lib
    for fn in ("sgr_splat_mesh", "sgr_mesh_raster_scratch_bytes", "sgr_mesh_raster"):
        assert fn in _lib.PROTOTYPES and hasattr(L, fn)
    names = [L.sgr_kernel_name(k).decode() for k in range(L.sgr_num_kernel_kinds())]
    assert "misc" in names and names[-2:] == ["mesh_nc_forward", "mesh_nc_backward"]   # no kind was added
    assert L.sgr_mesh_raster_scratch_bytes(-1, 10, 10) == 0
    assert L.sgr_mesh_raster_scratch_bytes(1000, 640, 480) >= 8 * 640 * 480 + 64 * 1000
    assert L.sgr_mesh_raster_scratch_bytes(1000, 640, 480) < L.sgr_mesh_raster_scratch_bytes(100_000, 640, 480)
    dummy = ctypes.c_void_p(256)
    assert L.sgr_splat_mesh(0, *([None] * 5), 2.0, None, None) == 0                 # P = 0: nothing to do
    assert L.sgr_splat_mesh(-1, *([dummy] * 5), 2.0, dummy, None) == -1 and b"bad size" in L.sgr_last_error()
    assert L.sgr_splat_mesh(4, *([dummy] * 4), None, 2.0, dummy, None) == -1 and b"null" in L.sgr_last_error()
    assert L.sgr_splat_mesh(4, *([dummy] * 5), 2.0, ctypes.c_void_p(264), None) == -1           # misaligned verts
    assert L.sgr_mesh_raster(3, -1, *([dummy] * 4), 8, 8, dummy, dummy, dummy, None) == -1
    assert L.sgr_mesh_raster(3, 1, *([dummy] * 4), 70000, 8, dummy, dummy, dummy, None) == -1
    assert b"bad sizes" in L.sgr_last_error()
    assert L.sgr_mesh_raster(3, 1, *([dummy] * 4), 8, 8, dummy, None, dummy, None) == -1
    assert b"null pointer" in L.sgr_last_error()
    assert L.sgr_mesh_raster(3, 1, *([dummy] * 4), 0, 8, None, None, None, None) == 0     # no pixels


def test_python_entry_points_validate_arguments():
    from sugar_b200 import levelset, splatmesh, steps
    cam = steps.camera_from_scene(camera(), "cpu")
    v = torch.zeros(6, 3)
    f = torch.tensor([[0, 1, 2], [3, 4, 5]])
    with pytest.raises(ValueError, match="faces must be int64"):
        splatmesh.rasterize_mesh(v, f.int(), cam)
    with pytest.raises(ValueError, match="verts must be float32"):
        splatmesh.rasterize_mesh(v.double(), f, cam)
    with pytest.raises(ValueError, match=r"faces must be int64 \[F,3\]"):
        splatmesh.rasterize_mesh(v, f[:, :2], cam)
    with pytest.raises(ValueError, match="outside"):
        splatmesh.rasterize_mesh(v, torch.tensor([[0, 1, 6]]), cam)
    with pytest.raises(ValueError, match="outside"):
        splatmesh.rasterize_mesh(v, torch.tensor([[0, -1, 2]]), cam)
    with pytest.raises(ValueError, match="image"):
        splatmesh.rasterize_mesh(v, f, SimpleNamespace(**{**vars(cam), "width": 0}))
    with pytest.raises(ValueError, match="projmatrix"):
        splatmesh.rasterize_mesh(v, f, SimpleNamespace(**{**vars(cam), "projmatrix": cam.projmatrix.double()}))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        splatmesh.rasterize_mesh(v, f, cam)
    p, s, q = torch.zeros(4, 3), torch.ones(4, 3), torch.tensor([[1.0, 0, 0, 0]]).repeat(4, 1)
    with pytest.raises(ValueError, match="quaternions"):
        splatmesh.splat_mesh(p, s, q[:, :3], cam)
    with pytest.raises(ValueError, match="scaling"):
        splatmesh.splat_mesh(p, s[:3], q, cam)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        splatmesh.splat_mesh(p, s, q, cam)
    strengths = torch.ones(4)
    with pytest.raises(ValueError, match="knn_idx"):
        levelset.level_surface_points_from_camera(p, s, q, strengths, cam, use_gaussian_depth=False)
    with pytest.raises(ValueError, match="knn_idx must be int64"):
        levelset.level_surface_points_from_camera(p, s, q, strengths, cam, use_gaussian_depth=False,
                                                  knn_idx=torch.zeros(4, 16, dtype=torch.int32))
