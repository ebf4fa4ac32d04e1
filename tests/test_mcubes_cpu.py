"""CPU checks of the marching-cubes extraction: the generated case table (against the committed header and by its
properties), the numpy oracle's meshes, the golden's vertex mapping, the ABI's argument validation and the PLY writer."""
import ctypes
import glob
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import mcubes_oracle as mo  # noqa: E402

GOLDEN = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "mcubes_*.npz")))


def test_generated_table_equals_the_committed_header():
    with open(mo.HEADER) as fh:
        assert fh.read() == mo.header_text()


def test_every_case_uses_each_crossed_edge_and_winds_outward():
    ntri, tab = mo.table()
    for case in range(256):
        tris = tab[case, :3 * ntri[case]].reshape(-1, 3)
        crossed = mo.crossed_edges(case)
        assert sorted(set(tris.reshape(-1).tolist())) == crossed, case
        loops = mo.case_loops(case)
        assert sorted(e for lp in loops for e in lp) == crossed, case      # each crossed edge in exactly one loop
        assert len(tris) == sum(len(lp) - 2 for lp in loops)
        ins = [(case >> c) & 1 for c in range(8)]
        for lp in loops:
            pts = [mo._mid(e) for e in lp]
            n = sum(np.cross(a, b) for a, b in zip(pts, pts[1:] + pts[:1]))
            out = sum(mo._outward(e, ins) for e in lp)
            assert n @ out > 0, (case, lp)
        for t in tris:   # every triangle's normal points from the inside corners of its edges to the outside ones
            a, b, c = (mo._mid(e) for e in t)
            out = sum(mo._outward(e, ins) for e in t)
            assert np.cross(b - a, c - a) @ out > 0, (case, t)
    assert ntri[0] == 0 and ntri[255] == 0


@pytest.mark.parametrize("seed", range(4))
def test_random_sign_volumes_give_closed_consistently_wound_meshes(seed):
    rng = np.random.default_rng(seed)
    vol = np.pad(rng.choice([-1.0, 1.0], (11, 13, 12)), 1, constant_values=-1.0).astype(np.float32)
    v, f = mo.marching_cubes(vol, 0.0)
    counts, each_directed_once = mo.directed_edge_counts(f)
    assert len(f) > 1000 and set(counts.tolist()) == {2} and each_directed_once


def _grid(R):
    x = np.linspace(-1.0, 1.0, R)
    return np.meshgrid(x, x, x, indexing="ij"), 2.0 / (R - 1)


def test_sphere_and_torus_topology_and_area():
    (X, Y, Z), h = _grid(64)
    r = 0.7
    v, f = mo.marching_cubes((r * r - (X * X + Y * Y + Z * Z)).astype(np.float32), 0.0)
    assert mo.euler_characteristic(len(v), f) == 2
    assert abs(mo.mesh_area(v * h, f) / (4 * np.pi * r * r) - 1) < 0.01
    v, f = mo.marching_cubes((0.2 ** 2 - (np.sqrt(X * X + Y * Y) - 0.6) ** 2 - Z * Z).astype(np.float32), 0.0)
    assert mo.euler_characteristic(len(v), f) == 0


def test_vertices_lie_on_crossed_edges_in_the_documented_order():
    rng = np.random.default_rng(5)
    vol = rng.normal(size=(6, 7, 5)).astype(np.float32)
    v, f = mo.marching_cubes(vol, 0.1)
    frac = v - np.floor(v)
    assert ((frac > 0).sum(1) <= 1).all()                      # on one grid edge each
    key = np.floor(v).astype(np.int64)
    axis = np.argmax(frac, 1)
    order = (key[:, 0] * 7 + key[:, 1]) * 5 + key[:, 2]
    assert (np.diff(order * 3 + axis) > 0).all()
    assert f.min() >= 0 and f.max() < len(v)


@pytest.mark.parametrize("path", GOLDEN, ids=os.path.basename)
def test_golden_mapping_and_meshes_agree_with_the_oracle(path):
    from sugar_b200 import mcubes
    g = np.load(path)
    e, R = float(g["extent"]), int(g["resolution"])
    for pre, ext in (("fg", e), ("bg", 4 * e)):
        v, f = mo.marching_cubes(g[f"{pre}_volume"], float(g["level"]))
        np.testing.assert_array_equal(f, g[f"{pre}_faces"])
        np.testing.assert_array_equal(mcubes.grid_to_world(torch.from_numpy(v), ext, R).numpy(), g[f"{pre}_verts"])
    # the background grid's exclusion: every voxel strictly inside (-e, e)^3 is 0
    X = (torch.linspace(-1, 1, R) * 4 * e).numpy()
    inside = (X > -np.float32(e)) & (X < np.float32(e))
    assert inside.any() and (g["bg_volume"][np.ix_(inside, inside, inside)] == 0).all()


def test_camera_extent_and_vertex_normals():
    from sugar_b200 import mcubes
    c = torch.tensor([[0.0, 0, 0], [2.0, 0, 0], [1.0, 1.0, 0]])
    assert mcubes.camera_spatial_extent(c) == pytest.approx(1.1 * float(torch.norm(c - c.mean(0), dim=-1).max()))
    verts = torch.tensor([[0.0, 0, 0], [1.0, 0, 0], [0, 1.0, 0], [0, 0, 1.0], [5.0, 5, 5]])
    faces = torch.tensor([[0, 1, 2], [0, 3, 1]])      # normals +z (area 1/2) and +y... (0,3,1): (0,0,1)x(1,0,0) = +y
    n = mcubes.vertex_normals(verts, faces)
    s = np.sqrt(0.5)
    np.testing.assert_allclose(n[0].numpy(), [0, s, s], atol=1e-7)
    np.testing.assert_allclose(n[2].numpy(), [0, 0, 1], atol=1e-7)
    np.testing.assert_allclose(n[3].numpy(), [0, 1, 0], atol=1e-7)
    assert (n[4] == 0).all()


def read_ply(path):
    with open(path, "rb") as fh:
        data = fh.read()
    head, body = data.split(b"end_header\n", 1)
    lines = head.decode().splitlines()
    assert lines[:2] == ["ply", "format binary_little_endian 1.0"]
    nv = int(next(x for x in lines if x.startswith("element vertex")).split()[-1])
    nf = int(next(x for x in lines if x.startswith("element face")).split()[-1])
    tmap = {"double": "<f8", "uchar": "u1"}
    props = [(x.split()[2], tmap[x.split()[1]]) for x in lines if x.startswith("property ") and "list" not in x]
    vd = np.dtype(props)
    verts = np.frombuffer(body[:nv * vd.itemsize], vd)
    faces = np.frombuffer(body[nv * vd.itemsize:], [("n", "u1"), ("i", "<i4", (3,))], count=nf)
    assert len(body) == nv * vd.itemsize + nf * 13
    return verts, faces


def test_ply_round_trip(tmp_path):
    from sugar_b200 import mcubes
    g = torch.Generator().manual_seed(1)
    v = torch.randn(20, 3, generator=g)
    f = torch.randint(0, 20, (30, 3), generator=g)
    c = torch.rand(20, 3, generator=g)
    n = torch.nn.functional.normalize(torch.randn(20, 3, generator=g), dim=-1)
    p = str(tmp_path / "m.ply")
    mcubes.write_ply(p, v, f, c, n)
    rv, rf = read_ply(p)
    np.testing.assert_array_equal(np.stack([rv["x"], rv["y"], rv["z"]], 1), v.double().numpy())
    np.testing.assert_array_equal(np.stack([rv["nx"], rv["ny"], rv["nz"]], 1), n.double().numpy())
    np.testing.assert_array_equal(np.stack([rv["red"], rv["green"], rv["blue"]], 1),
                                  np.round(c.double().numpy() * 255).astype(np.uint8))
    assert (rf["n"] == 3).all() and (rf["i"] == f.numpy()).all()
    mcubes.write_ply(p, v, f)
    rv, rf = read_ply(p)
    assert rv.dtype.names == ("x", "y", "z") and len(rf) == 30
    with pytest.raises(ValueError):
        mcubes.write_ply(p, v, f + 20)


def test_entry_points_validate_arguments_without_gpu():
    from sugar_b200 import _lib
    L = _lib.lib
    for fn in ("sgr_density_grid", "sgr_mcubes_count", "sgr_mcubes_emit"):
        assert fn in _lib.PROTOTYPES and hasattr(L, fn)
    assert 0 < L.sgr_density_grid_workspace_bytes(1000) <= L.sgr_density_grid_workspace_bytes(100000)
    assert L.sgr_mcubes_scratch_bytes(64, 64, 64) >= 9 * 64 ** 3
    d = ctypes.c_void_p(256)
    args = lambda P, K, R: (P, d, d, d, d, K, 1.0, R, R, R, d, d, d, 0.0, d, d, None)
    assert L.sgr_density_grid(*args(10, 16, 8)) == -1                 # K > P
    assert b"sgr_density_grid" in L.sgr_last_error()
    assert L.sgr_density_grid(*args(100, 65, 8)) == -1                # K > 64
    assert L.sgr_density_grid(*args(100, 16, 1025)) == -1             # more than 2^30 voxels
    assert L.sgr_density_grid(100, None, d, d, d, 16, 1.0, 8, 8, 8, d, d, d, 0.0, d, d, None) == -1
    n = ctypes.c_int64()
    assert L.sgr_mcubes_count(0, 4, 4, d, 0.0, ctypes.byref(n), ctypes.byref(n), d, None) == -1
    assert L.sgr_mcubes_count(4, 4, 4, None, 0.0, ctypes.byref(n), ctypes.byref(n), d, None) == -1
    assert L.sgr_mcubes_emit(4, 4, 4, d, 0.0, 5, 0, None, None, d, None) == -1      # vertices without a buffer
    assert L.sgr_mcubes_emit(4, 4, 4, d, 0.0, -1, 0, d, d, d, None) == -1
    assert L.sgr_mcubes_emit(4, 4, 4, d, 0.0, 0, 0, None, None, d, None) == 0       # nothing to write


def test_python_entry_points_need_cuda():
    from sugar_b200 import mcubes
    with pytest.raises(RuntimeError, match="CUDA"):
        mcubes.marching_cubes(torch.zeros(4, 4, 4), 0.5)
    x = torch.zeros(4, 3)
    with pytest.raises(RuntimeError, match="CUDA"):
        mcubes.density_grid(x, x, torch.zeros(4, 4), torch.ones(4), torch.zeros(2), torch.zeros(2), torch.zeros(2))
