"""CPU checks of the quadric decimation: the round algorithm with one collapse per round against the sequential greedy
loop (oracle/decimate_oracle.py), the boundary quadrics on a planar square, the clean-up passes on hand-made meshes,
decimate.clean_mesh (torch) against the oracle's passes, and the ABI's argument validation."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import decimate_oracle as do  # noqa: E402
from oracle import mcubes_oracle as mo  # noqa: E402


def _mc(R, radius=0.8, noise=0.0, scale=1.0, seed=0):
    """Marching cubes of a (noisy) sphere on [-1, 1]^3 at R^3; radius > 1 cuts it open at the grid box."""
    g = np.linspace(-1, 1, R)
    X, Y, Z = np.meshgrid(g, g, g, indexing="ij")
    f = radius - np.sqrt(X ** 2 + Y ** 2 + Z ** 2)
    if noise:
        f = f + noise * np.random.default_rng(seed).standard_normal(f.shape)
    v, fc = mo.marching_cubes(f.astype(np.float32), 0.0)
    return (v * scale).astype(np.float32), fc


def _grid(n, jitter=0.0, seed=0):
    """A flat n x n vertex grid on the unit square (z = 0), two triangles per cell."""
    x = np.linspace(0, 1, n)
    X, Y = np.meshgrid(x, x, indexing="ij")
    v = np.stack([X.ravel(), Y.ravel(), np.zeros(n * n)], 1)
    if jitter:
        inner = (v[:, 0] > 0) & (v[:, 0] < 1) & (v[:, 1] > 0) & (v[:, 1] < 1)
        v[inner, :2] += jitter * np.random.default_rng(seed).uniform(-1, 1, (inner.sum(), 2)) / n
    i, j = np.meshgrid(np.arange(n - 1), np.arange(n - 1), indexing="ij")
    a = (i * n + j).ravel()
    f = np.concatenate([np.stack([a, a + n, a + n + 1], 1), np.stack([a, a + n + 1, a + 1], 1)])
    return v.astype(np.float32), f.astype(np.int64)


def _attrs(V, seed):
    rng = np.random.default_rng(seed)
    return rng.random((V, 3)).astype(np.float32), rng.standard_normal((V, 3)).astype(np.float32)


MESHES = {
    "sphere_r16": lambda: _mc(16),
    "sphere_r20_world": lambda: _mc(20, scale=0.05),          # small faces: |det| <= 1e-4, the non-invertible rule
    "cut_open_r18": lambda: _mc(18, radius=1.15),             # surface cut open by the grid box: boundary quadrics
    "noisy_sphere_r16": lambda: _mc(16, noise=0.05, seed=3),
    "flat_grid": lambda: _grid(14),
    "jittered_grid": lambda: _grid(12, jitter=0.3, seed=1),
}


def _same(x, y):
    for k in ("verts", "faces", "colors", "normals", "last_removed"):
        if isinstance(x[k], np.ndarray):
            np.testing.assert_array_equal(x[k], y[k], err_msg=k)
        else:
            assert x[k] == y[k], k


@pytest.mark.parametrize("name", sorted(MESHES))
@pytest.mark.parametrize("frac", [0.5, 0.1])
def test_rounds_with_one_collapse_per_round_equal_the_greedy_loop(name, frac):
    v, f = MESHES[name]()
    col, nrm = _attrs(len(v), 7)
    target = int(len(f) * frac)
    g = do.decimate_greedy(v, f, target, col, nrm)
    r = do.decimate_rounds(v, f, target, col, nrm, max_collapses_per_round=1)
    _same(g, r)
    assert len(g["faces"]) <= target and len(g["faces"]) > target - g["last_removed"]


def test_both_invertibility_branches_occur():
    """The index-space sphere solves for the optimum; the world-scale one (faces ~1e-3) never passes |det| > 1e-4."""
    for name, want in (("sphere_r16", True), ("sphere_r20_world", False)):
        v, f = MESHES[name]()
        P, F = do._check(v, f)
        Q = do.initial_quadrics(P, F)
        q = Q[F[:, 0]] + Q[F[:, 1]]
        A00, A01, A02, A11, A12, A22 = (q[:, i] for i in range(6))
        det = A00 * (A11 * A22 - A12 * A12) + A01 * (A02 * A12 - A01 * A22) + A02 * (A01 * A12 - A02 * A11)
        assert bool((np.abs(det) > do.INV_DET).any()) == want, name


def test_parallel_rounds_reach_the_target_in_fewer_rounds():
    v, f = _mc(20)
    r = do.decimate_rounds(v, f, len(f) // 10)
    assert len(r["faces"]) <= len(f) // 10 < len(r["faces"]) + r["last_removed"]
    assert 0 < r["rounds"] < len(f) // 20
    assert do.decimate_rounds(v, f, len(f))["rounds"] == 0


@pytest.mark.parametrize("algo", ["greedy", "rounds"])
def test_decimated_square_keeps_its_outline(algo):
    v, f = _grid(16, jitter=0.3, seed=2)
    fn = do.decimate_greedy if algo == "greedy" else do.decimate_rounds
    m = fn(v, f, 40)
    P, F = m["verts"], m["faces"]
    assert len(F) <= 40
    np.testing.assert_allclose(P[:, 2], 0.0, atol=1e-12)
    e = np.sort(np.concatenate([F[:, [0, 1]], F[:, [1, 2]], F[:, [2, 0]]]), 1)
    u, c = np.unique(e, axis=0, return_counts=True)
    on_boundary = np.unique(u[c == 1])
    d = np.min(np.abs(np.stack([P[:, 0], P[:, 0] - 1, P[:, 1], P[:, 1] - 1], 1)), 1)
    assert d[on_boundary].max() <= 1e-12
    for corner in ((0, 0), (0, 1), (1, 0), (1, 1)):
        assert np.abs(P[:, :2] - corner).max(1).min() <= 1e-12, corner
    assert np.isclose(do.triangle_areas(P, F).sum(), 1.0, atol=1e-9)


def test_decimation_rejects_bad_faces():
    v, f = _grid(4)
    with pytest.raises(ValueError):
        do.decimate_rounds(v, np.array([[0, 1, 1]]), 0)
    with pytest.raises(ValueError):
        do.decimate_greedy(v, np.array([[0, 1, 99]]), 0)


# ---------------------------------------------------------------------------------------------------------------------
# clean-up passes
# ---------------------------------------------------------------------------------------------------------------------
def test_duplicated_triangles_up_to_rotation_not_reflection():
    f = np.array([[0, 1, 2], [1, 2, 0], [2, 0, 1], [0, 2, 1], [1, 2, 3], [2, 1, 0]])
    np.testing.assert_array_equal(do.remove_duplicated_triangles(f), [[0, 1, 2], [0, 2, 1], [1, 2, 3]])
    np.testing.assert_array_equal(do.remove_degenerate_triangles([[0, 1, 1], [0, 1, 2], [3, 3, 3], [2, 0, 2]]),
                                  [[0, 1, 2]])


def test_coincident_vertices_are_merged_into_the_first():
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [1, 0, 0], [-0.0, 0, 0], [0, 0, 1]], np.float64)
    c = np.arange(18, dtype=np.float64).reshape(6, 3)
    P, F, C, _ = do.remove_duplicated_vertices(v, [[0, 1, 2], [4, 3, 5]], c, None)
    np.testing.assert_array_equal(P, v[[0, 1, 2, 5]])
    np.testing.assert_array_equal(F, [[0, 1, 2], [0, 1, 3]])
    np.testing.assert_array_equal(C, c[[0, 1, 2, 5]])


def _fan():
    """Four faces on edge (0, 1) with apex heights 1, 3, 2, 0.5: areas 0.5, 1.5, 1, 0.25."""
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 3], [0, -2, 0], [0, 0, -0.5]], np.float64)
    return v, np.array([[0, 1, 2], [1, 0, 3], [0, 1, 4], [1, 0, 5]])


def test_non_manifold_fan_keeps_the_two_largest_faces():
    v, f = _fan()
    np.testing.assert_array_equal(do.remove_non_manifold_edges(v, f), [[1, 0, 3], [0, 1, 4]])


def _messy_mesh():
    """A decimated sphere with every defect the passes remove added to it."""
    v, f = _mc(14)
    m = do.decimate_rounds(v, f, len(f) // 3)
    P, F = m["verts"].astype(np.float32).astype(np.float64), m["faces"]
    n = len(P)
    rng = np.random.default_rng(5)
    extra_v = P[rng.choice(n, 6, replace=False)]                   # coincident copies
    fv, ff = _fan()
    P = np.concatenate([P, extra_v, fv + 5.0])
    F = np.concatenate([F, F[:4][:, [1, 2, 0]], F[5:7][:, [0, 2, 1]], [[0, 0, 1], [2, 3, 3]],
                        [[n, n + 1, n + 2], [n + 3, n + 4, n + 5]], ff + n + 6])
    return P, F, rng.random((len(P), 3)), rng.standard_normal((len(P), 3))


def test_torch_clean_mesh_equals_the_oracle_passes():
    from sugar_b200 import decimate
    P, F, C, N = _messy_mesh()
    want = do.clean_mesh(P, F, C, N)
    got = decimate.clean_mesh(torch.from_numpy(P), torch.from_numpy(F), torch.from_numpy(C), torch.from_numpy(N))
    for w, k in zip(want, ("verts", "faces", "colors", "normals")):
        np.testing.assert_array_equal(got[k].numpy(), w, err_msg=k)
    e = np.sort(np.concatenate([want[1][:, [0, 1]], want[1][:, [1, 2]], want[1][:, [2, 0]]]), 1)
    assert np.unique(e, axis=0, return_counts=True)[1].max() <= 2


def test_torch_clean_mesh_on_empty_and_clean_meshes():
    from sugar_b200 import decimate
    v, f = _grid(5)
    got = decimate.clean_mesh(torch.from_numpy(v), torch.from_numpy(f))
    assert torch.equal(got["faces"], torch.from_numpy(f)) and torch.equal(got["verts"], torch.from_numpy(v))
    got = decimate.clean_mesh(torch.zeros(0, 3), torch.zeros(0, 3, dtype=torch.int64))
    assert got["verts"].shape == (0, 3) and got["faces"].shape == (0, 3)


# ---------------------------------------------------------------------------------------------------------------------
# ABI and Python surface without a GPU
# ---------------------------------------------------------------------------------------------------------------------
def test_decimate_entry_points_validate_before_touching_cuda():
    from sugar_b200 import _lib
    L = _lib.lib
    d = ctypes.c_void_p(16)
    res = (ctypes.c_int64 * 4)()
    assert 0 < L.sgr_decimate_scratch_bytes(1000, 2000) < L.sgr_decimate_scratch_bytes(100000, 200000)
    assert L.sgr_decimate(-1, 0, 0, *([None] * 8), res, d, None) == -1
    assert b"sgr_decimate" in L.sgr_last_error()
    assert L.sgr_decimate(10, -1, 0, *([None] * 8), res, d, None) == -1
    assert L.sgr_decimate(10, 4, -1, d, d, None, None, d, d, None, None, res, d, None) == -1   # target < 0
    assert L.sgr_decimate(0, 4, 0, d, d, None, None, d, d, None, None, res, d, None) == -1     # faces without verts
    assert L.sgr_decimate(10, 4, 0, d, None, None, None, d, d, None, None, res, d, None) == -1  # no faces pointer
    assert L.sgr_decimate(10, 4, 0, d, d, d, None, d, d, None, None, res, d, None) == -1       # colours without output
    assert L.sgr_decimate(10, 4, 0, d, d, None, None, d, d, None, None, None, d, None) == -1    # no result
    assert L.sgr_decimate(10, 4, 0, d, d, None, None, d, d, None, None, res, None, None) == -1  # no scratch
    assert b"null pointer" in L.sgr_last_error()
    assert L.sgr_decimate(0, 0, 0, *([None] * 8), res, None, None) == 0                         # nothing to do
    assert list(res) == [0, 0, 0, 0]


def test_python_surface_rejects_cpu_tensors_and_bad_shapes():
    from sugar_b200 import decimate
    v, f = _grid(4)
    with pytest.raises(RuntimeError):
        decimate.simplify_quadric_decimation(torch.from_numpy(v), torch.from_numpy(f), 4)
