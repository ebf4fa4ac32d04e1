"""CPU checks of the screened-Poisson reconstruction: the float64 oracle's system (symmetry, definiteness, the hat
gradients by finite differences, a sphere's mesh), the C entry points' argument checks, and the mesh trim rules."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import mcubes_oracle as mo  # noqa: E402
from oracle import poisson_oracle as po  # noqa: E402


def _sphere(n, seed, r=0.8):
    rng = np.random.default_rng(seed)
    d = rng.normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    return (r * d).astype(np.float32), d.astype(np.float32)


def test_oracle_matrix_is_symmetric_and_positive_definite():
    import scipy.sparse.linalg as spla
    p, nr = _sphere(300, 0)
    s = po.system(p, nr, 5)
    A = s["A"]
    assert (A - A.T).count_nonzero() == 0
    assert s["q"].min() >= 0 and s["q"].max() > 0
    # the smallest eigenvalue, by shift-invert around -1
    lam = spla.eigsh(A.tocsc(), k=1, sigma=-1.0, which="LM", return_eigenvectors=False)[0]
    assert lam > 0
    # every row sums to its q: the stiffness has zero row sums (zero flux at the faces)
    assert np.allclose(np.asarray(A.sum(1)).ravel(), s["q"].reshape(-1))


def test_oracle_b_matches_finite_differences_of_the_hats():
    rng = np.random.default_rng(1)
    N = 8
    g = rng.uniform(0.2, N - 1.2, size=(50, 3))
    nr = rng.normal(size=(50, 3))
    _, ids, ws, gr = po.hats(g, N)
    eps = 1e-6
    for a in range(3):
        e = np.zeros(3)
        e[a] = eps
        _, ip, wp, _ = po.hats(g + e, N)
        _, im, wm, _ = po.hats(g - e, N)
        same = (ip == ids).all(1) & (im == ids).all(1)           # away from a bin change
        fd = (wp - wm) / (2 * eps)
        assert np.allclose(fd[same], gr[same, :, a], atol=1e-6)
    assert np.allclose(ws.sum(1), 1.0)                          # partition of unity
    # the assembled b is -a sum_s n_s . grad phi_i(p_s), with the gradient by finite differences of the hats
    p, nrm = _sphere(40, 6)
    s = po.system(p, nrm, 5)
    gg = po.grid_coords(p, s["o32"], s["inv_h32"])
    want = np.zeros(32 ** 3)
    for k in range(len(p)):
        _, ids0, _, _ = po.hats(gg[k:k + 1], 32)
        for c in range(8):
            node = ids0[0, c]
            grad = np.zeros(3)
            for a in range(3):
                e = np.zeros(3)
                e[a] = eps
                hp = np.maximum(0, 1 - np.abs(gg[k] + e - np.array(np.unravel_index(node, (32,) * 3)))).prod()
                hm = np.maximum(0, 1 - np.abs(gg[k] - e - np.array(np.unravel_index(node, (32,) * 3)))).prod()
                grad[a] = (hp - hm) / (2 * eps)
            want[node] += -s["area"] * nrm[k].astype(np.float64) @ grad
    assert np.allclose(s["b"].reshape(-1), want, atol=1e-6)


def test_oracle_sphere_mesh_lies_within_h():
    p, nr = _sphere(20000, 2)
    r = po.reconstruct(p, nr, 5)
    v, f = r["verts"], r["faces"]
    h = r["system"]["h"]
    assert len(f) > 500
    d = np.abs(np.linalg.norm(v, axis=1) - 0.8)
    assert d.max() < h, (d.max(), h)
    assert mo.euler_characteristic(len(v), f) == 2


def test_entry_points_reject_bad_sizes_and_null_pointers():
    from sugar_b200 import _lib
    L = _lib.lib
    d = ctypes.c_void_p(256)
    occ = ctypes.c_int64(0)
    norm = ctypes.c_double(0)
    assert L.sgr_poisson_bin(0, d, 32, 0, 0, 0, 1, d, d, d, d, d, d, ctypes.byref(occ), None) == -1
    assert b"sgr_poisson_bin" in L.sgr_last_error()
    assert L.sgr_poisson_bin(10, d, 33, 0, 0, 0, 1, d, d, d, d, d, d, ctypes.byref(occ), None) == -1      # not a power of two
    assert L.sgr_poisson_bin(10, d, 2048, 0, 0, 0, 1, d, d, d, d, d, d, ctypes.byref(occ), None) == -1
    assert L.sgr_poisson_bin(10, None, 32, 0, 0, 0, 1, d, d, d, d, d, d, ctypes.byref(occ), None) == -1
    assert L.sgr_poisson_bin(10, d, 32, 0, 0, 0, 1, d, ctypes.c_void_p(264), d, d, d, d, ctypes.byref(occ), None) == -1
    assert b"misaligned" in L.sgr_last_error()
    assert L.sgr_poisson_bin(10, d, 32, 0, 0, 0, 1, d, d, d, ctypes.c_void_p(264), d, d, ctypes.byref(occ), None) == -1
    assert L.sgr_poisson_bin(10, d, 32, 0, 0, 0, 1, d, d, d, d, None, d, ctypes.byref(occ), None) == -1
    assert b"misaligned" in L.sgr_last_error()
    assert L.sgr_poisson_splat(32, 10, d, d, 3, d, 0, 1, 4, d, d, None) == -1                    # mode
    assert L.sgr_poisson_splat(32, 10, d, d, 2, d, 3, 1, 4, d, d, None) == -1                    # channel
    assert L.sgr_poisson_splat(32, 10, d, d, 0, d, 0, 1, 4, d, None, None) == -1                 # q output
    assert L.sgr_poisson_splat(32, 10, d, d, 2, None, 0, 1, 4, d, None, None) == -1              # attribute
    assert L.sgr_poisson_coarsen(4, d, d, None) == -1
    assert L.sgr_poisson_coarsen(32, d, None, None) == -1
    assert L.sgr_poisson_residual_norm(32, 0.0, None, d, None, d, ctypes.byref(norm), None) == -1
    assert L.sgr_poisson_residual_norm(32, 1.0, d, d, None, d, ctypes.byref(norm), None) == -1   # u without q
    lv = (ctypes.c_void_p * 4)(256, 256, None, 256)
    assert L.sgr_poisson_vcycle(5, lv, lv, lv, d, ctypes.byref(norm), None) == -1
    assert b"level 2" in L.sgr_last_error()
    assert L.sgr_poisson_vcycle(11, lv, lv, lv, d, ctypes.byref(norm), None) == -1
    assert L.sgr_poisson_interpolate(32, d, 5, d, 2, 1, 0, d, d, None, None) == -1               # stride
    assert L.sgr_poisson_interpolate(32, d, 5, d, 3, 1, 0, None, d, None, None) == -1            # no output
    assert L.sgr_poisson_interpolate(32, d, 5, None, 3, 1, 0, d, d, None, None) == -1


def test_remove_vertices_by_mask_on_hand_made_meshes():
    from sugar_b200.poisson import remove_vertices_by_mask
    verts = torch.arange(15, dtype=torch.float32).reshape(5, 3)
    faces = torch.tensor([[0, 1, 2], [1, 2, 3], [2, 3, 4], [0, 3, 4]])
    colors = verts * 0.01
    mask = torch.tensor([False, True, False, False, False])
    out = remove_vertices_by_mask(verts, faces, mask, colors)
    assert torch.equal(out["verts"], verts[[0, 2, 3, 4]])
    assert torch.equal(out["faces"], torch.tensor([[1, 2, 3], [0, 2, 3]]))
    assert torch.equal(out["colors"], colors[[0, 2, 3, 4]]) and out["normals"] is None
    ov, of = po.remove_vertices_by_mask(verts.numpy(), faces.numpy(), mask.numpy())
    assert np.array_equal(out["verts"].numpy(), ov) and np.array_equal(out["faces"].numpy(), of)
    # unreferenced vertices stay
    out = remove_vertices_by_mask(verts, faces, torch.tensor([False, False, False, True, False]))
    assert torch.equal(out["verts"], verts[[0, 1, 2, 4]]) and torch.equal(out["faces"], torch.tensor([[0, 1, 2]]))
    out = remove_vertices_by_mask(verts, faces, torch.tensor([False, False, True, True, False]))
    assert out["verts"].shape[0] == 3 and out["faces"].shape == (0, 3)
    # a mask that empties the mesh
    out = remove_vertices_by_mask(verts, faces, torch.ones(5, dtype=torch.bool))
    assert out["verts"].shape == (0, 3) and out["faces"].shape == (0, 3)
    with pytest.raises(ValueError, match="mask"):
        remove_vertices_by_mask(verts, faces, torch.ones(4, dtype=torch.bool))
    # random meshes against the oracle
    g = torch.Generator().manual_seed(3)
    for _ in range(5):
        V = 40
        vv = torch.rand(V, 3, generator=g)
        ff = torch.stack([torch.randperm(V, generator=g)[:3] for _ in range(60)])
        mm = torch.rand(V, generator=g) < 0.2
        out = remove_vertices_by_mask(vv, ff, mm)
        ov, of = po.remove_vertices_by_mask(vv.numpy(), ff.numpy(), mm.numpy())
        assert np.array_equal(out["verts"].numpy(), ov) and np.array_equal(out["faces"].numpy(), of)


def test_quantile_rule_matches_numpy():
    from sugar_b200.poisson import quantile, quantile_index
    rng = np.random.default_rng(4)
    cases = [np.array([3.0]), np.array([1.0, 2.0]), np.array([5.0, 1.0, 4.0, 4.0, 2.0]),
             rng.normal(size=1001), rng.integers(0, 5, 300).astype(np.float64), rng.random(7).astype(np.float32)]
    for x in cases:
        for q in (0.0, 0.1, 0.25, 0.5, 0.73, 0.9, 1.0):
            assert quantile(torch.from_numpy(x), q) == float(np.quantile(x.astype(np.float64), q)), (x, q)
    # the trim keeps everything at quantile 0 (nothing is below the minimum)
    x = torch.from_numpy(rng.random(100))
    assert int((x.double() < quantile(x, 0.0)).sum()) == 0
    # index arithmetic past 2^24 values (torch.quantile's limit), against exact fractions
    from fractions import Fraction
    for V in (2 ** 24 + 1, 2 ** 25 + 3, 3 * 2 ** 26 + 5):
        for q in (0.1, 0.5, 0.999):
            lo, hi, gamma = quantile_index(V, q)
            exact = Fraction(q) * (V - 1)
            assert lo == int(exact) and hi == min(lo + 1, V - 1)
            assert abs(gamma - float(exact - lo)) < 1e-6
    with pytest.raises(ValueError):
        quantile(torch.zeros(0), 0.1)


def test_outlier_rule_of_the_oracle_on_planted_floaters():
    rng = np.random.default_rng(5)
    p = np.concatenate([rng.normal(size=(400, 3)) * 0.05, np.array([[10.0, 0, 0], [0, -12.0, 3]])])
    kept = po.outlier_kept(p, 20, 2.0)
    assert 400 not in kept and 401 not in kept and len(kept) >= 380
    assert len(po.outlier_kept(p, 20, 20.0)) == 402
