"""Shared pieces of the mesh Laplacian smoothing tests (test_meshlap_cpu.py, test_gpu_meshlap.py): an independent
float64 dense-matrix construction of pytorch3d 0.7.4's rules, the meshes, and the per-row comparison.

Every method is written as y = s * (Lp x) - x (uniform, cot) or y = s * (Lp x - rowsum(Lp) x) (cotcurv), with Lp the
off-diagonal-style matrix the kernels gather over and s the row scale; the backward is then
g_x = Lp^T (s g) - d g, d = 1 (uniform, cot) or rowsum(Lp) s (cotcurv), g_v = c y_v / |y_v|.  `row_scale` is
c (sum_j |Lp_jv| s_j + |d_v|): the size of the terms a gradient row sums, which bounds its rounding.  `dense_parts`
loops over faces into dense matrices (small meshes, the oracle's independent check); `sparse_parts` is the same in
vectorised scipy.sparse form for the scales and margins of large meshes.
"""
import numpy as np
import scipy.sparse as sp

from sugar_b200 import scenes

METHODS = ("uniform", "cot", "cotcurv")


def dense_parts(verts, faces, method):
    """-> (Lp [V,V], s [V], d [V], y [V,3]) in float64, from per-face loops and dense matrices."""
    v = np.asarray(verts, np.float64)
    V = len(v)
    Lp = np.zeros((V, V))
    if method == "uniform":
        edges = {tuple(sorted((int(a), int(b)))) for f in faces for a, b in ((f[1], f[2]), (f[2], f[0]), (f[0], f[1]))}
        for a, b in edges:
            Lp[a, b] += 1.0
            Lp[b, a] += 1.0
        deg = Lp.sum(1)
        s = np.where(deg > 0, 1.0 / np.where(deg > 0, deg, 1.0), 0.0)
        return Lp, s, np.ones(V), s[:, None] * (Lp @ v) - v
    area_sum = np.zeros(V)
    for f in faces:
        p0, p1, p2 = v[f[0]], v[f[1]], v[f[2]]
        A, B, C = np.linalg.norm(p1 - p2), np.linalg.norm(p0 - p2), np.linalg.norm(p0 - p1)
        sp = (A + B + C) / 2
        area = np.sqrt(max(sp * (sp - A) * (sp - B) * (sp - C), 1e-12))
        Lp[f[1], f[2]] += (B * B + C * C - A * A) / area / 4
        Lp[f[2], f[0]] += (A * A + C * C - B * B) / area / 4
        Lp[f[0], f[1]] += (A * A + B * B - C * C) / area / 4
        for i in f:
            area_sum[i] += area
    Lp = Lp + Lp.T
    rs = Lp.sum(1)
    if method == "cot":
        s = np.where(rs > 0, 1.0 / np.where(rs > 0, rs, 1.0), rs)
        return Lp, s, np.ones(V), s[:, None] * (Lp @ v) - v
    s = 0.25 * np.where(area_sum > 0, 1.0 / np.where(area_sum > 0, area_sum, 1.0), 0.0)
    return Lp, s, rs * s, s[:, None] * (Lp @ v - rs[:, None] * v)


def dense_loss_and_grad(verts, faces, method, g=1.0):
    Lp, s, d, y = dense_parts(verts, faces, method)
    n = np.linalg.norm(y, axis=1)
    c = g / len(y)
    u = np.where(n[:, None] > 0, y / np.where(n > 0, n, 1.0)[:, None], 0.0)
    return n.sum() / len(y), c * (Lp.T @ (s[:, None] * u) - d[:, None] * u)


def sparse_parts(verts, faces, method):
    """dense_parts with Lp as a scipy CSR matrix, vectorised."""
    v = np.asarray(verts, np.float64)
    f = np.asarray(faces, np.int64)
    V = len(v)
    if method == "uniform":
        e = np.sort(np.stack([f[:, [1, 2, 0]].ravel(), f[:, [2, 0, 1]].ravel()], 1), axis=1)
        e = np.unique(e, axis=0)
        ones = np.ones(2 * len(e))
        Lp = sp.coo_matrix((ones, (np.r_[e[:, 0], e[:, 1]], np.r_[e[:, 1], e[:, 0]])), (V, V)).tocsr()
        deg = np.asarray(Lp.sum(1)).ravel()
        s = np.where(deg > 0, 1.0 / np.where(deg > 0, deg, 1.0), 0.0)
        return Lp, s, np.ones(V), s[:, None] * (Lp @ v) - v
    p0, p1, p2 = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    A, B, C = np.linalg.norm(p1 - p2, axis=1), np.linalg.norm(p0 - p2, axis=1), np.linalg.norm(p0 - p1, axis=1)
    q = (A + B + C) / 2
    area = np.sqrt(np.maximum(q * (q - A) * (q - B) * (q - C), 1e-12))
    cot = np.stack([B * B + C * C - A * A, A * A + C * C - B * B, A * A + B * B - C * C], 1) / area[:, None] / 4
    Lp = sp.coo_matrix((cot.ravel(), (f[:, [1, 2, 0]].ravel(), f[:, [2, 0, 1]].ravel())), (V, V)).tocsr()
    Lp = (Lp + Lp.T).tocsr()
    rs = np.asarray(Lp.sum(1)).ravel()
    if method == "cot":
        s = np.where(rs > 0, 1.0 / np.where(rs > 0, rs, 1.0), rs)
        return Lp, s, np.ones(V), s[:, None] * (Lp @ v) - v
    area_sum = np.bincount(f.ravel(), np.repeat(area, 3), minlength=V)
    s = 0.25 * np.where(area_sum > 0, 1.0 / np.where(area_sum > 0, area_sum, 1.0), 0.0)
    return Lp, s, rs * s, s[:, None] * (Lp @ v - rs[:, None] * v)


def row_scale(verts, faces, method, g=1.0):
    Lp, s, d, _ = sparse_parts(verts, faces, method)
    return g / len(s) * (abs(Lp).T @ np.abs(s) + np.abs(d))


def union_jack(n, spacing=1.0):
    """Flat n x n grid (n odd), each cell split by the diagonal that makes every interior vertex of degree 4 or 8:
    with integer-multiple coordinates the uniform rows of interior vertices are exactly 0."""
    ij = np.stack(np.meshgrid(np.arange(n), np.arange(n), indexing="ij"), -1).reshape(-1, 2)
    verts = np.concatenate([ij * spacing, np.zeros((n * n, 1))], 1).astype(np.float32)
    faces = []
    for i in range(n - 1):
        for j in range(n - 1):
            a, b, c, d = i * n + j, (i + 1) * n + j, (i + 1) * n + j + 1, i * n + j + 1
            faces += [[a, b, c], [a, c, d]] if (i + j) % 2 == 0 else [[a, b, d], [b, c, d]]
    return verts, np.array(faces, np.int64)


def open_cap(subdivisions=3):
    """The upper part (z > -0.3) of an icosphere: an open mesh with a boundary loop, unused vertices dropped."""
    v, f = scenes.icosphere(subdivisions)
    f = f[(v[f][:, :, 2] > -0.3).all(1)]
    used = np.unique(f)
    remap = np.full(len(v), -1)
    remap[used] = np.arange(len(used))
    return v[used], remap[f]


def jittered_grid(n, seed, permute=True):
    """A height-field grid with its vertices moved in-plane by up to 30 % of the spacing: obtuse triangles."""
    v, f = scenes.height_field_mesh(n, n, seed=seed, amplitude=0.1, noise=0.3, permute=permute)
    rng = np.random.default_rng(seed)
    v = v.copy()
    v[:, :2] += (0.3 / (n - 1)) * rng.uniform(-1, 1, size=(len(v), 2))
    return v.astype(np.float32), f


def with_unused(v, f, k, seed):
    """`k` extra vertices no face uses, spread among the ids."""
    rng = np.random.default_rng(seed)
    V = len(v) + k
    ids = rng.permutation(V)
    new_of_old = ids[:len(v)]
    out = np.empty((V, 3), np.float32)
    out[new_of_old] = v
    out[ids[len(v):]] = rng.normal(size=(k, 3))
    return out, new_of_old[f]


def slivers(n=24, seed=3):
    """A jittered grid where a few vertices sit almost on the line of two neighbours (needles and caps, aspect down to
    1e-4): Heron's formula in float32 loses most of its digits there."""
    v, f = scenes.height_field_mesh(n, n, seed=seed, amplitude=0.1, noise=0.3)
    v = v.copy()
    rng = np.random.default_rng(seed)
    h = 1.0 / (n - 1)
    for k, idx in enumerate(rng.choice([i * n + j for i in range(2, n - 2) for j in range(2, n - 2)], 12, replace=False)):
        # onto the segment between its left and right neighbours, off it by 10^-(2 + k % 3) of the spacing
        left, right = v[idx - 1], v[idx + 1]
        t = rng.uniform(0.3, 0.7)
        v[idx] = left + t * (right - left) + np.array([0.0, 10.0 ** -(2 + k % 3) * h, 0.0])
    return v.astype(np.float32), f


def y_scale(verts, faces, method):
    """Per row, the size of the terms y_v sums: |s_v| sum_j |Lp_vj| |x_j - x_v|.  Every method's row is
    s_v sum_j Lp_vj (x_j - x_v) up to where s_v rowsum_v differs from 1 (an unused vertex), so this is what the float32
    face values can move it by, a self-loop's weight, however large, included (it multiplies 0)."""
    Lp, s, _, _ = sparse_parts(verts, faces, method)
    v = np.asarray(verts, np.float64)
    Lc = Lp.tocoo()
    dist = np.linalg.norm(v[Lc.col] - v[Lc.row], axis=1)
    return np.abs(s) * np.bincount(Lc.row, np.abs(Lc.data) * dist, minlength=len(v))


def check_margin(verts, faces, method, margin=1e-4):
    """Each row |y_v| of the case must be exactly 0 or at least margin x the size of the terms it sums (y_scale):
    y / |y| is undefined at 0, and below the margin float32 face values alone could turn it."""
    n = np.linalg.norm(sparse_parts(verts, faces, method)[3], axis=1)
    bad = (n > 0) & (n < margin * y_scale(verts, faces, method))
    assert not bad.any(), f"{int(bad.sum())} rows with 0 < |y| < {margin} of their terms: not a usable case"
    return n


def row_errors(got, want, scale):
    """max over rows of |got_v - want_v| / (|want_v| + scale_v)."""
    e = np.linalg.norm(np.asarray(got, np.float64) - want, axis=1)
    return float((e / (np.linalg.norm(want, axis=1) + scale + 1e-300)).max())
