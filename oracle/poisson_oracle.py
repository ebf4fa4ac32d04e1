"""Float64 restatement of the screened-Poisson problem of sugar_b200/poisson.py (csrc/sgr_poisson.cu), for tests.

The system is assembled sample by sample (np.add.at over each sample's eight hats) as a scipy sparse matrix and solved
with spsolve up to 32^3 nodes, with CG at a relative residual of 1e-12 above.  Grid coordinates are rounded to
float32 exactly as the kernels round them (g = (p - o) * inv_h - 0.5, one rounding per operation); everything after
that is float64.  Also: the statistical outlier rule (cdist + sort) and open3d's remove_vertices_by_mask.
"""
import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla
from scipy.spatial.distance import cdist


def domain(points, depth):
    """(o float64[3], h, o32, inv_h32) of the cube of side 1.1 x the bounding box's largest side."""
    p = np.asarray(points, np.float32).astype(np.float64)
    lo, hi = p.min(0), p.max(0)
    L = 1.1 * float((hi - lo).max())
    N = 1 << depth
    o = 0.5 * (lo + hi) - 0.5 * L
    return o, L / N, o.astype(np.float32), np.float32(N / L)


def grid_coords(points, o32, inv_h32):
    p = np.asarray(points, np.float32)
    return ((p - o32) * inv_h32 - np.float32(0.5)).astype(np.float32).astype(np.float64)


def hats(g, N):
    """Per sample: lower corners [n,3], the 8 corner offsets' node ids [n,8], weights [n,8], gradients [n,8,3]."""
    L = np.clip(np.floor(g).astype(np.int64), 0, N - 2)
    t = g - L
    ids, ws, gr = [], [], []
    for dx in (0, 1):
        for dy in (0, 1):
            for dz in (0, 1):
                d = np.array([dx, dy, dz])
                w1 = np.where(d == 1, t, 1.0 - t)                     # [n,3]
                s1 = np.where(d == 1, 1.0, -1.0)
                node = L + d
                ids.append((node[:, 0] * N + node[:, 1]) * N + node[:, 2])
                ws.append(w1.prod(1))
                gr.append(np.stack([s1[0] * w1[:, 1] * w1[:, 2], s1[1] * w1[:, 0] * w1[:, 2],
                                    s1[2] * w1[:, 0] * w1[:, 1]], 1))
    return L, np.stack(ids, 1), np.stack(ws, 1), np.stack(gr, 1)


def splat(points, depth, o32, inv_h32, values=None):
    """sum_s phi_i(p_s) (values None) or sum_s phi_i(p_s) values[s] on the grid of `depth` with the given domain."""
    N = 1 << depth
    _, ids, ws, _ = hats(grid_coords(points, o32, inv_h32), N)
    out = np.zeros(N ** 3)
    v = ws if values is None else ws * np.asarray(values, np.float64)[:, None]
    np.add.at(out, ids.reshape(-1), v.reshape(-1))
    return out.reshape(N, N, N)


def system(points, normals, depth, alpha=4.0):
    """-> dict(A csr, b [N,N,N], q [N,N,N], area, domain)."""
    N = 1 << depth
    o, h, o32, ih = domain(points, depth)
    g = grid_coords(points, o32, ih)
    L, ids, ws, gr = hats(g, N)
    n = len(g)
    occupied = len(np.unique((L[:, 0] * N + L[:, 1]) * N + L[:, 2]))
    a = occupied / n
    nr = np.asarray(normals, np.float64)
    b = np.zeros(N ** 3)
    q = np.zeros(N ** 3)
    np.add.at(b, ids.reshape(-1), (-a * np.einsum("sc,skc->sk", nr, gr)).reshape(-1))
    np.add.at(q, ids.reshape(-1), (alpha * a * ws).reshape(-1))
    A = stiffness(N) + sp.diags(q)
    return {"A": A.tocsr(), "b": b.reshape(N, N, N), "q": q.reshape(N, N, N), "area": a, "o": o, "h": h,
            "o32": o32, "inv_h32": ih}


def stiffness(N, coeff=1.0):
    """7-point graph Laplacian of the N^3 grid with zero-flux faces (missing neighbours dropped)."""
    one = sp.diags([np.ones(N - 1), -2 * np.ones(N) + np.r_[1, np.zeros(N - 2), 1], np.ones(N - 1)], [-1, 0, 1])
    I = sp.identity(N)
    lap = sp.kron(sp.kron(one, I), I) + sp.kron(sp.kron(I, one), I) + sp.kron(sp.kron(I, I), one)
    return (-coeff * lap).tocsr()


def solve(A, b):
    n = b.size
    rhs = b.reshape(-1)
    if n <= 32 ** 3:
        return spla.spsolve(A.tocsc(), rhs).reshape(b.shape)
    M = sp.diags(1.0 / A.diagonal())
    x, info = spla.cg(A, rhs, rtol=1e-12, atol=0.0, maxiter=20000, M=M)
    assert info == 0, info
    return x.reshape(b.shape)


def interpolate(grid, g):
    """Trilinear interpolation of grid [N,N,N] at grid coordinates g [m,3] (clamped as the kernels clamp)."""
    N = grid.shape[0]
    L = np.clip(np.floor(g).astype(np.int64), 0, N - 2)
    t = np.clip(g - L, 0.0, 1.0)
    out = np.zeros(len(g))
    for dx in (0, 1):
        for dy in (0, 1):
            for dz in (0, 1):
                d = np.array([dx, dy, dz])
                w = np.where(d == 1, t, 1.0 - t).prod(1)
                out += w * grid[L[:, 0] + dx, L[:, 1] + dy, L[:, 2] + dz]
    return out


def reconstruct(points, normals, depth, alpha=4.0):
    """The whole problem in float64: -> dict(u, iso, verts (world), faces, system)."""
    from oracle import mcubes_oracle as mo
    s = system(points, normals, depth, alpha)
    u = solve(s["A"], s["b"])
    iso = interpolate(u, grid_coords(points, s["o32"], s["inv_h32"])).mean()
    v, f = mo.marching_cubes(u.astype(np.float32), iso)
    return {"u": u, "iso": iso, "verts": s["o"] + (np.asarray(v, np.float64) + 0.5) * s["h"], "faces": f,
            "system": s}


def outlier_kept(points, nb_neighbors=20, std_ratio=20.0):
    """open3d 0.17's statistical outlier rule as its source reads: mean distance over the K nearest (self included)."""
    p = np.asarray(points, np.float64)
    d = np.sort(cdist(p, p), axis=1)[:, :min(nb_neighbors, len(p))]
    avg = d.mean(1)
    pos = avg > 0
    if pos.sum() < 2:
        return np.nonzero(pos)[0]
    v = avg[pos]
    bound = v.mean() + std_ratio * v.std(ddof=1)
    return np.nonzero(pos & (avg < bound))[0]


def remove_vertices_by_mask(verts, faces, mask):
    """open3d's TriangleMesh.remove_vertices_by_mask, one face at a time."""
    new_id, kept = {}, []
    for i in range(len(verts)):
        if not mask[i]:
            new_id[i] = len(kept)
            kept.append(verts[i])
    out = [[new_id[int(x)] for x in f] for f in faces if all(not mask[int(x)] for x in f)]
    return np.asarray(kept).reshape(-1, 3), np.asarray(out, np.int64).reshape(-1, 3)
