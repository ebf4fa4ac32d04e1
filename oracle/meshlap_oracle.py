"""PyTorch restatement of pytorch3d 0.7.4's mesh_laplacian_smoothing for one mesh -- TEST INFRASTRUCTURE ONLY.

The refinement stage can add `surface_mesh_laplacian_smoothing_factor * mesh_laplacian_smoothing(sugar.surface_mesh,
method=...)` (sugar_trainers/refine.py:163-171, 778-780; off by default), where `surface_mesh` is a new
`Meshes(verts=[_points], faces=[_surface_mesh_faces])` on every call.  pytorch3d is not a dependency here (the
reference's environment.yml:161 pins it), so this file restates, op for op, its published algorithm:

    Meshes.laplacian_packed      ops.laplacian(verts, edges_packed): edges_packed the unique (min, max) edges of
                                 (e12, e20, e01) hashed V * v0 + v1 (self-loops (v, v) included); A has a 1 at
                                 (v0, v1) and at (v1, v0) for every edge, deg = the row sums of A (a self-loop counts
                                 2), L[i, j] = 1 / deg[i] (0 where deg is 0) at those entries, then L[i, i] -= 1
    cot_laplacian(eps=1e-12)     A = |v1 - v2|, B = |v0 - v2|, C = |v0 - v1|, s = 0.5 (A + B + C),
                                 area = sqrt(clamp(s (s - A)(s - B)(s - C), min=eps)), cot = [(B^2 + C^2 - A^2),
                                 (A^2 + C^2 - B^2), (A^2 + B^2 - C^2)] / area / 4 at (ii, jj) = (faces[:, [1, 2, 0]],
                                 faces[:, [2, 0, 1]]), L += L^T; inv_areas = 1 / (scatter-add of area onto every face
                                 vertex slot) where > 0, else 0
    mesh_laplacian_smoothing     L (and inv_areas) under no_grad; uniform: y = L x; cot: y = (L x) * norm_w - x with
                                 norm_w = 1 / rowsum(L) where > 0, else rowsum(L); cotcurv: y = (L x - rowsum(L) x) *
                                 0.25 inv_areas; loss = sum_v |y_v| * (1 / V) over every vertex, used or not

The sparse matrices take the dtype of `verts`, so the same chain runs in float32 (pytorch3d's own arithmetic) and in
float64 (the reference the kernels are checked against).  This oracle is pinned by an independent float64 dense-matrix
construction of the same rules and by invariance properties (tests/test_meshlap_cpu.py); there is no golden from the
reference.
"""
import torch

METHODS = ("uniform", "cot", "cotcurv")


def _coo(indices, values, size):
    """torch.sparse.FloatTensor(indices, values, size) as pytorch3d builds them (duplicates summed where used)."""
    return torch.sparse_coo_tensor(indices, values, size, check_invariants=False)


def edges_packed(faces, V):
    """Meshes.edges_packed: [E,2] int64 unique (min, max) edges of every face's e12, e20, e01, sorted by V * v0 + v1."""
    v0, v1, v2 = faces.chunk(3, dim=1)
    edges = torch.cat([torch.cat([v1, v2], 1), torch.cat([v2, v0], 1), torch.cat([v0, v1], 1)], dim=0)
    edges, _ = edges.sort(dim=1)
    u = torch.unique(V * edges[:, 0] + edges[:, 1])
    return torch.stack([u // V, u % V], dim=1)


def laplacian(V, edges, dtype, device):
    """pytorch3d.ops.laplacian: the uniform Laplacian as a sparse [V,V] tensor."""
    e0, e1 = edges.unbind(1)
    idx = torch.cat([torch.stack([e0, e1], 0), torch.stack([e1, e0], 0)], dim=1)
    A = _coo(idx, torch.ones(idx.shape[1], dtype=dtype, device=device), (V, V))
    deg = torch.sparse.sum(A, dim=1).to_dense()
    deg0, deg1 = deg[e0], deg[e1]
    deg0 = torch.where(deg0 > 0.0, 1.0 / deg0, deg0)
    deg1 = torch.where(deg1 > 0.0, 1.0 / deg1, deg1)
    L = _coo(idx, torch.cat([deg0, deg1]), (V, V))
    diag = torch.arange(V, device=device)
    return L - _coo(torch.stack([diag, diag], 0), torch.ones(V, dtype=dtype, device=device), (V, V))


def cot_laplacian(verts, faces, eps=1e-12):
    """pytorch3d.ops.cot_laplacian -> (L sparse [V,V], inv_areas [V,1])."""
    V, F = verts.shape[0], faces.shape[0]
    face_verts = verts[faces]
    v0, v1, v2 = face_verts[:, 0], face_verts[:, 1], face_verts[:, 2]
    A = (v1 - v2).norm(dim=1)
    B = (v0 - v2).norm(dim=1)
    C = (v0 - v1).norm(dim=1)
    s = 0.5 * (A + B + C)
    area = (s * (s - A) * (s - B) * (s - C)).clamp_(min=eps).sqrt()
    A2, B2, C2 = A * A, B * B, C * C
    cota = (B2 + C2 - A2) / area
    cotb = (A2 + C2 - B2) / area
    cotc = (A2 + B2 - C2) / area
    cot = torch.stack([cota, cotb, cotc], dim=1)
    cot /= 4.0
    ii = faces[:, [1, 2, 0]]
    jj = faces[:, [2, 0, 1]]
    idx = torch.stack([ii, jj], dim=0).view(2, F * 3)
    L = _coo(idx, cot.view(-1), (V, V))
    L = L + L.t()
    inv_areas = torch.zeros(V, dtype=verts.dtype, device=verts.device)
    inv_areas.scatter_add_(0, faces.reshape(-1), torch.stack([area] * 3, dim=1).view(-1))
    pos = inv_areas > 0
    inv_areas[pos] = 1.0 / inv_areas[pos]
    return L, inv_areas.view(-1, 1)


def laplacian_rows(verts, faces, method="uniform"):
    """The per-vertex vectors y [V,3] whose norms the loss averages (differentiable in verts, L constant)."""
    if method not in METHODS:
        raise ValueError("Method should be one of {uniform, cot, cotcurv}")
    V = verts.shape[0]
    with torch.no_grad():
        if method == "uniform":
            L = laplacian(V, edges_packed(faces, V), verts.dtype, verts.device)
        else:
            L, inv_areas = cot_laplacian(verts, faces)
            if method == "cot":
                norm_w = torch.sparse.sum(L, dim=1).to_dense().view(-1, 1)
                pos = norm_w > 0
                norm_w[pos] = 1.0 / norm_w[pos]
            else:
                L_sum = torch.sparse.sum(L, dim=1).to_dense().view(-1, 1)
                norm_w = 0.25 * inv_areas
    if method == "uniform":
        return L.mm(verts)
    if method == "cot":
        return L.mm(verts) * norm_w - verts
    return (L.mm(verts) - L_sum * verts) * norm_w


def mesh_laplacian_smoothing_torch(verts, faces, method="uniform"):
    """pytorch3d 0.7.4 mesh_laplacian_smoothing(Meshes(verts=[verts], faces=[faces]), method), the Laplacian rebuilt on
    every call: a 0-dim tensor."""
    y = laplacian_rows(verts, faces, method)
    weights = torch.full((verts.shape[0],), 1.0 / verts.shape[0], dtype=verts.dtype, device=verts.device)
    return (y.norm(dim=1) * weights).sum() / 1
