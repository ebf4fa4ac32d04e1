"""The refinement stage's mesh regularisers, normal consistency and Laplacian smoothing, as fused CUDA ops over tables
built once.

Every refinement iteration of the reference adds (sugar_trainers/refine.py:775-783, factor 0.1 from train.py:162)

    loss += 0.1 * mesh_normal_consistency(sugar.surface_mesh)       # pytorch3d 0.7.4, one mesh

whose vertices are the same `_points` tensor `meshbind.bind_to_mesh` takes.  pytorch3d rebuilds the edge table and
lists the pairs of faces sharing an edge with a Python loop over all 3F (face, edge) entries on every call.  The faces
never change during refinement, so here the pair table is built once on the device and kept by the caller:

    topo = mesh_topology(faces, n_verts)                                  # once
    loss = loss + 0.1 * mesh_normal_consistency(verts, topology=topo)     # every step: csrc/sgr_meshloss.cu

The result is a 0-dim float32 tensor, differentiable with respect to `verts`.  When no two faces share an edge (a
triangle soup) it is 0 with a zero gradient; pytorch3d returns tensor([0.]) (shape [1]) in that case.

The same stage can add pytorch3d's Laplacian smoothing (refine.py:163-171, 778-780, off by default in the reference,
factor 5 when on), which rebuilds its sparse Laplacian on every call.  Here the neighbour and corner lists are built
once and the Laplacian is applied as a gather (csrc/sgr_meshlap.cu):

    lap = laplacian_topology(faces, n_verts)                                                     # once
    loss = loss + 5.0 * mesh_laplacian_smoothing(verts, method="uniform", topology=lap)         # every step

There is no CPU fallback.
"""
from typing import NamedTuple

import torch

from ._lib import (SGR_MESH_LAP_COT, SGR_MESH_LAP_COTCURV, SGR_MESH_LAP_PARTIALS, SGR_MESH_LAP_UNIFORM, check, lib, ptr,
                   require_cuda, scratch, stream, tensor)

INT32_MAX = 2 ** 31 - 1


class MeshTopology(NamedTuple):
    """The pairs of faces sharing an edge, in pytorch3d's order (by edge, then by face-entry pair), and the vertex
    incidence list the backward sums over.  Built by `mesh_topology`; valid for any vertex positions."""
    pairs: torch.Tensor      # int32 [Q,4]: (v0, v1, a, b), the shared edge (v0 < v1) and the two opposite vertices
    vert_ptr: torch.Tensor   # int32 [V+1]: CSR offsets into vert_inc
    vert_inc: torch.Tensor   # int32 [4Q]: entries 4 * pair + slot of `pairs` naming each vertex, ascending
    n_verts: int
    n_faces: int

    @property
    def num_pairs(self) -> int:
        return int(self.pairs.shape[0])


def mesh_topology(faces: torch.Tensor, n_verts: int) -> MeshTopology:
    """Pair table and vertex incidence of the mesh `faces` [F,3] (integer, CUDA) over `n_verts` vertices.

    Sort / unique / scan on the device with one host read (the pair count, together with the count of face ids
    outside [0, n_verts), which raise ValueError).  The caller keeps the result for as long as the faces stay."""
    require_cuda("meshloss", faces)
    if faces.dim() != 2 or faces.shape[1] != 3 or faces.dtype.is_floating_point or faces.dtype == torch.bool:
        raise ValueError(f"faces must be an integer [F,3] tensor, got {faces.dtype} {tuple(faces.shape)}")
    with torch.cuda.device(faces.device):
        return _build_topology(faces, n_verts)


def _build_topology(faces, n_verts):
    """mesh_topology's tensor program; device-agnostic so that the CPU tests can run it against the oracle."""
    V, F = int(n_verts), int(faces.shape[0])
    if V <= 0 or V > INT32_MAX or 3 * F > INT32_MAX:
        raise ValueError(f"{V} vertices / {F} faces: need 0 < V <= 2^31 - 1 and 3F <= 2^31 - 1")
    dev = faces.device
    f = faces.long()
    # entry 3 f + m: edge m of face f is (f1, f2), (f2, f0), (f0, f1) for m = 0, 1, 2 (pytorch3d's e12, e20, e01),
    # its opposite vertex f_m
    ea, eb = f[:, [1, 2, 0]].reshape(-1), f[:, [2, 0, 1]].reshape(-1)
    lo, hi = torch.minimum(ea, eb), torch.maximum(ea, eb)
    h, order = torch.sort(lo * V + hi, stable=True)
    lo, hi, opp = lo[order], hi[order], f.reshape(-1)[order]
    n = 3 * F
    idx = torch.arange(n, device=dev)
    starts = torch.ones(n, dtype=torch.bool, device=dev)
    starts[1:] = h[1:] != h[:-1]
    group = torch.cumsum(starts, 0) - 1
    rank = idx - torch.cummax(torch.where(starts, idx, torch.zeros_like(idx)), 0).values if n else idx
    size = torch.zeros(n, dtype=torch.int64, device=dev).scatter_add_(0, group, torch.ones_like(group))[group]
    per = size - 1 - rank                      # an entry pairs with the entries after it on its edge
    n_bad, Q = (int(v) for v in torch.stack([((f < 0) | (f >= V)).sum(), per.sum()]).tolist())  # the one host read
    if n_bad:
        raise ValueError(f"{n_bad} face vertex ids outside [0, {V})")
    if 4 * Q > INT32_MAX:
        raise ValueError(f"{Q} face pairs: at most (2^31 - 1) / 4")
    first = torch.repeat_interleave(idx, per, output_size=Q)
    offset = (torch.cumsum(per, 0) - per)[first]
    second = first + 1 + (torch.arange(Q, device=dev) - offset)
    pairs = torch.stack([lo[first], hi[first], opp[first], opp[second]], dim=1).int().contiguous()
    inc_vert, inc = torch.sort(pairs.reshape(-1).long(), stable=True)
    vert_ptr = torch.searchsorted(inc_vert, torch.arange(V + 1, device=dev)).int()
    return MeshTopology(pairs, vert_ptr, inc.int().contiguous(), V, F)


class _MeshNormalConsistency(torch.autograd.Function):
    @staticmethod
    def forward(ctx, verts, pairs, vert_ptr, vert_inc):
        verts = verts.detach().contiguous()
        Q, V, dev = pairs.shape[0], verts.shape[0], verts.device
        with torch.cuda.device(dev):
            out = torch.empty((), device=dev)
            ws = scratch(lib.sgr_mesh_nc_forward_scratch_bytes(Q), dev)
            check(lib.sgr_mesh_nc_forward(Q, V, ptr(verts), ptr(pairs), out.data_ptr(), ptr(ws), stream(dev)))
        ctx.save_for_backward(verts, pairs, vert_ptr, vert_inc)
        return out

    @staticmethod
    def backward(ctx, g):
        verts, pairs, vert_ptr, vert_inc = ctx.saved_tensors
        Q, V, dev = pairs.shape[0], verts.shape[0], verts.device
        with torch.cuda.device(dev):
            g = g.detach().float().contiguous()
            g_verts = torch.empty_like(verts)
            ws = scratch(lib.sgr_mesh_nc_backward_scratch_bytes(Q), dev)
            check(lib.sgr_mesh_nc_backward(Q, V, ptr(verts), ptr(pairs), ptr(vert_ptr), ptr(vert_inc), g.data_ptr(),
                                           ptr(g_verts), ptr(ws), stream(dev)))
        return g_verts, None, None, None


def mesh_normal_consistency(verts, faces=None, topology=None):
    """pytorch3d 0.7.4 mesh_normal_consistency of the one mesh (verts [V,3] float32 CUDA, faces [F,3]): the mean over
    the pairs of faces sharing an edge of 1 - cos(n_a, -n_b).  Pass `topology` (from `mesh_topology`) to skip the
    per-call table build (`faces` is then not read); without it one is built from `faces` on the device.
    -> 0-dim tensor."""
    require_cuda("meshloss", verts)
    tensor(verts, "verts", torch.float32, ("V", 3))
    if topology is None:
        if faces is None:
            raise ValueError("mesh_normal_consistency needs `faces` or a `topology`")
        if faces.device != verts.device:
            raise ValueError(f"faces on {faces.device}, verts on {verts.device}")
        topology = mesh_topology(faces, verts.shape[0])
    if topology.n_verts != verts.shape[0]:
        raise ValueError(f"the topology was built for {topology.n_verts} vertices, verts has {verts.shape[0]}")
    if topology.pairs.device != verts.device:
        raise ValueError(f"topology on {topology.pairs.device}, verts on {verts.device}")
    return _MeshNormalConsistency.apply(verts, topology.pairs, topology.vert_ptr, topology.vert_inc)


# ---- Laplacian smoothing -------------------------------------------------------------------------------------------

LAPLACIAN_METHODS = {"uniform": SGR_MESH_LAP_UNIFORM, "cot": SGR_MESH_LAP_COT, "cotcurv": SGR_MESH_LAP_COTCURV}


class LaplacianTopology(NamedTuple):
    """The vertex lists mesh_laplacian_smoothing gathers over, for each method.  Built by `laplacian_topology`; valid
    for any vertex positions."""
    faces: torch.Tensor        # int32 [F,3]
    corner_ptr: torch.Tensor   # int32 [V+1]: CSR offsets into corner_inc
    corner_inc: torch.Tensor   # int32 [3F]: the face corners 3 f + k at each vertex, ascending (cot, cotcurv)
    nbr_ptr: torch.Tensor      # int32 [V+1]: CSR offsets into nbr_idx
    nbr_idx: torch.Tensor      # int32 [2E]: the neighbours over the E unique edges, ascending, a self-loop twice (uniform)
    n_verts: int
    n_faces: int

    @property
    def degree(self) -> torch.Tensor:
        """int32 [V]: pytorch3d's uniform-Laplacian degree (the row sums of the adjacency; a self-loop counts 2)."""
        return self.nbr_ptr[1:] - self.nbr_ptr[:-1]


def laplacian_topology(faces: torch.Tensor, n_verts: int) -> LaplacianTopology:
    """Neighbour and corner lists of the mesh `faces` [F,3] (integer, CUDA) over `n_verts` vertices.

    Sort / scan on the device with one host read (the unique-edge count, together with the count of face ids outside
    [0, n_verts), which raise ValueError, as an empty mesh does).  The caller keeps the result for as long as the faces
    stay."""
    require_cuda("meshloss", faces)
    if faces.dim() != 2 or faces.shape[1] != 3 or faces.dtype.is_floating_point or faces.dtype == torch.bool:
        raise ValueError(f"faces must be an integer [F,3] tensor, got {faces.dtype} {tuple(faces.shape)}")
    with torch.cuda.device(faces.device):
        return _build_laplacian_topology(faces, n_verts)


def _build_laplacian_topology(faces, n_verts):
    """laplacian_topology's tensor program; device-agnostic so that the CPU tests can run it against the oracle."""
    V, F = int(n_verts), int(faces.shape[0])
    if V <= 0 or V > INT32_MAX or F <= 0 or 3 * F > INT32_MAX:
        raise ValueError(f"{V} vertices / {F} faces: need 0 < V <= 2^31 - 1 and 0 < 3F <= 2^31 - 1")
    dev = faces.device
    f = faces.long()
    # pytorch3d's edges_packed: the unique (min, max) of e12, e20, e01, hashed V * lo + hi; self-loops kept
    ea, eb = f[:, [1, 2, 0]].reshape(-1), f[:, [2, 0, 1]].reshape(-1)
    h = torch.sort(torch.minimum(ea, eb) * V + torch.maximum(ea, eb)).values
    starts = torch.ones(3 * F, dtype=torch.bool, device=dev)
    starts[1:] = h[1:] != h[:-1]
    n_bad, E = (int(v) for v in torch.stack([((f < 0) | (f >= V)).sum(), starts.sum()]).tolist())  # the one host read
    if n_bad:
        raise ValueError(f"{n_bad} face vertex ids outside [0, {V})")
    if 2 * E > INT32_MAX:
        raise ValueError(f"{E} unique edges: at most (2^31 - 1) / 2")
    # the members of a run all write the run's hash: the same value, whichever lands
    u = torch.empty(E, dtype=torch.int64, device=dev).scatter_(0, torch.cumsum(starts, 0) - 1, h)
    lo, hi = u // V, u % V
    # both directions of every edge, by (row, column): the uniform Laplacian's entries, a self-loop twice
    key = torch.sort(torch.cat([lo * V + hi, hi * V + lo])).values
    nbr_ptr = torch.searchsorted(key // V, torch.arange(V + 1, device=dev)).int()
    corner_vert, corner_inc = torch.sort(f.reshape(-1), stable=True)
    corner_ptr = torch.searchsorted(corner_vert, torch.arange(V + 1, device=dev)).int()
    return LaplacianTopology(faces.int().contiguous(), corner_ptr, corner_inc.int().contiguous(), nbr_ptr,
                             (key % V).int().contiguous(), V, F)


class _MeshLaplacianSmoothing(torch.autograd.Function):
    @staticmethod
    def forward(ctx, verts, method, faces, vert_ptr, vert_inc):
        verts = verts.detach().contiguous()
        V, F, dev = verts.shape[0], faces.shape[0], verts.device
        with torch.cuda.device(dev):
            out = torch.empty((), device=dev)
            face_w = torch.empty((F if method != SGR_MESH_LAP_UNIFORM else 0, 4), device=dev)
            ys = torch.empty((V, 4), device=dev)
            partials = torch.empty(SGR_MESH_LAP_PARTIALS, dtype=torch.float64, device=dev)
            check(lib.sgr_mesh_lap_forward(method, V, F, ptr(verts), ptr(faces), ptr(vert_ptr), ptr(vert_inc),
                                           ptr(face_w), ptr(ys), ptr(partials), out.data_ptr(), stream(dev)))
        ctx.method = method
        ctx.save_for_backward(faces, vert_ptr, vert_inc, face_w, ys)
        return out

    @staticmethod
    def backward(ctx, g):
        faces, vert_ptr, vert_inc, face_w, ys = ctx.saved_tensors
        V, F, dev = ys.shape[0], faces.shape[0], ys.device
        with torch.cuda.device(dev):
            g = g.detach().float().contiguous()
            g_verts = torch.empty((V, 3), device=dev)
            check(lib.sgr_mesh_lap_backward(ctx.method, V, F, ptr(faces), ptr(vert_ptr), ptr(vert_inc), ptr(face_w),
                                            ptr(ys), g.data_ptr(), ptr(g_verts), stream(dev)))
        return g_verts, None, None, None, None


def mesh_laplacian_smoothing(verts, faces=None, method="uniform", topology=None):
    """pytorch3d 0.7.4 mesh_laplacian_smoothing of the one mesh (verts [V,3] float32 CUDA, faces [F,3]) with `method`
    "uniform", "cot" or "cotcurv": the mean over all V vertices of |y_v|, y the Laplacian rows (see
    include/sugar_b200.h), L held constant.  Pass `topology` (from `laplacian_topology`) to skip the per-call list build
    (`faces` is then not read); without it one is built from `faces` on the device.  -> 0-dim tensor."""
    if method not in LAPLACIAN_METHODS:
        raise ValueError(f"method must be one of {sorted(LAPLACIAN_METHODS)}, got {method!r}")
    require_cuda("meshloss", verts)
    tensor(verts, "verts", torch.float32, ("V", 3))
    if topology is None:
        if faces is None:
            raise ValueError("mesh_laplacian_smoothing needs `faces` or a `topology`")
        if faces.device != verts.device:
            raise ValueError(f"faces on {faces.device}, verts on {verts.device}")
        topology = laplacian_topology(faces, verts.shape[0])
    if topology.n_verts != verts.shape[0]:
        raise ValueError(f"the topology was built for {topology.n_verts} vertices, verts has {verts.shape[0]}")
    if topology.faces.device != verts.device:
        raise ValueError(f"topology on {topology.faces.device}, verts on {verts.device}")
    if method == "uniform":
        lists = (topology.nbr_ptr, topology.nbr_idx)
    else:
        lists = (topology.corner_ptr, topology.corner_inc)
    return _MeshLaplacianSmoothing.apply(verts, LAPLACIAN_METHODS[method], topology.faces, *lists)
