"""The refinement stage's mesh normal-consistency regulariser as a fused CUDA op over a cached pair table.

Every refinement iteration of the reference adds (sugar_trainers/refine.py:775-783, factor 0.1 from train.py:162)

    loss += 0.1 * mesh_normal_consistency(sugar.surface_mesh)       # pytorch3d 0.7.4, one mesh

whose vertices are the same `_points` tensor `meshbind.bind_to_mesh` takes.  pytorch3d rebuilds the edge table and
lists the pairs of faces sharing an edge with a Python loop over all 3F (face, edge) entries on every call.  The faces
never change during refinement, so here the pair table is built once on the device and kept by the caller:

    topo = mesh_topology(faces, n_verts)                                  # once
    loss = loss + 0.1 * mesh_normal_consistency(verts, topology=topo)     # every step: csrc/sgr_meshloss.cu

The result is a 0-dim float32 tensor, differentiable with respect to `verts`.  When no two faces share an edge (a
triangle soup) it is 0 with a zero gradient; pytorch3d returns tensor([0.]) (shape [1]) in that case.  There is no CPU
fallback.
"""
from typing import NamedTuple

import torch

from ._lib import check, lib

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
    if not faces.is_cuda:
        raise RuntimeError("sugar_b200.meshloss needs CUDA tensors: there is no CPU fallback")
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
            scratch = torch.empty(lib.sgr_mesh_nc_forward_scratch_bytes(Q), dtype=torch.uint8, device=dev)
            check(lib.sgr_mesh_nc_forward(Q, V, verts.data_ptr(), pairs.data_ptr(), out.data_ptr(), scratch.data_ptr(),
                                          torch.cuda.current_stream(dev).cuda_stream))
        ctx.save_for_backward(verts, pairs, vert_ptr, vert_inc)
        return out

    @staticmethod
    def backward(ctx, g):
        verts, pairs, vert_ptr, vert_inc = ctx.saved_tensors
        Q, V, dev = pairs.shape[0], verts.shape[0], verts.device
        with torch.cuda.device(dev):
            g = g.detach().float().contiguous()
            g_verts = torch.empty_like(verts)
            scratch = torch.empty(lib.sgr_mesh_nc_backward_scratch_bytes(Q), dtype=torch.uint8, device=dev)
            check(lib.sgr_mesh_nc_backward(Q, V, verts.data_ptr(), pairs.data_ptr(), vert_ptr.data_ptr(),
                                           vert_inc.data_ptr(), g.data_ptr(), g_verts.data_ptr(), scratch.data_ptr(),
                                           torch.cuda.current_stream(dev).cuda_stream))
        return g_verts, None, None, None


def mesh_normal_consistency(verts, faces=None, topology=None):
    """pytorch3d 0.7.4 mesh_normal_consistency of the one mesh (verts [V,3] float32 CUDA, faces [F,3]): the mean over
    the pairs of faces sharing an edge of 1 - cos(n_a, -n_b).  Pass `topology` (from `mesh_topology`) to skip the
    per-call table build (`faces` is then not read); without it one is built from `faces` on the device.
    -> 0-dim tensor."""
    if not verts.is_cuda:
        raise RuntimeError("sugar_b200.meshloss needs CUDA tensors: there is no CPU fallback")
    if verts.dtype != torch.float32 or verts.dim() != 2 or verts.shape[1] != 3:
        raise ValueError(f"verts must be float32 [V,3], got {verts.dtype} {tuple(verts.shape)}")
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
