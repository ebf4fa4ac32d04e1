"""PyTorch restatement of pytorch3d 0.7.4's mesh_normal_consistency for one mesh -- TEST INFRASTRUCTURE ONLY.

The refinement stage adds `surface_mesh_normal_consistency_factor * mesh_normal_consistency(sugar.surface_mesh)`
(sugar_trainers/refine.py:775-783, factor 0.1 from train.py:162), where `surface_mesh` is a new
`Meshes(verts=[_points], faces=[_surface_mesh_faces])` on every call (sugar_scene/sugar_model.py:551-560).
pytorch3d is not under /root/reference (environment.yml:161 pins it), so this file restates, op for op, its
published algorithm:

    Meshes._compute_edges_packed   edges e12, e20, e01 of every face concatenated in that order ([3F, 2]), each
                                   sorted to (min, max), hashed V * v0 + v1, torch.unique(return_inverse=True):
                                   edges_packed sorted by hash, faces_packed_to_edges_packed = inverse.reshape(3, F).t()
    mesh_normal_consistency        edge_idx = face_to_edge.reshape(3F) sorted (stably here; the value does not depend
                                   on the order inside an edge), each entry carrying its face's three vertex ids;
                                   every pair i < j of the entries of one edge is a pair (split_list over
                                   range(3F) + a nested comprehension, the faithful Python loop below);
                                   n = sum_m (v1 - v0) x (face_vert_m - v0) per entry, (v0, v1) the sorted edge;
                                   loss = 1 - cosine_similarity(n_i, -n_j) per pair, weighted by 1 / num_pairs
                                   (float32) and summed; no pairs -> tensor([0.]).

This oracle is pinned only by property tests (tests/test_meshloss_cpu.py: flat sheets, hinges, fans, duplicated
faces, permutation invariance, the two pair builders agreeing); there is no golden from the reference.
"""
from itertools import islice

import torch


def split_list(input, length_to_split):
    """pytorch3d's split_list: consecutive slices of the given lengths."""
    inputt = iter(input)
    return [list(islice(inputt, elem)) for elem in length_to_split]


def edges_packed(faces, V):
    """-> (edges_packed [E,2] int64 sorted by V * v0 + v1, faces_packed_to_edges_packed [F,3] (e12, e20, e01))."""
    F = faces.shape[0]
    v0, v1, v2 = faces.chunk(3, dim=1)
    e01 = torch.cat([v0, v1], dim=1)
    e12 = torch.cat([v1, v2], dim=1)
    e20 = torch.cat([v2, v0], dim=1)
    edges = torch.cat([e12, e20, e01], dim=0)
    edges, _ = edges.sort(dim=1)
    edges_hash = V * edges[:, 0] + edges[:, 1]
    u, inverse_idxs = torch.unique(edges_hash, return_inverse=True)
    return torch.stack([u // V, u % V], dim=1), inverse_idxs.reshape(3, F).t()


def sorted_entries(faces, V):
    """-> (edges [E,2], edge_idx [3F] sorted, vert_idx [3F,3]: each sorted entry's face vertex ids)."""
    edges, face_to_edge = edges_packed(faces, V)
    F = faces.shape[0]
    edge_idx = face_to_edge.reshape(F * 3)
    vert_idx = faces.view(1, F, 3).expand(3, F, 3).transpose(0, 1).reshape(3 * F, 3)
    edge_idx, edge_sort_idx = edge_idx.sort(stable=True)
    return edges, edge_idx, vert_idx[edge_sort_idx]


def pairs_comprehension(edge_idx, E):
    """pytorch3d's own pair builder (a host loop over all 3F entries) -> [Q,2] int64 of sorted-entry indices."""
    edge_num = edge_idx.bincount(minlength=E)
    vert_edge_pair_idx = split_list(list(range(edge_idx.shape[0])), edge_num.tolist())
    vert_edge_pair_idx = [
        [e[i], e[j]]
        for e in vert_edge_pair_idx
        for i in range(len(e) - 1)
        for j in range(1, len(e))
        if i < j
    ]
    return torch.tensor(vert_edge_pair_idx, device=edge_idx.device, dtype=torch.int64).reshape(-1, 2)


def pairs_vectorised(edge_idx, E):
    """The same pair list as pairs_comprehension, in the same order, from tensor ops."""
    n = edge_idx.shape[0]
    counts = edge_idx.bincount(minlength=E)
    start = torch.cumsum(counts, 0) - counts
    rank = torch.arange(n, device=edge_idx.device) - start[edge_idx]
    per = counts[edge_idx] - 1 - rank                    # entry i pairs with the entries after it on its edge
    rep = torch.repeat_interleave(torch.arange(n, device=edge_idx.device), per)
    offset = (torch.cumsum(per, 0) - per)[rep]
    second = rep + 1 + (torch.arange(rep.shape[0], device=edge_idx.device) - offset)
    return torch.stack([rep, second], dim=1)


BUILDERS = {"comprehension": pairs_comprehension, "vectorised": pairs_vectorised}


def pair_table(faces, V, builder="vectorised"):
    """[Q,4] int64 rows (v0, v1, a, b): the shared sorted edge and the opposite vertex of each of the two faces."""
    edges, edge_idx, vert_idx = sorted_entries(faces, V)
    pairs = BUILDERS[builder](edge_idx, edges.shape[0])
    v0, v1 = edges[edge_idx, 0], edges[edge_idx, 1]
    opp = vert_idx.sum(dim=1) - v0 - v1                  # the face's vertex that is not on the edge
    return torch.stack([v0[pairs[:, 0]], v1[pairs[:, 0]], opp[pairs[:, 0]], opp[pairs[:, 1]]], dim=1)


def mesh_normal_consistency_torch(verts, faces, builder="comprehension"):
    """pytorch3d 0.7.4 mesh_normal_consistency(Meshes(verts=[verts], faces=[faces])), the edges rebuilt on every
    call: a 0-dim tensor, or tensor([0.]) (shape [1], float32) when no two faces share an edge."""
    V = verts.shape[0]
    with torch.no_grad():
        edges, edge_idx, vert_idx = sorted_entries(faces, V)
        vert_edge_pair_idx = BUILDERS[builder](edge_idx, edges.shape[0])
    if vert_edge_pair_idx.shape[0] == 0:
        return torch.tensor([0.0], dtype=torch.float32, device=verts.device, requires_grad=True)
    v0 = verts[edges[edge_idx, 0]]
    v1 = verts[edges[edge_idx, 1]]
    n_temp0 = (v1 - v0).cross(verts[vert_idx[:, 0]] - v0, dim=1)
    n_temp1 = (v1 - v0).cross(verts[vert_idx[:, 1]] - v0, dim=1)
    n_temp2 = (v1 - v0).cross(verts[vert_idx[:, 2]] - v0, dim=1)
    n = n_temp0 + n_temp1 + n_temp2
    n0 = n[vert_edge_pair_idx[:, 0]]
    n1 = -n[vert_edge_pair_idx[:, 1]]
    loss = 1 - torch.cosine_similarity(n0, n1, dim=1)
    num_normals = torch.full((1,), vert_edge_pair_idx.shape[0], dtype=torch.int64, device=verts.device)
    weights = 1.0 / num_normals[torch.zeros_like(vert_edge_pair_idx[:, 0])].float()
    return (loss * weights).sum() / 1
