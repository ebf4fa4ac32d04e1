"""Exact K-nearest neighbours on the GPU (uniform grid), standing in for pytorch3d.ops.knn_points as
SuGaR uses it (sugar_scene/sugar_model.py:1013-1030 reset_neighbors, :1335-1343).

    dists, idx = knn_points(queries, points, K)     # [Q,K] squared distances (ascending), [Q,K] int64
    knn_dists, knn_idx = reset_neighbors(points, K=16)   # the tables SuGaR keeps (neighbour 0 is the smallest index
                                                         # at distance 0: self unless the point is duplicated)
    dist2 = dist_cuda2(points)                       # simple-knn's distCUDA2: vanilla 3DGS's initial scales

Equal distances come in index order, so every row is a function of the input alone; the distances are float32
((dx*dx + dy*dy) + dz*dz) with d = point - query, each step rounded, which a float32 brute force reproduces to the bit.
"""
import torch

from ._lib import check, lib, ptr, require_cuda, scratch, stream, tensor


def _cloud(p, name, dev=None):
    """[N,3] or pytorch3d's batched [1,N,3] -> float32 [N,3]."""
    p = p.float()
    return tensor(p[0] if p.dim() == 3 and p.shape[0] == 1 else p, name, torch.float32, ("N", 3), dev, "p1")


def knn_points(p1: torch.Tensor, p2: torch.Tensor, K: int):
    """K nearest points of p2 for every point of p1.  Accepts [N,3] or pytorch3d's batched [1,N,3].  Shapes and
    devices are checked (ValueError)."""
    batched = p1.dim() == 3
    q = _cloud(p1, "p1")
    dev = q.device
    r = _cloud(p2, "p2", dev)
    require_cuda("knn", q, r)
    Q, P = q.shape[0], r.shape[0]
    with torch.cuda.device(dev):
        idx = torch.empty((Q, K), dtype=torch.int64, device=dev)
        d2 = torch.empty((Q, K), dtype=torch.float32, device=dev)
        ws = scratch(lib.sgr_knn_workspace_bytes(P), dev)
        check(lib.sgr_knn(P, r.data_ptr(), Q, ptr(q), K, ptr(idx), ptr(d2), ptr(ws), stream(dev)))
    return (d2[None], idx[None]) if batched else (d2, idx)


def reset_neighbors(points: torch.Tensor, K: int = 16):
    """SuGaR.reset_neighbors: (knn_dists [P,K], knn_idx [P,K]) of the cloud against itself, no grad."""
    with torch.no_grad():
        return knn_points(points, points, K)


def dist_cuda2(points: torch.Tensor) -> torch.Tensor:
    """simple-knn's distCUDA2 (vanilla 3DGS's create_from_pcd): float32 [P], per point the mean of the squared
    distances to its 3 nearest other points (other by index, so a duplicate position is a neighbour at 0), the
    reference's value to the bit.  With P <= 3 its FLT_MAX sentinels stay in the mean: inf for P <= 2, about
    FLT_MAX / 3 for P = 3.  `points`: [P,3] CUDA tensor (converted to float32).  No host synchronisation."""
    r = _cloud(points, "points")
    require_cuda("knn", r)
    dev, P = r.device, r.shape[0]
    out = torch.empty((P,), dtype=torch.float32, device=dev)
    if P == 0:
        return out
    with torch.cuda.device(dev):
        ws = scratch(lib.sgr_knn_workspace_bytes(P), dev)
        check(lib.sgr_dist_cuda2(P, ptr(r), ptr(out), ptr(ws), stream(dev)))
    return out
