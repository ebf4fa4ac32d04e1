"""Brute-force K nearest neighbours in sgr_knn's float32 arithmetic and order, for tests/test_gpu_knn.py and
tests/test_gpu_mcubes.py.

    d2, idx = knn_f32(queries, points, K)     # torch tensors on one device; [Q,K] float32, [Q,K] int64

Every query is compared with every point.  The distance is one tensor op per rounding, d = point - query, then
((dx*dx + dy*dy) + dz*dz), which is knn_dist2 in csrc/sgr_knn.cuh to the bit.  A row is the first K points in
(distance, index) order: topk finds the K-th distance, every point at or below it is a candidate, and a stable sort of
the candidates (taken in index order) by distance puts equal distances in index order.  Queries go in chunks so that
no temporary exceeds about `chunk_bytes`.
"""
import torch


def pair_d2(queries, points):
    """[Q,P] float32 squared distances, rounded as knn_dist2 rounds them."""
    d = points[None, :, 0] - queries[:, None, 0]
    d2 = d * d
    d = points[None, :, 1] - queries[:, None, 1]
    d2 = d2 + d * d
    d = points[None, :, 2] - queries[:, None, 2]
    return d2 + d * d


def knn_f32(queries, points, K, chunk_bytes=1 << 28):
    queries, points = queries.float().contiguous(), points.float().contiguous()
    Q, P = queries.shape[0], points.shape[0]
    assert 0 < K <= P
    dev = queries.device
    d2_out = torch.empty((Q, K), dtype=torch.float32, device=dev)
    idx_out = torch.empty((Q, K), dtype=torch.int64, device=dev)
    rows = max(1, chunk_bytes // (4 * P))
    for i in range(0, Q, rows):
        d2 = pair_d2(queries[i:i + rows], points)
        n = d2.shape[0]
        kth = d2.topk(K, dim=1, largest=False).values[:, K - 1:]
        r, c = (d2 <= kth).nonzero(as_tuple=True)          # row-major: each row's candidates in index order
        val = d2[r, c]
        del d2
        o = torch.sort(val, stable=True).indices            # by distance, equal distances keep index order
        o = o[torch.sort(r[o], stable=True).indices]        # then by row, keeping that order within each row
        r, c, val = r[o], c[o], val[o]
        start = torch.zeros(n + 1, dtype=torch.int64, device=dev)
        start[1:] = torch.bincount(r, minlength=n).cumsum(0)
        pos = torch.arange(r.shape[0], device=dev) - start[r]
        keep = pos < K
        d2_out[i:i + n][r[keep], pos[keep]] = val[keep]
        idx_out[i:i + n][r[keep], pos[keep]] = c[keep]
    return d2_out, idx_out

