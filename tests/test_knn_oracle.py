"""CPU: the float32 brute-force K-NN (oracle/knn_oracle.py) that the GPU K-NN tests hold the kernel to, against a
per-row sort in numpy float32 by (distance, index), on clouds with exact duplicates and tied distances, across chunk
boundaries."""
import numpy as np
import pytest
import torch

from oracle import knn_oracle as ko


def _rows(q, p, K):
    f = np.float32
    out_d, out_i = [], []
    for x in q:
        d = (p - x).astype(f)
        d2 = ((d[:, 0] * d[:, 0]).astype(f) + (d[:, 1] * d[:, 1]).astype(f)).astype(f) + (d[:, 2] * d[:, 2]).astype(f)
        o = np.lexsort((np.arange(len(p)), d2))[:K]
        out_d.append(d2[o])
        out_i.append(o)
    return np.array(out_d, np.float32), np.array(out_i, np.int64)


@pytest.mark.parametrize("K,chunk", [(1, 1 << 28), (5, 1 << 28), (16, 4 * 1500 * 7), (40, 4 * 1500)])
def test_brute_force_orders_ties_by_index(K, chunk):
    g = torch.Generator().manual_seed(K)
    pts = torch.cat([torch.randn(900, 3, generator=g), torch.randn(30, 3, generator=g).repeat(20, 1)])
    pts = torch.round(pts[torch.randperm(pts.shape[0], generator=g)] * 8) / 8      # coarse: many equal distances
    qs = torch.cat([pts[:200], torch.round(torch.randn(100, 3, generator=g) * 8) / 8])
    d2, idx = ko.knn_f32(qs, pts, K, chunk_bytes=chunk)
    want_d2, want_idx = _rows(qs.numpy(), pts.numpy(), K)
    assert np.array_equal(idx.numpy(), want_idx)
    assert np.array_equal(d2.numpy().view(np.int32), want_d2.view(np.int32))
    exact = ((pts.double()[idx] - qs.double()[:, None]) ** 2).sum(-1)
    assert bool(((d2.double() - exact).abs() <= 2.0 ** -21 * exact).all())
