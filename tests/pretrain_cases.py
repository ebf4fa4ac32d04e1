"""Point clouds for the distCUDA2 goldens and tests, built from seeded CPU torch generators (the same values on every
machine): a uniform cloud, a clustered one with exact duplicates, a planar one (a zero-extent axis), the sizes around
simple-knn's 1024-point boxes, the P <= 3 clouds whose FLT_MAX sentinels stay in the mean, a Gaussian bulk with 1%
floaters 6 sigma to 1e4 sigma out on both sides of every axis (beyond the K-NN grid's 4-sigma clip), and a unit cloud
centred far from the origin (coordinates quantised at 2^-13)."""
import math

import torch


def _g(seed):
    return torch.Generator().manual_seed(seed)


def clouds():
    """-> {name: float32 [P,3] CPU tensor}."""
    out = {"uniform_100k": torch.rand(100_000, 3, generator=_g(1)) * 4.0 - 2.0}
    centres = torch.randn(40, 3, generator=_g(2)) * 3.0
    pts = centres[torch.randint(0, 40, (20_000,), generator=_g(3))] + 0.02 * torch.randn(20_000, 3, generator=_g(4))
    dup = torch.randint(0, 20_000, (3_000,), generator=_g(5))
    out["clustered_dups"] = torch.cat([pts, pts[dup]])[torch.randperm(23_000, generator=_g(6))].contiguous()
    plane = torch.rand(30_000, 3, generator=_g(7)) * 2.0
    plane[:, 2] = 0.25
    out["planar"] = plane
    for P in (4, 1023, 1024, 1025, 2049):
        out[f"p{P}"] = torch.randn(P, 3, generator=_g(100 + P))
    bulk = torch.randn(30_000, 3, generator=_g(8))
    F = 300
    mag = 6.0 * torch.exp(torch.rand(F, generator=_g(9)) * math.log(1e4 / 6.0))
    sign = torch.where((torch.arange(F) // 3) % 2 == 0, 1.0, -1.0)
    bulk[torch.arange(F), torch.arange(F) % 3] = sign * mag
    out["floaters"] = bulk[torch.randperm(30_000, generator=_g(10))].contiguous()
    out["offset"] = torch.rand(30_000, 3, generator=_g(11)) - 0.5 + torch.tensor([3e3, -2e3, 1e3])
    for P in (1, 2, 3):
        out[f"p{P}"] = torch.randn(P, 3, generator=_g(200 + P))
    return out
