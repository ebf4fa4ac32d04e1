"""The trainers' photometric loss (L1 + D-SSIM) restated -- TEST INFRASTRUCTURE and the bench's reference arm.

Two independent formulations of `sugar_utils/loss_utils.py:17-62` (l1_loss, gaussian, create_window, ssim, _ssim):

* `ssim_torch` / `l1_dssim_torch`: the reference's sequence of PyTorch operations -- the window recipe, five grouped
  11x11 `conv2d` with zero padding and the elementwise chain -- for any dtype and device.  This is what
  `bench_workloads.reference_ops` plugs into the composed steps, so the reference arm times the reference's chain.
* `ssim_numpy`: float64 NumPy, the windowed moments as sums of shifted zero-padded copies, and the gradient of the
  trainers' loss by the closed form the fused kernels implement (DESIGN section 3).  It is the precision yardstick.

tests/golden/ssim_*.npz come from the reference's OWN functions (tests/golden/make_ssim_golden.py);
tests/test_loss_cpu.py pins both formulations to them.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

C1 = 0.01 ** 2
C2 = 0.03 ** 2


def gaussian_1d(window_size=11, sigma=1.5):
    """1-D weights exp(-(x - w//2)^2 / (2 sigma^2)) evaluated in double by math.exp, stored as float32 and
    normalised by their float32 sum (the window recipe of the trainers' loss)."""
    g = torch.tensor([math.exp(-(x - window_size // 2) ** 2 / float(2 * sigma ** 2)) for x in range(window_size)],
                     dtype=torch.float32)
    return g / g.sum()


def window_2d(window_size=11):
    """float32 [w, w]: the outer product of the 1-D weights, rounded to float32 (not separable bit for bit)."""
    g = gaussian_1d(window_size).unsqueeze(1)
    return g.mm(g.t()).float()


def ssim_torch(img1, img2, window_size=11, size_average=True):
    channel = img1.size(-3)
    window = window_2d(window_size).expand(channel, 1, window_size, window_size).contiguous()
    window = window.to(device=img1.device, dtype=img1.dtype)
    pad = window_size // 2
    conv = lambda t: F.conv2d(t, window, padding=pad, groups=channel)
    mu1, mu2 = conv(img1), conv(img2)
    mu1_sq, mu2_sq, mu1_mu2 = mu1.pow(2), mu2.pow(2), mu1 * mu2
    sigma1_sq = conv(img1 * img1) - mu1_sq
    sigma2_sq = conv(img2 * img2) - mu2_sq
    sigma12 = conv(img1 * img2) - mu1_mu2
    ssim_map = ((2 * mu1_mu2 + C1) * (2 * sigma12 + C2)) / ((mu1_sq + mu2_sq + C1) * (sigma1_sq + sigma2_sq + C2))
    if size_average:
        return ssim_map.mean()
    return ssim_map.mean(1).mean(1).mean(1)


def l1_dssim_torch(pred, gt, dssim_factor=0.2):
    """(1 - f) * l1_loss + f * (1 - ssim): the trainers' loss_fn."""
    return (1.0 - dssim_factor) * (pred - gt).abs().mean() + dssim_factor * (1.0 - ssim_torch(pred, gt))


def _corr(a, w2):
    """Zero-padded correlation of every [H, W] plane of a [..., H, W] float64 array with the [k, k] window, as the sum
    of k*k shifted copies."""
    k = w2.shape[0]
    r = k // 2
    H, W = a.shape[-2:]
    p = np.zeros(a.shape[:-2] + (H + 2 * r, W + 2 * r))
    p[..., r:r + H, r:r + W] = a
    out = np.zeros_like(a)
    for i in range(k):
        for j in range(k):
            out += w2[i, j] * p[..., i:i + H, j:j + W]
    return out


def ssim_numpy(img1, img2, dssim_factor=0.2, window=None):
    """float64 [B, C, H, W] (or [C, H, W]) -> dict(ssim [B], l1 [B], grad = d/d img1 of the trainers' loss
    (1 - f) * mean|img1 - img2| + f * (1 - mean S) over everything).  `window`: [11, 11], default the float32
    2-D window of the recipe."""
    x = np.asarray(img1, np.float64)
    y = np.asarray(img2, np.float64)
    squeeze = x.ndim == 3
    if squeeze:
        x, y = x[None], y[None]
    w2 = np.asarray(window_2d().numpy() if window is None else window, np.float64)
    mu1, mu2 = _corr(x, w2), _corr(y, w2)
    s1 = _corr(x * x, w2) - mu1 * mu1
    s2 = _corr(y * y, w2) - mu2 * mu2
    s12 = _corr(x * y, w2) - mu1 * mu2
    A1, A2 = 2 * mu1 * mu2 + C1, 2 * s12 + C2
    B1, B2 = mu1 * mu1 + mu2 * mu2 + C1, s1 + s2 + C2
    S = A1 * A2 / (B1 * B2)
    # dS/dE[x^2], dS/dE[xy], and dS/dmu1 with sigma1^2 and sigma12 expanded
    d1 = -S / B2
    d2 = 2 * A1 / (B1 * B2)
    d0 = 2 * mu2 * A2 / (B1 * B2) - 2 * mu1 * S / B1 - 2 * mu1 * d1 - mu2 * d2
    wt = w2[::-1, ::-1]   # the adjoint of a zero-padded correlation is the correlation with the flipped window
    n_all = x.size
    dS = (_corr(d0, wt) + 2 * x * _corr(d1, wt) + y * _corr(d2, wt)) / n_all
    grad = (1 - dssim_factor) * np.sign(x - y) / n_all - dssim_factor * dS
    red = tuple(range(1, x.ndim))
    out = dict(ssim=S.mean(axis=red), l1=np.abs(x - y).mean(axis=red), grad=grad[0] if squeeze else grad)
    return out
