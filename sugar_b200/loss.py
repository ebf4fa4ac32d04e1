"""The trainers' photometric loss, L1 + D-SSIM, as one fused forward and one fused backward (csrc/sgr_loss.cu).

Mirrors sugar_utils/loss_utils.py:17-62 as the three trainers use it (coarse_sdf.py:101-103, 452-457,
coarse_density.py:101-103, 456-461, refine.py:103-105, 499-504):

    loss = (1 - 0.2) * l1_loss(pred, gt) + 0.2 * (1 - ssim(pred, gt))      ==  l1_dssim_loss(pred, gt, 0.2)

`ssim` has the reference's signature and return.  Inputs are float32 CUDA tensors [C,H,W] or [B,C,H,W]; the second
image is the target and is not differentiated (it must not require grad).  The window is the reference's 11x11
Gaussian (sigma 1.5) and is applied separably; everything else -- zero padding, per-channel planes, C1 / C2 -- is the
reference's.  There is no CPU fallback.
"""
import ctypes as C
import math

import torch

from ._lib import SgrSsimParams, check, lib

C1 = 0.01 ** 2
C2 = 0.03 ** 2
MAX_ELEMENTS = 2 ** 31 - 1


def gaussian_window(window_size=11, sigma=1.5):
    """The reference's 1-D weights (loss_utils.py:23-25): exp(-(x - w//2)^2 / (2 sigma^2)) evaluated in double by
    math.exp, stored as float32, normalised by their float32 sum.  -> float32 tensor [window_size] on the CPU."""
    g = torch.tensor([math.exp(-(x - window_size // 2) ** 2 / float(2 * sigma ** 2)) for x in range(window_size)],
                     dtype=torch.float32)
    return g / g.sum()


_WINDOW = [float(v) for v in gaussian_window(11, 1.5)]


def _params(B, Cc, H, W):
    p = SgrSsimParams()
    p.B, p.C, p.H, p.W = int(B), int(Cc), int(H), int(W)
    p.c1, p.c2 = C1, C2
    for i, v in enumerate(_WINDOW):
        p.window[i] = v
    return p


def _ptr(t):
    return t.data_ptr()


class _L1Ssim(torch.autograd.Function):
    """(img1 [B,C,H,W], img2 [B,C,H,W]) -> (per-image mean |img1 - img2| [B], per-image mean SSIM [B])."""

    @staticmethod
    def forward(ctx, img1, img2):
        B, Cc, H, W = img1.shape
        dev = img1.device
        img1, img2 = img1.detach().contiguous(), img2.detach().contiguous()
        with torch.cuda.device(dev):
            maps = torch.empty((3,) + img1.shape, device=dev)
            out = torch.empty(B, 2, device=dev)
            scratch = torch.empty(lib.sgr_l1_ssim_scratch_bytes(B, Cc, H, W), dtype=torch.uint8, device=dev)
            p = _params(B, Cc, H, W)
            check(lib.sgr_l1_ssim_forward(C.byref(p), _ptr(img1), _ptr(img2), _ptr(maps), _ptr(out), _ptr(scratch),
                                          torch.cuda.current_stream(dev).cuda_stream))
        ctx.save_for_backward(img1, img2, maps)
        return out[:, 0], out[:, 1]

    @staticmethod
    def backward(ctx, g_l1, g_ssim):
        img1, img2, maps = ctx.saved_tensors
        B, Cc, H, W = img1.shape
        dev = img1.device
        with torch.cuda.device(dev):
            g = lambda t: torch.zeros(B, device=dev) if t is None else t.contiguous().float()
            g_l1, g_ssim = g(g_l1), g(g_ssim)
            grad = torch.empty_like(img1)
            p = _params(B, Cc, H, W)
            check(lib.sgr_l1_ssim_backward(C.byref(p), _ptr(img1), _ptr(img2), _ptr(maps), _ptr(g_l1), _ptr(g_ssim),
                                           _ptr(grad), torch.cuda.current_stream(dev).cuda_stream))
        return grad, None


def l1_ssim_per_image(img1, img2, window_size=11):
    """-> (l1 [B], ssim [B]): per image, the means of |img1 - img2| and of the SSIM map over its C*H*W elements.
    [C,H,W] inputs count as one image.  Differentiable with respect to img1 only."""
    if window_size != 11:
        raise NotImplementedError(f"window_size={window_size}: only the reference's 11x11 window is implemented")
    if not (img1.is_cuda and img2.is_cuda):
        raise RuntimeError("sugar_b200.loss needs CUDA tensors: there is no CPU fallback")
    if img2.requires_grad:
        raise RuntimeError("sugar_b200.loss differentiates the first image only: the second (the target) must not "
                           "require grad")
    if img1.shape != img2.shape:
        raise RuntimeError(f"images differ in shape: {tuple(img1.shape)} vs {tuple(img2.shape)}")
    if img1.dim() not in (3, 4):
        raise RuntimeError(f"expected [C,H,W] or [B,C,H,W] images, got {tuple(img1.shape)}")
    if img1.dtype != torch.float32 or img2.dtype != torch.float32:
        raise RuntimeError(f"sugar_b200.loss takes float32 images, got {img1.dtype} / {img2.dtype}")
    if img1.device != img2.device:
        raise RuntimeError(f"images on different devices: {img1.device} vs {img2.device}")
    if img1.numel() == 0:
        raise RuntimeError(f"empty images: {tuple(img1.shape)}")
    if img1.numel() > MAX_ELEMENTS:
        raise RuntimeError(f"{img1.numel()} elements: the fused loss takes at most 2^31 - 1")
    a, b = (img1, img2) if img1.dim() == 4 else (img1.unsqueeze(0), img2.unsqueeze(0))
    return _L1Ssim.apply(a, b)


def ssim(img1, img2, window_size=11, size_average=True):
    """sugar_utils/loss_utils.py:33-41: the mean SSIM over everything (size_average=True) or, for [B,C,H,W] inputs,
    the per-image means [B] (the reference's .mean(1).mean(1).mean(1)); a [C,H,W] input gives its one mean."""
    per_image = l1_ssim_per_image(img1, img2, window_size)[1]
    if size_average:
        return per_image.mean()
    return per_image if img1.dim() == 4 else per_image[0]


def l1_dssim_loss(pred, gt, dssim_factor=0.2):
    """The trainers' loss_fn: (1 - dssim_factor) * l1_loss(pred, gt) + dssim_factor * (1 - ssim(pred, gt)), from one
    forward and one backward launch pair."""
    l1, s = l1_ssim_per_image(pred, gt)
    return (1.0 - dssim_factor) * l1.mean() + dssim_factor * (1.0 - s.mean())
