"""LPIPS (VGG16, v0.1): the perceptual metric of metrics.py (gaussian_splatting/lpipsPyTorch), as sm_90a kernels
(csrc/sgr_lpips.cu).

    from sugar_b200.lpips import LPIPS, lpips
    metric = LPIPS("vgg16-397923af.pth", "vgg.pth")     # read and packed once
    d = metric(render, gt)                               # [N, 3, H, W] in [0, 1] -> [N]

The weights are the two files the reference's `torch.hub` directory holds after one run of its metrics.py:
torchvision's IMAGENET1K_V1 VGG16 (`features.{0,2,5,...,28}.{weight,bias}`) and the LPIPS v0.1 linear layers
(`lin{i}.model.1.weight`, [1, C, 1, 1]).  Nothing is downloaded.

The network is the reference's: z-score (x - mean) / std of the [0, 1] input (no 2x - 1), conv1_1 ... conv5_3 with
ReLU and 2x2 max pools, taps at relu1_2, relu2_2, relu3_3, relu4_3 and relu5_3; per tap the channel-normalised
features (eps 1e-10 outside the sqrt), their squared difference, the 1x1 linear layer and the mean over that tap's
H x W; LPIPS is the sum of the five.  Differences: a batch of N pairs gives N values (the reference sums them into
one), and the twelve tensor-core convs take TF32 operands with float32 accumulation (torch's default cuDNN
convolutions on an H100 are TF32 too).  Forward only.
"""
import ctypes as C
import os

import torch

from ._lib import check, lib, require_cuda, scratch, stream

# torchvision's vgg16().features indices of the 13 convs, their (Cout, Cin), and the convs the five taps follow
CONV_INDICES = (0, 2, 5, 7, 10, 12, 14, 17, 19, 21, 24, 26, 28)
CONV_SHAPES = ((64, 3), (64, 64), (128, 64), (128, 128), (256, 128), (256, 256), (256, 256), (512, 256), (512, 512),
               (512, 512), (512, 512), (512, 512), (512, 512))
TAP_CONVS = (1, 3, 6, 9, 12)
TAP_CHANNELS = (64, 128, 256, 512, 512)
MIN_SIZE = 16   # the fifth tap is 1/16 of the input

VGG_FILE = "vgg16-397923af.pth"
LIN_FILE = "vgg.pth"
DEFAULT_WEIGHTS_DIR = os.path.join(".", "lpipsPyTorch", "weights", "checkpoints")


def tf32_round(t: torch.Tensor) -> torch.Tensor:
    """float32 `t` rounded to TF32 (10 mantissa bits) to nearest, ties away from zero: cvt.rna.tf32.f32."""
    bits = t.contiguous().view(torch.int32).to(torch.int64)
    return ((bits + 0x1000) & ~0x1FFF).to(torch.int32).view(torch.float32)


def _load(path):
    try:
        return torch.load(path, map_location="cpu", weights_only=True)
    except FileNotFoundError:
        raise
    except Exception as e:
        raise ValueError(f"{path}: not a readable state dict ({e})") from e


def _take(sd, key, shape, path):
    if key not in sd:
        raise ValueError(f"{path}: missing key '{key}'")
    t = sd[key]
    if not torch.is_tensor(t) or tuple(t.shape) != tuple(shape):
        got = tuple(t.shape) if torch.is_tensor(t) else type(t).__name__
        raise ValueError(f"{path}: '{key}' has shape {got}, expected {tuple(shape)}")
    return t.detach().to(torch.float32)


def read_vgg16(path):
    """-> [(weight [Cout, Cin, 3, 3], bias [Cout])] * 13, float32, from torchvision's vgg16 state dict at `path`.
    Raises ValueError naming a missing key or a wrong shape."""
    sd = _load(path)
    return [(_take(sd, f"features.{i}.weight", (co, ci, 3, 3), path), _take(sd, f"features.{i}.bias", (co,), path))
            for i, (co, ci) in zip(CONV_INDICES, CONV_SHAPES)]


def read_lin(path):
    """-> [weight [C]] * 5, float32, from the LPIPS v0.1 linear layers at `path` (`lin{i}.model.1.weight`)."""
    sd = _load(path)
    return [_take(sd, f"lin{i}.model.1.weight", (1, c, 1, 1), path).reshape(c) for i, c in enumerate(TAP_CHANNELS)]


def pack_weights(convs, lins) -> torch.Tensor:
    """The kernels' weight blob (include/sugar_b200.h, LPIPS): per conv its weights KRSC then its bias, then the
    five linear vectors; the twelve tensor-core convs' weights rounded to TF32 once here.  -> float32 [n] (CPU)."""
    parts = []
    for l, (w, b) in enumerate(convs):
        w = w.permute(0, 2, 3, 1).contiguous()
        parts += [(w if l == 0 else tf32_round(w)).reshape(-1), b.reshape(-1)]
    parts += [v.reshape(-1) for v in lins]
    blob = torch.cat(parts)
    if blob.numel() != lib.sgr_lpips_weight_floats():
        raise ValueError(f"packed {blob.numel()} floats, the kernels take {lib.sgr_lpips_weight_floats()}")
    return blob


def conv_flops(H: int, W: int) -> int:
    """Multiply-adds x 2 of the 13 convs for one H x W image (the pools floor odd sizes)."""
    total = 0
    for l, (co, ci) in enumerate(CONV_SHAPES):
        total += 2 * H * W * co * ci * 9
        if l in TAP_CONVS[:4]:
            H, W = H // 2, W // 2
    return total


def pair_flops(H: int, W: int) -> int:
    """The conv FLOPs of one LPIPS value: both images of the pair."""
    return 2 * conv_flops(H, W)


class LPIPS:
    """LPIPS(vgg_path, lin_path)(x, y) -> [N]: the reference's LPIPS('vgg', '0.1') per pair of [N, 3, H, W] images.
    The weights are read, checked and packed once, onto `device` (default: the current CUDA device)."""

    def __init__(self, vgg_path, lin_path, device=None):
        convs, lins = read_vgg16(vgg_path), read_lin(lin_path)
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.weights = pack_weights(convs, lins).to(self.device)
        base, o = self.weights.data_ptr(), 0
        self._conv = []
        for co, ci in CONV_SHAPES:
            self._conv.append((base + 4 * o, base + 4 * (o + co * 9 * ci)))
            o += co * 9 * ci + co
        self._lin = []
        for c in TAP_CHANNELS:
            self._lin.append(base + 4 * o)
            o += c

    @torch.no_grad()
    def __call__(self, x, y, return_taps=False):
        """x, y float32 CUDA [N, 3, H, W] (renders and ground truths, values in [0, 1]), H, W >= 16 -> LPIPS [N];
        with return_taps, (LPIPS [N], the five tap means [N, 5])."""
        require_cuda("lpips", x, y)
        if x.dim() != 4 or x.shape[1] != 3 or x.shape != y.shape:
            raise ValueError(f"x, y must both be [N, 3, H, W], got {tuple(x.shape)} and {tuple(y.shape)}")
        if x.dtype != torch.float32 or y.dtype != torch.float32:
            raise ValueError(f"x, y must be float32, got {x.dtype} and {y.dtype}")
        if x.device != self.device or y.device != self.device:
            raise ValueError(f"x on {x.device}, y on {y.device}, the weights on {self.device}")
        N, _, H, W = x.shape
        if N < 1 or H < MIN_SIZE or W < MIN_SIZE:
            raise ValueError(f"LPIPS needs N >= 1 and H, W >= {MIN_SIZE}, got N={N}, H={H}, W={W}")
        x, y = x.contiguous(), y.contiguous()
        dev = self.device
        with torch.cuda.device(dev):
            st = stream(dev)
            off = (C.c_size_t * 8)()
            check(lib.sgr_lpips_scratch_layout(N, H, W, None, off))
            ws = scratch(off[7], dev)
            check(lib.sgr_lpips_scratch_layout(N, H, W, ws.data_ptr(), off))
            act = (ws.data_ptr() + off[0], ws.data_ptr() + off[1])
            out = torch.empty(N, device=dev)
            taps = torch.empty(N, 5, device=dev)
            w0, b0 = self._conv[0]
            check(lib.sgr_lpips_conv1(N, H, W, x.data_ptr(), y.data_ptr(), w0, b0, act[0], st))
            src, h, w = 0, H, W
            for l, (co, ci) in enumerate(CONV_SHAPES):
                if l > 0:
                    wl, bl = self._conv[l]
                    check(lib.sgr_lpips_conv3x3(2 * N, h, w, ci, co, act[src], wl, bl, act[1 - src], st))
                    src = 1 - src
                if l in TAP_CONVS:
                    t = TAP_CONVS.index(l)
                    pooled = act[1 - src] if t < 4 else None
                    check(lib.sgr_lpips_tap(N, h, w, co, act[src], self._lin[t], pooled, ws.data_ptr() + off[2 + t],
                                            st))
                    if t < 4:
                        src, h, w = 1 - src, h // 2, w // 2
            check(lib.sgr_lpips_reduce(N, H, W, ws.data_ptr() + off[2], taps.data_ptr(), out.data_ptr(), st))
        return (out, taps) if return_taps else out


_cache = {}


def lpips(x, y, net_type="vgg", version="0.1", weights_dir=DEFAULT_WEIGHTS_DIR):
    """gaussian_splatting/lpipsPyTorch.lpips with net_type 'vgg', version '0.1': LPIPS [N] per pair of [N, 3, H, W]
    images (the reference returns the sum over the batch, [1, 1, 1, 1]).  The weights are read from `weights_dir`
    (VGG_FILE and LIN_FILE, where the reference's torch.hub directory keeps them) once per directory and device."""
    if net_type != "vgg":
        raise NotImplementedError(f"net_type={net_type!r}: only 'vgg' is implemented (metrics.py uses vgg)")
    if version != "0.1":
        raise NotImplementedError(f"version={version!r}: only LPIPS v0.1 exists")
    key = (os.path.abspath(weights_dir), x.device)
    if key not in _cache:
        _cache[key] = LPIPS(os.path.join(weights_dir, VGG_FILE), os.path.join(weights_dir, LIN_FILE), x.device)
    return _cache[key](x, y)
