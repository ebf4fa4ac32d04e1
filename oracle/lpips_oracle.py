"""LPIPS (VGG16, v0.1) restated in float64 with plain F.conv2d, for the tests of csrc/sgr_lpips.cu.

lpips64(x, y, vgg, lin) takes the two state dicts as the files hold them (`features.{i}.weight|bias`,
`lin{i}.model.1.weight`) and [N, 3, H, W] images on any device (it computes there), and returns (LPIPS [N], tap
means [N, 5]) as float64 -- per pair, not summed over the batch as the reference's module does.  tf32=True rounds both operands of every conv but
conv1_1 to TF32 (to nearest, ties away) before it, as the kernels do, to tell TF32 rounding from other error.
"""
import torch
import torch.nn.functional as F

CONV_INDICES = (0, 2, 5, 7, 10, 12, 14, 17, 19, 21, 24, 26, 28)
TAP_CONVS = (1, 3, 6, 9, 12)
MEAN = (-.030, -.088, -.188)
STD = (.458, .448, .450)


def round_tf32(t):
    """float64 `t` -> float64 holding t's float32 value rounded to TF32 (10 mantissa bits), ties away from zero."""
    bits = t.to(torch.float32).view(torch.int32).to(torch.int64)
    return ((bits + 0x1000) & ~0x1FFF).to(torch.int32).view(torch.float32).to(torch.float64)


def features64(x, vgg, tf32=False):
    """The five tap activations (relu1_2 ... relu5_3) of [B, 3, H, W] images, float64."""
    dev = x.device
    mean = torch.tensor(MEAN, dtype=torch.float32, device=dev).view(1, 3, 1, 1)
    std = torch.tensor(STD, dtype=torch.float32, device=dev).view(1, 3, 1, 1)
    h = ((x.to(torch.float32) - mean) / std).to(torch.float64)   # the reference's z-score is float32
    taps = []
    for l, i in enumerate(CONV_INDICES):
        w = vgg[f"features.{i}.weight"].to(dev, torch.float64)
        b = vgg[f"features.{i}.bias"].to(dev, torch.float64)
        if tf32 and l > 0:
            h, w = round_tf32(h), round_tf32(w)
        h = F.relu(F.conv2d(h, w, b, padding=1))
        if l in TAP_CONVS:
            taps.append(h)
            if l != TAP_CONVS[-1]:
                h = F.max_pool2d(h, 2, 2)
    return taps


def lpips64(x, y, vgg, lin, tf32=False):
    """-> (LPIPS [N], taps [N, 5]) float64 of image pairs x, y [N, 3, H, W]."""
    N = x.shape[0]
    f = features64(torch.cat([x, y]), vgg, tf32)
    vals = []
    for t, a in enumerate(f):
        a = a / (torch.sqrt((a ** 2).sum(1, keepdim=True)) + 1e-10)
        d = (a[:N] - a[N:]) ** 2
        w = lin[f"lin{t}.model.1.weight"].to(a.device, torch.float64)
        vals.append(F.conv2d(d, w).mean((1, 2, 3)))
    taps = torch.stack(vals, 1)
    return taps.sum(1), taps
