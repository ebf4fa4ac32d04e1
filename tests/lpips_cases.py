"""Seeded LPIPS weights in the two files' formats (torchvision's vgg16 state dict and LPIPS v0.1's linear layers),
and seeded image pairs.  Shared by the LPIPS golden maker and the tests, so the ~59 MB of weights are never stored:
the golden keeps the seed and the digest of the float32 bytes."""
import hashlib
import os

import numpy as np
import torch

CONV_INDICES = (0, 2, 5, 7, 10, 12, 14, 17, 19, 21, 24, 26, 28)
CONV_SHAPES = ((64, 3), (64, 64), (128, 64), (128, 128), (256, 128), (256, 256), (256, 256), (512, 256), (512, 512),
               (512, 512), (512, 512), (512, 512), (512, 512))
TAP_CHANNELS = (64, 128, 256, 512, 512)
WEIGHT_SEED = 20261019


def make_state_dicts(seed=WEIGHT_SEED):
    """-> (vgg16 `features.*` state dict, LPIPS `lin{i}.model.1.weight` state dict), float32.  Convs are He-scaled
    normals (activations keep their scale through 13 layers) with small biases; linear weights are uniform [0, 1),
    non-negative as the trained ones are."""
    g = torch.Generator().manual_seed(seed)
    vgg = {}
    for i, (co, ci) in zip(CONV_INDICES, CONV_SHAPES):
        vgg[f"features.{i}.weight"] = torch.randn(co, ci, 3, 3, generator=g) * (2.0 / (9 * ci)) ** 0.5
        vgg[f"features.{i}.bias"] = (torch.rand(co, generator=g) - 0.5) * 0.1
    lin = {f"lin{i}.model.1.weight": torch.rand(1, c, 1, 1, generator=g) for i, c in enumerate(TAP_CHANNELS)}
    return vgg, lin


def digest(vgg, lin) -> str:
    h = hashlib.sha256()
    for sd in (vgg, lin):
        for k in sorted(sd):
            h.update(k.encode())
            h.update(sd[k].numpy().astype(np.float32).tobytes())
    return h.hexdigest()


def write_weight_files(directory, seed=WEIGHT_SEED):
    """Write vgg16-397923af.pth and vgg.pth into `directory` -> (vgg_path, lin_path)."""
    vgg, lin = make_state_dicts(seed)
    os.makedirs(directory, exist_ok=True)
    vp, lp = os.path.join(directory, "vgg16-397923af.pth"), os.path.join(directory, "vgg.pth")
    torch.save(vgg, vp)
    torch.save(lin, lp)
    return vp, lp


def image_pair(N, H, W, noise, seed):
    """A smooth random image and a copy with uniform noise of amplitude `noise`, clamped to [0, 1]: float32
    [N, 3, H, W] each."""
    g = torch.Generator().manual_seed(seed)
    base = torch.rand(N, 3, (H + 3) // 4, (W + 3) // 4, generator=g)
    x = torch.nn.functional.interpolate(base, size=(H, W), mode="bilinear", align_corners=False)
    y = (x + noise * (2 * torch.rand(x.shape, generator=g) - 1)).clamp(0, 1)
    return x.contiguous(), y.contiguous()


# (name, N, H, W, noise, seed) of the golden pairs
GOLDEN_CASES = (
    ("smooth_64x64", 1, 64, 64, 0.2, 1),
    ("close_64x96", 1, 64, 96, 0.01, 2),
    ("odd_37x53", 1, 37, 53, 0.1, 3),
    ("min_16x16", 1, 16, 16, 0.3, 4),
    ("batch2_48x40", 2, 48, 40, 0.05, 5),
)
