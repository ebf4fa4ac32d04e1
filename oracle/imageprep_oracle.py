"""numpy restatement of the reference's ground-truth image preparation (sugar_b200/csrc/sgr_image.cu is held to it
byte for byte).

The reference turns a decoded uint8 image into the float32 [3,H,W] image the trainers compare against in up to four
steps, each only where it runs:

1. alpha composite (readCamerasFromTransforms, gaussian_splatting/scene/dataset_readers.py:204-210, and
   load_gs_cameras with white_background, sugar_scene/cameras.py:102-107), in float64 as numpy evaluates it:
   n = u / 255.0, arr = n_c n_a + bg (1 - n_a), byte = trunc(arr 255.0) (np.array(.., dtype=np.byte) reinterpreted
   as RGB bytes by Pillow: a truncation, not a rounding);
2. Pillow's Image.resize(size) with its default filter (bicubic, a = -0.5, antialiased), from Pillow's
   libImaging/Resample.c: float64 coefficient tables per axis, 22-bit fixed point, int32 accumulation from 1 << 21,
   horizontal pass first into a uint8 intermediate, a pass only for an axis whose size changes;
3. an RGBA image resized without a composite goes through premultiplied RGBa (Image.resize converts RGBA to RGBa
   and back; libImaging/Convert.c rgbA2rgba / rgba2rgbA).  An RGBA image whose size does not change is copied
   as it is.  The alpha is then dropped: loadCam's mask test compares the height with 4 (camera_utils.py:47-50), so
   the mask is never applied to an image taller than 4 px;
4. uint8 -> float32 / 255, a correctly rounded float32 division (PILtoTorch on the CPU).
"""
import numpy as np

PRECISION_BITS = 22   # 32 - 8 - 2
BICUBIC_A = -0.5
BICUBIC_SUPPORT = 2.0

PLAIN, COMPOSITE, PREMULTIPLY = 0, 1, 2   # sgr_image_prepare's modes (include/sugar_b200.h)


def bicubic(x):
    """Resample.c bicubic_filter, elementwise, in its own evaluation order."""
    x = np.abs(np.asarray(x, np.float64))
    a = BICUBIC_A
    inner = ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    outer = (((x - 5) * x + 8) * x - 4) * a
    return np.where(x < 1.0, inner, np.where(x < 2.0, outer, 0.0))


def resample_coeffs(in_size: int, out_size: int):
    """Resample.c precompute_coeffs + normalize_coeffs_8bpc for the box (0, in_size) -> (bounds int32 [out,2] =
    (xmin, count), coeffs int32 [out, ksize], ksize).  Weights past a row's count are 0."""
    if in_size < 1 or out_size < 1:
        raise ValueError(f"resample sizes must be >= 1, got {in_size} -> {out_size}")
    scale = float(in_size) / out_size
    filterscale = max(scale, 1.0)
    support = BICUBIC_SUPPORT * filterscale
    ksize = int(np.ceil(support)) * 2 + 1
    ss = 1.0 / filterscale
    center = (np.arange(out_size, dtype=np.float64) + 0.5) * scale
    xmin = np.maximum(np.trunc(center - support + 0.5), 0).astype(np.int64)
    xmax = np.minimum(np.trunc(center + support + 0.5), in_size).astype(np.int64) - xmin
    kk = np.zeros((out_size, ksize), np.float64)
    ww = np.zeros(out_size, np.float64)
    for x in range(ksize):                        # left to right, as the C loop sums them
        live = x < xmax
        w = bicubic(((x + xmin) - center + 0.5) * ss)
        kk[:, x] = np.where(live, w, 0.0)
        ww = np.where(live, ww + w, ww)
    kk = np.where(ww[:, None] != 0.0, kk / np.where(ww != 0.0, ww, 1.0)[:, None], kk)
    one = float(1 << PRECISION_BITS)
    fixed = np.trunc(np.where(kk < 0, -0.5 + kk * one, 0.5 + kk * one)).astype(np.int32)
    fixed[np.arange(ksize)[None, :] >= xmax[:, None]] = 0
    bounds = np.stack([xmin, xmax], 1).astype(np.int32)
    return bounds, np.ascontiguousarray(fixed), ksize


def _clip8(acc):
    return np.clip(acc >> PRECISION_BITS, 0, 255).astype(np.uint8)


def resample_axis(img, bounds, coeffs, axis):
    """One Resample.c 8-bit pass of uint8 [H,W,C] along `axis` (1: horizontal, 0: vertical)."""
    n_in = img.shape[axis]
    acc = np.full(img.shape[:axis] + (len(bounds),) + img.shape[axis + 1:], 1 << (PRECISION_BITS - 1), np.int32)
    shape = [1, 1, 1]
    shape[axis] = len(bounds)
    for x in range(coeffs.shape[1]):
        idx = np.minimum(bounds[:, 0] + x, n_in - 1)
        w = coeffs[:, x].reshape(shape)
        acc += np.take(img, idx, axis=axis).astype(np.int32) * w
    return _clip8(acc)


def premultiply(rgba):
    """Convert.c rgbA2rgba: RGBA -> RGBa, c = MULDIV255(c, a)."""
    rgba = np.asarray(rgba, np.uint8)
    a = rgba[..., 3:4].astype(np.int32)
    tmp = rgba[..., :3].astype(np.int32) * a + 128
    out = rgba.copy()
    out[..., :3] = ((tmp >> 8) + tmp) >> 8
    return out


def unpremultiply(rgba):
    """Convert.c rgba2rgbA: RGBa -> RGBA, c = clip8(255 c / a) for 0 < a < 255, unchanged otherwise."""
    rgba = np.asarray(rgba, np.uint8)
    a = rgba[..., 3:4].astype(np.int32)
    c = rgba[..., :3].astype(np.int32)
    div = np.minimum(255 * c // np.maximum(a, 1), 255)
    out = rgba.copy()
    out[..., :3] = np.where((a == 0) | (a == 255), c, div)
    return out


def composite(rgba, white: bool):
    """The float64 composite over a white (1) or black (0) background -> uint8 [H,W,3]."""
    norm = np.asarray(rgba, np.uint8) / 255.0
    bg = np.array([1, 1, 1]) if white else np.array([0, 0, 0])
    arr = norm[:, :, :3] * norm[:, :, 3:4] + bg * (1 - norm[:, :, 3:4])
    return np.trunc(arr * 255.0).astype(np.uint8)


def prepare_bytes(img, out_w: int, out_h: int, background=None):
    """uint8 [H,W,C] (C = 3 or 4) -> the prepared uint8 [out_h, out_w, 3].  `background`: None (no composite), or
    "white" / "black" to composite an RGBA image first."""
    img = np.ascontiguousarray(img, np.uint8)
    if img.ndim != 3 or img.shape[2] not in (3, 4):
        raise ValueError(f"image must be uint8 [H,W,3|4], got {img.shape}")
    H, W, C = img.shape
    if background is not None:
        if C != 4:
            raise ValueError("the composite needs an RGBA image")
        img = composite(img, background == "white")
    elif C == 4:
        if (out_w, out_h) == (W, H):
            return np.ascontiguousarray(img[..., :3])
        img = premultiply(img)
    if out_w != W:
        img = resample_axis(img, *resample_coeffs(W, out_w)[:2], axis=1)
    if out_h != H:
        img = resample_axis(img, *resample_coeffs(H, out_h)[:2], axis=0)
    if img.shape[2] == 4:
        img = unpremultiply(img)
    return np.ascontiguousarray(img[..., :3])


def to_float(u8):
    """uint8 [H,W,3] -> float32 [3,H,W] = u / 255 (float32 division)."""
    return np.ascontiguousarray(np.transpose(u8, (2, 0, 1)).astype(np.float32) / np.float32(255.0))


def prepare(img, out_w: int, out_h: int, background=None):
    return to_float(prepare_bytes(img, out_w, out_h, background))
