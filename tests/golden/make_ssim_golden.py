"""Golden vectors for the trainers' photometric loss from the reference's OWN code.

Runs where the reference sources are present:  python tests/golden/make_ssim_golden.py
Imports sugar_utils/loss_utils.py from /root/reference by path at run time (it needs only torch) and calls its own
`ssim` and `l1_loss`; nothing of it is copied into the repository, only the resulting numbers are stored.
Outputs: tests/golden/ssim_<case>.npz, each holding
    code_pred, code_gt   int16 inputs as multiples of 2^-12 (exact in float32 and float64), or, for the
                         270x480 case, the digest of the inputs `make_inputs` regenerates from integers
    window_1d, window_2d the float32 window of the recipe
    ssim_f32/_f64, l1_f32/_f64   per-image SSIM and L1 means (the reference's ssim(size_average=False) / l1_loss)
    grad_f32, grad_f64           d/d pred of 0.8 * l1_loss + 0.2 * (1 - ssim), flattened: whole for small cases,
                                 else at the flat indices grad_idx (evenly spaced entries + the largest)
Float64 runs the reference's code unchanged on the float64 copies of the same inputs (its window follows the
input's dtype).  The inputs are integers, the RNG is numpy's PCG64 integer stream: the files regenerate
byte-identical.
"""
import hashlib
import importlib.util
import io
import os
import sys
import zipfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
REF = "/root/reference/sugar_utils/loss_utils.py"
SCALE = 4096.0      # inputs are code / SCALE
WHOLE_MAX = 6000    # gradients of at most this many entries are stored whole

# name -> (shape, kind, seed)
CASES = {
    "rand_1x3x37x53": ((1, 3, 37, 53), "random", 0),
    "rand_3x7x9": ((3, 7, 9), "random", 1),
    "batch_2x3x64x96": ((2, 3, 64, 96), "random", 2),
    "gray_1x1x48x80": ((1, 1, 48, 80), "random", 3),
    "equal_3x64x96": ((3, 64, 96), "equal", 4),
    "smooth_3x270x480": ((3, 270, 480), "smooth", 5),
}
STORE_INPUTS = {k for k, (s, _, _) in CASES.items() if np.prod(s) <= 40_000}


def make_inputs(name):
    """int16 codes (pred, gt) of a case; values = code / 4096."""
    shape, kind, seed = CASES[name]
    rng = np.random.default_rng(seed)
    if kind in ("random", "equal"):
        gt = rng.integers(0, 4097, size=shape, dtype=np.int64)
        pred = gt.copy() if kind == "equal" else rng.integers(0, 4097, size=shape, dtype=np.int64)
    else:
        # smooth ground truth: bilinear interpolation of a coarse grid (16-pixel cells) in integers, and the
        # render = ground truth + uniform noise of +-0.01
        C, H, W = shape
        g = rng.integers(64, 4033, size=(C, H // 16 + 2, W // 16 + 2), dtype=np.int64)
        yy, xx = np.arange(H), np.arange(W)
        y0, fy = (yy // 16)[:, None], (yy % 16)[:, None]
        x0, fx = (xx // 16)[None, :], (xx % 16)[None, :]
        gt = ((16 - fy) * (16 - fx) * g[:, y0, x0] + (16 - fy) * fx * g[:, y0, x0 + 1] +
              fy * (16 - fx) * g[:, y0 + 1, x0] + fy * fx * g[:, y0 + 1, x0 + 1]) // 256
        pred = gt + rng.integers(-41, 42, size=shape, dtype=np.int64)
    return pred.astype(np.int16), gt.astype(np.int16)


def inputs_digest(pred, gt):
    return np.frombuffer(hashlib.sha256(pred.tobytes() + gt.tobytes()).digest(), np.uint8)


def to_float(code, dtype):
    return code.astype(dtype) / dtype(SCALE)


def import_reference_losses():
    spec = importlib.util.spec_from_file_location("sugar_ref_loss_utils", REF)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def grad_index(g64):
    """Entries of a gradient a golden keeps: all of them for small cases (None), else 1024 evenly spaced ones and
    the 64 largest in magnitude of the float64 gradient, sorted."""
    a = g64.reshape(-1)
    if a.size <= WHOLE_MAX:
        return None
    strided = np.arange(1024, dtype=np.int64) * a.size // 1024
    top = np.argsort(-np.abs(a), kind="stable")[:64]
    return np.unique(np.concatenate([strided, top])).astype(np.int64)


def run_reference(ref, pred_code, gt_code, dtype):
    pred = torch.from_numpy(to_float(pred_code, dtype)).requires_grad_(True)
    gt = torch.from_numpy(to_float(gt_code, dtype))
    loss = 0.8 * ref.l1_loss(pred, gt) + 0.2 * (1.0 - ref.ssim(pred, gt))
    loss.backward()
    with torch.no_grad():
        if pred.dim() == 4:
            s = ref.ssim(pred, gt, size_average=False)
            l1 = torch.stack([ref.l1_loss(pred[b], gt[b]) for b in range(pred.shape[0])])
        else:
            s, l1 = ref.ssim(pred, gt).reshape(1), ref.l1_loss(pred, gt).reshape(1)
    return s.numpy(), l1.numpy(), pred.grad


def make_case(ref, name):
    pred_code, gt_code = make_inputs(name)
    out = {"inputs_digest": inputs_digest(pred_code, gt_code), "shape": np.asarray(CASES[name][0], np.int64)}
    if name in STORE_INPUTS:
        out["code_pred"], out["code_gt"] = pred_code, gt_code
    w1 = ref.gaussian(11, 1.5)
    out["window_1d"] = w1.numpy().astype(np.float32)
    out["window_2d"] = ref.create_window(11, 1)[0, 0].numpy().astype(np.float32)
    grads = {}
    for dt, tag in ((np.float32, "f32"), (np.float64, "f64")):
        s, l1, g = run_reference(ref, pred_code, gt_code, dt)
        out["ssim_" + tag], out["l1_" + tag] = s, l1
        grads[tag] = g.detach().numpy().reshape(-1)
    idx = grad_index(grads["f64"])
    if idx is not None:
        out["grad_idx"] = idx
    for tag, g in grads.items():
        out["grad_" + tag] = g if idx is None else g[idx]
    return out


def save_deterministic(path, arrays):
    """np.savez with fixed zip timestamps so that the file's bytes depend on its arrays only."""
    with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_DEFLATED) as z:
        for k in sorted(arrays):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(arrays[k]), allow_pickle=False)
            info = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            z.writestr(info, buf.getvalue())


def main():
    torch.set_num_threads(1)   # the summation order of the CPU convolutions does not depend on the host's cores
    ref = import_reference_losses()
    for name in CASES:
        path = os.path.join(HERE, f"ssim_{name}.npz")
        save_deterministic(path, make_case(ref, name))
        print(path, os.path.getsize(path))


if __name__ == "__main__":
    main()
