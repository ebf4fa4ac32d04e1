"""CPU checks of the fused L1 + D-SSIM loss's yardsticks and plumbing: both oracle formulations against the goldens the
reference's own loss_utils.py produced, the window recipe bit for bit, argument validation of the C entry points
without a GPU, and the composed coarse step with dssim_factor > 0 over the reference ops."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(HERE, "golden"))

from make_ssim_golden import CASES, STORE_INPUTS, inputs_digest, make_inputs, to_float  # noqa: E402
from oracle import ssim_oracle as so  # noqa: E402


def load_case(name):
    with np.load(os.path.join(HERE, "golden", f"ssim_{name}.npz")) as z:
        gold = {k: z[k] for k in z.files}
    pred, gt = make_inputs(name)
    assert np.array_equal(inputs_digest(pred, gt), gold["inputs_digest"]), "inputs do not regenerate"
    if name in STORE_INPUTS:
        assert np.array_equal(pred, gold["code_pred"]) and np.array_equal(gt, gold["code_gt"])
    return gold, pred, gt


def grad_err(g, gold, tag):
    """max |g - golden| over the golden's entries / max(|golden|_inf, 0.8 / N) (the L1 term's scale floors the
    denominator, so that pred == gt, whose true gradient is 0, is measured against the gradient's natural size)."""
    a = np.asarray(g, np.float64).reshape(-1)
    if "grad_idx" in gold:
        a = a[gold["grad_idx"]]
    b = gold["grad_" + tag].astype(np.float64)
    n = int(np.prod(gold["shape"]))
    return np.abs(a - b).max() / max(np.abs(b).max(), 0.8 / n)


@pytest.mark.parametrize("name", list(CASES))
def test_torch_oracle_reproduces_float32_goldens(name):
    gold, pc, gc = load_case(name)
    pred = torch.from_numpy(to_float(pc, np.float32)).requires_grad_(True)
    gt = torch.from_numpy(to_float(gc, np.float32))
    so.l1_dssim_torch(pred, gt, 0.2).backward()
    with torch.no_grad():
        if pred.dim() == 4:
            s = so.ssim_torch(pred, gt, size_average=False).numpy()
            l1 = (pred - gt).abs().mean(dim=(1, 2, 3)).numpy()
        else:
            s, l1 = np.array([float(so.ssim_torch(pred, gt))]), np.array([float((pred - gt).abs().mean())])
    np.testing.assert_allclose(s, gold["ssim_f32"], rtol=1e-6, atol=0)
    np.testing.assert_allclose(l1, gold["l1_f32"], rtol=1e-6, atol=1e-12)
    assert grad_err(pred.grad.numpy(), gold, "f32") <= 1e-5


@pytest.mark.parametrize("name", list(CASES))
def test_numpy_float64_formulation_reproduces_float64_goldens(name):
    gold, pc, gc = load_case(name)
    o = so.ssim_numpy(to_float(pc, np.float64), to_float(gc, np.float64), 0.2)
    np.testing.assert_allclose(o["ssim"], gold["ssim_f64"], rtol=1e-10, atol=0)
    np.testing.assert_allclose(o["l1"], gold["l1_f64"], rtol=1e-10, atol=1e-15)
    assert grad_err(o["grad"], gold, "f64") <= 1e-10


def test_window_equals_the_reference_recipe_bit_for_bit():
    from sugar_b200 import loss
    with np.load(os.path.join(HERE, "golden", "ssim_rand_3x7x9.npz")) as z:
        w1, w2 = z["window_1d"], z["window_2d"]
    assert w1.dtype == np.float32 and np.array_equal(loss.gaussian_window(11, 1.5).numpy(), w1)
    assert np.array_equal(np.asarray(loss._WINDOW, np.float32), w1)   # what the C ABI receives
    p = loss._params(1, 3, 8, 8)
    assert np.array_equal(np.asarray(list(p.window), np.float32), w1)
    assert np.float32(p.c1) == np.float32(0.01 ** 2) and np.float32(p.c2) == np.float32(0.03 ** 2)
    assert np.array_equal(so.window_2d().numpy(), w2) and np.array_equal(so.gaussian_1d().numpy(), w1)


def test_loss_entry_points_validate_without_gpu():
    from sugar_b200 import _lib
    L = _lib.lib
    assert L.sgr_struct_bytes(4) == ctypes.sizeof(_lib.SgrSsimParams) == 68
    names = {L.sgr_kernel_name(k).decode() for k in range(L.sgr_num_kernel_kinds())}
    assert {"loss_forward", "loss_backward"} <= names
    assert L.sgr_l1_ssim_scratch_bytes(0, 3, 10, 10) == 0
    assert 0 < L.sgr_l1_ssim_scratch_bytes(1, 3, 1080, 1920) <= L.sgr_l1_ssim_scratch_bytes(2, 3, 1080, 1920)
    dummy = ctypes.c_void_p(256)

    def params(B, C, H, W):
        p = _lib.SgrSsimParams()
        p.B, p.C, p.H, p.W = B, C, H, W
        return p
    fwd = lambda p, *ptrs: L.sgr_l1_ssim_forward(ctypes.byref(p) if p is not None else None, *ptrs)
    bwd = lambda p, *ptrs: L.sgr_l1_ssim_backward(ctypes.byref(p) if p is not None else None, *ptrs)
    assert fwd(None, *([dummy] * 5), None) == -1 and b"null params" in L.sgr_last_error()
    for bad in ((0, 3, 8, 8), (1, 0, 8, 8), (1, 3, 0, 8), (1, 3, 8, 0), (-1, 3, 8, 8)):
        assert fwd(params(*bad), *([dummy] * 5), None) == -1 and b"bad sizes" in L.sgr_last_error()
        assert bwd(params(*bad), *([dummy] * 6), None) == -1
    assert fwd(params(1, 3, 32768, 32768), *([dummy] * 5), None) == -1 and b"2^31" in L.sgr_last_error()
    assert fwd(params(70000, 1, 2, 2), *([dummy] * 5), None) == -1 and b"65535" in L.sgr_last_error()
    ok = params(2, 3, 8, 8)
    for i in range(5):
        ptrs = [dummy] * 5
        ptrs[i] = None
        assert fwd(ok, *ptrs, None) == -1 and b"null pointer" in L.sgr_last_error()
    for i in range(6):
        ptrs = [dummy] * 6
        ptrs[i] = None
        assert bwd(ok, *ptrs, None) == -1 and b"null pointer" in L.sgr_last_error()


class FakeRasterizerModule:
    """Differentiable stand-in with the rasterizer module's surface: image = mean colour plus a fixed ramp (so that the
    image has a non-trivial SSIM) plus zero-weight terms that give every input a gradient; radii = 1."""

    class GaussianRasterizationSettings:
        def __init__(self, **kw):
            self.__dict__.update(kw)

    class GaussianRasterizer:
        def __init__(self, st):
            self.st = st

        def __call__(self, means3D, means2D, opacities, scales, rotations, shs=None, colors_precomp=None):
            H, W = self.st.image_height, self.st.image_width
            c = colors_precomp if colors_precomp is not None else shs[:, 0]
            z = 0 * (opacities.sum() + scales.sum() + rotations.sum() + means3D.sum())
            ramp = torch.linspace(0, 0.3, H * W).view(1, H, W)
            return (c.mean(0)[:, None, None] + z + ramp) + 0 * self.st.bg[:, None, None], \
                torch.ones(means3D.shape[0], dtype=torch.int32)


def test_coarse_sdf_step_with_dssim_over_reference_ops():
    """dssim_factor=0.2: the photometric term is ops.l1_dssim, it equals 0.8 L1 + 0.2 (1 - ssim) of the oracle, the rest
    of the step is unchanged, and every parameter receives a gradient."""
    import bench
    import bench_workloads as bw
    from oracle import field_oracle as fo
    steps = bw._load_steps_without_package()
    scenes = bench.load_scenes()
    sc = scenes.make_scene(400, 40, 32, seed=3)
    cam = steps.camera_from_scene(sc, "cpu")
    ops = bw.reference_ops(torch, FakeRasterizerModule)
    seen = []

    def spy(pred, gt, f):
        out = so.l1_dssim_torch(pred, gt, f)
        seen.append((pred.detach().clone(), gt, f, out.detach()))
        return out
    ops.l1_dssim = spy
    gt = torch.rand(3, 32, 40, generator=torch.Generator().manual_seed(4))
    losses = {}
    for f in (0.0, 0.2):
        leaf = lambda t: t.clone().requires_grad_(True)
        raw = dict(points=leaf(torch.from_numpy(sc.means3D)), sh_dc=leaf(torch.from_numpy(sc.shs[:, :1].copy())),
                   sh_rest=leaf(torch.from_numpy(sc.shs[:, 1:].copy())),
                   densities=leaf(torch.logit(torch.from_numpy(sc.opacities).clamp(1e-4, 1 - 1e-4))),
                   scales=leaf(torch.from_numpy(sc.scales).log()), quaternions=leaf(torch.from_numpy(sc.rotations) * 1.3))
        knn = fo.knn_idx(raw["points"].detach(), 16)
        losses[f], _ = steps.coarse_sdf_step(raw, cam, gt, knn, ops, n_samples=1000,
                                             generator=torch.Generator().manual_seed(1), dssim_factor=f)
        for k, v in raw.items():
            assert v.grad is not None and bool(torch.isfinite(v.grad).all()), (f, k)
    assert len(seen) == 1 and seen[0][2] == 0.2           # plain L1 at 0.0: the oracle is not called
    img, g, _, val = seen[0]
    l1 = (img - g).abs().mean()
    want = 0.8 * l1 + 0.2 * (1 - so.ssim_torch(img[None], g[None]))
    assert abs(float(val) - float(want)) <= 1e-6 and 0.05 < float(so.ssim_torch(img, g)) < 0.99
    # the step's other terms are the same: the two losses differ by the photometric terms only
    assert abs(float(losses[0.2] - losses[0.0]) - float(val - l1)) <= 1e-5
