"""LPIPS on the GPU (csrc/sgr_lpips.cu through sugar_b200/lpips.py): each conv shape at odd and tiny sizes against
float64 F.conv2d on the device, the tap + pool kernel with its floors, the whole metric against the float64 oracle
(oracle/lpips_oracle.py) up to 1920x1080 and against the reference's own values (tests/golden/lpips_values.npz),
its determinism, and its agreement with torchvision's VGG16 on cuDNN at torch's default TF32."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import lpips_cases as lc  # noqa: E402
from oracle import lpips_oracle as lo  # noqa: E402
from sugar_b200 import _lib, lpips  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
U = 2.0 ** -11   # TF32's unit roundoff (10 mantissa bits, round to nearest)
EPS32 = 2.0 ** -24


def lpips_bound(v):
    """|sugar_b200 - float64| allowed for an LPIPS (or tap) value v: TF32 operands, float32 accumulation.  On one
    H100 80GB HBM3 the largest error measured was 6.3e-6 at 0.0097 (2x37x53), 1.0e-6 at 0.0027 (1920x1080) and
    1.4e-6 at 3.4e-7 (nearly equal images: the error is mostly absolute): a margin of about 5x."""
    return 2e-5 + 1e-3 * abs(v)


@pytest.fixture(scope="module")
def weights():
    return lc.make_state_dicts()


@pytest.fixture(scope="module")
def metric(tmp_path_factory):
    return lpips.LPIPS(*lc.write_weight_files(str(tmp_path_factory.mktemp("lpips"))), device=DEV)


def _nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous()


def _nchw(t):
    return t.permute(0, 3, 1, 2)


VGG_CONVS = sorted(set(lpips.CONV_SHAPES[1:]))


@pytest.mark.parametrize("cout,cin", VGG_CONVS)
@pytest.mark.parametrize("B,H,W", [(2, 1, 1), (2, 2, 3), (2, 37, 53), (1, 9, 130)])
def test_conv3x3_against_float64(cout, cin, B, H, W):
    g = torch.Generator(device=DEV).manual_seed(cin * 7 + cout + H)
    x = torch.rand(B, cin, H, W, device=DEV, generator=g)
    w = torch.randn(cout, cin, 3, 3, device=DEV, generator=g) * (2.0 / (9 * cin)) ** 0.5
    b = (torch.rand(cout, device=DEV, generator=g) - 0.5) * 0.1
    wk = lpips.tf32_round(w.permute(0, 2, 3, 1).contiguous())
    out = torch.empty(B, H, W, cout, device=DEV)
    _lib.check(_lib.lib.sgr_lpips_conv3x3(B, H, W, cin, cout, _nhwc(x).data_ptr(), wk.data_ptr(), b.data_ptr(),
                                          out.data_ptr(), _lib.stream(DEV)))
    w64 = wk.permute(0, 3, 1, 2).double()
    ref = F.relu(F.conv2d(x.double(), w64, b.double(), padding=1))
    # every product carries at most one TF32 rounding of x (the weights are TF32 already), the float32 sum at most
    # K of its own: a bound per output in terms of sum |x| |w|
    scale = F.conv2d(x.double().abs(), w64.abs(), b.double().abs(), padding=1)
    err = (_nchw(out).double() - ref).abs()
    bound = (U + 9 * cin * EPS32) * scale + 1e-30
    assert bool((err <= bound).all()), float((err / bound).max())
    assert float((err / scale.clamp_min(1e-30)).max()) < 2 * U


@pytest.mark.parametrize("N,H,W", [(1, 1, 1), (2, 2, 3), (2, 37, 53)])
def test_conv1_zscore_against_float64(N, H, W, weights):
    vgg, _ = weights
    g = torch.Generator(device=DEV).manual_seed(H * W)
    x, y = torch.rand(2, N, 3, H, W, device=DEV, generator=g)
    w, b = vgg["features.0.weight"].to(DEV), vgg["features.0.bias"].to(DEV)
    out = torch.empty(2 * N, H, W, 64, device=DEV)
    _lib.check(_lib.lib.sgr_lpips_conv1(N, H, W, x.data_ptr(), y.data_ptr(), w.permute(0, 2, 3, 1).contiguous().data_ptr(),
                                        b.data_ptr(), out.data_ptr(), _lib.stream(DEV)))
    mean = torch.tensor(lo.MEAN, dtype=torch.float32, device=DEV).view(1, 3, 1, 1)
    std = torch.tensor(lo.STD, dtype=torch.float32, device=DEV).view(1, 3, 1, 1)
    zin = ((torch.cat([x, y]) - mean) / std).double()
    ref = F.relu(F.conv2d(zin, w.double(), b.double(), padding=1))
    scale = F.conv2d(zin.abs(), w.double().abs(), b.double().abs(), padding=1)
    err = (_nchw(out).double() - ref).abs()
    assert bool((err <= 28 * EPS32 * scale + 1e-30).all())


@pytest.mark.parametrize("C", [64, 128, 256, 512])
@pytest.mark.parametrize("N,H,W", [(1, 1, 1), (2, 2, 3), (2, 5, 7), (2, 37, 53)])
def test_tap_and_pool(C, N, H, W):
    g = torch.Generator(device=DEV).manual_seed(C + H * W)
    feat = torch.rand(2 * N, H, W, C, device=DEV, generator=g)
    feat[0, 0, 0] = 0.0   # an all-zero pixel: the norm is eps alone
    lin = torch.rand(C, device=DEV, generator=g)
    nb = ((((H + 1) // 2) * ((W + 1) // 2)) + 31) // 32
    partials = torch.full((N, nb), float("nan"), dtype=torch.float64, device=DEV)
    pooled = torch.full((2 * N, H // 2, W // 2, C), float("nan"), device=DEV)
    _lib.check(_lib.lib.sgr_lpips_tap(N, H, W, C, feat.data_ptr(), lin.data_ptr(),
                                      pooled.data_ptr() if pooled.numel() else feat.data_ptr(),
                                      partials.data_ptr(), _lib.stream(DEV)))
    if pooled.numel():   # torch's max_pool2d refuses an empty output; the floored 1x1 input has none
        assert torch.equal(pooled, _nhwc(F.max_pool2d(_nchw(feat), 2, 2)))
    f = feat.double()
    f = f / (f.pow(2).sum(-1, keepdim=True).sqrt() + 1e-10)
    want = ((f[:N] - f[N:]) ** 2 * lin.double()).sum(-1).mean((1, 2))
    got = partials.sum(1) / (H * W)
    assert torch.allclose(got, want, rtol=1e-5, atol=1e-9), (got, want)


def test_unpooled_tap_only_at_512():
    feat = torch.zeros(2, 4, 4, 256, device=DEV)
    with pytest.raises(_lib.SgrError, match="pooled may be NULL at C = 512 only"):
        _lib.check(_lib.lib.sgr_lpips_tap(1, 4, 4, 256, feat.data_ptr(), feat.data_ptr(), None,
                                          feat.data_ptr(), _lib.stream(DEV)))


def test_against_reference_golden(metric, weights):
    gold = np.load(os.path.join(HERE, "golden", "lpips_values.npz"))
    assert int(gold["weight_seed"]) == lc.WEIGHT_SEED
    assert bytes(gold["weight_digest"]).hex() == lc.digest(*weights)
    for name, N, H, W, _, _ in lc.GOLDEN_CASES:
        x, y = (torch.from_numpy(gold[f"{name}_{k}"]).to(DEV) for k in "xy")
        got, taps = metric(x, y, return_taps=True)
        ref_taps = gold[f"{name}_taps_f64"]
        for n in range(N):
            for t in range(5):
                assert abs(float(taps[n, t]) - ref_taps[n, t]) <= lpips_bound(ref_taps[n, t]), (name, n, t)
            assert abs(float(got[n]) - ref_taps[n].sum()) <= lpips_bound(ref_taps[n].sum()), name
        # the reference's module sums a batch into one value
        assert abs(float(got.double().sum()) - float(gold[f"{name}_lpips_f64"][0])) <= N * lpips_bound(
            float(gold[f"{name}_lpips_f64"][0]))


@pytest.mark.parametrize("N,H,W,noise", [(1, 96, 128, 0.3), (1, 96, 128, 0.02), (2, 37, 53, 0.1),
                                         (1, 1080, 1920, 0.05), (1, 800, 800, 0.005)])
def test_against_float64_oracle(metric, weights, N, H, W, noise):
    x, y = (t.to(DEV) for t in lc.image_pair(N, H, W, noise, seed=H + W))
    got, taps = metric(x, y, return_taps=True)
    ref, ref_taps = lo.lpips64(x, y, *weights)
    for n in range(N):
        assert abs(float(got[n]) - float(ref[n])) <= lpips_bound(float(ref[n])), (float(got[n]), float(ref[n]))
        for t in range(5):
            assert abs(float(taps[n, t]) - float(ref_taps[n, t])) <= lpips_bound(float(ref_taps[n, t]))


def test_identical_images_give_zero(metric):
    x, _ = (t.to(DEV) for t in lc.image_pair(2, 40, 56, 0.1, seed=9))
    got, taps = metric(x, x.clone(), return_taps=True)
    assert torch.equal(got, torch.zeros_like(got)) and torch.equal(taps, torch.zeros_like(taps))


def test_deterministic_and_batch_independent(metric):
    x, y = (t.to(DEV) for t in lc.image_pair(3, 67, 45, 0.1, seed=11))
    a, ta = metric(x, y, return_taps=True)
    b, tb = metric(x, y, return_taps=True)
    assert torch.equal(a, b) and torch.equal(ta, tb)
    for n in range(3):
        s, ts = metric(x[n:n + 1], y[n:n + 1], return_taps=True)
        assert torch.equal(s[0], a[n]) and torch.equal(ts[0], ta[n])


def test_module_function_and_errors(tmp_path):
    lc.write_weight_files(str(tmp_path))
    x, y = (t.to(DEV) for t in lc.image_pair(1, 32, 32, 0.1, seed=3))
    d = lpips.lpips(x, y, net_type="vgg", weights_dir=str(tmp_path))
    assert d.shape == (1,) and float(d) > 0
    for kw in ({"net_type": "alex"}, {"net_type": "squeeze"}, {"version": "0.0"}):
        with pytest.raises(NotImplementedError):
            lpips.lpips(x, y, weights_dir=str(tmp_path), **kw)
    m = lpips.LPIPS(os.path.join(tmp_path, lpips.VGG_FILE), os.path.join(tmp_path, lpips.LIN_FILE), DEV)
    with pytest.raises(ValueError, match="H, W >= 16"):
        m(x[..., :15, :], y[..., :15, :])
    with pytest.raises(ValueError, match=r"\[N, 3, H, W\]"):
        m(x, y[:, :2])


def test_agrees_with_torchvision_cudnn_tf32(metric, weights):
    import scripts.bench_lpips as bl
    assert torch.backends.cudnn.allow_tf32
    theirs = bl.cudnn_lpips(torch, *weights, DEV)
    for N, H, W, noise in ((1, 256, 384, 0.2), (1, 540, 960, 0.02), (2, 37, 53, 0.1)):
        x, y = (t.to(DEV) for t in lc.image_pair(N, H, W, noise, seed=W))
        ref = lo.lpips64(x, y, *weights)[0]
        ours, cud = metric(x, y).double(), theirs(x, y).double()
        for n in range(N):
            assert abs(float(ours[n] - cud[n])) <= 2 * lpips_bound(float(ref[n])), (float(ours[n]), float(cud[n]))
