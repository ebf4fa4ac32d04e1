"""The SH colour's view-direction Jacobian (dRGB/dx, dRGB/dy, dRGB/dz per Gaussian) is computed by the forward and kept
in the geometry state; the per-Gaussian backward takes the view-direction term of dL/dmeans3D from it and builds
dL/dsh from the basis alone.  So the backward must not depend on the values of the SH coefficients it is handed (only
on their shape), and where the direction term is most of dL/dmeans3D it must still match the CPU oracle."""
import ctypes as C

import numpy as np
import pytest

import helpers as h

pytestmark = pytest.mark.gpu

GRAD_RTOL = 1e-4
ORACLE_GRAD_RTOL = 5e-4
# two backwards of one forward differ only by the order of the blend backward's fp32 atomics: up to ~1.5e-6 in
# raw-parameter mode's dL/dscales on these scenes (the chain rule of exp multiplies by the scale)
RERUN_RTOL = 1e-5
LAYOUTS = [(16, 0), (16, 1), (16, 2), (16, 3), (9, 0), (9, 1), (9, 2)]
BG = (0.1, 0.2, 0.3)


def _at_offset12(x):
    """x's values in a tensor that starts 12 bytes into a larger allocation: contiguous, not 16-byte aligned."""
    import torch
    buf = torch.zeros(x.numel() + 3, dtype=x.dtype, device=x.device)
    v = buf[3:].view(x.shape)
    v.copy_(x)
    return v


def _inputs(M, raw, offset):
    """Seeded scene tensors for _C: combined SH rows [P,M,3], or (raw-parameter mode) logits / log-scales /
    un-normalised quaternions and the (dc [P,1,3], rest [P,M-1,3]) pair.  `offset`: every per-Gaussian input starts
    12 bytes into its allocation (the word-by-word staging paths)."""
    import torch
    from sugar_b200 import scenes
    P, W, H = 3001, 150, 90
    sc = scenes.make_scene(P, W, H, seed=70 + M, camera="posed")
    t = h.to_torch(sc)
    g = dict(means3D=t["means3D"], opacity=t["opacities"], scales=t["scales"], rotations=t["rotations"])
    if raw:
        g.update(opacity=torch.logit(g["opacity"].clamp(1e-4, 1 - 1e-4)), scales=g["scales"].log(),
                 rotations=g["rotations"] * 1.7, sh=t["shs"][:, :1].contiguous(), sh_rest=t["shs"][:, 1:M].contiguous())
    else:
        g["sh"] = t["shs"][:, :M].contiguous()
    if offset:
        g = {k: _at_offset12(v) for k, v in g.items()}
        assert all(v.data_ptr() % 16 != 0 for v in g.values())
    dL = torch.from_numpy(scenes.upstream_grad(W, H, seed=4)).cuda()
    return sc, t, g, dL


def _forward(sc, t, g, deg):
    import torch
    from sugar_b200 import _C
    absent = torch.Tensor([])
    return _C.rasterize_gaussians(torch.tensor(BG, device="cuda"), g["means3D"], absent, g["opacity"], g["scales"],
                                  g["rotations"], 1.0, absent, t["viewmatrix"], t["projmatrix"], sc.tanfovx, sc.tanfovy,
                                  sc.height, sc.width, g["sh"], deg, t["campos"], False, False, sh_rest=g.get("sh_rest"))


def _backward(sc, t, g, deg, fw, dL, sh, sh_rest):
    import torch
    from sugar_b200 import _C
    R, _color, radii, geom, binning, img = fw
    absent = torch.Tensor([])
    out = _C.rasterize_gaussians_backward(torch.tensor(BG, device="cuda"), g["means3D"], radii, absent, g["scales"],
                                          g["rotations"], 1.0, absent, t["viewmatrix"], t["projmatrix"], sc.tanfovx,
                                          sc.tanfovy, dL, sh, deg, t["campos"], geom, R, binning, img, False,
                                          sh_rest=sh_rest)
    names = ["means2D", "colors", "opacity", "means3D", "cov3D", "sh", "scales", "rotations"]
    return dict(zip(names + (["sh_rest"] if sh_rest is not None else []), out))


def _nan_like(x):
    """A tensor of x's shape and alignment filled with NaN."""
    import torch
    y = _at_offset12(torch.zeros_like(x)) if x.data_ptr() % 16 else torch.empty_like(x)
    return y.fill_(float("nan"))


@pytest.mark.parametrize("offset", [False, True], ids=["aligned", "offset12"])
@pytest.mark.parametrize("raw", [False, True], ids=["combined", "raw"])
@pytest.mark.parametrize("M,deg", LAYOUTS)
def test_backward_reads_no_sh_coefficients(M, deg, raw, offset):
    """One forward with real SH, then two backwards: one handed the real coefficients, one handed NaN-filled tensors
    of the same shapes.  Every gradient must be finite and agree to the atomics-order noise of two backwards."""
    import torch
    sc, t, g, dL = _inputs(M, raw, offset)
    fw = _forward(sc, t, g, deg)
    assert int((fw[2] > 0).sum()) > 1000
    real = _backward(sc, t, g, deg, fw, dL, g["sh"], g.get("sh_rest"))
    nan = _backward(sc, t, g, deg, fw, dL, _nan_like(g["sh"]), _nan_like(g["sh_rest"]) if raw else None)
    assert set(real) == set(nan)
    for k in real:
        a, b = nan[k], real[k]
        assert a.shape == b.shape, k
        assert bool(torch.isfinite(a).all()), f"{k} is not finite with NaN coefficients"
        assert bool(torch.isfinite(b).all()), k
        assert h.rel_err(a.cpu().numpy(), b.cpu().numpy()) <= RERUN_RTOL, k
    assert float(real["means3D"].abs().max()) > 0.0


def _direction_dominated_scene():
    """Degree-1 coefficients of magnitude 200 perpendicular to each Gaussian's view direction: they leave the colours
    as they are (the band-1 term is their dot product with the direction) but make dRGB/d(dir) large, so the
    view-direction term is most of dL/dmeans3D."""
    from sugar_b200 import scenes
    P, W, H = 2000, 160, 96
    sc = scenes.make_scene(P, W, H, seed=5, camera="posed")
    rng = np.random.default_rng(9)
    d = sc.means3D.astype(np.float64) - sc.campos.astype(np.float64).reshape(1, 3)
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    sh = sc.shs.astype(np.float64).copy()
    for c in range(3):
        a = np.cross(d, rng.normal(size=(P, 3)))
        a *= 200.0 / np.linalg.norm(a, axis=1, keepdims=True)
        # band 1 = C1 (-y sh_1 + z sh_2 - x sh_3) = C1 <a, dir> with a = (-sh_3, -sh_1, sh_2)
        sh[:, 3, c], sh[:, 1, c], sh[:, 2, c] = -a[:, 0], -a[:, 1], a[:, 2]
    return sc._replace(shs=sh.astype(np.float32)), scenes.upstream_grad(W, H)


def _oracle_dmeans3D_without_direction_term(fw, bw):
    """The oracle's per-Gaussian backward with dL/dRGB = 0: dL/dmeans3D without the view-direction term."""
    from oracle import raster_oracle as ro
    L, i, _p = ro.lib(), fw["_in"], ro._p
    P, W, H, M, D = fw["P"], fw["W"], fw["H"], fw["M"], fw["D"]
    g = [np.zeros(s, np.float32) for s in ((P, 3), (P, 6), (P, M, 3), (P, 3), (P, 4))]
    L.oracle_preprocess_backward(
        C.c_int(P), C.c_int(D), C.c_int(M), _p(i["means3D"]), _p(fw["radii"]), _p(i["shs"]), _p(fw["clamped"]),
        _p(i["scales"]), _p(i["rotations"]), C.c_float(i["scale_modifier"]), _p(fw["cov3D"]), _p(i["viewmatrix"]),
        _p(i["projmatrix"]), C.c_int(W), C.c_int(H), C.c_float(i["tanfovx"]), C.c_float(i["tanfovy"]),
        _p(i["campos"]), _p(bw["dL_dmeans2D"].copy()), _p(bw["dL_dconic"].copy()), _p(np.zeros((P, 3), np.float32)),
        *(_p(x) for x in g))
    return g[0]


def test_direction_dominated_means_gradient_matches_oracle():
    from sugar_b200 import diff_gaussian_rasterization as ours
    sc, dL = _direction_dominated_scene()
    fw, bw = h.run_oracle(sc, np.asarray(BG, np.float32), dL, use_sh=True, sh_degree=3)
    rest = _oracle_dmeans3D_without_direction_term(fw, bw)
    direction = bw["dL_dmeans3D"].astype(np.float64) - rest
    assert np.abs(direction).max() > 4.0 * np.abs(rest).max()
    a = h.run_module(ours, sc, BG, dL, use_sh=True, sh_degree=3)
    assert np.array_equal(a["radii"].cpu().numpy(), fw["radii"])
    err = h.rel_err(a["grads"]["means3D"].cpu().numpy(), bw["dL_dmeans3D"])
    assert err <= GRAD_RTOL, f"grad means3D: {err:.2e}"
    # the other gradients at the bar of the suite's whole-tensor oracle comparison
    for k, name in (("shs", "dL_dsh"), ("means2D", "dL_dmeans2D"), ("opacities", "dL_dopacity"),
                    ("scales", "dL_dscales"), ("rotations", "dL_drotations")):
        err = h.rel_err(a["grads"][k].cpu().numpy().reshape(bw[name].shape), bw[name])
        assert err <= ORACLE_GRAD_RTOL, f"grad {k}: {err:.2e}"
