"""Raw-parameter mode (sugar_b200/fused.py, SURVEY 8f-1): SuGaR's activations + SH colours inside the kernels.
Checked against (a) "activate in PyTorch, then the drop-in rasterizer with shs=" (same kernels, activations
outside) and (b) the reference's own python colour path (get_points_rgb / eval_sh restated in oracle/, pinned
there) feeding colors_precomp -- the path the reference trainers take (coarse_sdf.py:51)."""
import numpy as np
import pytest

import helpers as h

pytestmark = pytest.mark.gpu


def _raw_params(sc, M=16):
    import torch
    t = h.to_torch(sc)
    r = dict(points=t["means3D"].clone(), sh_dc=t["shs"][:, :1].contiguous().clone(),
             sh_rest=t["shs"][:, 1:M].contiguous().clone(),
             densities=torch.logit(t["opacities"].clamp(1e-4, 1 - 1e-4)), scales=t["scales"].log(),
             quaternions=t["rotations"] * 1.7)
    return t, {k: v.requires_grad_(True) for k, v in r.items()}


def _settings(mod, sc, t, deg, bg):
    import torch
    return mod.GaussianRasterizationSettings(
        image_height=sc.height, image_width=sc.width, tanfovx=sc.tanfovx, tanfovy=sc.tanfovy,
        bg=torch.tensor(bg, device="cuda"), scale_modifier=1.0, viewmatrix=t["viewmatrix"], projmatrix=t["projmatrix"],
        sh_degree=deg, campos=t["campos"], prefiltered=False, debug=False)


@pytest.mark.parametrize("deg,M,P", [(3, 16, 6000), (1, 4, 4001), (0, 1, 3000), (2, 16, 257)])
def test_raw_mode_matches_activations_in_pytorch(deg, M, P):
    import torch
    from sugar_b200 import diff_gaussian_rasterization as mod, fused, scenes
    W, H = 200, 120
    sc = scenes.make_scene(P, W, H, seed=11 + deg, camera="posed")
    dL = torch.from_numpy(scenes.upstream_grad(W, H, seed=3)).cuda()
    bg = (0.1, 0.2, 0.3)
    t, a = _raw_params(sc, M)
    st = _settings(mod, sc, t, deg, bg)
    m2a = torch.zeros_like(a["points"], requires_grad=True)
    img_a, radii_a = fused.rasterize_raw(a["points"], m2a, a["sh_dc"], a["sh_rest"], a["densities"], a["scales"],
                                         a["quaternions"], st)
    (img_a * dL).sum().backward()
    _, b = _raw_params(sc, M)
    m2b = torch.zeros_like(b["points"], requires_grad=True)
    img_b, radii_b = mod.GaussianRasterizer(st)(
        means3D=b["points"], means2D=m2b, opacities=torch.sigmoid(b["densities"]),
        shs=torch.cat([b["sh_dc"], b["sh_rest"]], dim=1), scales=torch.exp(b["scales"]),
        rotations=torch.nn.functional.normalize(b["quaternions"], dim=-1))
    (img_b * dL).sum().backward()
    # the activations differ from PyTorch's at most in the last ulp (norm reduction order), which can move a radius
    # across an integer in rare cases: compare on the Gaussians whose radii agree, and demand that almost all do
    same = radii_a == radii_b
    assert float(same.float().mean()) > 0.999
    assert float((img_a - img_b).abs().max()) <= 1e-4
    assert float((img_a - img_b).abs().mean()) <= 1e-6
    for k in a:
        ga, gb = a[k].grad, b[k].grad
        assert ga is not None and ga.shape == gb.shape, k
        assert h.rel_err(ga.cpu().numpy(), gb.cpu().numpy()) <= 2e-4, k
    assert h.rel_err(m2a.grad.cpu().numpy(), m2b.grad.cpu().numpy()) <= 2e-4


RAW_INPUTS = ("points", "sh_dc", "sh_rest", "densities", "scales", "quaternions")


def _run_raw(sc, r, deg, dL, bg=(0.1, 0.2, 0.3)):
    """rasterize_raw on the raw tensors r (leaves); returns image, radii and the gradients of r and means2D."""
    import torch
    from sugar_b200 import diff_gaussian_rasterization as mod, fused
    t = h.to_torch(sc)
    m2 = torch.zeros_like(t["means3D"], requires_grad=True)
    img, radii = fused.rasterize_raw(r["points"], m2, r["sh_dc"], r["sh_rest"], r["densities"], r["scales"],
                                     r["quaternions"], _settings(mod, sc, t, deg, bg))
    (img * dL).sum().backward()
    return img.detach(), radii, dict({k: r[k].grad for k in r}, means2D=m2.grad)


def _at_offset12(x):
    """x's values in a leaf that starts 12 bytes into a larger allocation: contiguous, not 16-byte aligned."""
    import torch
    buf = torch.zeros(x.numel() + 3, dtype=x.dtype, device=x.device)
    v = buf[3:].view(x.shape)
    v.copy_(x.detach())
    return v.detach().requires_grad_(True)


@pytest.mark.parametrize("deg,M", [(3, 16), (2, 9), (1, 4), (0, 1)])
def test_raw_mode_without_bulk_copies_computes_the_same(deg, M):
    """Raw inputs that are not 16-byte aligned cannot be staged with TMA bulk copies: the per-Gaussian passes stage them
    word by word instead.  Staging is all that changes, so radii and image must be identical to the aligned run's and
    the gradients equal up to fp32 atomics order -- for each raw input misaligned alone, then for all of them."""
    import torch
    from sugar_b200 import scenes
    P, W, H = 4001, 200, 120
    sc = scenes.make_scene(P, W, H, seed=60 + M, camera="posed")
    dL = torch.from_numpy(scenes.upstream_grad(W, H, seed=6)).cuda()
    _, r0 = _raw_params(sc, M)
    assert all(v.data_ptr() % 16 == 0 for v in r0.values())
    img0, radii0, g0 = _run_raw(sc, r0, deg, dL)
    cases = [(k,) for k in RAW_INPUTS if r0[k].numel()] + [RAW_INPUTS]
    for moved in cases:
        _, r = _raw_params(sc, M)
        r = {k: _at_offset12(v) if k in moved else v for k, v in r.items()}
        assert all(r[k].data_ptr() % 16 != 0 for k in moved if r[k].numel())
        img, radii, g = _run_raw(sc, r, deg, dL)
        assert torch.equal(radii, radii0), moved
        assert torch.equal(img, img0), moved
        for k in g0:
            assert g[k].shape == g0[k].shape, (moved, k)
            assert h.rel_err(g[k].cpu().numpy(), g0[k].cpu().numpy()) <= 1e-4, (moved, k)


def test_raw_mode_with_saturated_logits_and_short_quaternions():
    """Logits at +-30 (opacity 1 -> alpha held at 0.99; opacity ~1e-13 -> never reaches 1/255) and raw quaternions of
    norm ~1e-3, against the activations evaluated in float64 PyTorch feeding the drop-in rasterizer."""
    import torch
    from sugar_b200 import diff_gaussian_rasterization as mod, scenes
    P, W, H, deg = 5000, 200, 120, 3
    sc = scenes.make_scene(P, W, H, seed=7, camera="posed")
    dL = torch.from_numpy(scenes.upstream_grad(W, H, seed=8)).cuda()

    def params():
        t, r = _raw_params(sc)
        with torch.no_grad():
            i = torch.arange(P, device="cuda")
            r["densities"][i % 3 == 0] = 30.0
            r["densities"][i % 3 == 1] = -30.0
            r["quaternions"][i % 2 == 0] *= 1e-3 / 1.7
        return t, r
    t, a = params()
    assert float(a["quaternions"][::2].norm(dim=1).max()) < 2e-3
    img_a, radii_a, ga = _run_raw(sc, a, deg, dL)
    _, b = params()
    m2b = torch.zeros_like(b["points"], requires_grad=True)
    img_b, radii_b = mod.GaussianRasterizer(_settings(mod, sc, t, deg, (0.1, 0.2, 0.3)))(
        means3D=b["points"], means2D=m2b, opacities=torch.sigmoid(b["densities"].double()).float(),
        shs=torch.cat([b["sh_dc"], b["sh_rest"]], dim=1), scales=torch.exp(b["scales"].double()).float(),
        rotations=torch.nn.functional.normalize(b["quaternions"].double(), dim=-1).float())
    (img_b * dL).sum().backward()
    assert float((radii_a == radii_b).float().mean()) > 0.999
    assert float((img_a - img_b).abs().max()) <= 1e-4
    assert float((img_a - img_b).abs().mean()) <= 1e-6
    for k in b:
        assert h.rel_err(ga[k].cpu().numpy(), b[k].grad.cpu().numpy()) <= 2e-4, k
    assert h.rel_err(ga["means2D"].cpu().numpy(), m2b.grad.cpu().numpy()) <= 2e-4
    # the -30 logits never reach alpha 1/255: nothing flows back to them
    assert float(ga["densities"][1::3].abs().max()) == 0.0 and float(ga["sh_dc"][1::3].abs().max()) == 0.0


def test_raw_mode_matches_the_reference_python_colour_path():
    """The trainers' path: python SH colours (sugar_model.py:839-883) -> colors_precomp."""
    import torch
    from oracle import field_oracle as fo
    from sugar_b200 import diff_gaussian_rasterization as mod, fused, scenes
    P, W, H, deg = 5000, 200, 120, 3
    sc = scenes.make_scene(P, W, H, seed=5, camera="posed")
    dL = torch.from_numpy(scenes.upstream_grad(W, H, seed=4)).cuda()
    t, a = _raw_params(sc)
    st = _settings(mod, sc, t, deg, (0.0, 0.0, 0.0))
    m2 = torch.zeros_like(a["points"], requires_grad=True)
    img_a, _ = fused.rasterize_raw(a["points"], m2, a["sh_dc"], a["sh_rest"], a["densities"], a["scales"],
                                   a["quaternions"], st)
    (img_a * dL).sum().backward()
    _, b = _raw_params(sc)
    colors = fo.points_rgb_torch(b["points"], torch.cat([b["sh_dc"], b["sh_rest"]], dim=1), t["campos"], deg + 1)
    m2b = torch.zeros_like(b["points"], requires_grad=True)
    img_b, _ = mod.GaussianRasterizer(st)(
        means3D=b["points"], means2D=m2b, opacities=torch.sigmoid(b["densities"]), colors_precomp=colors,
        scales=torch.exp(b["scales"]), rotations=torch.nn.functional.normalize(b["quaternions"], dim=-1))
    (img_b * dL).sum().backward()
    assert float((img_a - img_b).abs().max()) <= 1e-4
    for k in a:
        assert h.rel_err(a[k].grad.cpu().numpy(), b[k].grad.cpu().numpy()) <= 5e-4, k
