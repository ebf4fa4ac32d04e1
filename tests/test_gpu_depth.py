"""Colour and depth in one rasterizer call (sugar_b200/depth.py) against the two calls it replaces: an RGB call and a
depth call with colors_precomp = value in every channel and bg = depth_bg in every channel.

Forward: image, depth (vs the depth call's channel 0), radii, num_rendered, n_contrib and final_T bit-identical.
Backward: every gradient equal to the sum of the two calls' gradients within the suite's 1e-4 per-tensor rel_err
(summation order), dL/dvalues equal to the depth call's dL_dcolors[:, 0]."""
import numpy as np
import pytest

import helpers as h

pytestmark = pytest.mark.gpu

GRAD_RTOL = 1e-4


def view_z(means3D, viewmatrix):
    return (means3D @ viewmatrix[:3, :3] + viewmatrix[3, :3])[:, 2]


def run_pair(sc, bg, depth_bg, dL, dD, use_sh=True, sh_degree=3, use_cov_precomp=False, cov3D=None, pad_to=None,
             device="cuda"):
    """The fused call and the two separate calls on the same seeded tensors (separate leaves).  Returns
    (fused, two): dicts with image, depth, radii, num_rendered, state (inspect_state) and grads."""
    import torch
    from sugar_b200 import _C, depth, diff_gaussian_rasterization as dgr
    t = h.to_torch(sc, device)
    names = ["means3D", "opacities", "shs" if use_sh else "colors_precomp", "scales", "rotations"]
    if pad_to:
        t.update(h.pad_culled(t, names, pad_to))
    P = t["means3D"].shape[0]
    if use_cov_precomp:
        t["cov3D_precomp"] = torch.from_numpy(cov3D).to(device)
    values0 = view_z(t["means3D"], t["viewmatrix"]).contiguous()
    col = "shs" if use_sh else "colors_precomp"
    geo = ["cov3D_precomp"] if use_cov_precomp else ["scales", "rotations"]
    dLt, dDt = torch.from_numpy(dL).to(device), torch.from_numpy(dD).to(device)
    bgt = torch.tensor(bg, dtype=torch.float32, device=device)
    dbg = torch.tensor([depth_bg], dtype=torch.float32, device=device)

    def settings(b):
        return dgr.GaussianRasterizationSettings(
            image_height=sc.height, image_width=sc.width, tanfovx=sc.tanfovx, tanfovy=sc.tanfovy, bg=b,
            scale_modifier=1.0, viewmatrix=t["viewmatrix"], projmatrix=t["projmatrix"], sh_degree=sh_degree,
            campos=t["campos"], prefiltered=False, debug=False)

    def leaves():
        return {k: t[k].detach().clone().requires_grad_(True) for k in ["means3D", "opacities", col] + geo}

    def state(grad_fn, R):
        g, b, i = grad_fn.saved_tensors[7:10]
        st = _C.inspect_state(P, sc.width, sc.height, R, g, b, i)
        return {k: st[k].clone() for k in ("n_contrib", "final_T")}

    # fused
    L = leaves()
    m2 = torch.zeros_like(L["means3D"], requires_grad=True)
    vals = values0.clone().requires_grad_(True)
    kw = {k: L[k] for k in [col] + geo}
    image, dmap, radii = depth.rasterize_with_depth(L["means3D"], m2, L["opacities"], vals, settings(bgt), dbg, **kw)
    fused = dict(image=image.detach().clone(), depth=dmap.detach().clone(), radii=radii.clone(),
                 num_rendered=image.grad_fn.num_rendered, state=state(image.grad_fn, image.grad_fn.num_rendered))
    ((image * dLt).sum() + (dmap * dDt).sum()).backward()
    fused["grads"] = dict({k: v.grad for k, v in L.items()}, means2D=m2.grad, values=vals.grad)

    # two calls
    L = leaves()
    m2a = torch.zeros_like(L["means3D"], requires_grad=True)
    m2b = torch.zeros_like(L["means3D"], requires_grad=True)
    cb = values0[:, None].expand(-1, 3).contiguous().requires_grad_(True)
    kw = {k: L[k] for k in [col] + geo}
    img_a, rad_a = dgr.GaussianRasterizer(settings(bgt))(means3D=L["means3D"], means2D=m2a, opacities=L["opacities"],
                                                         **kw)
    kw_b = {k: L[k] for k in geo}
    img_b, rad_b = dgr.GaussianRasterizer(settings(dbg.expand(3).contiguous()))(
        means3D=L["means3D"], means2D=m2b, opacities=L["opacities"], colors_precomp=cb, **kw_b)
    two = dict(image=img_a.detach().clone(), depth=img_b[0].detach().clone(), radii=rad_a.clone(), radii_b=rad_b.clone(),
               num_rendered=img_a.grad_fn.num_rendered, num_rendered_b=img_b.grad_fn.num_rendered,
               state=state(img_a.grad_fn, img_a.grad_fn.num_rendered))
    ((img_a * dLt).sum() + (img_b[0] * dDt).sum()).backward()
    two["grads"] = dict({k: v.grad for k, v in L.items()}, means2D=m2a.grad + m2b.grad, values=cb.grad[:, 0])
    two["dcolors_b"] = cb.grad
    if pad_to:
        n = sc.means3D.shape[0]
        assert not fused["radii"][n:].any() and not fused["grads"]["values"][n:].any()
    return fused, two


def assert_forward_identical(f, t):
    import torch
    assert f["num_rendered"] == t["num_rendered"] == t["num_rendered_b"]
    assert torch.equal(f["radii"], t["radii"]) and torch.equal(f["radii"], t["radii_b"])
    assert torch.equal(f["image"], t["image"])
    assert torch.equal(f["depth"], t["depth"])
    for k in ("n_contrib", "final_T"):
        assert torch.equal(f["state"][k], t["state"][k]), k


def grad_errors(f, t):
    assert set(f["grads"]) == set(t["grads"])
    return {k: h.rel_err(f["grads"][k].cpu().numpy(), t["grads"][k].cpu().numpy()) for k in f["grads"]}


CASES = [
    # id, P, W, H, camera, use_sh, sh_degree, cov3D, depth_bg, extra scene kwargs
    ("identity_sh3", 20000, 320, 240, "identity", True, 3, False, 0.0, {}),
    ("posed_sh0", 20000, 320, 240, "posed", True, 0, False, 7.5, {}),
    ("posed_sh1", 20000, 320, 240, "posed", True, 1, False, 7.5, {}),
    ("posed_sh2", 20000, 333, 197, "posed", True, 2, False, 7.5, {}),
    ("posed_sh3", 20000, 320, 240, "posed", True, 3, False, 7.5, {}),
    ("posed_colors", 20000, 320, 240, "posed", False, 3, False, 7.5, {}),
    ("posed_cov3D", 20000, 320, 240, "posed", True, 3, True, 7.5, {}),
    ("negative_bg", 20000, 320, 240, "posed", True, 3, False, -3.25, {}),
    ("dense_T_stop", 120000, 256, 160, "posed", True, 3, False, 12.0, dict(px_sigma=6.0)),
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_fused_equals_two_calls(case):
    from sugar_b200 import scenes
    name, P, W, H, camera, use_sh, deg, cov, dbg, skw = case
    sc = scenes.make_scene(P, W, H, seed=3, camera=camera, **skw)
    cov3D = None
    if cov:
        fw, _ = h.run_oracle(sc, np.zeros(3, np.float32), None, use_sh=use_sh, sh_degree=deg)
        cov3D = fw["cov3D"].astype(np.float32)
    dL, dD = scenes.upstream_grad(W, H, seed=1), scenes.upstream_grad(W, H, seed=2)[0]
    f, t = run_pair(sc, (0.1, 0.2, 0.3), dbg, dL, dD, use_sh=use_sh, sh_degree=deg, use_cov_precomp=cov, cov3D=cov3D)
    assert_forward_identical(f, t)
    if name == "dense_T_stop":   # the early stop is reached: some pixel ends below the 1e-4 transmittance bar
        assert float(f["state"]["final_T"].min()) < 1e-3
    errs = grad_errors(f, t)
    assert max(errs.values()) <= GRAD_RTOL, errs


def test_plain_ids():
    """The plain-id instance lists (P >= 2^24): the scene padded with culled Gaussians (helpers.pad_culled)."""
    import torch
    from sugar_b200 import scenes
    sc = scenes.make_scene(20000, 320, 240, seed=4, camera="posed")
    dL, dD = scenes.upstream_grad(320, 240, seed=1), scenes.upstream_grad(320, 240, seed=2)[0]
    f, t = run_pair(sc, (0.1, 0.2, 0.3), 5.0, dL, dD, use_sh=False, pad_to=h.PACKED_MAX_P)
    assert_forward_identical(f, t)
    n = sc.means3D.shape[0]
    errs = {k: h.rel_err(f["grads"][k][:n].cpu().numpy(), t["grads"][k][:n].cpu().numpy()) for k in f["grads"]}
    assert max(errs.values()) <= GRAD_RTOL, errs
    del f, t
    torch.cuda.empty_cache()


def test_mesh_bound_scene():
    """Surface-aligned Gaussians (a 1e-6 axis): dL_dscales / dL_drotations are held to 5x the per-Gaussian chain's
    sensitivity to 1e-6 accumulator noise (helpers.grad_sensitivity), as in test_gpu_configs.py."""
    from sugar_b200 import scenes
    W, H = 240, 150
    sc = scenes.make_scene(40000, W, H, seed=0, mesh_bound=True)
    dL, dD = scenes.upstream_grad(W, H, seed=1), scenes.upstream_grad(W, H, seed=2)[0]
    f, t = run_pair(sc, (0.0, 0.0, 0.0), 9.0, dL, dD)
    assert_forward_identical(f, t)
    errs = grad_errors(f, t)
    bad = {k: e for k, e in errs.items() if e > GRAD_RTOL}
    if bad:
        sens = h.grad_sensitivity(sc, (0.0, 0.0, 0.0), dL, use_sh=True, sh_degree=3)
        bad = {k: e for k, e in bad.items() if k not in ("scales", "rotations") or e > 5.0 * sens.get(k, 0.0)}
    assert not bad, (bad, errs)


def test_headline_config():
    """3M Gaussians at 1920x1080, SH degree 3 (bench.py's workload), depth = view-space z over max z."""
    import torch
    from sugar_b200 import scenes
    W, H = 1920, 1080
    sc = scenes.make_scene(3_000_000, W, H, seed=0)
    z = sc.means3D @ sc.viewmatrix[:3, :3] + sc.viewmatrix[3, :3]
    dL, dD = scenes.upstream_grad(W, H, seed=1), scenes.upstream_grad(W, H, seed=2)[0]
    f, t = run_pair(sc, (0.0, 0.0, 0.0), float(z[:, 2].max()), dL, dD)
    assert_forward_identical(f, t)
    errs = grad_errors(f, t)
    assert max(errs.values()) <= GRAD_RTOL, errs
    del f, t
    torch.cuda.empty_cache()


def test_values_gradient_and_depth_match_the_oracle():
    """The depth map and dL/dvalues against the CPU oracle run with colours = value in every channel."""
    from sugar_b200 import scenes
    W, H = 96, 64
    sc = scenes.make_scene(1500, W, H, seed=6, camera="posed")
    vm = sc.viewmatrix
    z = (sc.means3D @ vm[:3, :3] + vm[3, :3])[:, 2].astype(np.float32)
    dbg = float(z.max())
    dL, dD = scenes.upstream_grad(W, H, seed=1), scenes.upstream_grad(W, H, seed=2)[0]
    f, t = run_pair(sc, (0.1, 0.2, 0.3), dbg, dL, dD, use_sh=False)
    scd = sc._replace(colors_precomp=np.repeat(z[:, None], 3, 1))
    dL3 = np.zeros((3, H, W), np.float32)
    dL3[0] = dD
    fw, bw = h.run_oracle(scd, np.full(3, dbg, np.float32), dL3, use_sh=False)
    assert np.array_equal(f["radii"].cpu().numpy(), fw["radii"])
    assert h.rel_err(f["depth"].cpu().numpy(), fw["color"][0]) < 1e-5
    assert h.rel_err(f["grads"]["values"].cpu().numpy(), bw["dL_dcolors"][:, 0]) < GRAD_RTOL
    assert h.rel_err(f["grads"]["values"].cpu().numpy(), t["dcolors_b"][:, 0].cpu().numpy()) < GRAD_RTOL


def _fused_once(sc, dbg=6.0, seed=7):
    import torch
    from sugar_b200 import depth, diff_gaussian_rasterization as dgr
    t = h.to_torch(sc)
    st = dgr.GaussianRasterizationSettings(
        image_height=sc.height, image_width=sc.width, tanfovx=sc.tanfovx, tanfovy=sc.tanfovy,
        bg=torch.zeros(3, device="cuda"), scale_modifier=1.0, viewmatrix=t["viewmatrix"], projmatrix=t["projmatrix"],
        sh_degree=3, campos=t["campos"], prefiltered=False, debug=False)
    leaf = lambda x: x.detach().clone().requires_grad_(True)
    L = dict(means3D=leaf(t["means3D"]), opacities=leaf(t["opacities"]), shs=leaf(t["shs"]), scales=leaf(t["scales"]),
             rotations=leaf(t["rotations"]), values=leaf(view_z(t["means3D"], t["viewmatrix"])))
    m2 = torch.zeros_like(L["means3D"], requires_grad=True)
    out = depth.rasterize_with_depth(L["means3D"], m2, L["opacities"], L["values"], st,
                                     torch.tensor([dbg], device="cuda"), shs=L["shs"], scales=L["scales"],
                                     rotations=L["rotations"])
    return out, L, m2


def test_two_runs_identical_forward():
    from sugar_b200 import scenes
    sc = scenes.make_scene(30000, 320, 240, seed=8, camera="posed")
    (a, _, _), (b, _, _) = _fused_once(sc), _fused_once(sc)
    for x, y in zip(a, b):
        assert x.dtype == y.dtype and bool((x == y).all())


def test_none_gradient_on_either_output():
    import torch
    from sugar_b200 import diff_gaussian_rasterization as dgr, scenes
    sc = scenes.make_scene(20000, 320, 240, seed=9, camera="posed")
    dL = torch.from_numpy(scenes.upstream_grad(320, 240, seed=1)).cuda()
    # image only: the depth's gradient is None, so dL/dvalues is zero and the rest is the RGB call's backward
    (img, dmap, _), L, m2 = _fused_once(sc)
    (img * dL).sum().backward()
    assert L["values"].grad is not None and not L["values"].grad.any()
    f = h.run_module(dgr, sc, (0.0, 0.0, 0.0), dL.cpu().numpy(), use_sh=True, sh_degree=3)
    for k in ("means3D", "opacities", "shs", "scales", "rotations"):
        assert h.rel_err(L[k].grad.cpu().numpy(), f["grads"][k].cpu().numpy()) <= GRAD_RTOL, k
    assert h.rel_err(m2.grad.cpu().numpy(), f["grads"]["means2D"].cpu().numpy()) <= GRAD_RTOL
    # depth only: the image's gradient is None
    (img, dmap, _), L, m2 = _fused_once(sc)
    dmap.sum().backward()
    assert L["values"].grad.abs().sum() > 0 and L["shs"].grad is not None
    assert not L["shs"].grad.any()   # colours take no part in the depth


def test_empty_cloud_returns_zeros():
    import torch
    from sugar_b200 import depth, diff_gaussian_rasterization as dgr, scenes
    sc = scenes.make_scene(10, 64, 48, seed=1)
    t = h.to_torch(sc)
    st = dgr.GaussianRasterizationSettings(
        image_height=48, image_width=64, tanfovx=sc.tanfovx, tanfovy=sc.tanfovy, bg=torch.ones(3, device="cuda"),
        scale_modifier=1.0, viewmatrix=t["viewmatrix"], projmatrix=t["projmatrix"], sh_degree=0, campos=t["campos"],
        prefiltered=False, debug=False)
    e = lambda *s: torch.zeros(s, device="cuda", requires_grad=True)
    means3D, vals = e(0, 3), e(0)
    img, dmap, radii = depth.rasterize_with_depth(means3D, e(0, 3), e(0, 1), vals, st, torch.ones(1, device="cuda"),
                                                  colors_precomp=e(0, 3), scales=e(0, 3), rotations=e(0, 4))
    assert img.shape == (3, 48, 64) and dmap.shape == (48, 64) and radii.shape == (0,)
    assert not img.any() and not dmap.any()
    (img.sum() + dmap.sum()).backward()
    assert means3D.grad.shape == (0, 3) and vals.grad.shape == (0,)


def test_view_parallel_exchange_is_refused():
    import torch
    from sugar_b200 import _C, scenes

    class Exchange:
        def enabled(self):
            return True
    ctx = _C.Context()
    ctx.exchange = Exchange()
    sc = scenes.make_scene(1000, 64, 48, seed=2)
    with _C.use_context(ctx), pytest.raises(NotImplementedError, match="view-parallel"):
        _fused_once(sc)
    torch.cuda.synchronize()


def test_coarse_sdf_step_fused_depth():
    """coarse_sdf_step(fused_depth=True): the same loss bit for bit, the raw-parameter gradients within tolerance."""
    import torch
    from sugar_b200 import knn, scenes, steps
    dev = torch.device("cuda")
    W, H = 480, 270
    sc = scenes.make_scene(100_000, W, H, seed=0)
    cam = steps.camera_from_scene(sc, dev)
    gt = torch.rand(3, H, W, generator=torch.Generator().manual_seed(0)).to(dev)
    leaf = lambda x: x.to(dev).requires_grad_(True)

    def raw():
        return dict(points=leaf(torch.from_numpy(sc.means3D)), sh_dc=leaf(torch.from_numpy(sc.shs[:, :1].copy())),
                    sh_rest=leaf(torch.from_numpy(sc.shs[:, 1:].copy())),
                    densities=leaf(torch.logit(torch.from_numpy(sc.opacities).clamp(1e-4, 1 - 1e-4))),
                    scales=leaf(torch.from_numpy(sc.scales).log()),
                    quaternions=leaf(torch.from_numpy(sc.rotations) * 1.3))
    ra, rb = raw(), raw()
    knn_idx = knn.reset_neighbors(ra["points"].detach(), 16)[1]
    ops = steps.ours_ops()
    g = torch.Generator(device=dev)
    la, sa = steps.coarse_sdf_step(ra, cam, gt, knn_idx, ops, n_samples=200_000, generator=g.manual_seed(1))
    lb, sb = steps.coarse_sdf_step(rb, cam, gt, knn_idx, ops, n_samples=200_000, generator=g.manual_seed(1),
                                   fused_depth=True)
    assert sa == sb and sa["sampled_gaussians"] > 0
    assert torch.equal(la, lb), (float(la), float(lb))
    errs = {k: h.rel_err(rb[k].grad.cpu().numpy(), ra[k].grad.cpu().numpy()) for k in ra}
    assert max(errs.values()) <= 1e-3, errs
