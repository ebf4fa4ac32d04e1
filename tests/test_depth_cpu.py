"""CPU checks of colour + depth in one rasterizer call (sugar_b200/depth.py): the C entry points' argument
validation, the Python signature, and that coarse_sdf_step(fused_depth=True) hands one call exactly the inputs of
the two separate calls."""
import ctypes
import inspect
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def test_feature_entry_points_validate_arguments_without_gpu():
    from sugar_b200 import _lib
    L = _lib.lib
    cb = _lib.SgrAlloc(lambda ctx, n: 0)
    n = ctypes.c_int64(0)
    nz = ctypes.c_void_p(16)   # never dereferenced: every case below fails validation first

    def fwd(v, g, values=nz, fbg=nz, color=nz, feature=nz, radii=nz):
        return L.sgr_rasterize_forward_feature(ctypes.byref(v), ctypes.byref(g), cb, None, cb, None, cb, None, values,
                                               fbg, color, feature, radii, 0, ctypes.byref(n), None)

    def bwd(v, g, **null):
        names = ["radii", "geom", "binning", "image", "dL_dout_color", "values", "feature_bg", "dL_dout_feature",
                 "dL_dmeans2D", "dL_dcolors", "dL_dopacity", "dL_dmeans3D", "dL_dcov3D", "dL_dsh", "dL_dscales",
                 "dL_drotations", "dL_dvalues", "grad_scratch"]
        p = {k: (None if null.get(k) else nz) for k in names}
        return L.sgr_rasterize_backward_feature(ctypes.byref(v), ctypes.byref(g), *[p[k] for k in names[:4]], 10,
                                                *[p[k] for k in names[4:]], None)

    v, g = _lib.SgrView(), _lib.SgrGaussians()
    v.image_width, v.image_height, g.P = 0, 0, 5
    assert fwd(v, g) == -1 and b"bad sizes" in L.sgr_last_error()
    assert bwd(v, g) == -1 and b"bad sizes" in L.sgr_last_error()

    # a well-formed scene description with fake (never dereferenced) device pointers
    v.image_width, v.image_height, v.sh_degree = 64, 48, 0
    v.bg = v.viewmatrix = v.projmatrix = v.campos = 16
    g.P, g.M = 5, 0
    g.means3D = g.opacities = g.colors_precomp = g.scales = g.rotations = 16
    for kw, what in ((dict(feature=None), b"null output"), (dict(color=None), b"null output"),
                     (dict(values=None), b"values"), (dict(fbg=None), b"feature_bg"), (dict(radii=None), b"radii")):
        L.sgr_last_error()
        assert fwd(v, g, **kw) == -1 and what in L.sgr_last_error(), kw
    for name in ("values", "feature_bg", "dL_dout_feature", "dL_dvalues", "grad_scratch", "dL_dmeans2D"):
        assert bwd(v, g, **{name: True}) == -1 and b"null pointer" in L.sgr_last_error(), name
    # ambiguous colours are rejected by the shared validation
    g.shs, g.M = 16, 1
    assert fwd(v, g) == -1 and b"excatly one" in L.sgr_last_error()
    assert bwd(v, g) == -1 and b"excatly one" in L.sgr_last_error()
    g.shs, g.M = None, 0
    # raw-parameter mode is out of scope
    g.activations = 1
    assert fwd(v, g) == -1 and b"raw-parameter" in L.sgr_last_error()
    assert bwd(v, g) == -1 and b"raw-parameter" in L.sgr_last_error()


def test_rasterize_with_depth_signature():
    from sugar_b200 import depth
    assert list(inspect.signature(depth.rasterize_with_depth).parameters) == [
        "means3D", "means2D", "opacities", "point_values", "raster_settings", "depth_bg", "shs", "colors_precomp",
        "scales", "rotations", "cov3D_precomp"]
    from sugar_b200 import steps
    assert inspect.signature(steps.coarse_sdf_step).parameters["fused_depth"].default is False


class _Settings:
    def __init__(self, **kw):
        self.__dict__.update(kw)


def _recording_ops(bw):
    """Reference ops with a recording, differentiable stand-in rasterizer (image = mean colour) and a recording
    rasterize_with_depth built from the same stand-in."""
    calls = []

    class Raster:
        GaussianRasterizationSettings = _Settings

        class GaussianRasterizer:
            def __init__(self, st):
                self.st = st

            def __call__(self, means3D, means2D, opacities, scales, rotations, shs=None, colors_precomp=None):
                calls.append(dict(kind="render", st=self.st, means3D=means3D, opacities=opacities, scales=scales,
                                  rotations=rotations, shs=shs, colors=colors_precomp))
                H, W = self.st.image_height, self.st.image_width
                c = colors_precomp if colors_precomp is not None else shs[:, 0]
                z = 0 * (opacities.sum() + scales.sum() + rotations.sum() + means3D.sum() + means2D.sum())
                return ((c.mean(0)[:, None, None] + z).expand(3, H, W) + 0 * self.st.bg[:, None, None],
                        torch.ones(means3D.shape[0], dtype=torch.int32))

    def rasterize_with_depth(means3D, means2D, opacities, point_values, raster_settings, depth_bg, shs=None,
                             colors_precomp=None, scales=None, rotations=None, cov3D_precomp=None):
        calls.append(dict(kind="fused", st=raster_settings, means3D=means3D, opacities=opacities, scales=scales,
                          rotations=rotations, shs=shs, colors=colors_precomp, values=point_values, depth_bg=depth_bg))
        H, W = raster_settings.image_height, raster_settings.image_width
        c = colors_precomp if colors_precomp is not None else shs[:, 0]
        z = 0 * (opacities.sum() + scales.sum() + rotations.sum() + means3D.sum() + means2D.sum())
        return ((c.mean(0)[:, None, None] + z).expand(3, H, W) + 0 * raster_settings.bg[:, None, None],
                (point_values.mean() + z).expand(H, W) + 0 * depth_bg, torch.ones(means3D.shape[0], dtype=torch.int32))

    ops = bw.reference_ops(torch, Raster)
    return ops, rasterize_with_depth, calls


def _inputs():
    import bench
    from oracle import field_oracle as fo
    sc = bench.load_scenes().make_scene(300, 64, 48, seed=0)
    leaf = lambda t: t.clone().requires_grad_(True)
    raw = dict(points=leaf(torch.from_numpy(sc.means3D)), sh_dc=leaf(torch.from_numpy(sc.shs[:, :1].copy())),
               sh_rest=leaf(torch.from_numpy(sc.shs[:, 1:].copy())),
               densities=leaf(torch.logit(torch.from_numpy(sc.opacities).clamp(1e-4, 1 - 1e-4))),
               scales=leaf(torch.from_numpy(sc.scales).log()), quaternions=leaf(torch.from_numpy(sc.rotations) * 1.3))
    return sc, raw, fo.knn_idx(raw["points"].detach(), 16)


def test_fused_depth_step_makes_one_call_with_the_two_calls_inputs():
    import bench_workloads as bw
    steps = bw._load_steps_without_package()
    sc, raw, knn = _inputs()
    cam = steps.camera_from_scene(sc, "cpu")
    gt = torch.rand(3, 48, 64, generator=torch.Generator().manual_seed(3))

    ops, fused_op, calls = _recording_ops(bw)
    loss_two, _ = steps.coarse_sdf_step(raw, cam, gt, knn, ops, n_samples=500, generator=torch.Generator().manual_seed(1),
                                        backward=False)
    two = list(calls)
    calls.clear()
    ops.rasterize_with_depth = fused_op
    loss_one, _ = steps.coarse_sdf_step(raw, cam, gt, knn, ops, n_samples=500, generator=torch.Generator().manual_seed(1),
                                        backward=False, fused_depth=True)
    assert [c["kind"] for c in two] == ["render", "render"] and [c["kind"] for c in calls] == ["fused"]
    rgb, dep, one = two[0], two[1], calls[0]
    same = lambda a, b: a is None and b is None or (a is not None and b is not None and torch.equal(a, b))
    for k in ("means3D", "opacities", "scales", "rotations"):
        assert same(one[k], rgb[k]) and same(one[k], dep[k]), k
    for k in ("shs", "colors"):   # the image's colours are the RGB call's
        assert same(one[k], rgb[k]), k
    for f in ("image_height", "image_width", "tanfovx", "tanfovy", "scale_modifier", "sh_degree", "prefiltered",
              "debug"):
        assert getattr(one["st"], f) == getattr(rgb["st"], f), f
    for f in ("bg", "viewmatrix", "projmatrix", "campos"):
        assert torch.equal(getattr(one["st"], f), getattr(rgb["st"], f)), f
    # the depth call's colours are the value in every channel and its background the depth background in every one
    assert torch.equal(dep["colors"], one["values"][:, None].expand(-1, 3))
    assert torch.equal(dep["st"].bg, one["depth_bg"].expand(3))
    assert not one["depth_bg"].requires_grad and one["values"].requires_grad
    assert torch.equal(loss_one, loss_two)


def test_fused_depth_needs_the_op():
    import bench_workloads as bw
    steps = bw._load_steps_without_package()
    sc, raw, knn = _inputs()
    ops, _, calls = _recording_ops(bw)   # the reference arm: no rasterize_with_depth
    with pytest.raises(ValueError, match="rasterize_with_depth"):
        steps.coarse_sdf_step(raw, steps.camera_from_scene(sc, "cpu"), torch.rand(3, 48, 64), knn, ops,
                              n_samples=500, fused_depth=True)
    assert calls == []
