"""Drop-in `diff_gaussian_rasterization` module backed by libsugar_b200 (sm_90a).

Public surface identical to the module SuGaR imports (`from diff_gaussian_rasterization import
GaussianRasterizationSettings, GaussianRasterizer`, sugar_scene/sugar_model.py:10; reference
implementation: gaussian_splatting/submodules/diff-gaussian-rasterization/
diff_gaussian_rasterization/__init__.py):

    GaussianRasterizationSettings   12-field NamedTuple, same order            (:157-169)
    GaussianRasterizer(nn.Module)   .forward(...) -> (color[3,H,W], radii[P])  (:171-220)
                                    .markVisible(positions) -> bool[P]
    rasterize_gaussians(...)        9 positional arguments                      (:21-42)

To use it in place of the reference build put `sugar_b200/` first on sys.path (or
`import sugar_b200; sugar_b200.install()`), see INTEGRATION.md.
"""
from typing import NamedTuple

import torch
import torch.nn as nn

from .. import _C


class GaussianRasterizationSettings(NamedTuple):
    image_height: int
    image_width: int
    tanfovx: float
    tanfovy: float
    bg: torch.Tensor
    scale_modifier: float
    viewmatrix: torch.Tensor
    projmatrix: torch.Tensor
    sh_degree: int
    campos: torch.Tensor
    prefiltered: bool
    debug: bool


def _optional_inputs(shs, colors_precomp, scales, rotations, cov3D_precomp):
    """The reference's "exactly one of" checks (:191-195); absent optionals then travel as empty tensors, as in the
    reference (:197-206).  -> (shs, colors_precomp, scales, rotations, cov3D_precomp)"""
    if (shs is None) == (colors_precomp is None):
        raise Exception('Please provide excatly one of either SHs or precomputed colors!')
    has_sr = scales is not None or rotations is not None
    if ((scales is None or rotations is None) and cov3D_precomp is None) or (has_sr and cov3D_precomp is not None):
        raise Exception('Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!')
    absent = torch.Tensor([])
    return tuple(absent if t is None else t for t in (shs, colors_precomp, scales, rotations, cov3D_precomp))


def _snapshot(args):
    """debug=True keeps a CPU copy of the arguments so a failing call can be dumped (reference :17-19)."""
    return tuple(a.detach().cpu().clone() if isinstance(a, torch.Tensor) else a for a in args)


def _call_with_dump(fn, args, debug, dump_name, what, **kw):
    """fn(*args, **kw); with debug, a failing call dumps `args` followed by the keyword tensors."""
    if not debug:
        return fn(*args, **kw)
    saved = _snapshot(args + tuple(v for v in kw.values() if isinstance(v, torch.Tensor)))
    try:
        return fn(*args, **kw)
    except Exception:
        torch.save(saved, dump_name)
        print(f"\nAn error occured in {what}. Please forward {dump_name} for debugging.")
        raise


class _RasterizeGaussians(torch.autograd.Function):
    """autograd boundary: forward keeps the three opaque state buffers, backward returns one
    gradient per forward input in input order."""

    @staticmethod
    def forward(ctx, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                raster_settings):
        rs = raster_settings
        args = (rs.bg, means3D, colors_precomp, opacities, scales, rotations, rs.scale_modifier, cov3Ds_precomp,
                rs.viewmatrix, rs.projmatrix, rs.tanfovx, rs.tanfovy, rs.image_height, rs.image_width, sh,
                rs.sh_degree, rs.campos, rs.prefiltered, rs.debug)
        # the op's cross-call state (capacity hint, view-parallel exchange) travels with the autograd
        # node: the backward runs on autograd's engine thread, where thread-local selection is not visible
        ctx.sgr_context = _C.current_context()
        num_rendered, color, radii, geom, binning, img = _call_with_dump(
            _C.rasterize_gaussians, args, rs.debug, "snapshot_fw.dump", "forward", context=ctx.sgr_context)
        ctx.raster_settings = rs
        ctx.num_rendered = num_rendered
        ctx.save_for_backward(colors_precomp, means3D, scales, rotations, cov3Ds_precomp, radii, sh, geom, binning,
                              img)
        ctx.mark_non_differentiable(radii)
        # radii never receives a gradient; without this autograd would fill a [P] zeros tensor for it on every backward
        ctx.set_materialize_grads(False)
        return color, radii

    @staticmethod
    def backward(ctx, grad_out_color, _grad_radii):
        if grad_out_color is None:   # the image took no part in the loss
            return (None,) * 9
        rs = ctx.raster_settings
        colors_precomp, means3D, scales, rotations, cov3Ds_precomp, radii, sh, geom, binning, img = ctx.saved_tensors
        args = (rs.bg, means3D, radii, colors_precomp, scales, rotations, rs.scale_modifier, cov3Ds_precomp,
                rs.viewmatrix, rs.projmatrix, rs.tanfovx, rs.tanfovy, grad_out_color, sh, rs.sh_degree, rs.campos,
                geom, ctx.num_rendered, binning, img, rs.debug)
        (g_means2D, g_colors, g_opacities, g_means3D, g_cov3D, g_sh, g_scales, g_rotations) = _call_with_dump(
            _C.rasterize_gaussians_backward, args, rs.debug, "snapshot_bw.dump", "backward", context=ctx.sgr_context)
        return (g_means3D, g_means2D, g_sh, g_colors, g_opacities, g_scales, g_rotations, g_cov3D, None)


def rasterize_gaussians(means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                        raster_settings):
    return _RasterizeGaussians.apply(means3D, means2D, sh, colors_precomp, opacities, scales, rotations,
                                     cov3Ds_precomp, raster_settings)


class GaussianRasterizer(nn.Module):
    def __init__(self, raster_settings):
        super().__init__()
        self.raster_settings = raster_settings

    def markVisible(self, positions):
        """Boolean mask of points in front of the near plane of this camera."""
        rs = self.raster_settings
        with torch.no_grad():
            return _C.mark_visible(positions, rs.viewmatrix, rs.projmatrix)

    def forward(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None,
                cov3D_precomp=None):
        shs, colors_precomp, scales, rotations, cov3D_precomp = _optional_inputs(shs, colors_precomp, scales,
                                                                                 rotations, cov3D_precomp)
        return rasterize_gaussians(means3D, means2D, shs, colors_precomp, opacities, scales, rotations,
                                   cov3D_precomp, self.raster_settings)
