"""Colour and a per-Gaussian scalar (e.g. depth) in one rasterizer pass.

Once SDF regularisation starts, the reference's coarse trainers rasterize every view twice with the same geometry:
the RGB render, then a depth render whose colours are the Gaussians' view-space z in all three channels over a
background of max z, of which channel 0 is kept (sugar_trainers/coarse_sdf.py:506-518, 578-590).
`rasterize_with_depth` does both in one call: one preprocess, one binning, one forward and one backward blend that
carries a fourth channel.

    image, depth, radii = rasterize_with_depth(means3D, means2D, opacities, point_values, raster_settings, depth_bg,
                                               shs=..., scales=..., rotations=...)

* `image` [3,H,W] is bit-identical to GaussianRasterizer(raster_settings)(...) with the same arguments, and `depth`
  [H,W] to channel 0 of a second call with colors_precomp = point_values expanded to 3 channels and
  bg = depth_bg in every channel.  `radii` is the shared [P] radii.
* `point_values` [P] (or [P,1]) is any per-Gaussian scalar.  It is an input, not something the kernel derives, so
  its gradient flows back through whatever produced it (e.g. the view transform of the points).
* `depth_bg` is a one-element tensor on the device (no host read), e.g. `point_values.max().detach()`.  It gets no
  gradient.
* Gradients reach every other input and equal the sum of the two calls' gradients up to fp32 summation order.  In
  particular `means2D.grad` is the sum over both channels: a caller that needs the RGB-only screen-space gradient
  (densification statistics) must still render twice.  The reference's depth render used a throw-away means2D, and
  its trainers stop densifying before the depth render starts.
* A gradient of None for the image or the depth counts as zero.

The op is `_C.rasterize_gaussians` / `_C.rasterize_gaussians_backward` with the keyword `values` (the C entry points
sgr_rasterize_forward_feature / sgr_rasterize_backward_feature).  Raw-parameter mode (fused.py) and use under a
view-parallel exchange (parallel.py) are not supported; the latter raises NotImplementedError, since the exchange sums
only the rasterizer's own gradients.
"""
import torch

from . import _C
from .diff_gaussian_rasterization import _call_with_dump, _optional_inputs


class _RasterizeWithDepth(torch.autograd.Function):
    @staticmethod
    def forward(ctx, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, point_values,
                depth_bg, raster_settings):
        rs = raster_settings
        bg1 = depth_bg.detach().reshape(1)
        args = (rs.bg, means3D, colors_precomp, opacities, scales, rotations, rs.scale_modifier, cov3Ds_precomp,
                rs.viewmatrix, rs.projmatrix, rs.tanfovx, rs.tanfovy, rs.image_height, rs.image_width, sh,
                rs.sh_degree, rs.campos, rs.prefiltered, rs.debug)
        ctx.sgr_context = _C.current_context()
        num_rendered, color, radii, geom, binning, img, depth = _call_with_dump(
            _C.rasterize_gaussians, args, rs.debug, "snapshot_fw.dump", "forward", context=ctx.sgr_context,
            values=point_values, feature_bg=bg1)
        ctx.raster_settings = rs
        ctx.num_rendered = num_rendered
        ctx.save_for_backward(colors_precomp, means3D, scales, rotations, cov3Ds_precomp, radii, sh, geom, binning,
                              img, point_values, bg1)
        ctx.mark_non_differentiable(radii)
        ctx.set_materialize_grads(False)
        return color, depth, radii

    @staticmethod
    def backward(ctx, grad_color, grad_depth, _grad_radii):
        if grad_color is None and grad_depth is None:
            return (None,) * 11
        rs = ctx.raster_settings
        (colors_precomp, means3D, scales, rotations, cov3Ds_precomp, radii, sh, geom, binning, img, point_values,
         bg1) = ctx.saved_tensors
        H, W = int(rs.image_height), int(rs.image_width)
        dev = means3D.device
        if grad_color is None:
            grad_color = torch.zeros((3, H, W), dtype=torch.float32, device=dev)
        if grad_depth is None:
            grad_depth = torch.zeros((H, W), dtype=torch.float32, device=dev)
        args = (rs.bg, means3D, radii, colors_precomp, scales, rotations, rs.scale_modifier, cov3Ds_precomp,
                rs.viewmatrix, rs.projmatrix, rs.tanfovx, rs.tanfovy, grad_color, sh, rs.sh_degree, rs.campos,
                geom, ctx.num_rendered, binning, img, rs.debug)
        (g_means2D, g_colors, g_opacities, g_means3D, g_cov3D, g_sh, g_scales, g_rotations, g_values) = \
            _call_with_dump(_C.rasterize_gaussians_backward, args, rs.debug, "snapshot_bw.dump", "backward",
                            context=ctx.sgr_context, values=point_values, feature_bg=bg1, dL_dout_feature=grad_depth)
        return (g_means3D, g_means2D, g_sh, g_colors, g_opacities, g_scales, g_rotations, g_cov3D, g_values, None,
                None)


def rasterize_with_depth(means3D, means2D, opacities, point_values, raster_settings, depth_bg, shs=None,
                         colors_precomp=None, scales=None, rotations=None, cov3D_precomp=None):
    """-> (image [3,H,W], depth [H,W], radii [P]); see the module docstring."""
    shs, colors_precomp, scales, rotations, cov3D_precomp = _optional_inputs(shs, colors_precomp, scales, rotations,
                                                                             cov3D_precomp)
    P = means3D.shape[0]
    if point_values.numel() != P or (point_values.dim() == 2 and point_values.shape[1] != 1) or point_values.dim() > 2:
        raise ValueError(f"point_values must be [P] or [P,1] with P = {P}, got {tuple(point_values.shape)}")
    if not torch.is_tensor(depth_bg) or depth_bg.numel() != 1:
        raise ValueError("depth_bg must be a one-element tensor")
    return _RasterizeWithDepth.apply(means3D, means2D, shs, colors_precomp, opacities, scales, rotations,
                                     cov3D_precomp, point_values.reshape(P), depth_bg, raster_settings)
