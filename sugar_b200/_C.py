"""`_C`-compatible shim: the three symbols the reference's pybind module exports
(diff-gaussian-rasterization/ext.cpp:15-19, rasterize_points.h:19-67), same positional
signatures and return tuples, implemented over the C ABI of libsugar_b200.so.  Keyword-only extras of
`rasterize_gaussians` / `rasterize_gaussians_backward` select raw-parameter mode (`sh_rest`, sugar_b200/fused.py) and
one more blended channel (`values`, sugar_b200/depth.py).  Each appends its gradient to the backward's tuple;
`values` also appends the blended map to the forward's.

torch is used only for device memory (caching allocator), the current stream and the device
guard; all arithmetic happens in the hand-written sm_90a kernels.
"""
import contextlib
import ctypes as C
import threading
from typing import Tuple

import torch

from . import _lib
from ._lib import SgrGaussians, SgrView, check, f32_ptr, lib, require_cuda, stream


class Context:
    """Mutable state of the op that outlives one call.  Nothing here is process-global: a model (or a
    thread, or a view-parallel exchange) can own its context and select it with `use_context`;
    calls made outside any `use_context` block share `default_context()`.

    capacity_hint  (device, H, W) -> instance capacity.  After the first forward the binning buffer is
                   sized from the previous view's instance count (x1.25 + slack) so the whole forward is
                   enqueued without waiting for the device; the C side re-runs binning on overflow
                   (include/sugar_b200.h).
    exchange       None, or the view-parallel exchange (sugar_b200.parallel.ViewParallel) that the
                   backward hands its per-Gaussian gradients to before returning them to autograd.

    The forward stores the context it ran under in the autograd node, so the backward -- which autograd
    runs on its own engine thread -- uses the same one."""

    def __init__(self):
        self.capacity_hint = {}
        self.exchange = None
        self.lock = threading.Lock()


_default_context = Context()
_tls = threading.local()


def default_context() -> Context:
    return _default_context


def current_context() -> Context:
    return getattr(_tls, "ctx", None) or _default_context


@contextlib.contextmanager
def use_context(ctx: Context):
    """Calls made by this thread inside the block use `ctx` (nestable)."""
    prev = getattr(_tls, "ctx", None)
    _tls.ctx = ctx
    try:
        yield ctx
    finally:
        _tls.ctx = prev


_ROUND = 64 << 20  # arena sizes are rounded up to 64 MiB so the caching allocator sees few distinct sizes


def _round_up(n: int, a: int) -> int:
    return (n + a - 1) // a * a


class _Arena:
    """Allocator-callback state.  One torch allocation backs all three opaque buffers of a forward
    (carved at 256-byte offsets): per-step allocations of stable, rounded sizes keep the caching
    allocator from fragmenting (and from calling cudaMalloc, a device-wide stall) in steady state."""

    def __init__(self, device, reserve_bytes: int):
        self.device = device
        self.block = (torch.empty(_round_up(reserve_bytes, _ROUND), dtype=torch.uint8, device=device)
                      if reserve_bytes else None)
        self.used = 0
        self.parts = {}
        self.error = None   # an exception raised inside a callback (e.g. torch OOM): re-raised after the C call returns
        self.cbs = {name: _lib.SgrAlloc(lambda _ctx, n, name=name: self._alloc(name, n)) for name in ("geom", "binning", "img")}

    def _alloc(self, name, nbytes):
        try:
            nbytes = int(nbytes)
            if self.block is not None and self.used + nbytes + 256 <= self.block.numel():
                off = _round_up(self.block.data_ptr() + self.used, 256) - self.block.data_ptr()
                t = self.block[off:off + nbytes]
                self.used = off + nbytes
            else:  # no (or too small a) reservation: plain allocation, still rounded
                t = torch.empty(_round_up(nbytes, _ROUND), dtype=torch.uint8, device=self.device)[:nbytes]
            self.parts[name] = t
            return t.data_ptr()
        except BaseException as e:  # never unwind through the C frame: NULL makes the library stop with an error status
            self.error = e
            return None

    def get(self, name):
        return self.parts.get(name, torch.empty(0, dtype=torch.uint8, device=self.device))

    def release(self):
        """Break the arena <-> callback reference cycle so the block is released by reference
        counting as soon as the autograd graph lets go of the views (not at the next cyclic GC).
        Blocks left to the cyclic GC come back in bursts, and the caching allocator then splits them and
        calls cudaMalloc inside the training loop, a device-wide stall (scripts/step_times.py)."""
        self.cbs = None
        self.block = None
        self.parts = {}


def _view_struct(bg, scale_modifier, viewmatrix, projmatrix, tan_fovx, tan_fovy, H, W, degree, campos, prefiltered,
                 debug) -> SgrView:
    v = SgrView()
    v.image_height, v.image_width = int(H), int(W)
    v.tanfovx, v.tanfovy = float(tan_fovx), float(tan_fovy)
    v.bg = f32_ptr(bg, "bg")
    v.scale_modifier = float(scale_modifier)
    v.viewmatrix = f32_ptr(viewmatrix, "viewmatrix")
    v.projmatrix = f32_ptr(projmatrix, "projmatrix")
    v.sh_degree = int(degree)
    v.campos = f32_ptr(campos, "campos")
    v.prefiltered, v.debug = int(bool(prefiltered)), int(bool(debug))
    return v


def _gauss_struct(P, M, means3D, opacity, sh, colors, scales, rotations, cov3D_precomp, sh_rest=None) -> SgrGaussians:
    g = SgrGaussians()
    g.activations = _lib.SGR_ACT_RAW if sh_rest is not None else 0   # raw SuGaR parameters, (dc, rest) SH arrays
    g.sh_rest = f32_ptr(sh_rest, "sh_rest") if sh_rest is not None else None
    g.P, g.M = int(P), int(M)
    g.means3D = f32_ptr(means3D, "means3D")
    g.opacities = f32_ptr(opacity, "opacity")
    g.shs = f32_ptr(sh, "sh")
    g.colors_precomp = f32_ptr(colors, "colors")
    g.scales = f32_ptr(scales, "scales")
    g.rotations = f32_ptr(rotations, "rotations")
    g.cov3D_precomp = f32_ptr(cov3D_precomp, "cov3D_precomp")
    return g


def _c(t):
    return t if (t is None or t.is_contiguous()) else t.contiguous()


def _no_exchange(context: Context):
    if context.exchange is not None and context.exchange.enabled():
        raise NotImplementedError("rasterize_with_depth under a view-parallel exchange: the exchange sums only the "
                                  "rasterizer's own gradients, dL/dvalues would reach the points unsummed")


def rasterize_gaussians(background, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp,
                        viewmatrix, projmatrix, tan_fovx, tan_fovy, image_height, image_width, sh, degree, campos,
                        prefiltered, debug, *, context: Context = None, sh_rest: torch.Tensor = None,
                        values: torch.Tensor = None, feature_bg: torch.Tensor = None) -> Tuple:
    """RasterizeGaussiansCUDA (rasterize_points.cu:36-115) -> (R, color[3,H,W], radii, geom, binning, img).
    Keyword-only extras that are not part of the reference signature: `context` selects whose capacity hint is used
    (default: the calling thread's current one); `sh_rest` selects raw-parameter mode (sugar_b200/fused.py): `sh` is
    then the model's DC array [P,1,3], `sh_rest` [P,M-1,3], and opacity / scales / rotations are the RAW parameters,
    activated in the kernel; `values` f32[P] blends one extra channel over `feature_bg` (device f32[1])
    (sgr_rasterize_forward_feature, sugar_b200/depth.py) and appends that map [H,W] to the returned tuple."""
    context = context or current_context()
    feature = values is not None
    if feature:
        _no_exchange(context)
    if means3D.dim() != 2 or means3D.size(1) != 3:
        raise RuntimeError("means3D must have dimensions (num_points, 3)")
    require_cuda("diff_gaussian_rasterization", means3D)
    dev = means3D.device
    P, H, W = means3D.size(0), int(image_height), int(image_width)
    if feature and (values.numel() != P or feature_bg.numel() != 1):
        raise RuntimeError(f"values must hold one scalar per Gaussian ({P}, got {values.numel()}) and feature_bg one")
    M = sh.size(1) if (sh is not None and sh.numel() != 0) else 0
    if sh_rest is not None:
        if M != 1 or sh_rest.dim() != 3 or sh_rest.size(0) != P:
            raise RuntimeError("raw-parameter mode: sh must be [P,1,3] and sh_rest [P,M-1,3]")
        M = 1 + sh_rest.size(1)
        sh_rest = _c(sh_rest)
    with torch.cuda.device(dev):
        out_color = torch.empty((3, H, W), dtype=torch.float32, device=dev)
        out_feature = torch.empty((H, W), dtype=torch.float32, device=dev) if feature else None
        radii = torch.empty((P,), dtype=torch.int32, device=dev)
        key = (dev.index, H, W)
        hint = context.capacity_hint.get(key, 0)
        reserve = lib.sgr_geometry_bytes(P) + lib.sgr_image_bytes(W, H) + 1024
        if hint:
            reserve += lib.sgr_binning_bytes(hint)
        arena = _Arena(dev, reserve if P else 0)
        means3D, colors, opacity, scales, rotations, cov3D_precomp, sh, values, feature_bg = map(
            _c, (means3D, colors, opacity, scales, rotations, cov3D_precomp, sh, values, feature_bg))
        background, viewmatrix, projmatrix, campos = map(_c, (background, viewmatrix, projmatrix, campos))
        view = _view_struct(background, scale_modifier, viewmatrix, projmatrix, tan_fovx, tan_fovy, H, W, degree,
                            campos, prefiltered, debug)
        g = _gauss_struct(P, M, means3D, opacity, sh, colors, scales, rotations, cov3D_precomp, sh_rest)
        rendered = C.c_int64(0)
        allocs = (arena.cbs["geom"], None, arena.cbs["binning"], None, arena.cbs["img"], None)
        tail = (radii.data_ptr() if P else None, hint, C.byref(rendered), stream(dev))
        if feature:
            status = lib.sgr_rasterize_forward_feature(
                C.byref(view), C.byref(g), *allocs, f32_ptr(values, "values"), f32_ptr(feature_bg, "feature_bg"),
                out_color.data_ptr(), out_feature.data_ptr(), *tail)
        else:
            status = lib.sgr_rasterize_forward(C.byref(view), C.byref(g), *allocs, out_color.data_ptr(), *tail)
        if arena.error is not None:   # the allocator callback failed (e.g. out of memory): its own exception, not
            err = arena.error         # the library's generic "allocator returned NULL"
            arena.release()
            raise err
        check(status)
        R = int(rendered.value)
        if P:
            # next view's optimistic capacity: 25% headroom, rounded to 1M instances (stable sizes)
            context.capacity_hint[key] = _round_up(int(R * 1.25) + 65536, 1 << 20)
    geom_t, binning_t, img_t = arena.get("geom"), arena.get("binning"), arena.get("img")
    arena.release()
    out = (R, out_color, radii, geom_t, binning_t, img_t)
    return out + (out_feature,) if feature else out


_PART_ALIGN = 16  # floats: every gradient array starts on a 64-byte boundary (TMA bulk stores need 16)


def _alloc_backward(P: int, M: int, dev, with_records: bool, split_sh: bool = False):
    """All eight gradients (+ the 44-byte reduce records of the view-parallel step) + the accumulator scratch in
    ONE rounded allocation: a stable size for the caching allocator, one free when autograd lets go."""
    widths = [("means3D", 3), ("opacity", 1), ("scales", 3), ("rotations", 4), ("sh", 3 if split_sh else 3 * M),
              ("means2D", 3), ("colors", 3), ("cov3D", 6)]
    if with_records:
        widths.append(("records", 11))
    if split_sh:
        widths.append(("sh_rest", 3 * (M - 1)))
    n_scratch = (lib.sgr_backward_scratch_bytes(P) + 3) // 4 if P else 0
    offs, o = {}, 0
    for name, w in widths:
        offs[name] = o
        # dL_dcolors is followed by 4 spare floats: the view-parallel exchange appends the camera position there,
        # so that one all-gather carries a view's SH factors and its camera
        o = _round_up(o + P * w + (4 if name == "colors" else 0), _PART_ALIGN)
    total = o + n_scratch + 64
    flat = torch.empty(_round_up(4 * total, _ROUND) // 4, dtype=torch.float32, device=dev)
    skew = (-(flat.data_ptr() // 4)) % _PART_ALIGN  # the allocator aligns to 512 B; be explicit anyway
    shapes = {"means3D": (P, 3), "opacity": (P, 1), "scales": (P, 3), "rotations": (P, 4),
              "sh": (P, 1 if split_sh else M, 3), "sh_rest": (P, max(M - 1, 0), 3), "means2D": (P, 3), "colors": (P, 3),
              "cov3D": (P, 6), "records": (P, 11)}
    bufs = {name: flat[skew + offs[name]:skew + offs[name] + P * w].view(shapes[name]) for name, w in widths}
    bufs["scratch"] = flat[skew + o:skew + o + n_scratch]
    bufs["colors_block"] = flat[skew + offs["colors"]:skew + offs["colors"] + 3 * P + 4]
    return bufs


def rasterize_gaussians_backward(background, means3D, radii, colors, scales, rotations, scale_modifier,
                                 cov3D_precomp, viewmatrix, projmatrix, tan_fovx, tan_fovy, dL_dout_color, sh,
                                 degree, campos, geomBuffer, R, binningBuffer, imageBuffer, debug, *,
                                 context: Context = None, sh_rest: torch.Tensor = None, values: torch.Tensor = None,
                                 feature_bg: torch.Tensor = None, dL_dout_feature: torch.Tensor = None):
    """RasterizeGaussiansBackwardCUDA (rasterize_points.cu:118-196).  With a view-parallel exchange attached to
    `context` (sugar_b200/parallel.py) the gradients come back already summed over the ranks.  With `sh_rest`
    (raw-parameter mode, see rasterize_gaussians) a ninth tensor dL_dsh_rest is returned and dL_dopacity /
    dL_dscales / dL_drotations / dL_dsh are gradients of the raw parameters.  With `values` (the extra channel of
    rasterize_gaussians, gradient `dL_dout_feature` [H,W]; sgr_rasterize_backward_feature) each of the eight
    gradients holds both channels' terms and a ninth tensor dL_dvalues [P] is returned."""
    context = context or current_context()
    feature = values is not None
    if feature:
        _no_exchange(context)
    dev = means3D.device
    P, H, W = means3D.size(0), dL_dout_color.size(1), dL_dout_color.size(2)
    M = sh.size(1) if (sh is not None and sh.numel() != 0) else 0
    raw = sh_rest is not None
    if raw:
        M = 1 + sh_rest.size(1)
        sh_rest = _c(sh_rest)
    ex = context.exchange if (context.exchange is not None and context.exchange.enabled()) else None
    if raw and ex is not None:
        raise NotImplementedError("raw-parameter mode under a view-parallel exchange: activate in PyTorch instead "
                                  "(the exchange acts on the op's output gradients either way)")
    with torch.cuda.device(dev):
        has_cov = cov3D_precomp is not None and cov3D_precomp.numel() != 0
        # the peer-memory exchange keeps its records in its own peer-visible buffer
        b = _alloc_backward(P, M, dev, with_records=ex is not None and not ex.uses_peer_memory(M, has_cov), split_sh=raw)
        dL_dvalues = torch.empty((P,), dtype=torch.float32, device=dev) if feature else None  # every row written
        if P != 0:
            means3D, colors, scales, rotations, cov3D_precomp, sh, dL_dout_color = map(
                _c, (means3D, colors, scales, rotations, cov3D_precomp, sh, dL_dout_color))
            values, feature_bg, dL_dout_feature = map(_c, (values, feature_bg, dL_dout_feature))
            background, viewmatrix, projmatrix, campos = map(_c, (background, viewmatrix, projmatrix, campos))
            view = _view_struct(background, scale_modifier, viewmatrix, projmatrix, tan_fovx, tan_fovy, H, W, degree,
                                campos, False, debug)
            # opacities are not an input of the reference's backward; the forward stored them
            g = _gauss_struct(P, M, means3D, None, sh, colors, scales, rotations, cov3D_precomp, sh_rest)
            st = stream(dev)
            # the SH exchange rebuilds the summed dL_dsh from the views' colour gradients: the pass does not write it
            dsh = b["sh"].data_ptr() if (M and not (ex is not None and ex.sh_factors)) else None
            inputs = (C.byref(view), C.byref(g), radii.data_ptr(), geomBuffer.data_ptr(), binningBuffer.data_ptr(),
                      imageBuffer.data_ptr(), int(R), f32_ptr(dL_dout_color, "dL_dout_color"))

            def grads(dL_dcolors, dL_dsh):   # the eight gradient arrays in the C argument order
                return (b["means2D"].data_ptr(), dL_dcolors, b["opacity"].data_ptr(), b["means3D"].data_ptr(),
                        b["cov3D"].data_ptr(), dL_dsh, b["scales"].data_ptr(), b["rotations"].data_ptr())

            def launch(plan, *, dL_dcolors=b["colors"].data_ptr(), dL_dsh=dsh):
                """Enqueue sgr_rasterize_backward_staged under `plan` (None: no stages); the view-parallel peer
                exchange points the two outputs it sums itself into its own buffers."""
                check(lib.sgr_rasterize_backward_staged(*inputs, *grads(dL_dcolors, dL_dsh), b["scratch"].data_ptr(),
                                                        st, None if plan is None else C.byref(plan)))

            if feature:
                check(lib.sgr_rasterize_backward_feature(
                    *inputs, f32_ptr(values, "values"), f32_ptr(feature_bg, "feature_bg"),
                    f32_ptr(dL_dout_feature, "dL_dout_feature"), *grads(b["colors"].data_ptr(), dsh),
                    dL_dvalues.data_ptr(), b["scratch"].data_ptr(), st))
            elif ex is not None:
                ex.run_backward(launch, b, P, M, int(degree), means3D, campos, has_cov_precomp=has_cov)
            elif raw:   # the plan carries the second SH gradient array
                launch(_lib.SgrBackwardPlan(num_chunks=1, dL_dsh_rest=b["sh_rest"].data_ptr() if M > 1 else None))
            else:
                launch(None)
    out = (b["means2D"], b["colors"], b["opacity"], b["means3D"], b["cov3D"], b["sh"], b["scales"], b["rotations"])
    return out + ((b["sh_rest"],) if raw else (dL_dvalues,) if feature else ())


def mark_visible(means3D, viewmatrix, projmatrix) -> torch.Tensor:
    """markVisible (rasterize_points.cu:198-216)."""
    P = means3D.size(0)
    present = torch.zeros((P,), dtype=torch.bool, device=means3D.device)
    if P != 0:
        with torch.cuda.device(means3D.device):
            means3D, viewmatrix, projmatrix = map(_c, (means3D, viewmatrix, projmatrix))
            check(lib.sgr_mark_visible(P, f32_ptr(means3D, "means3D"), f32_ptr(viewmatrix, "viewmatrix"),
                                       f32_ptr(projmatrix, "projmatrix"), present.data_ptr(),
                                       stream(means3D.device)))
    return present


def inspect_state(P, W, H, R, geomBuffer, binningBuffer, imageBuffer):
    """Decode the opaque buffers into the reference's named arrays (parity tests only)."""
    dev = geomBuffer.device
    T = ((W + 15) // 16) * ((H + 15) // 16)
    f = lambda *s: torch.zeros(s, dtype=torch.float32, device=dev)
    out = dict(depths=f(P), means2D=f(P, 2), conic_opacity=f(P, 4), rgb=f(P, 3),
               clamped=torch.zeros((P, 3), dtype=torch.uint8, device=dev),
               tiles_touched=torch.zeros(P, dtype=torch.int32, device=dev),
               keys=torch.zeros(max(R, 1), dtype=torch.int64, device=dev),
               point_list=torch.zeros(max(R, 1), dtype=torch.int32, device=dev),
               ranges=torch.zeros((T, 2), dtype=torch.int32, device=dev),
               final_T=f(H, W), n_contrib=torch.zeros((H, W), dtype=torch.int32, device=dev),
               footprint=torch.zeros(max(R, 1), dtype=torch.uint8, device=dev))
    with torch.cuda.device(dev):
        check(lib.sgr_inspect_state(P, W, H, R, geomBuffer.data_ptr(), binningBuffer.data_ptr(), imageBuffer.data_ptr(),
                                    out["depths"].data_ptr(), out["means2D"].data_ptr(),
                                    out["conic_opacity"].data_ptr(), out["rgb"].data_ptr(), out["clamped"].data_ptr(),
                                    out["tiles_touched"].data_ptr(), out["keys"].data_ptr(),
                                    out["point_list"].data_ptr(), out["ranges"].data_ptr(), out["final_T"].data_ptr(),
                                    out["n_contrib"].data_ptr(), out["footprint"].data_ptr(), stream(dev)))
    out["keys"] = out["keys"][:R]
    out["point_list"] = out["point_list"][:R]
    out["footprint"] = out["footprint"][:R]
    return out
