"""ctypes binding of libsugar_b200.so (the C ABI declared in include/sugar_b200.h).

There is no CPU fallback: if the CUDA library is missing this module raises at import, and every
call raises on a non-zero status with the library's own message.
"""
import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("SGR_LIB_PATH", os.path.join(_HERE, "lib", "libsugar_b200.so"))  # override: the stats build (scripts/blend_stats.py)


class SgrError(RuntimeError):
    pass


class SgrView(C.Structure):
    _fields_ = [
        ("image_height", C.c_int32), ("image_width", C.c_int32),
        ("tanfovx", C.c_float), ("tanfovy", C.c_float),
        ("bg", C.c_void_p), ("scale_modifier", C.c_float),
        ("viewmatrix", C.c_void_p), ("projmatrix", C.c_void_p),
        ("sh_degree", C.c_int32), ("campos", C.c_void_p),
        ("prefiltered", C.c_int32), ("debug", C.c_int32),
    ]


class SgrGaussians(C.Structure):
    _fields_ = [
        ("P", C.c_int32), ("M", C.c_int32),
        ("means3D", C.c_void_p), ("opacities", C.c_void_p), ("shs", C.c_void_p),
        ("colors_precomp", C.c_void_p), ("scales", C.c_void_p), ("rotations", C.c_void_p),
        ("cov3D_precomp", C.c_void_p), ("activations", C.c_int32), ("sh_rest", C.c_void_p),
    ]


class SgrFieldParams(C.Structure):
    _fields_ = [("N", C.c_int32), ("K", C.c_int32), ("P", C.c_int32), ("density_factor", C.c_float),
                ("density_threshold", C.c_float), ("opacity_min_clamp", C.c_float), ("samples_per_idx_row", C.c_int32)]


class SgrSsimParams(C.Structure):
    _fields_ = [("B", C.c_int32), ("C", C.c_int32), ("H", C.c_int32), ("W", C.c_int32), ("c1", C.c_float),
                ("c2", C.c_float), ("window", C.c_float * 11)]


class SgrDensifyGates(C.Structure):
    _fields_ = [("max_grad", C.c_float), ("clone_scale", C.c_float), ("big_scale", C.c_float),
                ("min_opacity", C.c_float), ("screen_size", C.c_float), ("inv_split", C.c_float),
                ("use_screen", C.c_int32)]


class SgrDensifyColumn(C.Structure):
    _fields_ = [("src", C.c_void_p), ("dst", C.c_void_p), ("width", C.c_int32), ("kind", C.c_int32)]


class SgrAdamSegment(C.Structure):
    _fields_ = [("param", C.c_void_p), ("grad", C.c_void_p), ("exp_avg", C.c_void_p), ("exp_avg_sq", C.c_void_p),
                ("n", C.c_int64), ("one_minus_beta1", C.c_float), ("beta2", C.c_float), ("one_minus_beta2", C.c_float),
                ("bias_correction2_sqrt", C.c_float), ("eps", C.c_float), ("step_size", C.c_float)]


ALLOC_FN = C.CFUNCTYPE(C.c_void_p, C.c_void_p, C.c_size_t)
STAGE_HOOK = C.CFUNCTYPE(None, C.c_void_p, C.c_int32)


class SgrPeerPlan(C.Structure):
    _fields_ = [("peer_flag_tab", C.c_void_p), ("peer_nranks", C.c_int32), ("peer_rank", C.c_int32),
                ("peer_slot_blend", C.c_int32), ("peer_slot_chunk0", C.c_int32), ("peer_seq", C.c_uint32),
                ("peer_view_blocks", C.c_void_p), ("peer_flags", C.c_void_p), ("peer_dsh_scale", C.c_float),
                ("peer_timeout_s", C.c_double), ("peer_record_stages", C.c_void_p), ("peer_signal_stream", C.c_void_p),
                ("peer_side_stream", C.c_void_p), ("peer_rec_tab", C.c_void_p), ("peer_sum_tab", C.c_void_p),
                ("peer_sums", C.c_void_p), ("peer_slot_reduced0", C.c_int32), ("peer_emulate_ranks", C.c_uint64)]


class SgrBackwardPlan(C.Structure):
    _fields_ = [("hook", STAGE_HOOK), ("hook_ctx", C.c_void_p), ("num_chunks", C.c_int32),
                ("reduce_records", C.c_void_p), ("dL_dsh_rest", C.c_void_p), ("chunk_taper", C.c_int32),
                ("peer", C.POINTER(SgrPeerPlan))]


# name -> (restype, argtypes); kept in one table so tests can check it against the header
PROTOTYPES = {
    "sgr_rasterize_forward": (C.c_int, [C.POINTER(SgrView), C.POINTER(SgrGaussians), ALLOC_FN, C.c_void_p, ALLOC_FN,
                                        C.c_void_p, ALLOC_FN, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64,
                                        C.POINTER(C.c_int64), C.c_void_p]),
    "sgr_rasterize_backward": (C.c_int, [C.POINTER(SgrView), C.POINTER(SgrGaussians)] + [C.c_void_p] * 4 +
                               [C.c_int64] + [C.c_void_p] * 11),
    "sgr_rasterize_backward_staged": (C.c_int, [C.POINTER(SgrView), C.POINTER(SgrGaussians)] + [C.c_void_p] * 4 +
                                      [C.c_int64] + [C.c_void_p] * 11 + [C.POINTER(SgrBackwardPlan)]),
    "sgr_rasterize_forward_feature": (C.c_int, [C.POINTER(SgrView), C.POINTER(SgrGaussians), ALLOC_FN, C.c_void_p,
                                                ALLOC_FN, C.c_void_p, ALLOC_FN, C.c_void_p] + [C.c_void_p] * 5 +
                                      [C.c_int64, C.POINTER(C.c_int64), C.c_void_p]),
    "sgr_rasterize_backward_feature": (C.c_int, [C.POINTER(SgrView), C.POINTER(SgrGaussians)] + [C.c_void_p] * 4 +
                                       [C.c_int64] + [C.c_void_p] * 15),
    "sgr_backward_chunk_range": (C.c_int, [C.c_int32] * 4 + [C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    "sgr_view_grad_finalize": (C.c_int, [C.c_int32] * 6 + [C.c_void_p] * 3 + [C.c_int64, C.c_int32] + [C.c_void_p] * 2 +
                               [C.c_float] + [C.c_void_p] * 5),
    "sgr_peer_alloc": (C.c_int, [C.c_size_t, C.POINTER(C.c_void_p)]),
    "sgr_peer_free": (C.c_int, [C.c_void_p]),
    "sgr_peer_export": (C.c_int, [C.c_void_p, C.c_void_p]),
    "sgr_peer_import": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p)]),
    "sgr_peer_close": (C.c_int, [C.c_void_p]),
    "sgr_peer_flag_bytes": (C.c_size_t, []),
    "sgr_peer_signal": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_uint32, C.c_void_p]),
    "sgr_peer_wait": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_uint32, C.c_double, C.c_void_p]),
    "sgr_peer_reduce_records_synced": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                                 C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_uint32, C.c_void_p,
                                                 C.c_double, C.c_void_p]),
    "sgr_mark_visible": (C.c_int, [C.c_int32] + [C.c_void_p] * 5),
    "sgr_geometry_bytes": (C.c_size_t, [C.c_int32]),
    "sgr_binning_bytes": (C.c_size_t, [C.c_int64]),
    "sgr_image_bytes": (C.c_size_t, [C.c_int32, C.c_int32]),
    "sgr_backward_scratch_bytes": (C.c_size_t, [C.c_int32]),
    "sgr_inspect_state": (C.c_int, [C.c_int32, C.c_int32, C.c_int32, C.c_int64] + [C.c_void_p] * 16),
    "sgr_field_scratch_bytes": (C.c_size_t, [C.c_int32]),
    "sgr_normal_scratch_bytes": (C.c_size_t, [C.c_int32]),
    "sgr_normal_loss_forward": (C.c_int, [C.c_int32] * 3 + [C.c_void_p] * 10),
    "sgr_normal_loss_backward": (C.c_int, [C.c_int32] * 3 + [C.c_void_p] * 11),
    "sgr_field_forward": (C.c_int, [C.POINTER(SgrFieldParams)] + [C.c_void_p] * 12),
    "sgr_field_backward": (C.c_int, [C.POINTER(SgrFieldParams)] + [C.c_void_p] * 17),
    "sgr_density_estimation_forward": (C.c_int, [C.POINTER(SgrFieldParams)] + [C.c_void_p] * 11),
    "sgr_density_estimation_backward": (C.c_int, [C.POINTER(SgrFieldParams)] + [C.c_void_p] * 15),
    "sgr_meshbind_forward": (C.c_int, [C.c_int32] * 3 + [C.c_void_p] * 5 + [C.c_float] + [C.c_void_p] * 4),
    "sgr_meshbind_backward": (C.c_int, [C.c_int32] * 3 + [C.c_void_p] * 12),
    "sgr_meshbind_edited_forward": (C.c_int, [C.c_int32] * 3 + [C.c_void_p] * 6 + [C.c_float] + [C.c_void_p] * 5),
    "sgr_sh_colors_rotated": (C.c_int, [C.c_int32] * 3 + [C.c_void_p] * 3 + [C.c_int32] + [C.c_void_p] * 4),
    "sgr_knn_workspace_bytes": (C.c_size_t, [C.c_int32]),
    "sgr_knn": (C.c_int, [C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                          C.c_void_p]),
    "sgr_dist_cuda2": (C.c_int, [C.c_int32] + [C.c_void_p] * 4),
    "sgr_l1_ssim_scratch_bytes": (C.c_size_t, [C.c_int32] * 4),
    "sgr_l1_ssim_forward": (C.c_int, [C.POINTER(SgrSsimParams)] + [C.c_void_p] * 6),
    "sgr_l1_ssim_backward": (C.c_int, [C.POINTER(SgrSsimParams)] + [C.c_void_p] * 7),
    "sgr_mesh_nc_forward_scratch_bytes": (C.c_size_t, [C.c_int32]),
    "sgr_mesh_nc_backward_scratch_bytes": (C.c_size_t, [C.c_int32]),
    "sgr_mesh_nc_forward": (C.c_int, [C.c_int32, C.c_int32] + [C.c_void_p] * 5),
    "sgr_mesh_nc_backward": (C.c_int, [C.c_int32, C.c_int32] + [C.c_void_p] * 8),
    "sgr_border_peel": (C.c_int, [C.c_int32, C.c_int32] + [C.c_void_p] * 6),
    "sgr_splat_mesh": (C.c_int, [C.c_int32] + [C.c_void_p] * 5 + [C.c_float, C.c_void_p, C.c_void_p]),
    "sgr_mesh_raster_scratch_bytes": (C.c_size_t, [C.c_int32] * 3),
    "sgr_mesh_raster": (C.c_int, [C.c_int32, C.c_int32] + [C.c_void_p] * 4 + [C.c_int32, C.c_int32] +
                        [C.c_void_p] * 4),
    "sgr_texture_init": (C.c_int, [C.c_int32] * 5 + [C.c_void_p] * 8),
    "sgr_texture_bake_view": (C.c_int, [C.c_int32] * 4 + [C.c_void_p] * 6 + [C.c_int32, C.c_int32] +
                              [C.c_void_p] * 8),
    "sgr_texture_render": (C.c_int, [C.c_int32] * 5 + [C.c_void_p] * 7 + [C.c_int32] * 2 + [C.c_void_p] * 2 +
                           [C.c_int32] + [C.c_float] * 3 + [C.c_double] * 2 + [C.c_void_p] * 2),
    "sgr_density_grid_workspace_bytes": (C.c_size_t, [C.c_int32]),
    "sgr_density_grid": (C.c_int, [C.c_int32] + [C.c_void_p] * 4 + [C.c_int32, C.c_float] + [C.c_int32] * 3 +
                         [C.c_void_p] * 3 + [C.c_float] + [C.c_void_p] * 3),
    "sgr_mcubes_scratch_bytes": (C.c_size_t, [C.c_int32] * 3),
    "sgr_mcubes_count": (C.c_int, [C.c_int32] * 3 + [C.c_void_p, C.c_double] + [C.c_void_p] * 4),
    "sgr_mcubes_emit": (C.c_int, [C.c_int32] * 3 + [C.c_void_p, C.c_double, C.c_int64, C.c_int64] + [C.c_void_p] * 4),
    "sgr_poisson_bin": (C.c_int, [C.c_int32, C.c_void_p, C.c_int32] + [C.c_float] * 4 + [C.c_void_p] * 8),
    "sgr_poisson_splat": (C.c_int, [C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32,
                                    C.c_float, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p]),
    "sgr_poisson_coarsen": (C.c_int, [C.c_int32] + [C.c_void_p] * 3),
    "sgr_poisson_residual_norm": (C.c_int, [C.c_int32, C.c_float] + [C.c_void_p] * 6),
    "sgr_poisson_vcycle": (C.c_int, [C.c_int32] + [C.c_void_p] * 6),
    "sgr_poisson_interpolate": (C.c_int, [C.c_int32, C.c_void_p, C.c_int64, C.c_void_p, C.c_int32, C.c_float, C.c_float] +
                                [C.c_void_p] * 4),
    "sgr_decimate_scratch_bytes": (C.c_size_t, [C.c_int32, C.c_int32]),
    "sgr_decimate": (C.c_int, [C.c_int32, C.c_int32, C.c_int64] + [C.c_void_p] * 11),
    "sgr_densify_stats": (C.c_int, [C.c_int32, C.c_void_p, C.c_int32] + [C.c_void_p] * 6),
    "sgr_densify_classify": (C.c_int, [C.c_int32] + [C.c_void_p] * 4 + [C.POINTER(SgrDensifyGates)] +
                             [C.c_void_p] * 2),
    "sgr_densify_emit": (C.c_int, [C.c_int32] * 5 + [C.c_void_p, C.c_int32, C.POINTER(SgrDensifyColumn)] +
                         [C.c_void_p] * 4 + [C.c_float, C.c_void_p, C.c_void_p]),
    "sgr_adam_step": (C.c_int, [C.c_int32, C.POINTER(SgrAdamSegment), C.c_void_p]),
    "sgr_struct_bytes": (C.c_size_t, [C.c_int32]),
    "sgr_launch_count": (C.c_ulonglong, []),
    "sgr_num_kernel_kinds": (C.c_int, []),
    "sgr_kernel_name": (C.c_char_p, [C.c_int]),
    "sgr_profile_enable": (C.c_int, [C.c_int]),
    "sgr_profile_read": (C.c_int, [C.c_void_p, C.c_void_p]),
    "sgr_profile_timeline": (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "sgr_last_error": (C.c_char_p, []),
    "sgr_version": (C.c_char_p, []),
}


def _load():
    if not os.path.exists(LIB_PATH):
        raise SgrError(
            f"{LIB_PATH} not found: build it with `python sugar_b200/build.py` (needs nvcc). "
            "sugar_b200 has no CPU or PyTorch fallback.")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in PROTOTYPES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is missing
        fn.restype = res
        fn.argtypes = args
    return lib


lib = _load()
for _i, _t in enumerate((SgrView, SgrGaussians, SgrBackwardPlan, SgrFieldParams, SgrSsimParams, SgrDensifyGates,
                          SgrDensifyColumn, SgrAdamSegment, SgrPeerPlan)):
    if lib.sgr_struct_bytes(_i) != C.sizeof(_t):   # a stale library or a binding edited without the header
        raise SgrError(f"{LIB_PATH}: struct {_t.__name__} is {lib.sgr_struct_bytes(_i)} bytes in the library, "
                       f"{C.sizeof(_t)} in this binding -- rebuild with `python sugar_b200/build.py`")


def check(status: int) -> None:
    if status != 0:
        raise SgrError(lib.sgr_last_error().decode(errors="replace") or f"libsugar_b200 error {status}")


# How the op wrappers pass tensors to the library.  Argument checks run first, so that they work on CPU tensors too.

def ptr(t):
    """Device pointer of an optional tensor: None or an empty tensor gives NULL."""
    return None if t is None or t.numel() == 0 else t.data_ptr()


def f32_ptr(t, name: str):
    """ptr() of an optional float32 CUDA tensor, checked (the rasterizer's arguments)."""
    if t is None or t.numel() == 0:
        return None
    if t.dtype != torch.float32:
        raise TypeError(f"{name} must be float32, got {t.dtype}")
    if not t.is_cuda:
        raise SgrError(f"{name} must be a CUDA tensor (sugar_b200 has no CPU path)")
    return t.data_ptr()


def stream(dev):
    """The current CUDA stream of `dev` as the library takes it."""
    return torch.cuda.current_stream(dev).cuda_stream


def scratch(nbytes: int, dev) -> torch.Tensor:
    """Device scratch of `nbytes`, the answer of one of the library's size queries."""
    return torch.empty(nbytes, dtype=torch.uint8, device=dev)


def require_cuda(module: str, *ts) -> None:
    for t in ts:
        if t is not None and not (torch.is_tensor(t) and t.is_cuda):
            raise SgrError(f"sugar_b200.{module} needs CUDA tensors: there is no CPU fallback")


def tensor(t, name: str, dtype, shape, device=None, ref: str = "verts", align: int = 0):
    """-> `t` as the kernel may read it: contiguous, and copied when `align` (bytes) is given and not met.
    Raises ValueError unless `t` is a `dtype` tensor of `shape` on `device` (when given; `ref` names the argument
    that fixed it).  `shape` entries are sizes, or names of free dimensions (str)."""
    want = ",".join(str(s) for s in shape)
    if not torch.is_tensor(t) or t.dtype != dtype or t.dim() != len(shape) or \
            any(isinstance(s, int) and t.shape[i] != s for i, s in enumerate(shape)):
        got = f"{t.dtype} {tuple(t.shape)}" if torch.is_tensor(t) else type(t).__name__
        raise ValueError(f"{name} must be {str(dtype).replace('torch.', '')} [{want}], got {got}")
    if device is not None and t.device != device:
        raise ValueError(f"{name} on {t.device}, {ref} on {device}")
    t = t.contiguous()
    if align and t.data_ptr() % align:
        t = t.clone()
    return t


def same_device(dev, ref: str = "verts", **ts) -> None:
    for name, t in ts.items():
        if t is not None and t.device != dev:
            raise ValueError(f"{name} on {t.device}, {ref} on {dev}")


def check_ids(*checks) -> None:
    """checks: (ids, lo, hi, what).  Raises ValueError naming each check with ids outside [lo, hi), after one host
    read for all of them."""
    checks = [c for c in checks if c[0].numel()]
    if not checks:
        return
    counts = torch.stack([((ids < lo) | (ids >= hi)).sum() for ids, lo, hi, _ in checks]).tolist()
    for n, (_, lo, hi, what) in zip(counts, checks):
        if n:
            raise ValueError(f"{n} {what} outside [{lo}, {hi})")


def profile(on: bool) -> None:
    check(lib.sgr_profile_enable(int(on)))


def profile_read():
    """-> {kernel name: (total_ms, launches)} since profiling was enabled / last read."""
    n = lib.sgr_num_kernel_kinds()
    ms = (C.c_float * n)()
    cnt = (C.c_int * n)()
    check(lib.sgr_profile_read(ms, cnt))
    return {lib.sgr_kernel_name(k).decode(): (float(ms[k]), int(cnt[k])) for k in range(n) if cnt[k]}


def profile_timeline(max_records: int = 4096):
    """-> [(kernel name, begin_ms, end_ms)] of every launch since profiling was enabled."""
    kinds = (C.c_int * max_records)()
    tb = (C.c_float * max_records)()
    te = (C.c_float * max_records)()
    n = lib.sgr_profile_timeline(max_records, kinds, tb, te)
    if n < 0:
        check(n)
    return [(lib.sgr_kernel_name(kinds[i]).decode(), float(tb[i]), float(te[i])) for i in range(n)]
