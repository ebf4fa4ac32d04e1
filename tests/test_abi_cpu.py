"""CPU checks of the C ABI: libsugar_b200.so loads without a GPU and exports every function
include/sugar_b200.h declares (no compute calls here)."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_functions():
    text = open(os.path.join(ROOT, "include", "sugar_b200.h")).read()
    return sorted(set(re.findall(r"SGR_API[^;(]*?\b(sgr_[a-z_0-9]+)\s*\(", text)))


def test_library_exports_every_declared_symbol():
    from sugar_b200 import _lib
    names = declared_functions()
    assert len(names) >= 15
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/sugar_b200.h but not exported"
    assert set(_lib.PROTOTYPES) == set(names), (set(names) ^ set(_lib.PROTOTYPES))


def test_sizes_and_errors_without_gpu():
    from sugar_b200 import _lib
    L = _lib.lib
    assert b"sm_90a" in L.sgr_version()
    assert L.sgr_geometry_bytes(1000) >= 1000 * 60
    assert L.sgr_binning_bytes(0) > 0
    assert L.sgr_image_bytes(1920, 1080) >= 1920 * 1080 * 8
    assert L.sgr_backward_scratch_bytes(10) >= 320
    # argument validation happens before any CUDA call
    v = _lib.SgrView(); g = _lib.SgrGaussians()
    v.image_width, v.image_height, g.P = 0, 0, 5
    n = ctypes.c_int64(0)
    cb = _lib.SgrAlloc(lambda ctx, n: 0)
    rc = L.sgr_rasterize_forward(ctypes.byref(v), ctypes.byref(g), cb, None, cb, None, cb, None, None, None, 0,
                                 ctypes.byref(n), None)
    assert rc == -1 and b"bad sizes" in L.sgr_last_error()


def test_dropin_module_surface():
    from sugar_b200 import diff_gaussian_rasterization as m
    assert m.GaussianRasterizationSettings._fields == (
        "image_height", "image_width", "tanfovx", "tanfovy", "bg", "scale_modifier", "viewmatrix", "projmatrix",
        "sh_degree", "campos", "prefiltered", "debug")
    import inspect
    sig = inspect.signature(m.GaussianRasterizer.forward)
    assert list(sig.parameters) == ["self", "means3D", "means2D", "opacities", "shs", "colors_precomp", "scales",
                                    "rotations", "cov3D_precomp"]
    assert list(inspect.signature(m.rasterize_gaussians).parameters) == [
        "means3D", "means2D", "sh", "colors_precomp", "opacities", "scales", "rotations", "cov3Ds_precomp",
        "raster_settings"]
    assert hasattr(m.GaussianRasterizer, "markVisible")


def test_entry_points_validate_arguments_without_gpu():
    """Factor-mode rebuild, normal loss, K-NN and field entry points reject bad sizes / null pointers before
    touching CUDA (status -1 + message), and their workspace queries are monotone."""
    from sugar_b200 import _lib
    L = _lib.lib
    dummy = ctypes.c_void_p(16)

    def sh_from_factors(P, M, degree, views, means3D, campos, dRGB, dL_dsh):   # parallel.sh_grad_from_factors
        return L.sgr_view_grad_finalize(P, 0, P, M, degree, views, means3D, campos, dRGB, 3 * P, 3, dL_dsh, None, 1.0,
                                        *([None] * 5))
    assert sh_from_factors(10, 0, 0, 1, dummy, dummy, dummy, dummy) == -1      # M must be > 0
    assert sh_from_factors(10, 16, 4, 1, dummy, dummy, dummy, dummy) == -1     # degree > 3
    assert sh_from_factors(10, 16, 3, 1, None, None, None, dummy) == -1        # null pointers
    assert sh_from_factors(10, 16, 3, 1, None, None, None, None) == -1
    assert b"sgr_view_grad_finalize" in L.sgr_last_error()
    assert sh_from_factors(0, 16, 3, 1, None, None, None, None) == -1          # nothing to write into
    assert L.sgr_normal_loss_forward(5, 0, 10, *([None] * 10)) == -1                        # K must be > 0
    assert L.sgr_normal_loss_forward(5, 16, 10, *([None] * 10)) == -1                       # null pointers
    assert L.sgr_normal_loss_backward(5, 16, 10, *([None] * 11)) == -1
    p = _lib.SgrFieldParams()
    p.N, p.K, p.P = 4, 0, 10
    assert L.sgr_field_forward(ctypes.byref(p), *([None] * 12)) == -1
    for fn in (L.sgr_field_scratch_bytes, L.sgr_normal_scratch_bytes, L.sgr_knn_workspace_bytes):
        assert 0 < fn(1000) <= fn(100000)
    # the staged backward shares the plain one's validation
    v = _lib.SgrView(); g = _lib.SgrGaussians()
    v.image_width, v.image_height, g.P = 0, 0, 5
    hook = _lib.SgrStageHook(lambda ctx, stage: None)
    plan = _lib.SgrBackwardPlan(hook=hook, num_chunks=4)
    assert L.sgr_rasterize_backward_staged(ctypes.byref(v), ctypes.byref(g), *([None] * 4), 0, *([None] * 11),
                                           ctypes.byref(plan)) == -1
    # chunk ranges of the per-Gaussian pass: contiguous, cover [0, P), boundaries on CTA multiples
    p0, p1 = ctypes.c_int32(), ctypes.c_int32()
    for P, nch in ((1000, 4), (64, 4), (3_000_000, 4), (1, 1), (129, 3)):
        prev, seen = 0, 0
        for c in range(nch):
            assert L.sgr_backward_chunk_range(P, nch, c, 0, ctypes.byref(p0), ctypes.byref(p1)) == 0
            assert p0.value == min(prev, P) and p0.value <= p1.value <= P
            assert p0.value % 64 == 0 or p0.value == P
            prev, seen = p1.value, seen + (p1.value - p0.value)
        assert seen == P and prev == P
    assert L.sgr_backward_chunk_range(10, 2, 2, 0, ctypes.byref(p0), ctypes.byref(p1)) == -1
    assert L.sgr_view_grad_finalize(10, 0, 10, 16, 3, 1, None, None, None, 30, 3, None, None, 1.0, *([None] * 5)) == -1


def test_struct_layouts_match_the_library():
    """The ctypes structs of the binding have the sizes the library was compiled with (sgr_struct_bytes)."""
    from sugar_b200 import _lib
    for i, t in enumerate((_lib.SgrView, _lib.SgrGaussians, _lib.SgrBackwardPlan, _lib.SgrFieldParams,
                           _lib.SgrSsimParams, _lib.SgrDensifyGates, _lib.SgrDensifyColumn, _lib.SgrAdamSegment,
                           _lib.SgrPeerPlan)):
        assert _lib.lib.sgr_struct_bytes(i) == ctypes.sizeof(t), t.__name__
    assert [f for f, _ in _lib.SgrBackwardPlan._fields_] == ["hook", "hook_ctx", "num_chunks", "reduce_records",
                                                              "dL_dsh_rest", "chunk_taper", "peer"]
    assert _lib.lib.sgr_struct_bytes(9) == 0 and _lib.lib.sgr_struct_bytes(99) == 0


def test_every_integer_define_is_exported():
    from sugar_b200 import _lib
    text = open(os.path.join(ROOT, "include", "sugar_b200.h")).read()
    defines = re.findall(r"^#define[ \t]+(SGR_\w+)[ \t]+\(?(-?\d+)\)?", text, re.M)
    assert len(defines) >= 15
    for name, value in defines:
        assert getattr(_lib, name, None) == int(value), name


def test_header_parser_rejects_unknown_types():
    """A type outside the binding's vocabulary is an import error that names its declaration, not a guessed width."""
    import pytest
    from sugar_b200 import _lib
    for decl, what in (("SGR_API int sgr_bad(int32_t n, half_t *x);", "sgr_bad(half_t *x)"),
                       ("typedef struct SgrBad { float a; bfloat16 b; } SgrBad;", "SgrBad.b"),
                       ("SGR_API long sgr_long(void);", "sgr_long")):
        with pytest.raises(_lib.SgrError, match=re.escape(what)):
            _lib.parse_header(decl)


def test_chunk_ranges_cover_and_halve():
    """SgrBackwardPlan.chunk_taper: contiguous cover of [0, P), boundaries on 64-Gaussian blocks, every chunk about half
    of the one before it; taper 0 is the plain equal split."""
    from sugar_b200 import _lib
    L = _lib.lib
    p0, p1 = ctypes.c_int32(), ctypes.c_int32()
    for P, n in ((3_000_000, 4), (6_000_000, 3), (6001, 3), (129, 3), (64, 4), (1000, 1), (257, 16)):
        prev, sizes = 0, []
        for c in range(n):
            assert L.sgr_backward_chunk_range(P, n, c, 1, ctypes.byref(p0), ctypes.byref(p1)) == 0
            assert p0.value == min(prev, P) and p0.value <= p1.value <= P
            assert p0.value % 64 == 0 or p0.value == P
            prev = p1.value
            sizes.append(p1.value - p0.value)
        assert prev == P and sum(sizes) == P
        if P >= 64 * 64 * n:
            for a, b in zip(sizes, sizes[1:]):
                assert 0.4 * a <= b <= 0.6 * a, sizes
        blocks = (P + 63) // 64
        for c in range(n):   # taper 0: the equal split of the 64-Gaussian blocks
            assert L.sgr_backward_chunk_range(P, n, c, 0, ctypes.byref(p0), ctypes.byref(p1)) == 0
            m = min(n, blocks)
            want = (P, P) if c >= m else (min(P, blocks * c // m * 64), min(P, blocks * (c + 1) // m * 64))
            assert (p0.value, p1.value) == want


def test_peer_entry_points_reject_bad_arguments_without_cuda():
    from sugar_b200 import _lib
    L = _lib.lib
    assert L.sgr_peer_flag_bytes() == 64 * 64 * 4
    assert L.sgr_peer_alloc(0, None) == -1 and b"sgr_peer_alloc" in L.sgr_last_error()
    assert L.sgr_peer_export(None, None) == -1 and L.sgr_peer_import(None, None) == -1
    assert L.sgr_peer_free(None) == 0 and L.sgr_peer_close(None) == 0          # nothing to do
    assert L.sgr_peer_signal(None, 2, 0, 0, 1, None) == -1                     # no flag table
    assert L.sgr_peer_wait(None, 2, 0, 1, 1, 1.0, None) == -1
    dummy = ctypes.c_void_p(16)
    assert L.sgr_peer_signal(dummy, 65, 0, 0, 1, None) == -1                   # more ranks than flag columns
    assert L.sgr_peer_signal(dummy, 2, 64, 0, 1, None) == -1                   # slot out of range
    assert L.sgr_peer_signal(dummy, 2, 0, 2, 1, None) == -1                    # rank out of range
    assert L.sgr_peer_wait(dummy, 2, 60, 5, 1, 1.0, None) == -1                # slots run past the table
    assert L.sgr_peer_reduce_records_synced(None, None, 2, 0, 0, 64, None, 0, None, 0, 0, None, 0.0, None) == -1
    assert L.sgr_peer_reduce_records_synced(dummy, dummy, 2, 0, 32, 64, None, 0, None, 0, 0, None, 0.0,
                                            None) == -1   # p0 not on a 64-record block
    assert L.sgr_peer_reduce_records_synced(dummy, dummy, 2, 0, 0, 64, None, 0, dummy, 3, 1, None, 1.0, None) == -1  # signal without counter


def test_backward_plan_is_checked_before_anything_is_enqueued():
    """A malformed SgrBackwardPlan / SgrPeerPlan is rejected with the backward's other arguments, naming the field,
    before the first launch: in peer mode the BLEND signal would otherwise have gone out to the other ranks already."""
    from sugar_b200 import _lib
    L = _lib.lib
    d = ctypes.c_void_p(256)   # a non-null, aligned dummy: nothing is dereferenced before the checks reject the plan
    P = 17 * 64                # 17 CTAs of the per-Gaussian pass: 17 chunks survive the clamp to one per CTA
    v = _lib.SgrView(image_height=16, image_width=16, bg=d, viewmatrix=d, projmatrix=d, campos=d, sh_degree=3)

    def peer(**kw):
        return ctypes.pointer(_lib.SgrPeerPlan(**{**dict(peer_flag_tab=d, peer_nranks=2, peer_slot_chunk0=1,
                                                         peer_slot_reduced0=20), **kw}))

    side = dict(peer_side_stream=d, peer_rec_tab=d, peer_sum_tab=d, peer_sums=d, peer_flags=d)
    for field, raw, plan in (
            ("dL_dsh_rest", 1, _lib.SgrBackwardPlan(num_chunks=1)),
            ("peer_view_blocks", 0, _lib.SgrBackwardPlan(peer=peer(peer_view_blocks=d))),
            ("peer_record_stages", 0, _lib.SgrBackwardPlan(peer=peer(peer_view_blocks=d, peer_flags=d,
                                                                     peer_record_stages=d))),
            ("peer_side_stream", 0, _lib.SgrBackwardPlan(reduce_records=d, peer=peer(**{**side, "peer_sum_tab": None}))),
            ("peer_side_stream", 0, _lib.SgrBackwardPlan(num_chunks=17, reduce_records=d, peer=peer(**side))),
            ("peer_flag_tab", 0, _lib.SgrBackwardPlan(peer=peer(peer_flag_tab=None)))):
        g = _lib.SgrGaussians(P=P, M=16, means3D=d, shs=d, scales=d, rotations=d, activations=raw)
        launches = L.sgr_launch_count()
        rc = L.sgr_rasterize_backward_staged(ctypes.byref(v), ctypes.byref(g), *([d] * 4), 1, *([d] * 10), None,
                                             ctypes.byref(plan))
        assert (rc, L.sgr_launch_count()) == (-1, launches) and field in L.sgr_last_error().decode(), field


def test_allocator_callback_exception_is_kept_for_the_caller():
    """_Arena._alloc never unwinds through the C frame: it records the exception and hands the library NULL."""
    import torch
    from sugar_b200 import _C
    arena = _C._Arena(torch.device("cpu"), 0)
    assert arena._alloc("geom", "not a size") is None and isinstance(arena.error, ValueError)
    arena.release()
