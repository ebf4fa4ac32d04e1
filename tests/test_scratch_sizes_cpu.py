"""Every scratch and workspace size query of the C ABI over several shapes (no GPU needed).

The values pin the buffer layouts: a layout change that moves a size shows up here.  Sizes an entry point rejects
give 0, never a wrapped or clamped size.  The 3M-Gaussian / 1920x1080 rows are the flagship scale."""
import ctypes

import pytest

INT32_MAX = 2 ** 31 - 1

SIZES = {
    "sgr_geometry_bytes": [((0,), 256), ((1,), 1280), ((7,), 1536), ((1000,), 96768), ((3000000,), 288000256)],
    "sgr_binning_bytes": [((0,), 1024), ((1,), 1024), ((7,), 1024), ((12345,), 247296), ((60000000,), 1200000256)],
    "sgr_image_bytes": [((1, 1), 2048), ((17, 9), 3072), ((1920, 1080), 16720384)],
    "sgr_backward_scratch_bytes": [((0,), 256), ((1,), 512), ((7,), 512), ((3000000,), 96000256)],
    "sgr_field_scratch_bytes": [((1,), 768), ((7,), 1280), ((3000000,), 288000256)],
    "sgr_normal_scratch_bytes": [((1,), 768), ((7,), 768), ((3000000,), 144000256)],
    "sgr_knn_workspace_bytes": [((1,), 2048), ((7,), 2048), ((1000,), 24320), ((3000000,), 66030336)],
    "sgr_density_grid_workspace_bytes": [((1,), 2560), ((7,), 2816), ((1000,), 76544), ((3000000,), 222030592)],
    "sgr_mcubes_scratch_bytes": [((1, 1, 1), 1536), ((3, 5, 7), 2048), ((512, 512, 512), 1208091392)],
    "sgr_decimate_scratch_bytes": [((0, 0), 1536), ((1, 0), 4352), ((3, 1), 6144), ((1000, 1999), 407552),
                                   ((1200000, 2400000), 486003968)],
    "sgr_l1_ssim_scratch_bytes": [((1, 1, 1, 1), 512), ((2, 3, 17, 9), 512), ((1, 3, 1080, 1920), 196096)],
    "sgr_mesh_nc_forward_scratch_bytes": [((0,), 0), ((1,), 512), ((7,), 512), ((3000000,), 94208)],
    "sgr_mesh_nc_backward_scratch_bytes": [((0,), 0), ((1,), 512), ((7,), 768), ((3000000,), 144000256)],
    "sgr_mesh_raster_scratch_bytes": [((0, 1, 1), 1024), ((1, 1, 1), 1536), ((7, 17, 9), 2816),
                                      ((6000000, 1920, 1080), 472612864), ((5, 0, 7), 1536)],
}

REJECTED = {
    "sgr_geometry_bytes": [(-1,)],
    "sgr_binning_bytes": [(-1,)],
    "sgr_image_bytes": [(0, 5), (-1, 5), (5, 0), (65535 * 16 + 1, 5)],
    "sgr_backward_scratch_bytes": [(-1,)],
    "sgr_field_scratch_bytes": [(0,), (-1,)],
    "sgr_normal_scratch_bytes": [(0,), (-1,)],
    "sgr_knn_workspace_bytes": [(0,), (-1,)],
    "sgr_density_grid_workspace_bytes": [(0,), (-1,)],
    "sgr_mcubes_scratch_bytes": [(0, 1, 1), (-1, 1, 1), (1025, 1024, 1024)],
    "sgr_decimate_scratch_bytes": [(-1, -1), (0, 1), ((1 << 30) + 1, 0), (8, (1 << 29) + 1)],
    "sgr_l1_ssim_scratch_bytes": [(0, 3, 5, 5), (1, -3, 5, 5), (65536, 1, 4, 4)],
    "sgr_mesh_nc_forward_scratch_bytes": [(-1,), (INT32_MAX // 4 + 1,)],
    "sgr_mesh_nc_backward_scratch_bytes": [(-1,), (INT32_MAX // 4 + 1,)],
    "sgr_mesh_raster_scratch_bytes": [(-1, 1, 1), (1, -1, 1), (1, 65536, 1), (1, 65535, 65535)],
}


def _lib():
    from sugar_b200 import _lib
    return _lib.lib


@pytest.mark.parametrize("name", sorted(SIZES))
def test_size_queries_match_the_table(name):
    fn = getattr(_lib(), name)
    got = [(args, fn(*args)) for args, _ in SIZES[name]]
    assert got == SIZES[name]


@pytest.mark.parametrize("name", sorted(REJECTED))
def test_rejected_sizes_give_zero(name):
    fn = getattr(_lib(), name)
    assert [fn(*args) for args in REJECTED[name]] == [0] * len(REJECTED[name])


def test_every_size_query_is_tabulated():
    from sugar_b200 import _lib as L
    queries = {n for n, (res, _) in L.PROTOTYPES.items() if res is ctypes.c_size_t and n.endswith("_bytes")}
    assert queries - {"sgr_struct_bytes", "sgr_peer_flag_bytes"} == set(SIZES) == set(REJECTED)
