"""CPU checks of bench.py's host-side pieces: the algorithmic-byte model (DESIGN.md section 3 / SURVEY.md 8d),
the nvidia-smi clock-sample parser and its load-window filter, the peak loader.  No GPU, no timing."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def test_algorithmic_bytes_model_headline():
    import bench
    P, V, R, W, H = 3_000_000, 2_509_989, 11_414_139, 1920, 1080
    b = bench.algorithmic_bytes(P, V, R, W, H, 16, 3)
    assert set(b) == {"preprocess", "tile_scan", "scatter", "tile_sort_smem", "tile_sort_global", "blend_forward",
                      "blend_backward", "preprocess_backward"}
    # the GB/s bench.py reports (bytes / ms) come from exactly these
    assert b["blend_backward"] == R * 40 + W * H * 20 + V * 72 == 678_756_768
    assert b["preprocess"] == P * (44 + 192) + P * 12 + V * 56 + R * 4
    assert b["preprocess_backward"] == V * (80 + 192) + P * (92 + 192)
    # colours_precomp-style degree 0 reads 12 B of SH per Gaussian
    assert bench.algorithmic_bytes(P, V, R, W, H, 16, 0)["preprocess"] == P * (44 + 12) + P * 12 + V * 56 + R * 4


def test_clock_sampler_parses_rows_and_filters_the_load_window():
    import bench
    s = bench.ClockSampler.__new__(bench.ClockSampler)

    class P:
        def terminate(self):
            pass
    s.proc = P()
    row = "0, {sm}, 1965, 700.1, 0x0000000000000004, Not Active, Not Active, Not Active, {cap}"
    s.rows = [(0.5, row.format(sm=1200, cap="Not Active")),      # before the load window: ignored
              (1.2, row.format(sm=1965, cap="Not Active")),
              (1.6, row.format(sm=1950, cap="Active")),          # inside the timed region
              (2.1, row.format(sm=1965, cap="Not Active")),
              (2.2, "garbage"),
              (9.0, row.format(sm=300, cap="Not Active"))]       # after the window: ignored
    out = s.stop(load=(1.0, 2.5), timed=(1.5, 1.8))
    assert out["samples"] == 3 and out["samples_in_timed_region"] == 1
    assert out["sm_mhz"] == 1965.0 and out["sm_max_mhz"] == 1965.0
    assert out["reasons"] == ["sw_power_cap"]
    s.proc = None
    assert s.stop()["sm_mhz"] is None


def test_load_peaks_returns_a_positive_hbm_peak():
    import bench
    peak, src = bench.load_peaks()
    assert peak > 1000 and isinstance(src, str)


def test_reference_arm_helpers_do_not_map_the_product_library():
    """bench.py --impl reference must not import sugar_b200 (which maps libsugar_b200.so): the scene generator is
    loaded by path and tests/helpers.py stays import-free of the package at module level."""
    import subprocess
    code = ("import sys; sys.path.insert(0, %r); sys.path.insert(0, %r + '/tests'); import bench, helpers; "
            "sc = bench.load_scenes().make_scene(100, 32, 16, seed=0); assert sc.means3D.shape == (100, 3); "
            "assert not any(m == 'sugar_b200' or m.startswith('sugar_b200.') for m in sys.modules), "
            "[m for m in sys.modules if 'sugar' in m]; "
            "maps = open('/proc/self/maps').read(); assert 'libsugar_b200' not in maps") % (ROOT, ROOT)
    subprocess.run([sys.executable, "-c", code], check=True, timeout=120)


def test_cpu_sample_worker_and_factor_mode_bytes():
    import bench
    dt = bench._cpu_sample((0, 300, 48, 32, 3))
    assert 0 < dt < 30
    P, V, R, W, H = 1000, 800, 3000, 64, 64
    full = bench.algorithmic_bytes(P, V, R, W, H, 16, 3)["preprocess_backward"]
    fac = bench.algorithmic_bytes(P, V, R, W, H, 16, 3, sh_written=False)["preprocess_backward"]
    assert full - fac == P * 192
    assert bench.KERNEL_BOUND["blend_backward"] == "fp32-issue" and bench.KERNEL_BOUND["preprocess"] == "hbm"
