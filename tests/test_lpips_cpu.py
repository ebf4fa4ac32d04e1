"""LPIPS and the evaluation driver without a GPU: the float64 oracle against the reference's own values
(tests/golden/make_lpips_golden.py), the weight-file readers and the packed layout the kernels take, their errors,
TF32 rounding, the scratch carve, the FLOP model, and metrics.py's command line, result file names, keys and the
model paths for every flag."""
import ctypes as C
import json
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import lpips_cases as lc  # noqa: E402
from oracle import lpips_oracle as lo  # noqa: E402
from sugar_b200 import _lib, lpips, metrics, pipeline  # noqa: E402


@pytest.fixture(scope="module")
def weights():
    return lc.make_state_dicts()


@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(HERE, "golden", "lpips_values.npz"))


def test_golden_weights_regenerate(gold, weights):
    assert int(gold["weight_seed"]) == lc.WEIGHT_SEED
    assert bytes(gold["weight_digest"]).hex() == lc.digest(*weights)


@pytest.mark.parametrize("case", lc.GOLDEN_CASES, ids=[c[0] for c in lc.GOLDEN_CASES])
def test_oracle_matches_reference(case, gold, weights):
    name, N = case[0], case[1]
    x, y = torch.from_numpy(gold[name + "_x"]), torch.from_numpy(gold[name + "_y"])
    total, taps = lo.lpips64(x, y, *weights)
    ref64, ref32 = gold[name + "_taps_f64"], gold[name + "_taps_f32"]
    # the reference's float64 run z-scores in float64, the oracle (like the float32 reference) in float32
    assert np.allclose(taps.numpy(), ref64, rtol=1e-6, atol=1e-9)
    assert np.allclose(taps.numpy(), ref32, rtol=1e-4, atol=1e-7)
    # the reference's module returns the sum over the batch
    assert np.allclose(total.sum().numpy(), gold[name + "_lpips_f64"][0], rtol=1e-6, atol=1e-9)
    # TF32 operands move the value by what the kernels' bound allows
    t32 = lo.lpips64(x, y, *weights, tf32=True)[0]
    assert bool(((t32 - total).abs() <= 5e-5 + 2e-3 * total.abs()).all())


def test_tf32_round():
    g = torch.Generator().manual_seed(0)
    v = torch.randn(10_000, generator=g) * torch.exp(torch.randn(10_000, generator=g) * 5)
    ties = torch.tensor([1 + 2 ** -11, -(1 + 2 ** -11), 1 + 3 * 2 ** -11, 1 + 2 ** -12, 0.0, -0.0])
    v = torch.cat([v, ties])
    r = lpips.tf32_round(v)
    assert torch.equal(r.double(), lo.round_tf32(v.double()))
    assert bool(((r.view(torch.int32) & 0x1FFF) == 0).all())
    assert bool(((r - v).abs() <= v.abs() * 2 ** -11).all())
    assert r[-6:].tolist() == [1 + 2 ** -10, -(1 + 2 ** -10), 1 + 2 ** -9, 1.0, 0.0, -0.0]


def test_readers_and_packed_layout(tmp_path, weights):
    vgg, lin = weights
    vp, lp = lc.write_weight_files(str(tmp_path))
    convs, lins = lpips.read_vgg16(vp), lpips.read_lin(lp)
    blob = lpips.pack_weights(convs, lins)
    assert blob.dtype == torch.float32 and blob.numel() == _lib.lib.sgr_lpips_weight_floats() == 14_716_160
    o = 0
    for l, (i, (co, ci)) in enumerate(zip(lc.CONV_INDICES, lc.CONV_SHAPES)):
        w = vgg[f"features.{i}.weight"].permute(0, 2, 3, 1).reshape(-1)
        n = co * 9 * ci
        assert torch.equal(blob[o:o + n], w if l == 0 else lpips.tf32_round(w)), l
        assert torch.equal(blob[o + n:o + n + co], vgg[f"features.{i}.bias"]), l
        o += n + co
    for t, c in enumerate(lc.TAP_CHANNELS):
        assert torch.equal(blob[o:o + c], lin[f"lin{t}.model.1.weight"].reshape(-1))
        assert o % 4 == 0   # every array 16-byte aligned in the blob
        o += c
    assert o == blob.numel()


def test_reader_errors(tmp_path, weights):
    vgg, lin = weights
    bad = dict(vgg)
    del bad["features.17.bias"]
    torch.save(bad, tmp_path / "a.pth")
    with pytest.raises(ValueError, match=r"missing key 'features\.17\.bias'"):
        lpips.read_vgg16(str(tmp_path / "a.pth"))
    bad = dict(vgg)
    bad["features.5.weight"] = torch.zeros(128, 64, 5, 5)
    torch.save(bad, tmp_path / "b.pth")
    with pytest.raises(ValueError, match=r"'features\.5\.weight' has shape \(128, 64, 5, 5\), expected "
                                         r"\(128, 64, 3, 3\)"):
        lpips.read_vgg16(str(tmp_path / "b.pth"))
    bad = dict(lin)
    bad["lin3.model.1.weight"] = torch.zeros(1, 256, 1, 1)
    torch.save(bad, tmp_path / "c.pth")
    with pytest.raises(ValueError, match=r"'lin3\.model\.1\.weight' has shape \(1, 256, 1, 1\)"):
        lpips.read_lin(str(tmp_path / "c.pth"))
    torch.save({k: v for k, v in lin.items() if not k.startswith("lin0")}, tmp_path / "d.pth")
    with pytest.raises(ValueError, match=r"missing key 'lin0\.model\.1\.weight'"):
        lpips.read_lin(str(tmp_path / "d.pth"))
    (tmp_path / "e.pth").write_bytes(b"not a checkpoint")
    with pytest.raises(ValueError, match="not a readable state dict"):
        lpips.read_vgg16(str(tmp_path / "e.pth"))


def test_net_type_and_version_refused():
    x = torch.zeros(1, 3, 16, 16)
    for kw in ({"net_type": "alex"}, {"net_type": "squeeze"}, {"net_type": "vgg", "version": "0.0"}):
        with pytest.raises(NotImplementedError):
            lpips.lpips(x, x, **kw)


def test_scratch_layout():
    N, H, W = 2, 37, 53
    size = (C.c_size_t * 8)()
    _lib.check(_lib.lib.sgr_lpips_scratch_layout(N, H, W, None, size))
    off = (C.c_size_t * 8)()
    _lib.check(_lib.lib.sgr_lpips_scratch_layout(N, H, W, 4096 + 8, off))   # an unaligned base
    assert off[7] == size[7] and all((4096 + 8 + o) % 256 == 0 for o in off[:3])
    act = 2 * N * H * W * 64 * 4
    assert off[1] - off[0] >= act and off[2] - off[1] >= act
    blocks = [(((H >> t) + 1) // 2 * (((W >> t) + 1) // 2) + 31) // 32 for t in range(5)]
    for t in range(4):
        assert off[3 + t] - off[2 + t] == 8 * N * blocks[t]
    assert off[6] + 8 * N * blocks[4] <= size[7]
    with pytest.raises(_lib.SgrError, match="H, W >= 16"):
        _lib.check(_lib.lib.sgr_lpips_scratch_layout(1, 64, 15, None, off))


def test_flop_model():
    # an independent count: each conv's output pixels x Cout x 9 Cin multiply-adds, sizes halved (floored) after
    # conv1_2, 2_2, 3_3 and 4_3
    def count(H, W):
        sizes = [(H >> s, W >> s) for s in (0, 0, 1, 1, 2, 2, 2, 3, 3, 3, 4, 4, 4)]
        return sum(2 * h * w * co * 9 * ci for (h, w), (co, ci) in zip(sizes, lc.CONV_SHAPES))
    for H, W in ((1080, 1920), (800, 800), (37, 53)):
        assert lpips.conv_flops(H, W) == count(H, W)
    assert lpips.pair_flops(1080, 1920) == 2 * count(1080, 1920)
    assert round(lpips.conv_flops(1080, 1920) / 2e9) == 634          # GMAC per image
    assert abs(lpips.pair_flops(1080, 1920) / 1e12 - 2.535) < 1e-3    # TFLOP per pair


# ------------------------------------------------------------------------------------------------------ metrics.py
def test_cli_defaults_and_presets():
    a = metrics.parse_args(["--scene_config", "s.json", "-r", "sdf"])
    assert (a.iteration_to_load, a.estimation_factor, a.surface_level, a.n_vertices_in_mesh, a.gaussians_per_triangle,
            a.refinement_iterations, a.gpu) == (7000, 0.2, 0.3, 1_000_000, 1, 15_000, 0)
    assert not (a.evaluate_vanilla or a.use_uv_texture or a.use_diffuse_color_only or a.use_poisson_center or
                a.use_marching_cubes)
    assert a.compute_lpips is True and a.output_dir == "./output"
    assert a.lpips_weights_dir == os.path.join(".", "lpipsPyTorch", "weights", "checkpoints")
    a = metrics.parse_args(["--scene_config", "s.json", "-r", "density", "--low_poly", "True", "-f", "123"])
    assert (a.n_vertices_in_mesh, a.gaussians_per_triangle, a.refinement_iterations) == (200_000, 6, 123)
    a = metrics.parse_args(["--scene_config", "s.json", "-r", "sdf", "--low_poly", "True", "--high_poly", "yes",
                            "--refinement_time", "medium"])
    assert (a.n_vertices_in_mesh, a.gaussians_per_triangle, a.refinement_iterations) == (1_000_000, 1, 7_000)
    for t, f in (("short", 2000), ("long", 15_000), ("other", 15_000)):
        assert metrics.parse_args(["--scene_config", "s", "-r", "sdf", "--refinement_time", t]).refinement_iterations == f
    a = metrics.parse_args(["--scene_config", "s", "-r", "sdf", "--compute_lpips", "False", "--evaluate_vanilla", "1"])
    assert a.compute_lpips is False and a.evaluate_vanilla is True
    with pytest.raises(SystemExit):
        metrics.parse_args(["--scene_config", "s", "-r", "nerf"])


def test_result_file_names_and_keys():
    f = metrics.result_file_name
    assert f("sdf") == "results_sdf02_normal02.json"
    assert f("density", 0.5) == "results_density05_normal02.json"
    assert f("sdf", use_uv_texture=True, use_diffuse_color_only=True) == "results_sdf02_normal02_uvtexture.json"
    assert f("sdf", use_diffuse_color_only=True, use_marching_cubes=True) == "results_sdf02_normal02_diffuseonly.json"
    assert f("sdf", use_poisson_center=True, use_marching_cubes=True) == "results_sdf02_normal02_poissoncenter.json"
    assert f("sdf", use_marching_cubes=True) == "results_sdf02_normal02_marchingcubes.json"
    assert metrics.sugar_key(0.3, 1_000_000, 15_000) == "sugar_03_1000000_15000"
    assert metrics.sugar_key(0.25, 200_000, 2000) == "sugar_025_200000_2000"


def test_model_paths_for_every_flag():
    p = metrics.model_paths("garden", "sdf", output_dir="out")
    mesh = "sugarmesh_3Dgs7000_sdfestim02_sdfnorm02_level03_decim1000000"
    fine = "sugarfine_3Dgs7000_sdfestim02_sdfnorm02_level03_decim1000000_normalconsistency01_gaussperface1"
    assert p.mesh == f"out/coarse_mesh/garden/{mesh}.ply"
    assert p.refined == f"out/refined/garden/{fine}/15000.pt"
    assert p.textured_mesh == f"out/refined_mesh/garden/{fine}.obj"
    # where they coincide, the pipeline's own names
    for kw in (dict(), dict(surface_level=0.1, n_vertices_in_mesh=200_000, gaussians_per_triangle=6,
                            refinement_iterations=2000, iteration_to_load=30_000)):
        q = metrics.model_paths("garden", "density", output_dir="out", **kw)
        o = pipeline.output_paths("data/garden/", "density", output_dir="out", **kw)
        assert (q.mesh, q.refined, q.textured_mesh) == (o.mesh, o.refined, o.textured_mesh)
    mc = metrics.model_paths("garden", "sdf", use_marching_cubes=True, output_dir="out")
    assert mc.mesh == "out/coarse_mesh/garden/sugarmesh_3Dgs7000_sdfestim02_sdfnorm02marchingcubes_level03_decim1000000.ply"
    assert mc.refined == ("out/refined/garden/sugarfine_3Dgs7000_sdfestim02_sdfnorm02marchingcubes_level03_decim1000000"
                          "_normalconsistency01_gaussperface1/15000.pt")
    assert mc.textured_mesh == p.textured_mesh
    pc = metrics.model_paths("garden", "sdf", use_poisson_center=True, use_marching_cubes=False, output_dir="out",
                             estimation_factor=0.5, gaussians_per_triangle=3)
    assert pc.mesh == "out/coarse_mesh/garden/sugarmesh_3Dgs7000_sdfestim05_sdfnorm02_poissoncenters_decim1000000.ply"
    assert pc.refined == ("out/refined/garden/sugarfine_3Dgs7000_sdfestim05_sdfnorm02_poissoncenters_decim1000000"
                          "_normalconsistency01_gaussperface3/15000.pt")
    assert pc.textured_mesh == ("out/refined_mesh/garden/sugarfine_3Dgs7000_sdfestim05_sdfnorm02_level03_decim1000000"
                                "_normalconsistency01_gaussperface3.obj")
    # marching cubes wins over the Poisson centres, as in the reference's if / elif
    both = metrics.model_paths("garden", "sdf", use_poisson_center=True, use_marching_cubes=True, output_dir="out")
    assert both.mesh == mc.mesh


def test_missing_lpips_weights_named_before_rendering(tmp_path):
    cfg = tmp_path / "scenes.json"
    cfg.write_text(json.dumps({str(tmp_path / "no_scene"): str(tmp_path / "no_gs")}))
    (tmp_path / "w").mkdir()
    lc.write_weight_files(str(tmp_path / "w"))
    os.remove(tmp_path / "w" / "vgg.pth")
    with pytest.raises(FileNotFoundError) as e:
        metrics.main(["--scene_config", str(cfg), "-r", "sdf", "--lpips_weights_dir", str(tmp_path / "w"),
                      "--output_dir", str(tmp_path / "out")])
    assert "vgg16-397923af.pth" in str(e.value) and "vgg.pth" in str(e.value) and "missing" in str(e.value)
    assert not (tmp_path / "out").exists()
