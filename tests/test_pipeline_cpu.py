"""The pipeline's CPU side: the refined model built from a mesh against the reference constructor's goldens
(tests/golden/make_pipeline_golden.py), SuGaR checkpoints both ways, the mesh PLY reader on write_ply's and open3d-style
files, the reference's output names and train.py's command line."""
import math
import os
import struct
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from sugar_b200 import checkpoint, mcubes, pipeline, train  # noqa: E402

GOLDEN = os.path.join(HERE, "golden")


def _load(name):
    return checkpoint.load_file(os.path.join(GOLDEN, name), "cpu")


def _same(a, b):
    """Same dtype, shape and bits."""
    assert a.dtype == b.dtype and a.shape == b.shape, (a.dtype, b.dtype, a.shape, b.shape)
    assert torch.equal(a.view(torch.uint8) if a.dim() else a.reshape(1).view(torch.uint8),
                       b.view(torch.uint8) if b.dim() else b.reshape(1).view(torch.uint8))


def _same_state(sd, ref):
    assert list(sd.keys()) == list(ref.keys())
    for k in ref:
        _same(sd[k].detach().cpu(), ref[k])


# ------------------------------------------------------------------------------------------- the model from a mesh
@pytest.mark.parametrize("name", ["pipeline_bound_n1.pt", "pipeline_bound_n3.pt", "pipeline_bound_n4.pt",
                                  "pipeline_bound_n6.pt", "pipeline_bound_degenerate_n4.pt"])
def test_init_refined_from_mesh_equals_the_reference_constructor(name):
    g = _load(name)
    inp, ref = g["inputs"], g["state_dict"]
    n = ref["_scales"].shape[0] // ref["_surface_mesh_faces"].shape[0]
    colors = (inp["vertex_colors_u8"].double() / 255.0).float()
    raw, mesh = train.init_refined_from_mesh(inp["verts"], inp["faces"], colors, n, inp["extent"] / 1_000_000)
    assert mesh.faces.dtype == torch.int64 and mesh.n == n and mesh.topology is None
    _same_state(checkpoint.state_dict(raw, mesh), ref)
    assert all(t.requires_grad and t.is_leaf for t in raw.values())
    if "degenerate" in name:
        assert float(raw["scales"][0, 0].detach()) == float(torch.tensor(1e-7).log())


@pytest.mark.parametrize("n", [0, 2, 5, 7])
def test_init_refined_from_mesh_rejects_other_counts(n):
    with pytest.raises(ValueError, match="1, 3, 4 or 6"):
        train.init_refined_from_mesh(torch.rand(3, 3), torch.tensor([[0, 1, 2]]), torch.rand(3, 3), n, 1e-6)


# ------------------------------------------------------------------------------------------------- checkpoints
def test_reference_checkpoint_loads_and_saves_back_identically(tmp_path):
    path = os.path.join(GOLDEN, "pipeline_save_model_bound.pt")
    ref = checkpoint.load_file(path, "cpu")
    raw, mesh, extra = checkpoint.load_checkpoint(path, "cpu")
    assert mesh.n == 3 and mesh.faces.dtype == torch.int64 and set(raw) == {"verts", "sh_dc", "sh_rest", "densities",
                                                                          "scales", "quaternions"}
    assert extra["train_losses"] == [0.25, 0.125] and extra["epoch"] == 2 and extra["iteration"] == 2
    out = str(tmp_path / "again.pt")
    checkpoint.save_checkpoint(out, raw, mesh, **extra)
    back = checkpoint.load_file(out, "cpu")
    assert list(back.keys()) == list(ref.keys())
    _same_state(back["state_dict"], ref["state_dict"])
    assert back["optimizer_state_dict"]["param_groups"] == ref["optimizer_state_dict"]["param_groups"]
    for k, s in ref["optimizer_state_dict"]["state"].items():
        for name, t in s.items():
            _same(back["optimizer_state_dict"]["state"][k][name], t)


def test_coarse_round_trip_is_exact(tmp_path):
    g = _load("pipeline_unbound.pt")
    ref, gs = g["state_dict"], g["inputs"]
    raw = dict(points=gs["xyz"], densities=gs["opacity"], scales=gs["scaling"], quaternions=gs["rotation"],
               sh_dc=gs["features_dc"], sh_rest=gs["features_rest"])
    _same_state(checkpoint.state_dict(raw), ref)
    path = str(tmp_path / "15000.pt")
    checkpoint.save_checkpoint(path, raw, train_losses=[1.0], epoch=1, iteration=15000)
    back, mesh, extra = checkpoint.load_checkpoint(path, "cpu")
    assert mesh is None and extra == {"train_losses": [1.0], "epoch": 1, "iteration": 15000}
    _same_state(checkpoint.state_dict(back), ref)


def test_bound_round_trip_is_exact(tmp_path):
    g = _load("pipeline_bound_n6.pt")
    inp = g["inputs"]
    raw, mesh = train.init_refined_from_mesh(inp["verts"], inp["faces"], torch.rand(12, 3), 6, 3.7e-6)
    path = str(tmp_path / "m.pt")
    checkpoint.save_checkpoint(path, raw, mesh)
    sd = checkpoint.load_file(path, "cpu")["state_dict"]
    assert sd["_surface_mesh_faces"].dtype == torch.int32 and sd["surface_mesh_thickness"].dtype == torch.float32
    back, mesh2, _ = checkpoint.load_checkpoint(path, "cpu")
    assert mesh2.n == 6 and torch.equal(mesh2.faces, mesh.faces) and mesh2.thickness == mesh.thickness
    assert torch.equal(mesh2.bary, mesh.bary)
    _same_state(checkpoint.state_dict(back, mesh2), checkpoint.state_dict(raw, mesh))


def test_optimizer_state_survives_save_and_load(tmp_path):
    """SugarOptimizer's state (torch's Adam layout) through a checkpoint file, without a GPU: the state dict is built
    by hand in the layout SugarOptimizer.state_dict() gives, and the reference optimizer's own file loads."""
    ref = _load("pipeline_save_model_bound.pt")["optimizer_state_dict"]
    assert [g["name"] for g in ref["param_groups"]] == ["points", "sh_coordinates_dc", "sh_coordinates_rest",
                                                        "all_densities", "scales", "quaternions"]
    from sugar_b200.optim import group_table
    assert [name for name, _, _ in group_table(1.0, bound=True)] == [g["name"] for g in ref["param_groups"]]
    g = _load("pipeline_bound_n3.pt")
    raw, mesh = train.init_refined_from_mesh(g["inputs"]["verts"], g["inputs"]["faces"], torch.rand(12, 3), 3, 1e-6)
    # a torch Adam over the same groups stands in for SugarOptimizer (CUDA only) to make the state
    opt = torch.optim.Adam([{"params": [raw[k]], "lr": lr, "name": name} for name, k, lr in group_table(0.5, True)],
                           lr=0.0, eps=1e-15)
    for p in raw.values():
        p.grad = torch.ones_like(p)
    opt.step()
    path = str(tmp_path / "o.pt")
    checkpoint.save_checkpoint(path, raw, mesh, optimizer_state_dict=opt.state_dict())
    back, _, extra = checkpoint.load_checkpoint(path, "cpu")
    opt2 = torch.optim.Adam([{"params": [back[k]], "lr": 0.0, "name": name} for name, k, _ in group_table(1, True)],
                            lr=0.0, eps=1e-15)
    opt2.load_state_dict(extra["optimizer_state_dict"])
    for p, q in zip((raw[k] for _, k, _ in group_table(1, True)), (back[k] for _, k, _ in group_table(1, True))):
        for name in ("exp_avg", "exp_avg_sq", "step"):
            assert torch.equal(opt.state[p][name], opt2.state[q][name])
    assert [g["lr"] for g in opt2.param_groups] == [g["lr"] for g in opt.param_groups]


# ------------------------------------------------------------------------------------------------------ mesh PLY
def test_read_mesh_ply_inverts_write_ply(tmp_path):
    g = torch.Generator().manual_seed(2)
    v = torch.randn(30, 3, generator=g)
    f = torch.randint(0, 30, (50, 3), generator=g)
    c = torch.rand(30, 3, generator=g)
    n = torch.nn.functional.normalize(torch.randn(30, 3, generator=g), dim=-1)
    for colors, normals in ((c, n), (c, None), (None, n), (None, None)):
        path = str(tmp_path / "m.ply")
        mcubes.write_ply(path, v, f, colors, normals)
        m = mcubes.read_mesh_ply(path)
        assert m["verts"].dtype == torch.float32 and torch.equal(m["verts"], v)
        assert m["faces"].dtype == torch.int64 and torch.equal(m["faces"], f)
        if colors is None:
            assert m["colors"] is None
        else:
            u8 = np.round(np.clip(c.double().numpy(), 0, 1) * 255).astype(np.uint8)
            assert torch.equal(m["colors"], torch.from_numpy((u8 / 255.0).astype(np.float32)))
        assert (m["normals"] is None) == (normals is None)
        if normals is not None:
            assert torch.equal(m["normals"], normals)


def _open3d_style(path, verts, faces, vtype="double", itype="int", normals=None, colors=None, fmt="binary_little_endian",
                  count=3, cut=0):
    """A PLY laid out as open3d's write_triangle_mesh writes one."""
    fields = [(a, "<f8" if vtype == "double" else "<f4") for a in "xyz"]
    if normals is not None:
        fields += [(a, "<f8" if vtype == "double" else "<f4") for a in ("nx", "ny", "nz")]
    if colors is not None:
        fields += [(a, "u1") for a in ("red", "green", "blue")]
    rec = np.empty(len(verts), fields)
    for i, a in enumerate("xyz"):
        rec[a] = verts[:, i]
    if normals is not None:
        for i, a in enumerate(("nx", "ny", "nz")):
            rec[a] = normals[:, i]
    if colors is not None:
        for i, a in enumerate(("red", "green", "blue")):
            rec[a] = colors[:, i]
    head = ["ply", f"format {fmt} 1.0", "comment Created by Open3D", f"element vertex {len(verts)}"]
    head += [f"property {'double' if t == '<f8' else 'float' if t == '<f4' else 'uchar'} {a}" for a, t in fields]
    head += [f"element face {len(faces)}", f"property list uchar {itype} vertex_indices", "end_header"]
    body = rec.tobytes()
    for fc in faces:
        ids = list(fc) + [fc[0]] * (count - 3)
        body += struct.pack("<B" + ("i" if itype == "int" else "I") * count, count, *ids)
    with open(path, "wb") as fh:
        fh.write(("\n".join(head) + "\n").encode() + (body[:-cut] if cut else body))


@pytest.mark.parametrize("vtype", ["double", "float"])
@pytest.mark.parametrize("itype", ["int", "uint"])
@pytest.mark.parametrize("with_normals,with_colors", [(True, True), (False, True), (True, False), (False, False)])
def test_read_mesh_ply_reads_open3d_files(tmp_path, vtype, itype, with_normals, with_colors):
    rng = np.random.default_rng(4)
    v = rng.standard_normal((9, 3))
    f = rng.integers(0, 9, (7, 3))
    nr = rng.standard_normal((9, 3)) if with_normals else None
    c = rng.integers(0, 256, (9, 3), dtype=np.uint8) if with_colors else None
    path = str(tmp_path / "o3d.ply")
    _open3d_style(path, v, f, vtype, itype, nr, c)
    m = mcubes.read_mesh_ply(path)
    assert torch.equal(m["verts"], torch.from_numpy(v.astype(np.float32 if vtype == "float" else np.float64)
                                                    .astype(np.float32)))
    assert torch.equal(m["faces"], torch.from_numpy(f.astype(np.int64)))
    if with_colors:
        assert torch.equal(m["colors"], torch.from_numpy((c / 255.0).astype(np.float32)))
    else:
        assert m["colors"] is None
    assert (m["normals"] is None) == (not with_normals)


@pytest.mark.parametrize("kind,match", [("ascii", "binary_little_endian"), ("big", "binary_little_endian"),
                                        ("quad", "triangles only"), ("short", "bytes"),
                                        ("short_vertices", "bytes"), ("bad_id", "outside")])
def test_read_mesh_ply_rejects(tmp_path, kind, match):
    v = np.zeros((4, 3))
    f = np.array([[0, 1, 2], [1, 2, 3]])
    path = str(tmp_path / "bad.ply")
    if kind == "ascii":
        _open3d_style(path, v, f, fmt="ascii")
    elif kind == "big":
        _open3d_style(path, v, f, fmt="binary_big_endian")
    elif kind == "quad":
        _open3d_style(path, v, f, count=4)
    elif kind == "short":
        _open3d_style(path, v, f, cut=5)
    elif kind == "short_vertices":
        _open3d_style(path, v, np.zeros((0, 3), np.int64), cut=10)
    else:
        _open3d_style(path, v, np.array([[0, 1, 4]]))
    with pytest.raises(ValueError, match=match):
        mcubes.read_mesh_ply(path)


# ------------------------------------------------------------------------------------------------------ names
def test_output_names_sdf_defaults():
    p = pipeline.output_paths("data/garden", "sdf")
    assert p.coarse == "./output/coarse/garden/sugarcoarse_3Dgs7000_sdfestim02_sdfnorm02/15000.pt"
    assert p.mesh == "./output/coarse_mesh/garden/sugarmesh_3Dgs7000_sdfestim02_sdfnorm02_level03_decim1000000.ply"
    assert p.refined == ("./output/refined/garden/sugarfine_3Dgs7000_sdfestim02_sdfnorm02_level03_decim1000000_"
                         "normalconsistency01_gaussperface1/15000.pt")
    assert p.refined_ply == ("./output/refined_ply/garden/sugarfine_3Dgs7000_sdfestim02_sdfnorm02_level03_"
                             "decim1000000_normalconsistency01_gaussperface1.ply")
    assert p.textured_mesh == ("./output/refined_mesh/garden/sugarfine_3Dgs7000_sdfestim02_sdfnorm02_level03_"
                               "decim1000000_normalconsistency01_gaussperface1.obj")


def test_output_names_density_low_poly_postprocessed():
    p = pipeline.output_paths("data/garden/", "density", surface_level=0.5, n_vertices_in_mesh=200000,
                              gaussians_per_triangle=6, refinement_iterations=2000, postprocess_mesh=True,
                              output_dir="out")
    assert p.coarse == "out/coarse/garden/sugarcoarse_3Dgs7000_densityestim02_sdfnorm02/15000.pt"
    assert p.mesh == "out/coarse_mesh/garden/sugarmesh_3Dgs7000_densityestim02_sdfnorm02_level05_decim200000.ply"
    assert p.refined == ("out/refined/garden/sugarfine_3Dgs7000_densityestim02_sdfnorm02_level05_decim200000_"
                         "normalconsistency01_gaussperface6/2000.pt")
    assert p.refined_ply == ("out/refined_ply/garden/sugarfine_3Dgs7000_densityestim02_sdfnorm02_level05_"
                             "decim200000_normalconsistency01_gaussperface6.ply")
    assert p.textured_mesh == ("out/refined_mesh/garden/sugarfine_3Dgs7000_densityestim02_sdfnorm02_level05_"
                               "decim200000_normalconsistency01_gaussperface6_postprocessed.obj")


def test_output_names_other_combinations():
    p = pipeline.output_paths("/abs/scenes/kitchen", "sdf", iteration_to_load=30000, surface_level=0.3,
                              n_vertices_in_mesh=200000, gaussians_per_triangle=1)
    assert p.mesh == "./output/coarse_mesh/kitchen/sugarmesh_3Dgs30000_sdfestim02_sdfnorm02_level03_decim200000.ply"
    assert p.textured_mesh.endswith("/sugarfine_3Dgs30000_sdfestim02_sdfnorm02_level03_decim200000_"
                                    "normalconsistency01_gaussperface1.obj")
    p = pipeline.output_paths("kitchen", "density", surface_level=0.5, n_vertices_in_mesh=1000000,
                              gaussians_per_triangle=6)
    assert p.refined == ("./output/refined/kitchen/sugarfine_3Dgs7000_densityestim02_sdfnorm02_level05_"
                         "decim1000000_normalconsistency01_gaussperface6/15000.pt")
    assert pipeline.scene_name("a/b/") == "b" and pipeline.scene_name("a/b") == "b"
    with pytest.raises(ValueError):
        pipeline.output_paths("a", "rgb")


# ------------------------------------------------------------------------------------------------------ command line
BASE = ["-s", "data/garden", "-c", "gs/garden", "-r", "sdf"]


def test_command_line_defaults():
    kw = pipeline.parse_args(BASE)
    assert kw == dict(scene_path="data/garden", checkpoint_path="gs/garden", regularization_type="sdf",
                      iteration_to_load=7000, surface_level=0.3, n_vertices_in_mesh=1_000_000, center_bbox=True,
                      gaussians_per_triangle=1, refinement_iterations=15_000, export_uv_textured_mesh=True,
                      square_size=10, postprocess_mesh=False, postprocess_density_threshold=0.1,
                      postprocess_iterations=5, export_ply=True, eval=True, gpu=0, output_dir="./output")
    import inspect
    assert set(kw) <= set(inspect.signature(pipeline.run).parameters)


def test_command_line_flags_and_presets():
    kw = pipeline.parse_args(BASE + ["-i", "30000", "-l", "0.5", "-v", "300000", "-g", "4", "-f", "900", "-t",
                                     "False", "--square_size", "8", "--postprocess_mesh", "True",
                                     "--postprocess_density_threshold", "0.2", "--postprocess_iterations", "3",
                                     "--export_ply", "no", "--eval", "False", "--gpu", "1", "--center_bbox", "f",
                                     "--output_dir", "out"])
    assert kw["iteration_to_load"] == 30000 and kw["surface_level"] == 0.5 and kw["n_vertices_in_mesh"] == 300000
    assert kw["gaussians_per_triangle"] == 4 and kw["refinement_iterations"] == 900
    assert kw["export_uv_textured_mesh"] is False and kw["square_size"] == 8 and kw["postprocess_mesh"] is True
    assert kw["postprocess_density_threshold"] == 0.2 and kw["postprocess_iterations"] == 3
    assert kw["export_ply"] is False and kw["eval"] is False and kw["gpu"] == 1 and kw["center_bbox"] is False
    assert kw["output_dir"] == "out"
    kw = pipeline.parse_args(BASE + ["--low_poly", "True"])
    assert (kw["n_vertices_in_mesh"], kw["gaussians_per_triangle"]) == (200_000, 6)
    kw = pipeline.parse_args(BASE + ["-v", "5", "-g", "3", "--high_poly", "True"])
    assert (kw["n_vertices_in_mesh"], kw["gaussians_per_triangle"]) == (1_000_000, 1)
    kw = pipeline.parse_args(BASE + ["--low_poly", "True", "--high_poly", "True"])   # train.py applies high_poly last
    assert (kw["n_vertices_in_mesh"], kw["gaussians_per_triangle"]) == (1_000_000, 1)
    for t, n in (("short", 2000), ("medium", 7000), ("long", 15000)):
        assert pipeline.parse_args(BASE + ["-f", "5", "--refinement_time", t])["refinement_iterations"] == n


@pytest.mark.parametrize("extra,word", [(["-b", "(0,0,0)"], "bboxmin"), (["-B", "1,1,1"], "bboxmax"),
                                        (["--white_background", "True"], "white_background")])
def test_command_line_refuses(capsys, extra, word):
    with pytest.raises(SystemExit):
        pipeline.parse_args(BASE + extra)
    assert word in capsys.readouterr().err
    pipeline.parse_args(BASE + ["--white_background", "False"])


def test_extraction_keeps_strength_above_one_half_strictly():
    """The extraction keeps strength > 0.5; the coarse trainer's prune removes strength < 0.5.  A Gaussian at exactly
    0.5 (density logit 0) survives the prune and is left out of the mesh."""
    d = torch.tensor([[-1e-3], [0.0], [1e-3], [4.0], [-4.0]])
    assert pipeline.extraction_mask(d).tolist() == [False, False, True, True, False]
    pruned = torch.sigmoid(d).view(-1) < 0.5          # train.train_coarse's prune rule at prune_threshold 0.5
    assert pruned.tolist() == [True, False, False, False, True]
