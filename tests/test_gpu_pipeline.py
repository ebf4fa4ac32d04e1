"""The whole pipeline on the GPU: a COLMAP-text scene of a closed object rendered by this package's rasterizer, a
perturbed 3DGS checkpoint of it, then pipeline.run with short schedules.  Every file must exist under the reference's
name and load back through this package's readers; the coarse checkpoint must hold the trained model bit for bit; the
mesh must lie near the true surface; refinement must raise the train views' PSNR; the textured mesh must render the
object; and the refined model's start and the texture must come back bit for bit from the files alone."""
import math
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import dataset_cases as dc  # noqa: E402
from sugar_b200 import checkpoint, dataset, gsply, mcubes, meshbind, objfile, pipeline, steps, texture, train  # noqa

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
RADIUS = 1.0                 # the object: a sphere of Gaussian disks
W, H, FX = 160, 120, 150.0
FACES = 3000                 # -v: the decimation target of each part
COARSE_LAST = 7299           # 300 coarse iterations from 7000
REFINE_ITERS = 300
# Bounds set from the first run on one H100 80GB HBM3 (DESIGN.md section 16), measured value -> bound:
SURFACE_MEDIAN, SURFACE_Q90 = 0.03, 0.04   # | |v| - R | / R of the foreground vertices: 0.0145, 0.0186 -> about 2x
REFINED_PSNR = 28.0                          # refined model over the train views: 13.2 -> 32.8 dB, bound 4.8 dB below
TEXTURE_PSNR = 20.0                          # textured mesh against the ground truth, mean over train views: 22.9 dB


def sphere_model(P=20_000, seed=0):
    """Flat Gaussians tangent to the sphere, coloured by position: the surface-shaped model the images come from."""
    i = torch.arange(P, dtype=torch.float64) + 0.5
    z = 1 - 2 * i / P
    phi = math.pi * (1 + 5 ** 0.5) * i
    r = torch.sqrt(1 - z * z)
    n = torch.stack([r * torch.cos(phi), r * torch.sin(phi), z], 1).float()
    q = torch.nn.functional.normalize(torch.stack([1 + n[:, 2], -n[:, 1], n[:, 0], torch.zeros(P)], 1), dim=-1)
    rgb = 0.5 + 0.35 * torch.stack([torch.sin(3 * n[:, 0]), torch.cos(2 * n[:, 1]), torch.sin(4 * n[:, 2] + 1)], 1)
    raw = dict(points=n * RADIUS, sh_dc=((rgb - 0.5) / train.SH_C0)[:, None], sh_rest=torch.zeros(P, 15, 3),
               densities=torch.full((P, 1), 3.0), scales=torch.log(torch.tensor([[0.035, 0.035, 0.004]])).repeat(P, 1),
               quaternions=q)
    return {k: v.to(DEV).contiguous() for k, v in raw.items()}


def render(raw, cam):
    with torch.no_grad():
        return steps.render(steps.ours_ops(), steps.activate(raw), cam, torch.zeros(3, device=DEV), sh_deg=0)[0]


def psnr(a, b):
    return float(-10 * torch.log10(((a.clamp(0, 1) - b) ** 2).mean()))


@pytest.fixture(scope="module")
def scene(tmp_path_factory):
    """A COLMAP-text scene of 24 views, the ground truth the package's renders, and a 3DGS output directory holding
    the perturbed model at iteration 7000 and cameras.json."""
    root = tmp_path_factory.mktemp("pipeline")
    scene_dir, gs_dir = str(root / "scenes" / "sphere"), str(root / "gs" / "sphere")
    os.makedirs(os.path.join(scene_dir, "images"))
    truth = sphere_model()
    poses = dc.ring_poses(12, radius=4.0, height=1.6, seed=1) + dc.ring_poses(12, radius=4.0, height=-1.6, seed=2)
    cams, images = [], []
    for i, (Rwc, t) in enumerate(poses):
        name = f"view_{i:02d}"
        cam = dataset.make_camera(Rwc.T, t, dataset.focal2fov(FX, W), dataset.focal2fov(FX, H), W, H, device=DEV,
                                  name=name, orig_width=W, orig_height=H)
        px = (render(truth, cam).clamp(0, 1) * 255.0).round().to(torch.uint8).permute(1, 2, 0).cpu().numpy()
        dc.write_png(os.path.join(scene_dir, "images", name + ".png"), px)
        images.append((i + 1, dc.rotmat2qvec(Rwc), t, 1, name + ".png"))
        cams.append(cam)
    pts = truth["points"][::50].cpu().double().numpy()
    dc.write_colmap(os.path.join(scene_dir, "sparse", "0"), [(1, "PINHOLE", W, H, [FX, FX, W / 2, H / 2])], images,
                    (pts, np.full((len(pts), 3), 128, np.uint8)), binary=False)
    os.makedirs(gs_dir)
    dataset.write_cameras_json(os.path.join(gs_dir, "cameras.json"), cams)
    g = torch.Generator(device=DEV).manual_seed(7)
    noisy = {k: v.clone() for k, v in truth.items()}
    noisy["points"] += 0.01 * torch.randn(noisy["points"].shape, device=DEV, generator=g)
    noisy["scales"] += 0.15 * torch.randn(noisy["scales"].shape, device=DEV, generator=g)
    noisy["sh_dc"] += 0.3 * torch.randn(noisy["sh_dc"].shape, device=DEV, generator=g)
    noisy["densities"] = torch.full_like(noisy["densities"], 1.0)
    gsply.save_gaussians_ply(os.path.join(gs_dir, "point_cloud", "iteration_7000", "point_cloud.ply"), noisy)
    out_dir = str(root / "output")
    out = pipeline.run(
        scene_dir, gs_dir, "sdf", n_vertices_in_mesh=FACES, refinement_iterations=REFINE_ITERS, output_dir=out_dir,
        coarse_kwargs=dict(num_iterations=COARSE_LAST, regularize_from=7000, entropy_window=(7000, 7100),
                           prune_at=(7100,), sdf_from=7100, reset_neighbors_every=100, n_samples=100_000),
        surface_kwargs=dict(n_total_points=200_000), poisson_kwargs=dict(poisson_depth=7))
    return dict(scene=scene_dir, gs=gs_dir, out_dir=out_dir, out=out)


def test_files_at_the_reference_names_and_readable(scene):
    out = scene["out"]
    names = pipeline.output_paths(scene["scene"], "sdf", 7000, 0.3, FACES, 1, REFINE_ITERS,
                                  output_dir=scene["out_dir"], coarse_iterations=COARSE_LAST)
    assert out.coarse == names.coarse and out.mesh == names.mesh and out.refined == names.refined
    assert out.refined_ply == names.refined_ply and out.textured_mesh == names.textured_mesh
    assert names.mesh.endswith("/coarse_mesh/sphere/sugarmesh_3Dgs7000_sdfestim02_sdfnorm02_level03_decim3000.ply")
    for p in (names.coarse, names.mesh, names.refined, names.refined_ply, names.textured_mesh):
        assert os.path.isfile(p), p
    raw, mesh, extra = checkpoint.load_checkpoint(out.coarse, DEV)
    assert mesh is None and extra["iteration"] == COARSE_LAST and len(extra["train_losses"]) == 6   # 7050 ... 7250
    assert all(math.isfinite(x) for x in extra["train_losses"])
    n_views = len(dataset.load_gs_cameras(scene["scene"], scene["gs"], eval_split=True, device=DEV)[0])
    assert n_views == 21 and extra["epoch"] == math.ceil(300 / 21)
    raw_r, mesh_r, extra_r = checkpoint.load_checkpoint(out.refined, DEV)
    sd = checkpoint.load_file(out.refined, "cpu")["state_dict"]
    assert sd["_surface_mesh_faces"].dtype == torch.int32 and mesh_r.faces.dtype == torch.int64 and mesh_r.n == 1
    assert len(extra_r["train_losses"]) == 1 + REFINE_ITERS // 50 and extra_r["iteration"] == REFINE_ITERS
    m = mcubes.read_mesh_ply(out.mesh)
    assert m["colors"] is not None and m["normals"] is not None
    assert torch.equal(mesh_r.faces.cpu(), m["faces"])
    v, f, vuv, fuv, tex = objfile.load_textured_mesh(out.textured_mesh)
    assert f.shape[0] == m["faces"].shape[0] and tex.shape[0] == texture.texture_size(f.shape[0], 10)
    ply = gsply.load_gaussians_ply(out.refined_ply, sh_degree=3, device=DEV)
    assert ply["points"].shape[0] == m["faces"].shape[0]
    # a refined optimizer's state loads back into a SugarOptimizer over the loaded model
    from sugar_b200.optim import SugarOptimizer
    opt = SugarOptimizer(raw_r, spatial_lr_scale=1.0, bound=True)
    opt.load_state_dict(extra_r["optimizer_state_dict"])
    ref = out.stages.refine.optimizer
    for p, q in zip((g["params"][0] for g in opt.param_groups), (g["params"][0] for g in ref.param_groups)):
        for k in ("exp_avg", "exp_avg_sq"):
            assert torch.equal(opt.state[p][k], ref.state[q][k])


def test_coarse_checkpoint_is_the_trained_model(scene):
    c = scene["out"].stages.coarse
    raw, _, _ = checkpoint.load_checkpoint(c.path, DEV)
    for k, t in c.raw.items():
        assert torch.equal(raw[k], t.detach()), k


def test_mesh_near_the_true_surface(scene):
    e = scene["out"].stages.extract
    F = e.mesh["faces"].shape[0]
    assert 0 < F <= 2 * FACES, F
    fg = e.foreground["verts"]
    assert fg.shape[0] > 100
    d = (fg.norm(dim=-1) - RADIUS).abs() / RADIUS
    med, q90 = float(d.median()), float(torch.quantile(d, 0.9))
    print(f"mesh: {F} faces, {fg.shape[0]} foreground vertices, | |v| - R | / R median {med:.4f} q90 {q90:.4f}")
    assert med < SURFACE_MEDIAN and q90 < SURFACE_Q90


def _render_bound(raw, mesh, cam, sh_deg):
    with torch.no_grad():
        b = meshbind.bind_to_mesh(raw["verts"], mesh.faces, mesh.bary, raw["scales"], raw["quaternions"],
                                  mesh.thickness)
        a = SimpleNamespace(points=b.points, scaling=b.scaling, quaternions=b.quaternions,
                                  strengths=torch.sigmoid(raw["densities"]).view(-1, 1),
                                  sh=torch.cat([raw["sh_dc"], raw["sh_rest"]], dim=1))
        return steps.render(steps.ours_ops(), a, cam, torch.zeros(3, device=DEV), sh_deg=sh_deg)[0]


def test_refinement_and_texture_reach_the_images(scene):
    r, t = scene["out"].stages.refine, scene["out"].stages.texture
    views, _ = pipeline.train_views(scene["scene"], scene["gs"], True, DEV)
    deg = train.refine_sh_degree(REFINE_ITERS)
    before = np.mean([psnr(_render_bound(r.initial, r.mesh, cam, deg), gt) for cam, gt in views])
    after = np.mean([psnr(_render_bound(r.raw, r.mesh, cam, deg), gt) for cam, gt in views])
    tex = np.mean([psnr(texture.render_textured_mesh(t.verts, t.faces, t.verts_uv, t.faces_uv, t.texture, cam), gt)
                   for cam, gt in views])
    print(f"train-view PSNR: refined model {before:.2f} -> {after:.2f} dB, textured mesh {tex:.2f} dB")
    assert after > before and after > REFINED_PSNR
    assert tex > TEXTURE_PSNR


def test_seams(scene):
    """The refined model starts from the mesh file (uint8 colours), -v is refine's n_vertices_in_fg, and the stages
    rerun from their input files alone give the same initial model and the same texture, bit for bit."""
    out = scene["out"]
    r, t, e = out.stages.refine, out.stages.texture, out.stages.extract
    views, extent = pipeline.train_views(scene["scene"], scene["gs"], True, DEV)
    raw, mesh = pipeline.refine_init(out.mesh, 1, extent, DEV)
    for k, v in r.initial.items():
        assert torch.equal(raw[k], v), k
    assert torch.equal(mesh.faces, r.mesh.faces) and mesh.thickness == r.mesh.thickness
    mem, _ = train.init_refined_from_mesh(e.mesh["verts"], e.mesh["faces"], e.mesh["colors"], 1, extent / 1e6)
    assert not torch.equal(mem["sh_dc"], r.initial["sh_dc"])     # the in-memory colours are not the file's
    assert r.optimizer.spatial_lr_scale == train.refine_spatial_lr_scale(FACES, extent)
    again = pipeline.texture_stage(scene["scene"], scene["gs"], out.refined, output_dir=scene["out_dir"] + "_again",
                                   device=DEV)
    assert torch.equal(again.texture, t.texture) and torch.equal(again.verts_uv, t.verts_uv)
    with open(again.path, "rb") as a, open(out.textured_mesh, "rb") as b:
        assert a.read() == b.read()
