"""The evaluation driver on the GPU (sugar_b200/metrics.py): a COLMAP-text scene of a sphere rendered by this
package's rasterizer, the true model as the 3DGS iteration 30000 and a perturbed one as iteration 7000, a refined
checkpoint bound to a sphere mesh and its textured .obj written through the package's own writers, and random LPIPS
weight files.  metrics.main must write the reference-named file with every key, each mean must match a
recomputation over every 8th view, and the 30k model must beat the 7k model on all three metrics."""
import json
import math
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch
from scipy.spatial import ConvexHull

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import dataset_cases as dc  # noqa: E402
import lpips_cases as lc  # noqa: E402
from sugar_b200 import (checkpoint, dataset, gsply, loss, lpips, meshbind, metrics, objfile, steps,  # noqa: E402
                        texture, train)

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
W, H, FX = 160, 120, 150.0
N_VIEWS = 16
LEVEL, VERTS, GPT, ITERS = 0.3, 1000, 1, 100     # -l -v -g -f of the refined model's names


def sphere_model(P=20_000):
    """Flat Gaussians tangent to the unit sphere, coloured by position."""
    i = torch.arange(P, dtype=torch.float64) + 0.5
    z = 1 - 2 * i / P
    phi = math.pi * (1 + 5 ** 0.5) * i
    r = torch.sqrt(1 - z * z)
    n = torch.stack([r * torch.cos(phi), r * torch.sin(phi), z], 1).float()
    q = torch.nn.functional.normalize(torch.stack([1 + n[:, 2], -n[:, 1], n[:, 0], torch.zeros(P)], 1), dim=-1)
    raw = dict(points=n, sh_dc=((colour(n) - 0.5) / train.SH_C0)[:, None], sh_rest=torch.zeros(P, 15, 3),
               densities=torch.full((P, 1), 3.0), scales=torch.log(torch.tensor([[0.035, 0.035, 0.004]])).repeat(P, 1),
               quaternions=q)
    return {k: v.to(DEV).contiguous() for k, v in raw.items()}


def colour(n):
    return 0.5 + 0.35 * torch.stack([torch.sin(3 * n[:, 0]), torch.cos(2 * n[:, 1]), torch.sin(4 * n[:, 2] + 1)], 1)


def sphere_mesh(n=800):
    """A closed triangle mesh of the unit sphere: the convex hull of Fibonacci points, faces wound outwards."""
    i = np.arange(n) + 0.5
    z = 1 - 2 * i / n
    phi = np.pi * (1 + 5 ** 0.5) * i
    r = np.sqrt(1 - z * z)
    v = np.stack([r * np.cos(phi), r * np.sin(phi), z], 1)
    f = ConvexHull(v).simplices.copy()
    nrm = np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]])
    flip = (nrm * v[f].mean(1)).sum(1) < 0
    f[flip] = f[flip][:, ::-1]
    return torch.from_numpy(v).float().to(DEV), torch.from_numpy(f.astype(np.int64)).to(DEV)


def render_vanilla(raw, cam):
    return steps.render(steps.ours_ops(), steps.activate(raw), cam, torch.zeros(3, device=DEV), sh_deg=3)[0]


def render_bound(raw, mesh, cam, sh_deg):
    b = meshbind.bind_to_mesh(raw["verts"], mesh.faces, mesh.bary, raw["scales"], raw["quaternions"], mesh.thickness)
    a = SimpleNamespace(points=b.points, scaling=b.scaling, quaternions=b.quaternions,
                        strengths=torch.sigmoid(raw["densities"]).view(-1, 1),
                        sh=torch.cat([raw["sh_dc"], raw["sh_rest"]], dim=1))
    return steps.render(steps.ours_ops(), a, cam, torch.zeros(3, device=DEV), sh_deg=sh_deg)[0]


@pytest.fixture(scope="module")
def scene(tmp_path_factory):
    root = tmp_path_factory.mktemp("metrics")
    scene_dir, gs_dir, out_dir = str(root / "scenes" / "ball"), str(root / "gs" / "ball"), str(root / "output")
    os.makedirs(os.path.join(scene_dir, "images"))
    truth = sphere_model()
    poses = dc.ring_poses(8, radius=4.0, height=1.4, seed=3) + dc.ring_poses(8, radius=4.0, height=-1.4, seed=4)
    cams, images = [], []
    with torch.no_grad():
        for i, (Rwc, t) in enumerate(poses):
            name = f"view_{i:02d}"
            cam = dataset.make_camera(Rwc.T, t, dataset.focal2fov(FX, W), dataset.focal2fov(FX, H), W, H,
                                      device=DEV, name=name, orig_width=W, orig_height=H)
            px = (render_vanilla(truth, cam).clamp(0, 1) * 255.0).round().to(torch.uint8).permute(1, 2, 0)
            dc.write_png(os.path.join(scene_dir, "images", name + ".png"), px.cpu().numpy())
            images.append((i + 1, dc.rotmat2qvec(Rwc), t, 1, name + ".png"))
            cams.append(cam)
    pts = truth["points"][::50].cpu().double().numpy()
    dc.write_colmap(os.path.join(scene_dir, "sparse", "0"), [(1, "PINHOLE", W, H, [FX, FX, W / 2, H / 2])], images,
                    (pts, np.full((len(pts), 3), 128, np.uint8)), binary=False)
    os.makedirs(gs_dir)
    dataset.write_cameras_json(os.path.join(gs_dir, "cameras.json"), cams)
    g = torch.Generator(device=DEV).manual_seed(5)
    noisy = {k: v.clone() for k, v in truth.items()}
    noisy["points"] += 0.02 * torch.randn(noisy["points"].shape, device=DEV, generator=g)
    noisy["sh_dc"] += 0.3 * torch.randn(noisy["sh_dc"].shape, device=DEV, generator=g)
    for it, model in ((30_000, truth), (7000, noisy)):
        gsply.save_gaussians_ply(os.path.join(gs_dir, "point_cloud", f"iteration_{it}", "point_cloud.ply"), model)
    # a refined model bound to a sphere mesh, and its textured mesh, under the names metrics.py reads
    paths = metrics.model_paths("ball", "sdf", 7000, 0.2, LEVEL, VERTS, GPT, ITERS, output_dir=out_dir)
    verts, faces = sphere_mesh()
    refined, mesh = train.init_refined_from_mesh(verts, faces, colour(verts), GPT, 1e-6)
    with torch.no_grad():
        refined["sh_rest"].normal_(0.0, 0.05, generator=g)   # view-dependent colour: SH degree 0 and 3 differ
    os.makedirs(os.path.dirname(paths.refined))
    checkpoint.save_checkpoint(paths.refined, refined, mesh, train_losses=[], epoch=1, iteration=ITERS)
    with torch.no_grad():
        b = meshbind.bind_to_mesh(refined["verts"], mesh.faces, mesh.bary, refined["scales"], refined["quaternions"],
                                  mesh.thickness)
        verts_uv, faces_uv, tex = texture.extract_texture_image_and_uv_from_gaussians(
            refined["verts"].detach(), mesh.faces, b.points, b.scaling, b.quaternions,
            torch.sigmoid(refined["densities"].detach()), refined["sh_dc"].detach(), cams, square_size=4)
    os.makedirs(os.path.dirname(paths.textured_mesh))
    objfile.save_textured_mesh(paths.textured_mesh, refined["verts"].detach(), mesh.faces, verts_uv, faces_uv, tex)
    wdir = str(root / "lpips_weights")
    lc.write_weight_files(wdir)
    cfg = str(root / "scenes.json")
    with open(cfg, "w") as f:
        json.dump({scene_dir: gs_dir}, f)
    args = ["--scene_config", cfg, "-r", "sdf", "-l", str(LEVEL), "-v", str(VERTS), "-g", str(GPT), "-f", str(ITERS),
            "--output_dir", out_dir, "--lpips_weights_dir", wdir]
    return SimpleNamespace(scene=scene_dir, gs=gs_dir, out=out_dir, cams=cams, truth=truth, noisy=noisy,
                           textured_mesh=paths.textured_mesh,
                           refined=refined, mesh=mesh, uv=(refined["verts"].detach(), mesh.faces, verts_uv, faces_uv,
                                                           tex), weights=wdir, args=args)


def recompute(scene, render, with_lpips=True):
    """The means over every 8th view of the ground truth, recomputed outside the driver from `render`."""
    views, _ = dataset.load_gs_cameras(scene.scene, scene.gs, eval_split=False, device=DEV)
    metric = lpips.LPIPS(os.path.join(scene.weights, lpips.VGG_FILE), os.path.join(scene.weights, lpips.LIN_FILE))
    vals = {"ssim": [], "psnr": [], "lpips": []}
    with torch.no_grad():
        for cam, gt in views[::8]:
            img = render(cam).clamp(0, 1)[None]
            vals["ssim"].append(float(loss.ssim(img, gt[None])))
            vals["psnr"].append(float(loss.psnr(img, gt[None])))
            vals["lpips"].append(float(metric(img, gt[None].contiguous())))
    if not with_lpips:
        del vals["lpips"]
    return {k: float(np.mean(v)) for k, v in vals.items()}


def check_means(got, want):
    assert set(got) == set(want)
    for k, v in want.items():
        assert abs(got[k] - v) <= 1e-5 * max(1.0, abs(v)), (k, got[k], v)


def test_gaussians_vanilla_and_every_key(scene):
    res = metrics.main(scene.args + ["--evaluate_vanilla", "True"])
    path = os.path.join(scene.out, "metrics", "results_sdf02_normal02.json")
    with open(path) as f:
        on_disk = json.load(f)
    assert on_disk == res and list(res) == ["ball"]
    key = f"sugar_03_{VERTS}_{ITERS}"
    assert set(res["ball"]) == {"3dgs_7k", "3dgs_30k", key}
    assert len(dataset.load_gs_cameras(scene.scene, scene.gs, eval_split=True, device=DEV)[1]) == N_VIEWS // 8
    check_means(res["ball"]["3dgs_30k"], recompute(scene, lambda c: render_vanilla(scene.truth, c)))
    check_means(res["ball"]["3dgs_7k"], recompute(scene, lambda c: render_vanilla(scene.noisy, c)))
    check_means(res["ball"][key], recompute(scene, lambda c: render_bound(scene.refined, scene.mesh, c, 3)))
    r30, r7 = res["ball"]["3dgs_30k"], res["ball"]["3dgs_7k"]
    print(f"3dgs_30k {r30}\n3dgs_7k {r7}\nsugar {res['ball'][key]}")
    assert r30["psnr"] > r7["psnr"] and r30["ssim"] > r7["ssim"] and r30["lpips"] < r7["lpips"]


def test_uv_texture(scene):
    res = metrics.main(scene.args + ["--use_uv_texture", "True"])
    assert os.path.isfile(os.path.join(scene.out, "metrics", "results_sdf02_normal02_uvtexture.json"))
    key = f"sugar_03_{VERTS}_{ITERS}"
    assert set(res["ball"]) == {key}
    # the .obj as written: its texture went through the 8-bit PNG, as the reference's save_obj / load_objs_as_meshes
    written = objfile.load_textured_mesh(scene.textured_mesh, DEV)
    assert torch.equal(written[1], scene.uv[1])
    assert float((scene.uv[4].clamp(0, 1) - written[4]).abs().max()) <= 1 / 255 + 1e-6   # truncated to bytes
    check_means(res["ball"][key], recompute(scene, lambda c: texture.render_textured_mesh(*written, c)))


def test_without_lpips_and_diffuse_only(scene):
    res = metrics.main(scene.args + ["--compute_lpips", "False", "--use_diffuse_color_only", "True",
                                     "--lpips_weights_dir", os.path.join(scene.out, "nowhere")])
    assert os.path.isfile(os.path.join(scene.out, "metrics", "results_sdf02_normal02_diffuseonly.json"))
    got = res["ball"][f"sugar_03_{VERTS}_{ITERS}"]
    assert set(got) == {"ssim", "psnr"}
    check_means(got, recompute(scene, lambda c: render_bound(scene.refined, scene.mesh, c, 0), with_lpips=False))
