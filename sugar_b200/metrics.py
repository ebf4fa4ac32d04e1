"""Evaluate trained scenes on their held-out views: the reference's metrics.py (PSNR, SSIM, LPIPS) over this
package's pieces.

    python -m sugar_b200.metrics --scene_config scenes.json -r sdf [--evaluate_vanilla True] [--use_uv_texture True]

scenes.json maps each scene's source directory to its 3DGS output directory, as the reference's does.  Per scene:

    views       the test split of dataset.load_gs_cameras(eval_split=True): every 8th view (i % 8 == 0); the ground
                truth as loaded (not clamped)
    3dgs_7k     with --evaluate_vanilla: point_cloud/iteration_7000/point_cloud.ply, rendered at SH degree 3
    3dgs_30k    and point_cloud/iteration_30000/point_cloud.ply
    sugar_<l>_<v>_<f>
                the refined checkpoint (pipeline.py's name for -i -e -r -l -v -g -f) rendered as the refinement
                renders a bound model, at SH degree 0 with --use_diffuse_color_only, else 3; with --use_uv_texture
                the textured .obj instead, through texture.render_textured_mesh

Every render is clamped to [0, 1] over a black background, then scored with loss.ssim, loss.psnr and lpips.LPIPS
(VGG, v0.1; `--lpips_weights_dir` holds vgg16-397923af.pth and vgg.pth); each model's numbers are the means over
its views.  The results of every scene so far are rewritten after each scene to
<output_dir>/metrics/results_<r><e>_normal02[_uvtexture|_diffuseonly|_poissoncenter|_marchingcubes].json.

Deliberate differences (DESIGN.md section 17): the scene name is pipeline.scene_name (a trailing '/' is allowed);
the refined model comes from its checkpoint alone (it holds the vertices and faces), so the mesh .ply is not read;
LPIPS is computed per pair with the weights loaded once; `--compute_lpips False` leaves 'lpips' out.
"""
import argparse
import json
import os
from types import SimpleNamespace

import torch

from . import checkpoint, dataset, gsply, loss, lpips, meshbind, objfile, pipeline, steps, texture
from .pipeline import _factor, _mesh_file, _refined_dir, str2bool

N_SKIP_IMAGES_FOR_EVAL_SPLIT = 8
VANILLA_ITERATIONS = {"3dgs_7k": 7000, "3dgs_30k": 30_000}
VANILLA_SH_DEGREE = 3


# ------------------------------------------------------------------------------------------------------ names
def result_file_name(regularization_type, estimation_factor=0.2, use_uv_texture=False, use_diffuse_color_only=False,
                     use_poisson_center=False, use_marching_cubes=False):
    """The reference's result file name; the first flag set in this order picks the suffix."""
    name = f"results_{regularization_type}{_factor(estimation_factor)}_normal{_factor(pipeline.NORMAL_FACTOR)}"
    for flag, suffix in ((use_uv_texture, "_uvtexture"), (use_diffuse_color_only, "_diffuseonly"),
                         (use_poisson_center, "_poissoncenter"), (use_marching_cubes, "_marchingcubes")):
        if flag:
            return name + suffix + ".json"
    return name + ".json"


def sugar_key(surface_level, n_vertices_in_mesh, refinement_iterations):
    return f"sugar_{_factor(surface_level)}_{n_vertices_in_mesh}_{refinement_iterations}"


def model_paths(scene, regularization_type, iteration_to_load=7000, estimation_factor=0.2, surface_level=0.3,
                n_vertices_in_mesh=1_000_000, gaussians_per_triangle=1, refinement_iterations=15_000,
                use_poisson_center=False, use_marching_cubes=False, output_dir="./output"):
    """The files metrics.py reads for a scene named `scene` -> namespace(mesh, refined, textured_mesh).  mesh is the
    coarse mesh the refined model was bound to: the default extraction's name, or with use_marching_cubes
    '...sdfnorm02marchingcubes_level<l>_decim<v>.ply' (no underscore before 'marchingcubes', as the reference
    writes it), or with use_poisson_center '..._poissoncenters_decim<v>.ply'; refined follows the mesh's name;
    textured_mesh always follows the default extraction's.  For estimation factor 0.2 and the default extraction
    these are pipeline.output_paths' names."""
    coarse_dir = f"sugarcoarse_3Dgs{iteration_to_load}_{regularization_type}estim{_factor(estimation_factor)}" \
                 f"_sdfnorm{_factor(pipeline.NORMAL_FACTOR)}"
    stem = "sugarmesh_" + coarse_dir.replace("sugarcoarse_", "")
    level_mesh = _mesh_file(coarse_dir, surface_level, n_vertices_in_mesh)
    if use_marching_cubes:
        mesh = stem + f"marchingcubes_level{_factor(surface_level)}_decim{_factor(n_vertices_in_mesh)}.ply"
    elif use_poisson_center:
        mesh = stem + f"_poissoncenters_decim{_factor(n_vertices_in_mesh)}.ply"
    else:
        mesh = level_mesh
    refined_dir = _refined_dir(mesh, gaussians_per_triangle)
    return SimpleNamespace(
        mesh=os.path.join(output_dir, "coarse_mesh", scene, mesh),
        refined=os.path.join(output_dir, "refined", scene, refined_dir, f"{refinement_iterations}.pt"),
        textured_mesh=os.path.join(output_dir, "refined_mesh", scene,
                                   _refined_dir(level_mesh, gaussians_per_triangle) + ".obj"))


def lpips_weight_paths(weights_dir):
    """-> (vgg_path, lin_path) in `weights_dir`; raises FileNotFoundError naming both files when either is missing."""
    vgg, lin = os.path.join(weights_dir, lpips.VGG_FILE), os.path.join(weights_dir, lpips.LIN_FILE)
    missing = [p for p in (vgg, lin) if not os.path.isfile(p)]
    if missing:
        raise FileNotFoundError(
            f"LPIPS needs {vgg} (torchvision's VGG16 IMAGENET1K_V1 weights) and {lin} (the LPIPS v0.1 linear "
            f"layers); missing: {', '.join(missing)}.  A run of the reference's metrics.py leaves both in its "
            "torch.hub directory; or pass --compute_lpips False")
    return vgg, lin


# ------------------------------------------------------------------------------------------------------ renders
def _black(device):
    return torch.zeros(3, device=device)


def vanilla_renderer(ply_path, device):
    raw = gsply.load_gaussians_ply(ply_path, sh_degree=VANILLA_SH_DEGREE, device=device)
    a = steps.activate(raw)
    return lambda cam: steps.render(steps.ours_ops(), a, cam, _black(device), sh_deg=VANILLA_SH_DEGREE)[0]


def refined_renderer(refined_path, sh_deg, device):
    raw, mesh, _ = checkpoint.load_checkpoint(refined_path, device)
    if mesh is None:
        raise ValueError(f"{refined_path}: a coarse checkpoint, not a refined (mesh-bound) one")
    b = meshbind.bind_to_mesh(raw["verts"], mesh.faces, mesh.bary, raw["scales"], raw["quaternions"], mesh.thickness)
    a = SimpleNamespace(points=b.points, scaling=b.scaling, quaternions=b.quaternions,
                        strengths=torch.sigmoid(raw["densities"]).view(-1, 1),
                        sh=torch.cat([raw["sh_dc"], raw["sh_rest"]], dim=1))
    return lambda cam: steps.render(steps.ours_ops(), a, cam, _black(device), sh_deg=sh_deg)[0]


def textured_renderer(obj_path, device):
    verts, faces, verts_uv, faces_uv, tex = objfile.load_textured_mesh(obj_path, device)
    return lambda cam: texture.render_textured_mesh(verts, faces, verts_uv, faces_uv, tex, cam)


def score(renders, views, metric):
    """renders: name -> cam -> image [3,H,W]; views: [(cam, gt)].  -> name -> {'ssim', 'psnr'[, 'lpips']}: the means
    over the views of each render clamped to [0, 1] against the ground truth."""
    per = {k: {"ssim": [], "psnr": []} | ({"lpips": []} if metric else {}) for k in renders}
    for cam, gt in views:
        g = gt[None]
        for k, render in renders.items():
            img = render(cam).clamp(min=0, max=1)[None]
            per[k]["ssim"].append(loss.ssim(img, g).reshape(()))
            per[k]["psnr"].append(loss.psnr(img, g).reshape(()))
            if metric:
                per[k]["lpips"].append(metric(img.contiguous(), g.contiguous()).reshape(()))
    return {k: {m: torch.stack(v).mean().item() for m, v in d.items()} for k, d in per.items()}


def evaluate_scene(source_path, gs_checkpoint_path, a, metric, device):
    """One scene's results as the reference's metrics.py computes them (see the module docstring)."""
    _, test_views = dataset.load_gs_cameras(source_path, gs_checkpoint_path, eval_split=True,
                                            eval_split_interval=N_SKIP_IMAGES_FOR_EVAL_SPLIT, device=device)
    if not test_views:
        raise ValueError(f"{gs_checkpoint_path}: no test views")
    results = {}
    with torch.no_grad():
        if a.evaluate_vanilla:
            renders = {k: vanilla_renderer(os.path.join(gs_checkpoint_path, "point_cloud", f"iteration_{it}",
                                                        "point_cloud.ply"), device)
                       for k, it in VANILLA_ITERATIONS.items()}
            results.update(score(renders, test_views, metric))
        paths = model_paths(pipeline.scene_name(source_path), a.regularization_type, a.iteration_to_load,
                            a.estimation_factor, a.surface_level, a.n_vertices_in_mesh, a.gaussians_per_triangle,
                            a.refinement_iterations, a.use_poisson_center, a.use_marching_cubes, a.output_dir)
        if a.use_uv_texture:
            render = textured_renderer(paths.textured_mesh, device)
        else:
            render = refined_renderer(paths.refined, 0 if a.use_diffuse_color_only else VANILLA_SH_DEGREE, device)
        key = sugar_key(a.surface_level, a.n_vertices_in_mesh, a.refinement_iterations)
        results[key] = score({key: render}, test_views, metric)[key]
    return results


# ------------------------------------------------------------------------------------------------------ command line
def parser():
    """metrics.py's flags and presets, plus --output_dir, --lpips_weights_dir and --compute_lpips."""
    p = argparse.ArgumentParser(prog="python -m sugar_b200.metrics",
                                description="Evaluate SuGaR (and vanilla 3DGS) models on the held-out views.")
    p.add_argument("--scene_config", type=str, required=True,
                   help="JSON file {source_images_dir_path: vanilla_gaussian_splatting_checkpoint_path}")
    p.add_argument("-i", "--iteration_to_load", type=int, default=7000, help="the 3DGS iteration the coarse model "
                   "started from")
    p.add_argument("-e", "--estimation_factor", type=float, default=0.2, help="the coarse estimation factor")
    p.add_argument("-r", "--regularization_type", type=str, required=True, choices=("sdf", "density"),
                   help="the coarse regularisation")
    p.add_argument("-l", "--surface_level", type=float, default=0.3, help="surface level of the mesh")
    p.add_argument("-v", "--n_vertices_in_mesh", type=int, default=1_000_000, help="decimation target of the mesh")
    p.add_argument("-g", "--gaussians_per_triangle", type=int, default=1, help="Gaussians per triangle")
    p.add_argument("-f", "--refinement_iterations", type=int, default=15_000, help="refinement iterations")
    p.add_argument("--gpu", type=int, default=0, help="CUDA device index")
    p.add_argument("--low_poly", type=str2bool, default=False, help="-v 200000 -g 6")
    p.add_argument("--high_poly", type=str2bool, default=False, help="-v 1000000 -g 1")
    p.add_argument("--refinement_time", type=str, default=None, help="short, medium or long: -f 2000, 7000 or 15000")
    p.add_argument("--evaluate_vanilla", type=str2bool, default=False, help="also evaluate the 3DGS models")
    p.add_argument("--use_uv_texture", type=str2bool, default=False, help="render the textured mesh")
    p.add_argument("--use_diffuse_color_only", type=str2bool, default=False, help="render SuGaR at SH degree 0")
    p.add_argument("--use_poisson_center", type=str2bool, default=False, help="the Poisson-centre mesh's model")
    p.add_argument("--use_marching_cubes", type=str2bool, default=False, help="the marching-cubes mesh's model")
    p.add_argument("--output_dir", type=str, default="./output", help="root of the outputs (and of metrics/)")
    p.add_argument("--lpips_weights_dir", type=str, default=lpips.DEFAULT_WEIGHTS_DIR,
                   help=f"directory holding {lpips.VGG_FILE} and {lpips.LIN_FILE}")
    p.add_argument("--compute_lpips", type=str2bool, default=True, help="compute LPIPS (needs its weight files)")
    return p


def parse_args(argv=None):
    """The command line with the presets applied as metrics.py applies them (low_poly, high_poly, refinement_time;
    an unknown refinement_time changes nothing)."""
    a = parser().parse_args(argv)
    if a.low_poly:
        a.n_vertices_in_mesh, a.gaussians_per_triangle = 200_000, 6
    if a.high_poly:
        a.n_vertices_in_mesh, a.gaussians_per_triangle = 1_000_000, 1
    a.refinement_iterations = {"short": 2_000, "medium": 7_000, "long": 15_000}.get(a.refinement_time,
                                                                                  a.refinement_iterations)
    return a


def main(argv=None):
    """Evaluate every scene of --scene_config -> {scene: results}; the file is rewritten after each scene."""
    a = parse_args(argv)
    with open(a.scene_config) as f:
        scenes = json.load(f)
    device = torch.device("cuda", a.gpu)
    metric = lpips.LPIPS(*lpips_weight_paths(a.lpips_weights_dir), device=device) if a.compute_lpips else None
    out_dir = os.path.join(a.output_dir, "metrics")
    os.makedirs(out_dir, exist_ok=True)
    path = os.path.join(out_dir, result_file_name(a.regularization_type, a.estimation_factor, a.use_uv_texture,
                                                  a.use_diffuse_color_only, a.use_poisson_center,
                                                  a.use_marching_cubes))
    results = {}
    with torch.cuda.device(device):
        for source_path, gs_checkpoint_path in scenes.items():
            results[pipeline.scene_name(source_path)] = evaluate_scene(source_path, gs_checkpoint_path, a, metric,
                                                                       device)
            with open(path, "w") as f:
                json.dump(results, f, indent=4)
            print(f"{pipeline.scene_name(source_path)}: {results[pipeline.scene_name(source_path)]} -> {path}")
    return results


if __name__ == "__main__":
    main()
