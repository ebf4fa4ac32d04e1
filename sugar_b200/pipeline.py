"""SuGaR end to end: the reference's train.py (coarse -> mesh -> refine -> textured mesh) over this package's stages,
reading and writing the reference's files under the reference's names.

    python -m sugar_b200.pipeline -s data/garden -c gs_out/garden -r sdf [-l 0.3 -v 1000000 -g 1 -f 15000 ...]

    out = run("data/garden", "gs_out/garden", "sdf")          # -> namespace of the paths, and each stage's result

Each stage reads only what the previous one wrote, as the reference's scripts do, so each can run alone:

    coarse_stage    coarse_sdf.py / coarse_density.py: the 3DGS checkpoint's point_cloud.ply and cameras.json ->
                    train.train_coarse from iteration 7000 -> checkpoint.save_checkpoint (coarse/.../15000.pt)
    extract_stage   coarse_mesh.py's default branch: the coarse checkpoint, Gaussians of strength > 0.5 ->
                    poisson.surface_point_cloud -> poisson.extract_mesh_poisson -> mcubes.write_ply (coarse_mesh/...ply)
    refine_stage    refine.py: mcubes.read_mesh_ply -> train.init_refined_from_mesh -> train.train_refined ->
                    save_checkpoint (refined/.../<-f>.pt), and with export_ply gsply.export_refined_ply (refined_ply/)
    texture_stage   refined_mesh.py: the refined checkpoint -> optionally postprocess.postprocess_mesh ->
                    texture.extract_texture_image_and_uv_from_gaussians -> objfile.save_textured_mesh (refined_mesh/)

The views are the train split of dataset.load_gs_cameras(scene, checkpoint, eval_split=eval), and the extent is
mcubes.camera_spatial_extent of their centres, in every stage.  `-v` is the decimation target in faces of the
foreground and of the background mesh, each, and refine.py's n_vertices_in_fg (its position learning-rate scale), as
train.py passes it.  The keyword dicts coarse_kwargs, surface_kwargs, poisson_kwargs and refine_kwargs are forwarded
to train_coarse, surface_point_cloud, extract_mesh_poisson and train_refined (schedules, sample counts, Poisson
depth, ...) for short runs; the command line does not expose them.

Not supported, with an error that says so: a custom foreground box (-b / -B) and a white background (the trainers
render over black).  DESIGN.md section 16 has the file formats and the differences from the reference.
"""
import argparse
import math
import os
from types import SimpleNamespace

import torch

from . import checkpoint, dataset, gsply, knn, mcubes, meshbind, objfile, poisson, postprocess, texture, train
from .optim import SugarOptimizer

COARSE_FIRST_ITERATION = 7000      # coarse_sdf.py:468-469: trained-3DGS runs start here, whatever -i is
COARSE_ITERATIONS = 15_000
PRINT_LOSS_EVERY = 50              # print_loss_every_n_iterations: the iterations whose loss train_losses holds
REFINE_MILESTONES = (2000, 7000, 15_000)
ESTIMATION_FACTOR = NORMAL_FACTOR = 0.2
NORMAL_CONSISTENCY_FACTOR = 0.1


# ------------------------------------------------------------------------------------------------------ names
def scene_name(scene_path):
    """The scene's name as the reference takes it: the last '/'-separated part, or the one before a trailing '/'."""
    parts = scene_path.split("/")
    return parts[-1] if len(parts[-1]) > 0 else parts[-2]


def _factor(x):
    return str(x).replace(".", "")


def _mesh_file(coarse_dir, surface_level, n_vertices_in_mesh):
    """coarse_mesh.py:478-485: the mesh's file name from the coarse checkpoint's directory name."""
    return "sugarmesh_" + coarse_dir.replace("sugarcoarse_", "") + \
        f"_level{_factor(surface_level)}_decim{_factor(n_vertices_in_mesh)}.ply"


def _refined_dir(mesh_file, gaussians_per_triangle):
    """refine.py:269-276: the refined checkpoints' directory name from the mesh's file name."""
    return "sugarfine_" + mesh_file.split(".")[0].replace("sugarmesh_", "") + \
        f"_normalconsistency{_factor(NORMAL_CONSISTENCY_FACTOR)}_gaussperface{_factor(gaussians_per_triangle)}"


def output_paths(scene_path, regularization_type="sdf", iteration_to_load=7000, surface_level=0.3,
                 n_vertices_in_mesh=1_000_000, gaussians_per_triangle=1, refinement_iterations=15_000,
                 postprocess_mesh=False, output_dir="./output", coarse_iterations=COARSE_ITERATIONS):
    """Every output name of the pipeline under `output_dir`, restated from the reference's lines -> namespace(coarse,
    mesh, refined, refined_ply, textured_mesh):

        coarse        coarse/<scene>/sugarcoarse_3Dgs<i>_{sdf|density}estim02_sdfnorm02/<15000>.pt
                      (coarse_sdf.py:241-246, coarse_density.py:245, :816)
        mesh          coarse_mesh/<scene>/sugarmesh_<coarse dir without 'sugarcoarse_'>_level<l>_decim<v>.ply
                      (coarse_mesh.py:69-73, 478-485)
        refined       refined/<scene>/sugarfine_<mesh name without 'sugarmesh_'>_normalconsistency01_gaussperface<g>/
                      <f>.pt (refine.py:231-235, 270-276, 866)
        refined_ply   refined_ply/<scene>/<refined dir>.ply (refine.py:877-885)
        textured_mesh refined_mesh/<scene>/<refined dir>[_postprocessed].obj (refined_mesh.py:36-47)

    Factors are written str(x).replace('.', ''): 0.3 -> 03, 0.2 -> 02; decim is the integer as given."""
    if regularization_type not in ("sdf", "density"):
        raise ValueError(f"regularization_type must be 'sdf' or 'density', got {regularization_type!r}")
    scene = scene_name(scene_path)
    coarse_dir = f"sugarcoarse_3Dgs{iteration_to_load}_{regularization_type}estim{_factor(ESTIMATION_FACTOR)}" \
                 f"_sdfnorm{_factor(NORMAL_FACTOR)}"
    coarse = os.path.join(output_dir, "coarse", scene, coarse_dir, f"{coarse_iterations}.pt")
    mesh_file = _mesh_file(coarse_dir, surface_level, n_vertices_in_mesh)
    mesh = os.path.join(output_dir, "coarse_mesh", scene, mesh_file)
    refined_dir = _refined_dir(mesh_file, gaussians_per_triangle)
    refined = os.path.join(output_dir, "refined", scene, refined_dir, f"{refinement_iterations}.pt")
    refined_ply = os.path.join(output_dir, "refined_ply", scene, refined_dir + ".ply")
    textured = os.path.join(output_dir, "refined_mesh", scene,
                            refined_dir + ("_postprocessed" if postprocess_mesh else "") + ".obj")
    return SimpleNamespace(coarse=coarse, mesh=mesh, refined=refined, refined_ply=refined_ply, textured_mesh=textured)


# ------------------------------------------------------------------------------------------------------ stages
def train_views(scene_path, checkpoint_path, eval=True, device="cuda"):
    """The train split of dataset.load_gs_cameras (every 8th view is a test view with `eval`) -> (views, extent):
    extent = mcubes.camera_spatial_extent of the views' centres."""
    views, _ = dataset.load_gs_cameras(scene_path, checkpoint_path, eval_split=eval, device=device)
    if not views:
        raise ValueError(f"{checkpoint_path}: no training views")
    extent = mcubes.camera_spatial_extent(torch.stack([cam.campos.detach().cpu() for cam, _ in views]))
    return views, extent


def _makedirs(path):
    d = os.path.dirname(path)
    if d:
        os.makedirs(d, exist_ok=True)


class _Recorder:
    """on_iteration for the trainers: the losses the reference records (iteration 1 and every PRINT_LOSS_EVERY, read
    to the host only then), the epoch count, and the reference's milestone saves."""

    def __init__(self, first, n_views, save=None, milestones=()):
        self.first, self.n_views, self.save, self.milestones = first, n_views, save, milestones
        self.losses, self.last = [], first - 1

    def __call__(self, it, loss, ev):
        self.last = it
        if it == 1 or it % PRINT_LOSS_EVERY == 0:
            self.losses.append(loss.item())
        if self.save is not None and it in self.milestones:
            self.save(it, (it - self.first) // self.n_views)

    def epochs(self):
        """Epochs begun, as the reference's counter reads after its loop (a partial epoch counts)."""
        return math.ceil((self.last - self.first + 1) / self.n_views)


def coarse_stage(scene_path, checkpoint_path, regularization_type, iteration_to_load=7000, eval=True,
                 output_dir="./output", device="cuda", coarse_kwargs=None):
    """coarse_sdf.py / coarse_density.py with train.py's arguments: the 3DGS model at iteration_to_load, the K = 16
    neighbour table, train.train_coarse(mode=regularization_type) from iteration 7000 to 15000 (both overridable in
    coarse_kwargs as first_iteration / num_iterations), then the checkpoint.  -> namespace(path, raw, optimizer,
    train_losses)."""
    kw = dict(coarse_kwargs or {})
    first = kw.pop("first_iteration", COARSE_FIRST_ITERATION)
    num_iterations = kw.pop("num_iterations", COARSE_ITERATIONS)
    path = output_paths(scene_path, regularization_type, iteration_to_load, output_dir=output_dir,
                        coarse_iterations=num_iterations).coarse
    views, extent = train_views(scene_path, checkpoint_path, eval, device)
    ply = os.path.join(checkpoint_path, "point_cloud", f"iteration_{iteration_to_load}", "point_cloud.ply")
    raw = gsply.load_gaussians_ply(ply, sh_degree=3, device=device)
    knn_idx = knn.reset_neighbors(raw["points"].detach(), 16)[1]
    rec = _Recorder(first, len(views))
    opt = train.train_coarse(raw, views, knn_idx, mode=regularization_type, spatial_extent=extent,
                             num_iterations=num_iterations, first_iteration=first, on_iteration=rec, **kw)
    _makedirs(path)
    checkpoint.save_checkpoint(path, raw, train_losses=rec.losses, epoch=rec.epochs(), iteration=num_iterations,
                               optimizer_state_dict=opt.state_dict())
    return SimpleNamespace(path=path, raw=raw, optimizer=opt, train_losses=rec.losses)


def extraction_mask(densities):
    """The Gaussians the extraction keeps: strength sigmoid(densities) > 0.5, strictly (drop_low_opacity_points,
    sugar_model.py:801-803).  The coarse trainer's prune at 9000 removes strength < 0.5, so a Gaussian at exactly 0.5
    survives the prune and is left out of the mesh."""
    return torch.sigmoid(densities.detach())[..., 0] > 0.5


def extract_stage(scene_path, checkpoint_path, coarse_path, surface_level=0.3, n_vertices_in_mesh=1_000_000,
                  center_bbox=True, eval=True, output_dir="./output", device="cuda", surface_kwargs=None,
                  poisson_kwargs=None):
    """coarse_mesh.py's default branch with train.py's arguments: the coarse checkpoint's Gaussians of strength > 0.5
    (drop_low_opacity_points), their level-set points over the train views at `surface_level`, the Poisson meshes of
    the foreground and background boxes (centred on the mean camera centre with center_bbox; depth 10, density
    quantile 0.1), each decimated to n_vertices_in_mesh faces, combined and written with colours and normals.  The
    mesh name follows the coarse checkpoint's directory.  -> namespace(path, mesh: the combined mesh dict)."""
    raw, mesh, _ = checkpoint.load_checkpoint(coarse_path, device)
    if mesh is not None:
        raise ValueError(f"{coarse_path}: a refined (mesh-bound) checkpoint, not a coarse one")
    coarse_dir = os.path.basename(os.path.dirname(os.path.abspath(coarse_path)))
    path = os.path.join(output_dir, "coarse_mesh", scene_name(scene_path),
                        _mesh_file(coarse_dir, surface_level, n_vertices_in_mesh))
    views, extent = train_views(scene_path, checkpoint_path, eval, device)
    cams = [cam for cam, _ in views]
    with torch.no_grad():
        strengths = torch.sigmoid(raw["densities"].detach())
        keep = extraction_mask(raw["densities"])
        points = raw["points"].detach()[keep].contiguous()
        scaling = torch.exp(raw["scales"].detach()[keep]).contiguous()
        quaternions = torch.nn.functional.normalize(raw["quaternions"].detach()[keep], dim=-1).contiguous()
        sh_dc = raw["sh_dc"].detach()[keep].contiguous()
        strengths = strengths[keep].contiguous()
        center = torch.stack([c.campos.detach().float().cpu() for c in cams]).mean(dim=0) if center_bbox else None
    cloud = poisson.surface_point_cloud(points, scaling, quaternions, strengths, sh_dc, cams,
                                        surface_level=surface_level, **(surface_kwargs or {}))
    pkw = dict(poisson_depth=10, vertices_density_quantile=0.1)
    pkw.update(poisson_kwargs or {})
    out = poisson.extract_mesh_poisson(cloud["points"], cloud["colors"], cloud["normals"], extent, center=center,
                                       decimation_target=n_vertices_in_mesh, **pkw)
    _makedirs(path)
    mcubes.write_ply(path, **out["combined"])
    return SimpleNamespace(path=path, mesh=out["combined"], foreground=out["foreground"],
                           background=out["background"])


def refine_init(mesh_path, gaussians_per_triangle, extent, device="cuda"):
    """The refinement's initial model from the mesh file alone: read_mesh_ply, then init_refined_from_mesh with
    thickness extent / 1e6 (sugar_model.py:165-166) -> (raw, mesh)."""
    m = mcubes.read_mesh_ply(mesh_path)
    if m["colors"] is None:
        raise ValueError(f"{mesh_path}: the mesh has no vertex colours (the refined model's initial colours)")
    return train.init_refined_from_mesh(m["verts"].to(device), m["faces"].to(device), m["colors"].to(device),
                                        gaussians_per_triangle, extent / 1_000_000)


def refine_stage(scene_path, checkpoint_path, mesh_path, gaussians_per_triangle=1, n_vertices_in_mesh=1_000_000,
                 refinement_iterations=15_000, export_ply=True, eval=True, output_dir="./output", device="cuda",
                 refine_kwargs=None):
    """refine.py with train.py's arguments: the model bound to the mesh file (refine_init), spatial_lr_scale =
    train.refine_spatial_lr_scale(n_vertices_in_mesh, extent), train.train_refined with normal consistency 0.1 for
    refinement_iterations, the checkpoints at the reference's milestones (2000, 7000) below the last iteration and at
    the last, and with export_ply the viewer's .ply.  The names follow the mesh file's.  -> namespace(path, ply_path
    (None without export_ply), initial (the initial raw, detached copies), raw, mesh, optimizer, train_losses)."""
    refined_dir = _refined_dir(os.path.basename(mesh_path), gaussians_per_triangle)
    scene = scene_name(scene_path)
    ckpt_dir = os.path.join(output_dir, "refined", scene, refined_dir)
    views, extent = train_views(scene_path, checkpoint_path, eval, device)
    raw, mesh = refine_init(mesh_path, gaussians_per_triangle, extent, device)
    initial = {k: v.detach().clone() for k, v in raw.items()}
    lr_scale = train.refine_spatial_lr_scale(n_vertices_in_mesh, extent)
    opt = SugarOptimizer(raw, spatial_lr_scale=lr_scale, bound=True)
    os.makedirs(ckpt_dir, exist_ok=True)

    def save(it, epoch):
        checkpoint.save_checkpoint(os.path.join(ckpt_dir, f"{it}.pt"), raw, mesh, train_losses=list(rec.losses),
                                   epoch=epoch, iteration=it, optimizer_state_dict=opt.state_dict())

    kw = dict(normal_consistency_factor=NORMAL_CONSISTENCY_FACTOR)
    kw.update(refine_kwargs or {})
    milestones = tuple(m for m in REFINE_MILESTONES if m < refinement_iterations)
    rec = _Recorder(kw.get("first_iteration", 1), len(views), save, milestones)
    train.train_refined(raw, mesh, views, lr_scale, num_iterations=refinement_iterations, on_iteration=rec,
                        optimizer=opt, **kw)
    path = os.path.join(ckpt_dir, f"{refinement_iterations}.pt")
    save(refinement_iterations, rec.epochs())
    ply_path = None
    if export_ply:
        ply_path = os.path.join(output_dir, "refined_ply", scene, refined_dir + ".ply")
        gsply.export_refined_ply(ply_path, raw, mesh)
    return SimpleNamespace(path=path, ply_path=ply_path, initial=initial, raw=raw, mesh=mesh, optimizer=opt,
                           train_losses=rec.losses)


def texture_stage(scene_path, checkpoint_path, refined_path, square_size=10, postprocess_mesh=False,
                  postprocess_density_threshold=0.1, postprocess_iterations=5, eval=True, output_dir="./output",
                  device="cuda"):
    """refined_mesh.py with train.py's arguments: the refined checkpoint (n = P // F), optionally the border-face
    post-processing, the UV texture baked over the train views with `square_size`, and the .obj / .mtl / .png.  The
    name follows the checkpoint's directory.  -> namespace(path, verts, faces, verts_uv, faces_uv, texture)."""
    raw, mesh, _ = checkpoint.load_checkpoint(refined_path, device)
    if mesh is None:
        raise ValueError(f"{refined_path}: a coarse checkpoint, not a refined (mesh-bound) one")
    refined_dir = os.path.basename(os.path.dirname(os.path.abspath(refined_path)))
    path = os.path.join(output_dir, "refined_mesh", scene_name(scene_path),
                        refined_dir + ("_postprocessed" if postprocess_mesh else "") + ".obj")
    views, _ = train_views(scene_path, checkpoint_path, eval, device)
    verts, faces = raw["verts"].detach(), mesh.faces
    scales, quats, dens, sh_dc = (raw[k].detach() for k in ("scales", "quaternions", "densities", "sh_dc"))
    if postprocess_mesh:
        pp = postprocess.postprocess_mesh(verts, faces, mesh.n, scales, quats, dens, sh_dc, raw["sh_rest"].detach(),
                                          mesh.thickness, density_threshold=postprocess_density_threshold,
                                          iterations=postprocess_iterations)
        faces, scales, quats, dens, sh_dc = pp.faces, pp.scales, pp.quaternions, pp.densities, pp.sh_dc
    with torch.no_grad():
        b = meshbind.bind_to_mesh(verts, faces, mesh.bary, scales, quats, mesh.thickness)
        verts_uv, faces_uv, tex = texture.extract_texture_image_and_uv_from_gaussians(
            verts, faces, b.points, b.scaling, b.quaternions, torch.sigmoid(dens), sh_dc, [cam for cam, _ in views],
            square_size=square_size)
    _makedirs(path)
    objfile.save_textured_mesh(path, verts, faces, verts_uv, faces_uv, tex)
    return SimpleNamespace(path=path, verts=verts, faces=faces, verts_uv=verts_uv, faces_uv=faces_uv, texture=tex)


def run(scene_path, checkpoint_path, regularization_type, iteration_to_load=7000, surface_level=0.3,
        n_vertices_in_mesh=1_000_000, center_bbox=True, gaussians_per_triangle=1, refinement_iterations=15_000,
        export_uv_textured_mesh=True, square_size=10, postprocess_mesh=False, postprocess_density_threshold=0.1,
        postprocess_iterations=5, export_ply=True, eval=True, gpu=0, output_dir="./output", coarse_kwargs=None,
        surface_kwargs=None, poisson_kwargs=None, refine_kwargs=None):
    """train.py: the four stages, each reading the files the one before wrote -> namespace(coarse, mesh, refined,
    refined_ply, textured_mesh: the paths written (refined_ply / textured_mesh None when not exported); stages: each
    stage's result namespace)."""
    if regularization_type not in ("sdf", "density"):
        raise ValueError(f"Unknown regularization type: {regularization_type!r} (sdf or density)")
    device = f"cuda:{int(gpu)}"
    with torch.cuda.device(device):
        common = dict(eval=eval, output_dir=output_dir, device=device)
        c = coarse_stage(scene_path, checkpoint_path, regularization_type, iteration_to_load,
                         coarse_kwargs=coarse_kwargs, **common)
        m = extract_stage(scene_path, checkpoint_path, c.path, surface_level, n_vertices_in_mesh, center_bbox,
                          surface_kwargs=surface_kwargs, poisson_kwargs=poisson_kwargs, **common)
        r = refine_stage(scene_path, checkpoint_path, m.path, gaussians_per_triangle, n_vertices_in_mesh,
                         refinement_iterations, export_ply, refine_kwargs=refine_kwargs, **common)
        t = None
        if export_uv_textured_mesh:
            t = texture_stage(scene_path, checkpoint_path, r.path, square_size, postprocess_mesh,
                              postprocess_density_threshold, postprocess_iterations, **common)
    return SimpleNamespace(coarse=c.path, mesh=m.path, refined=r.path, refined_ply=r.ply_path,
                           textured_mesh=None if t is None else t.path,
                           stages=SimpleNamespace(coarse=c, extract=m, refine=r, texture=t))


# ------------------------------------------------------------------------------------------------------ command line
def str2bool(v):
    if isinstance(v, bool):
        return v
    if v.lower() in ("yes", "true", "t", "y", "1"):
        return True
    if v.lower() in ("no", "false", "f", "n", "0"):
        return False
    raise argparse.ArgumentTypeError(f"a boolean is expected, got {v!r}")


def parser():
    """train.py's flags and presets (train.py:16-100), plus --output_dir."""
    p = argparse.ArgumentParser(prog="python -m sugar_b200.pipeline",
                                description="Optimize a full SuGaR model from a 3DGS checkpoint.")
    p.add_argument("-s", "--scene_path", type=str, required=True, help="path to the scene (images/ and sparse/)")
    p.add_argument("-c", "--checkpoint_path", type=str, required=True,
                   help="the 3DGS output directory (cameras.json, point_cloud/iteration_<i>/point_cloud.ply)")
    p.add_argument("-i", "--iteration_to_load", type=int, default=7000, help="the 3DGS iteration to load")
    p.add_argument("-r", "--regularization_type", type=str, required=True, choices=("sdf", "density"),
                   help="the coarse regularisation")
    p.add_argument("-l", "--surface_level", type=float, default=0.3, help="surface level of the mesh")
    p.add_argument("-v", "--n_vertices_in_mesh", type=int, default=1_000_000,
                   help="decimation target in faces, foreground and background each")
    p.add_argument("-b", "--bboxmin", type=str, default=None, help="not supported")
    p.add_argument("-B", "--bboxmax", type=str, default=None, help="not supported")
    p.add_argument("--center_bbox", type=str2bool, default=True, help="centre the boxes on the cameras")
    p.add_argument("-g", "--gaussians_per_triangle", type=int, default=1, help="Gaussians per triangle: 1, 3, 4, 6")
    p.add_argument("-f", "--refinement_iterations", type=int, default=15_000, help="refinement iterations")
    p.add_argument("-t", "--export_uv_textured_mesh", type=str2bool, default=True, help="write the textured .obj")
    p.add_argument("--square_size", type=int, default=10, help="texels per face pair square")
    p.add_argument("--postprocess_mesh", type=str2bool, default=False, help="remove low-density border faces")
    p.add_argument("--postprocess_density_threshold", type=float, default=0.1)
    p.add_argument("--postprocess_iterations", type=int, default=5)
    p.add_argument("--export_ply", type=str2bool, default=True, help="write the refined Gaussians for the viewer")
    p.add_argument("--low_poly", type=str2bool, default=False, help="-v 200000 -g 6")
    p.add_argument("--high_poly", type=str2bool, default=False, help="-v 1000000 -g 1")
    p.add_argument("--refinement_time", type=str, default=None, choices=(None, "short", "medium", "long"),
                   help="-f 2000, 7000 or 15000")
    p.add_argument("--eval", type=str2bool, default=True, help="hold out every 8th view")
    p.add_argument("--gpu", type=int, default=0, help="CUDA device index")
    p.add_argument("--white_background", type=str2bool, default=False, help="not supported")
    p.add_argument("--output_dir", type=str, default="./output", help="root of the outputs")
    return p


def parse_args(argv=None):
    """The command line -> run()'s keyword arguments, presets applied as train.py applies them (low_poly, then
    high_poly, then refinement_time).  Exits with an error naming -b / -B or --white_background when given."""
    p = parser()
    a = p.parse_args(argv)
    if a.bboxmin is not None or a.bboxmax is not None:
        p.error("-b/--bboxmin and -B/--bboxmax (a custom foreground box) are not supported")
    if a.white_background:
        p.error("--white_background True is not supported: the trainers render over black")
    if a.low_poly:
        a.n_vertices_in_mesh, a.gaussians_per_triangle = 200_000, 6
    if a.high_poly:
        a.n_vertices_in_mesh, a.gaussians_per_triangle = 1_000_000, 1
    if a.refinement_time is not None:
        a.refinement_iterations = {"short": 2_000, "medium": 7_000, "long": 15_000}[a.refinement_time]
    keys = ("scene_path", "checkpoint_path", "regularization_type", "iteration_to_load", "surface_level",
            "n_vertices_in_mesh", "center_bbox", "gaussians_per_triangle", "refinement_iterations",
            "export_uv_textured_mesh", "square_size", "postprocess_mesh", "postprocess_density_threshold",
            "postprocess_iterations", "export_ply", "eval", "gpu", "output_dir")
    return {k: getattr(a, k) for k in keys}


def main(argv=None):
    out = run(**parse_args(argv))
    for k in ("coarse", "mesh", "refined", "refined_ply", "textured_mesh"):
        if getattr(out, k) is not None:
            print(f"{k}: {getattr(out, k)}")


if __name__ == "__main__":
    main()
