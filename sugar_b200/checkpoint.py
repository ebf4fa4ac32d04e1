"""SuGaR's model checkpoints (the `.pt` files its trainers hand to each other), both ways.

    save_checkpoint(path, raw, train_losses=..., epoch=..., iteration=..., optimizer_state_dict=opt.state_dict())
    save_checkpoint(path, raw, mesh, ...)                 # a refined (mesh-bound) model
    raw, mesh, extra = load_checkpoint(path, "cuda")      # mesh is None for a coarse model
    opt.load_state_dict(extra["optimizer_state_dict"])    # a SugarOptimizer over raw

The file is SuGaR.save_model's (sugar_model.py:2296-2301): torch.save of {"state_dict": ..., **extra}.  The state dict
holds the module's parameters in their registration order (sugar_model.py:149-361):

    unbound   _points [P,3], all_densities [P,1], _scales [P,3], _quaternions [P,4], _sh_coordinates_dc [P,1,3],
              _sh_coordinates_rest [P,M,3]
    bound     _surface_mesh_faces int32 [F,3] (open3d's triangles), surface_mesh_thickness float32 0-dim, then the six
              above with _points the mesh vertices [V,3], _scales and _quaternions [F n,2]

This package's names are steps.py's raw dict (points or, bound, verts; densities; scales; quaternions; sh_dc; sh_rest)
and, for a bound model, the namespace steps.refine_step takes: faces int64, bary [n,3], thickness (a Python float,
the float32 value), n, and on a CUDA device the meshloss.mesh_topology of the faces.  n = P // F, as
load_refined_model derives it.  `extra` is every other entry of the file as saved: the trainers store train_losses,
epoch, iteration and optimizer_state_dict (coarse_sdf.py:782-790, refine.py:833-841); the optimizer state is torch's
Adam layout, which SugarOptimizer.load_state_dict takes as it is.
"""
from collections import OrderedDict
from types import SimpleNamespace

import numpy as np
import torch

# (state-dict name, raw key) in registration order; a bound model's _points is raw["verts"]
PARAMS = (("_points", "points"), ("all_densities", "densities"), ("_scales", "scales"),
          ("_quaternions", "quaternions"), ("_sh_coordinates_dc", "sh_dc"), ("_sh_coordinates_rest", "sh_rest"))


def mesh_namespace(faces, n, thickness, n_verts):
    """The mesh namespace of a bound model over `n_verts` vertices: faces int64 [F,3] on the faces' device, bary [n,3]
    (meshbind.bary_coords), thickness rounded to float32 as the checkpoint stores it, n, and `topology`
    (meshloss.mesh_topology) when the faces are on a CUDA device, else None (refine_step then builds it per call)."""
    from . import meshbind, meshloss
    if n not in (1, 3, 4, 6):
        raise ValueError(f"n_gaussians_per_surface_triangle must be 1, 3, 4 or 6, got {n!r}")
    faces = faces.long().contiguous()
    topology = meshloss.mesh_topology(faces, n_verts) if faces.is_cuda and faces.numel() else None
    return SimpleNamespace(faces=faces, bary=meshbind.bary_coords(n, faces.device),
                           thickness=float(np.float32(thickness)), n=n, topology=topology)


def state_dict(raw, mesh=None):
    """-> SuGaR.state_dict() of `raw` (and `mesh` for a bound model): an OrderedDict of detached tensors in the
    reference's order, names, dtypes and shapes."""
    sd = OrderedDict()
    if mesh is not None:
        if mesh.faces.numel() and int(mesh.faces.max()) > 2 ** 31 - 1:
            raise ValueError("face ids must fit in int32")
        sd["_surface_mesh_faces"] = mesh.faces.detach().to(torch.int32)
        sd["surface_mesh_thickness"] = torch.tensor(float(mesh.thickness), dtype=torch.float32,
                                                    device=mesh.faces.device)
    for name, key in PARAMS:
        k = "verts" if mesh is not None and key == "points" else key
        if k not in raw:
            raise ValueError(f"raw has no {k!r} ({name})")
        sd[name] = raw[k].detach()
    return sd


def save_checkpoint(path, raw, mesh=None, **extra):
    """SuGaR.save_model(path, **extra) of `raw` (and `mesh` for a bound model): torch.save of
    {"state_dict": state_dict(raw, mesh), **extra}."""
    ckpt = {"state_dict": state_dict(raw, mesh)}
    ckpt.update(extra)
    torch.save(ckpt, path)


def _numpy_scalar_globals():
    core = getattr(np, "_core", None) or np.core
    return [core.multiarray.scalar, np.dtype, type(np.dtype(np.float64))]


def load_file(path, device="cuda"):
    """torch.load(path, weights_only=True) that also admits numpy float64 scalars: the position learning rate in a
    saved optimizer's param_groups is get_expon_lr_func's numpy value, in the reference's files as in this
    package's (optim.expon_lr).  Nothing else beyond torch's weights-only set is allowed."""
    with torch.serialization.safe_globals(_numpy_scalar_globals()):
        return torch.load(path, map_location=device, weights_only=True)


def load_checkpoint(path, device="cuda"):
    """A SuGaR checkpoint -> (raw, mesh, extra): raw the dict of float32 leaf tensors on `device` (steps.activate's
    keys, or refine_step's for a bound model), mesh the bound model's namespace (see the module docstring) or None,
    extra the file's other entries.  Read with load_file (torch.load(weights_only=True)).  ValueError when a parameter
    is missing or the Gaussian count is not a multiple of the face count."""
    ckpt = load_file(path, device)
    if not isinstance(ckpt, dict) or "state_dict" not in ckpt:
        raise ValueError(f"{path}: not a SuGaR checkpoint (no 'state_dict')")
    sd = ckpt["state_dict"]
    missing = [name for name, _ in PARAMS if name not in sd]
    if missing:
        raise ValueError(f"{path}: state_dict lacks {missing}")
    bound = "_surface_mesh_faces" in sd
    raw, mesh = {}, None
    if bound:
        faces = sd["_surface_mesh_faces"]
        F, P = int(faces.shape[0]), int(sd["_scales"].shape[0])
        if F == 0 or P % F:
            raise ValueError(f"{path}: {P} Gaussians over {F} faces is not a whole number per face")
        mesh = mesh_namespace(faces, P // F, float(sd["surface_mesh_thickness"]), int(sd["_points"].shape[0]))
    for name, key in PARAMS:
        k = "verts" if bound and key == "points" else key
        raw[k] = sd[name].detach().to(device=device, dtype=torch.float32).contiguous().requires_grad_(True)
    extra = {k: v for k, v in ckpt.items() if k != "state_dict"}
    return raw, mesh, extra
