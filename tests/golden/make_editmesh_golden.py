"""Golden vectors for the editable mesh-bound model and the compositor's rotated colours, from the reference's OWN code.

Needs the reference sources (make_field_golden.import_reference_sugar):  python tests/golden/make_editmesh_golden.py
SuGaR.points / .scaling / .quaternions (sugar_scene/sugar_model.py:384-398, 415-479) are called UNBOUND on a duck-typed
object with editable=True, _reference_points and edited_cache=None, so they run get_edited_quaternions_and_scales
(:572-667) as the reference does after make_editable(); the module's missing third-party imports are stubbed
(tests/golden/make_field_golden.py), and the two pytorch3d functions the path calls -- Meshes.faces_normals_list and
matrix_to_quaternion -- are the restatements in oracle/meshbind_oracle.py.  Rotated colours are SuGaR.get_points_rgb
(:839-883) with the compositor's directions (sugar_compositor.py:146-150).
Outputs: tests/golden/editmesh_<case>.npz (inputs and outputs, float32).
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
from oracle import editmesh_oracle as eo  # noqa: E402
from oracle import meshbind_oracle as mo  # noqa: E402
from make_field_golden import import_reference_sugar  # noqa: E402

# name -> make_case arguments: every n_per of the reference's presets, each kind of edit, a soup and a connected mesh
CASES = {"identity_n6": dict(kind="identity", F=120, n_per=6, seed=0),
         "rigid_n1": dict(kind="rigid", F=150, n_per=1, seed=1),
         "jitter_n3": dict(kind="jitter", F=120, n_per=3, seed=2),
         "stretch_n4": dict(kind="stretch", F=100, n_per=4, seed=3),
         "bent_n6": dict(kind="bent", F=200, n_per=6, seed=4, mesh="height"),
         "jitter_height_n1": dict(kind="jitter", F=200, n_per=1, seed=5, mesh="height")}
# rotated colours: (points, SH degree, rotation axis, angle)
COLOR_CASES = {"shrot_deg3": (600, 3, [0.2, 1.0, -0.4], 0.9), "shrot_deg1": (300, 1, [1.0, 0.0, 0.0], -2.3)}


def edited(SuGaR, case):
    F, n = case["faces"].shape[0], case["bary"].shape[0]

    class Mesh:
        def faces_normals_list(self_inner):
            return [mo.faces_normals(case["verts"], case["faces"])]

    class Fake:
        binded_to_surface_mesh = True
        editable = True
        learnable_positions = True
        device = "cpu"
        _points = case["verts"]
        _reference_points = case["reference_verts"]
        _reference_normals = mo.faces_normals(case["reference_verts"], case["faces"])
        edited_cache = None
        _surface_mesh_faces = case["faces"]
        surface_triangle_bary_coords = case["bary"][..., None]
        n_gaussians_per_surface_triangle = n
        _n_points = F * n
        _scales = case["scales_raw"]
        _quaternions = case["complex_raw"]
        surface_mesh_thickness = torch.tensor(case["thickness"])
        scale_activation = staticmethod(torch.exp)
        surface_mesh = Mesh()

        def get_edited_quaternions_and_scales(self, verbose=False):
            return SuGaR.get_edited_quaternions_and_scales(self, verbose)

    fake = Fake()
    p = SuGaR.points.fget(fake)
    q = SuGaR.quaternions.fget(fake)   # computes both and caches the scales
    s = SuGaR.scaling.fget(fake)       # takes the cached scales
    return p.reshape(F * n, 3), s.reshape(F * n, 3), q.reshape(F * n, 4)


def main():
    sm = import_reference_sugar()
    sm.matrix_to_quaternion = mo.matrix_to_quaternion     # `from pytorch3d.transforms import ...` bound it at import
    assert not sm.use_old_method
    SuGaR = sm.SuGaR
    with torch.no_grad():
        for name, cfg in CASES.items():
            case = eo.make_case(**cfg)
            p, s, q = edited(SuGaR, case)
            inputs = {k: (v.numpy() if torch.is_tensor(v) else np.float32(v)) for k, v in case.items()}
            np.savez_compressed(os.path.join(HERE, f"editmesh_{name}.npz"), points=p.numpy(), scaling=s.numpy(),
                                quaternions=q.numpy(), **inputs)
            print(name, tuple(p.shape), "max |dot|", eo.max_axis_dot(case["verts"], case["faces"]))
        for name, (P, deg, axis, angle) in COLOR_CASES.items():
            g = torch.Generator().manual_seed(P + deg)
            points = torch.randn(P, 3, generator=g) * 2.0
            sh = torch.randn(P, 16, 3, generator=g) * 0.4
            campos = torch.tensor([0.7, -1.9, 6.5])
            R = eo.rotation(axis, angle)

            class Model:
                pass
            model = Model()
            model.points = points
            model.sh_coordinates = sh
            directions = (torch.nn.functional.normalize(points - campos, dim=-1).unsqueeze(1) @ R)[..., 0, :]
            colors = SuGaR.get_points_rgb(model, camera_centers=None, directions=directions, sh_levels=deg + 1)
            np.savez_compressed(os.path.join(HERE, f"editmesh_{name}.npz"), points=points.numpy(), sh=sh.numpy(),
                                campos=campos.numpy(), rotation=R.numpy(), sh_degree=np.int32(deg), colors=colors.numpy())
            print(name, tuple(colors.shape))


if __name__ == "__main__":
    main()
