"""Golden vectors for the splatted diamond mesh from the reference's OWN code.

Runs in the build container (needs /root/reference):  python tests/golden/make_splatmesh_golden.py
SuGaR.splat_mesh needs a model, a pytorch3d camera and pytorch3d's Meshes.  This script reads exactly
sugar_scene/sugar_model.py:490-513 (the body of the `triangle_vertices` property for the diamond primitive) and
:698-715 (splat_mesh up to the splatted vertices) from /root/reference at run time, dedents the lines and executes
them unchanged, in float64, with a duck-typed `self` (points, scaling, quaternions, primitive_verts = the diamond,
triangle_scale = 2) and a stand-in camera whose get_world_to_view_transform().transform_points / .inverse() and
get_camera_center come from this package's view matrix.  pytorch3d's quaternion helpers are the restatements of
oracle/field_oracle.py and oracle/meshbind_oracle.py.  Only numbers are stored: the float32 inputs and the float64
vertices.
Outputs: tests/golden/splatmesh_<case>.npz
"""
import os
import sys
import textwrap

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from oracle import field_oracle as fo  # noqa: E402
from oracle import meshbind_oracle as mbo  # noqa: E402
from sugar_b200 import scenes  # noqa: E402

SRC = "/root/reference/sugar_scene/sugar_model.py"
BLOCKS = ((490, 513), (698, 715))
# posed: random poses under a posed camera; flat: near-degenerate scales (one axis ~1e-6 of the others, the other two
# within 1e-4 of each other but never tied); offaxis: Gaussians far off the optical axis, up to 3x the field of view
CASES = {"posed_500": dict(P=500, seed=31, camera="posed"),
         "flat_2000": dict(P=2000, seed=32, camera="posed", flat=True),
         "offaxis_2000": dict(P=2000, seed=33, camera="identity", lateral=3.0)}
W, H = 320, 240


def make_inputs(P, seed, camera, flat=False, lateral=1.1):
    sc = scenes.make_scene(P, W, H, seed=seed, camera=camera, lateral=lateral, frac_behind=0.0)
    scales = sc.scales.copy()
    if flat:
        rng = np.random.Generator(np.random.PCG64(seed))
        k = rng.integers(0, 3, P)
        s = scales[np.arange(P), (k + 1) % 3]
        scales[np.arange(P), (k + 2) % 3] = s * (1.0 + rng.choice([-1.0, 1.0], P) * rng.uniform(2e-4, 1e-3, P))
        scales[np.arange(P), k] = s * 1e-6
    return dict(points=sc.means3D, scaling=scales.astype(np.float32), quaternions=sc.rotations,
                viewmatrix=sc.viewmatrix, projmatrix=sc.projmatrix, campos=sc.campos, width=W, height=H)


def reference_vertices(code_tv, code_splat, inp):
    d = lambda k: torch.from_numpy(inp[k]).double()
    view = d("viewmatrix")

    class Transform:
        def __init__(self, m):
            self.m = m

        def transform_points(self, p):
            return p @ self.m[:3, :3] + self.m[3, :3]

        def inverse(self):
            return Transform(torch.linalg.inv(self.m))

    class Camera:
        def get_world_to_view_transform(self):
            return Transform(view)

        def get_camera_center(self):
            return d("campos")[None]

    class Model:
        points = d("points")
        scaling = d("scaling")
        quaternions = torch.nn.functional.normalize(d("quaternions"), dim=-1)
        primitive_verts = torch.tensor([[0., -1., 0.], [0., 0, 1.], [0., 1., 0.], [0., 0., -1.]], dtype=torch.float64)
        triangle_scale = 2.0
        n_vertices_per_gaussian = 4

    model = Model()
    helpers = dict(torch=torch, quaternion_to_matrix=fo.quaternion_to_matrix, quaternion_apply=fo.quaternion_apply,
                   matrix_to_quaternion=mbo.matrix_to_quaternion)
    ns = dict(helpers, self=model)
    exec(code_tv, ns)
    model.triangle_vertices = ns["triangle_vertices"]
    ns = dict(helpers, self=model, p3d_camera=Camera(), mode="perspective")
    exec(code_splat, ns)
    return ns["splatted_verts"].numpy()


def main():
    lines = open(SRC).read().splitlines()
    codes = [compile(textwrap.dedent("\n".join(lines[a - 1:b])), f"sugar_model.py:{a}-{b}", "exec") for a, b in BLOCKS]
    for name, cfg in CASES.items():
        inp = make_inputs(**cfg)
        verts = reference_vertices(codes[0], codes[1], inp)
        print(name, verts.shape, float(np.abs(verts).max()))
        np.savez_compressed(os.path.join(HERE, f"splatmesh_{name}.npz"), verts=verts, **inp)


if __name__ == "__main__":
    main()
