"""Golden vectors for the UV texture's layout and initial texels from the reference's OWN code.

Runs in the build container (needs /root/reference):  python tests/golden/make_texture_golden.py
extract_texture_image_and_uv_from_gaussians needs a SuGaR model and pytorch3d.  This script reads exactly
sugar_scene/sugar_model.py:2478-2605 (square size check, UV layout, initial texels up to SH2RGB) and :730-736
(get_covariance up to its return_sqrt branch) from /root/reference at run time, dedents the lines and executes them
unchanged, in float32 on the CPU, with a duck-typed `rc` (surface_mesh.verts_list() / faces_list(), points, scaling,
quaternions, sh_coordinates [P,1,3], n_gaussians_per_surface_triangle, device) and SH2RGB(x) = x * C0 + 0.5.
pytorch3d's quaternion_to_matrix is the restatement of oracle/field_oracle.py.  The Gaussians are bound to the mesh
with oracle/meshbind_oracle.py (the reference's binding, restated), so their centres, in-plane scales and rotations are
the refined model's.  Only numbers are stored: the inputs, verts_uv, faces_uv and the texture.
Outputs: tests/golden/texture_<case>.npz
"""
import math
import os
import sys
import textwrap
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from oracle import field_oracle as fo  # noqa: E402
from oracle import meshbind_oracle as mbo  # noqa: E402
from sugar_b200 import meshbind, scenes  # noqa: E402

SRC = "/root/reference/sugar_scene/sugar_model.py"
BLOCKS = ((2478, 2605), (730, 736))
SH_C0 = 0.28209479177387814
# soup: random triangles of size ~1; heightfield: a permuted scenes.height_field_mesh
CASES = {"f1_n1_s10": dict(mesh="soup", F=1, n=1, s=10, seed=51),
         "f1_n6_s3": dict(mesh="soup", F=1, n=6, s=3, seed=52),
         "f7_n6_s10": dict(mesh="soup", F=7, n=6, s=10, seed=53),
         "f7_n1_s3": dict(mesh="soup", F=7, n=1, s=3, seed=54),
         "heightfield_n6_s10": dict(mesh="heightfield", F=None, n=6, s=10, seed=55),
         "heightfield_n1_s4": dict(mesh="heightfield", F=None, n=1, s=4, seed=56)}


def make_inputs(mesh, F, n, s, seed):
    g = torch.Generator().manual_seed(seed)
    if mesh == "soup":
        verts = torch.randn(3 * F, 3, generator=g)
        faces = torch.arange(3 * F).view(F, 3)
        size = 1.0
    else:
        v, f = scenes.height_field_mesh(12, 10, seed=seed, permute=True)
        verts, faces = torch.from_numpy(v), torch.from_numpy(f)
        F, size = faces.shape[0], 1.0 / 11
    P = F * n
    scales_raw = torch.randn(P, 2, generator=g) * 0.3 + math.log(0.3 * size)
    complex_raw = torch.randn(P, 2, generator=g)
    points, scaling, quats = mbo.bind_to_mesh_torch(verts, faces, meshbind.bary_coords(n), scales_raw, complex_raw,
                                                    1e-3 * size)
    sh_dc = torch.randn(P, 3, generator=g) * 0.8
    return dict(verts=verts.float(), faces=faces.long(), points=points.float(), scaling=scaling.float(),
                quaternions=quats.float(), sh_dc=sh_dc.float(), n=n, square_size=s)


def reference_texture(codes, inp):
    class Mesh:
        def verts_list(self):
            return [inp["verts"]]

        def faces_list(self):
            return [inp["faces"]]

    class Model:
        surface_mesh = Mesh()
        n_gaussians_per_surface_triangle = inp["n"]
        points = inp["points"]
        scaling = inp["scaling"]
        quaternions = inp["quaternions"]
        sh_coordinates = inp["sh_dc"][:, None, :]
        device = "cpu"

    rc = Model()
    ns = dict(torch=torch, quaternion_to_matrix=fo.quaternion_to_matrix)
    exec(codes[1], ns)
    rc.get_covariance = types.MethodType(ns["get_covariance"], rc)
    ns = dict(torch=torch, np=np, rc=rc, square_size=inp["square_size"], n_sh=1, texture_with_gaussian_renders=True,
              SH2RGB=lambda x: x * SH_C0 + 0.5)
    exec(codes[0], ns)
    return ns["verts_uv"], ns["faces_uv"], ns["texture_img"]


def main():
    lines = open(SRC).read().splitlines()
    codes = [compile(textwrap.dedent("\n".join(lines[a - 1:b])), f"sugar_model.py:{a}-{b}", "exec") for a, b in BLOCKS]
    for name, cfg in CASES.items():
        inp = make_inputs(**cfg)
        verts_uv, faces_uv, tex = reference_texture(codes, inp)
        print(name, tuple(tex.shape), int(inp["faces"].shape[0]), "faces",
              float((tex != 0.5).any(-1).float().mean()), "owned")
        np.savez_compressed(os.path.join(HERE, f"texture_{name}.npz"),
                            verts_uv=verts_uv.numpy(), faces_uv=faces_uv.numpy(), texture=tex.numpy(),
                            **{k: (v.numpy() if torch.is_tensor(v) else np.asarray(v)) for k, v in inp.items()})


if __name__ == "__main__":
    main()
