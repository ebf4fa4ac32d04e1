"""Golden vectors for the refined mesh's post-processing from the reference's OWN code.

Runs in the build container (needs /root/reference):  python tests/golden/make_postprocess_golden.py
The `--postprocess_mesh` branch needs a SuGaR model, pytorch3d and open3d.  This script reads exactly
sugar_extractors/refined_mesh.py:128-162 (edge entries, erosion, re-admission, compaction) and
sugar_scene/sugar_model.py:730-750 (get_covariance) and :1335-1368 (get_gaussians_closest_to_samples,
compute_density) from /root/reference at run time, dedents the lines and executes them unchanged, in float32 on the
CPU, with a duck-typed `refined_sugar` (surface_mesh.verts_list() / faces_list() / faces_normals_list(), strengths,
points, scaling, quaternions, _scales, _quaternions, all_densities, _sh_coordinates_dc, _sh_coordinates_rest, device)
and a stub CONSOLE.  pytorch3d's knn_points and quaternion_to_matrix are the restatements of
oracle/postprocess_oracle.py and oracle/field_oracle.py; the Gaussians are bound to the mesh with
oracle/meshbind_oracle.py.  n = 1 only: the reference's branch raises above that.

A case is rejected (and its seed advanced) when an eroded face's density is within 1e-4 relative of float32(threshold)
or a centre's 16th and 17th neighbour distances are within 1e-6 relative, so that a GPU evaluation in another order
decides every face as the reference does.  Only numbers are stored: the inputs, face_mask, the compacted tensors and
the eroded faces' densities.
Outputs: tests/golden/postprocess_<case>.npz
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
from oracle import postprocess_oracle as ppo  # noqa: E402
from sugar_b200 import meshbind, scenes  # noqa: E402

REF = "/root/reference"
BLOCKS = (("sugar_extractors/refined_mesh.py", 128, 162), ("sugar_scene/sugar_model.py", 730, 750),
          ("sugar_scene/sugar_model.py", 1335, 1368))
THRESHOLD = 0.1
# mesh: icosphere (closed, jittered), holes (icosphere minus a few faces), fan (icosphere with a 3-face fin on one edge, two
# faces with a repeated vertex id sharing their degenerate edge and one alone), heightfield (open, permuted,
# xy-jittered); nan: one strength is NaN
CASES = {"icosphere": dict(mesh="icosphere", iterations=5, seed=61),
         "holes": dict(mesh="holes", iterations=5, seed=62),
         "fan": dict(mesh="fan", iterations=5, seed=63),
         "heightfield_it0": dict(mesh="heightfield", iterations=0, seed=64),
         "heightfield_it1": dict(mesh="heightfield", iterations=1, seed=64),
         "heightfield_it5": dict(mesh="heightfield", iterations=5, seed=64),
         "heightfield_it12": dict(mesh="heightfield", iterations=12, seed=64),
         "nan": dict(mesh="heightfield", iterations=2, seed=65, nan=True)}


def make_mesh(mesh, seed):
    g = np.random.default_rng(seed)
    if mesh == "heightfield":
        v, f = scenes.height_field_mesh(9, 8, seed=seed, permute=True)
        v = v.copy()
        v[:, :2] += 0.1 / 8 * g.normal(size=(len(v), 2))            # grid spacing ~1/8: no tied distances
        return v.astype(np.float32), f, 1.0 / 8
    v, f = scenes.icosphere(2)
    v, f = v + 0.01 * g.normal(size=v.shape), f.copy()              # jittered: no tied distances
    if mesh == "holes":
        f = np.delete(f, g.choice(len(f), 6, replace=False), 0)
    elif mesh == "fan":
        a, b = f[0, 0], f[0, 1]
        c, d = next(g[:2] for g in f if a not in g and b not in g)
        tips = len(v) + np.arange(5)
        v = np.concatenate([v, 1.3 * v[[a, b, c, d, a]] + 0.05 * g.normal(size=(5, 3))]).astype(np.float32)
        fin = np.stack([np.full(3, a), np.full(3, b), tips[:3]], 1)                       # 3 more faces on (a, b)
        degenerate = np.array([[c, c, d], [c, c, tips[3]], [a, a, tips[4]]])            # (c, c) twice, (a, a) once
        f = np.concatenate([f, fin, degenerate])
    return v.astype(np.float32), f.astype(np.int64), 0.2


def make_inputs(mesh, iterations, seed, nan=False):
    verts, faces, size = make_mesh(mesh, seed)
    g = torch.Generator().manual_seed(seed)
    verts, faces = torch.from_numpy(verts), torch.from_numpy(faces)
    P = faces.shape[0]
    lo, hi = math.log(0.02 / 0.98), math.log(0.3 / 0.7)            # strengths spread over (0.02, 0.3)
    densities_raw = lo + (hi - lo) * torch.rand(P, 1, generator=g)
    if nan:
        densities_raw[P // 2] = float("nan")
    return dict(verts=verts, faces=faces, n=1, scales_raw=torch.randn(P, 2, generator=g) * 0.2 + math.log(0.3 * size),
                complex_raw=torch.randn(P, 2, generator=g), densities_raw=densities_raw,
                sh_dc=torch.randn(P, 1, 3, generator=g), sh_rest=torch.randn(P, 15, 3, generator=g) * 0.1,
                thickness=1e-3 * size, density_threshold=THRESHOLD, iterations=iterations)


def knn_points(p1, p2, K):
    d2, idx = ppo.knn_points(p1[0], p2[0], K)
    return types.SimpleNamespace(dists=d2.float()[None], idx=idx[None])


def reference_postprocess(codes, inp):
    verts, faces = inp["verts"], inp["faces"]
    points, scaling, quats = mbo.bind_to_mesh_torch(verts, faces, meshbind.bary_coords(1), inp["scales_raw"],
                                                    inp["complex_raw"], inp["thickness"])

    class Mesh:
        def verts_list(self):
            return [verts]

        def faces_list(self):
            return [faces]

        def faces_normals_list(self):
            return [mbo.faces_normals(verts, faces)]

    class Model:
        pass

    rs = Model()
    rs.surface_mesh, rs.device = Mesh(), "cpu"
    rs.points, rs.scaling, rs.quaternions = points.float(), scaling.float(), quats.float()
    rs._scales, rs._quaternions, rs.all_densities = inp["scales_raw"], inp["complex_raw"], inp["densities_raw"]
    rs._sh_coordinates_dc, rs._sh_coordinates_rest = inp["sh_dc"], inp["sh_rest"]
    rs.strengths = torch.sigmoid(rs.all_densities.view(-1, 1))
    ns = dict(torch=torch, quaternion_to_matrix=fo.quaternion_to_matrix, knn_points=knn_points)
    exec(codes[1], ns)
    exec(codes[2], ns)
    for name in ("get_covariance", "get_gaussians_closest_to_samples", "compute_density"):
        setattr(rs, name, types.MethodType(ns[name], rs))
    ns = dict(torch=torch, knn_points=knn_points, refined_sugar=rs, postprocess_iterations=inp["iterations"],
              postprocess_density_threshold=inp["density_threshold"],
              CONSOLE=types.SimpleNamespace(print=lambda *a, **k: None))
    density = rs.compute_density

    def compute_density(x, *a, **k):            # records the mask after the erosion rounds
        ns["eroded_mask"] = ns["face_mask"].clone()
        return density(x, *a, **k)
    rs.compute_density = compute_density
    exec(codes[0], ns)
    return ns, rs.points


def main():
    codes = []
    for path, a, b in BLOCKS:
        lines = open(os.path.join(REF, path)).read().splitlines()
        codes.append(compile(textwrap.dedent("\n".join(lines[a - 1:b])), f"{path}:{a}-{b}", "exec"))
    thr = float(np.float32(THRESHOLD))
    for name, cfg in CASES.items():
        cfg = dict(cfg)
        for attempt in range(20):
            inp = make_inputs(**cfg)
            ns, points = reference_postprocess(codes, inp)
            eroded = torch.nonzero(~ns["eroded_mask"])[:, 0]
            rho = ns["face_densities"]
            d2, _ = ppo.knn_points(inp["verts"][inp["faces"]].mean(-2)[eroded], points, 17)
            near_thr = ((rho.double() - thr).abs() <= 1e-4 * thr).any()
            near_tie = ((d2[:, 16] - d2[:, 15]) <= 1e-6 * d2[:, 16]).any() if len(d2) else False
            if not (near_thr or near_tie):
                break
            print(f"{name}: seed {cfg['seed']} rejected (threshold {bool(near_thr)}, K-NN tie {bool(near_tie)})")
            cfg["seed"] += 1000
        else:
            raise RuntimeError(f"{name}: no unambiguous seed")
        mask = ns["face_mask"]
        print(name, "seed", cfg["seed"], int(inp["faces"].shape[0]), "faces,", len(eroded), "eroded,",
              int((rho > thr).sum()), "re-admitted,", int(mask.sum()), "kept")
        out = dict(face_mask=mask, faces_out=ns["new_faces"], scales_out=ns["new_scales"],
                   quaternions_out=ns["new_quaternions"], densities_out=ns["new_densities"],
                   sh_dc_out=ns["new_sh_coordinates_dc"], sh_rest_out=ns["new_sh_coordinates_rest"],
                   eroded=eroded, eroded_density=rho)
        np.savez_compressed(os.path.join(HERE, f"postprocess_{name}.npz"),
                            **{k: (v.numpy() if torch.is_tensor(v) else np.asarray(v)) for k, v in inp.items()},
                            **{k: v.numpy() for k, v in out.items()})


if __name__ == "__main__":
    main()
