"""Golden SuGaR models and checkpoint files from the reference's OWN code.

Runs in the build container (needs /root/reference):  python tests/golden/make_pipeline_golden.py
SuGaR is imported through make_field_golden.import_reference_sugar's stubs and constructed on the CPU with a duck-typed
`nerfmodel` (device, training_cameras with get_spatial_extent, height, width, fx, fy and p3d_cameras.K) and an
open3d-like mesh (vertices float64, triangles int32, vertex_colors uint8 / 255 in float64), so the arithmetic of the
bound constructor (sugar_model.py:149-361) is the reference's.  Outputs, under tests/golden/:

    pipeline_bound_n{1,3,4,6}.pt  {"inputs": verts, faces, vertex_colors, extent; "state_dict": SuGaR.state_dict()}
                                  of refine.py's bound model (learn positions, opacities, scales), n Gaussians per face
    pipeline_bound_degenerate_n4.pt  the same over a mesh with a zero-length edge (the 1e-7 clamp)
    pipeline_unbound.pt           {"inputs": the 3DGS tensors; "state_dict"} of coarse_sdf.py's model: initialize=False,
                                  then the 3DGS parameters copied in as coarse_sdf.py:389-394 does
    pipeline_save_model_bound.pt  SuGaR.save_model's file of the n = 3 model, with train_losses, epoch, iteration and a
                                  SuGaROptimizer's state_dict after two Adam steps on fixed gradients
"""
import os
import sys
from types import SimpleNamespace

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_field_golden import import_reference_sugar  # noqa: E402


def fake_nerfmodel(extent, W=64, H=48, f=50.0):
    cams = SimpleNamespace(get_spatial_extent=lambda: extent, height=torch.tensor([H]), width=torch.tensor([W]),
                           fx=torch.tensor([f]), fy=torch.tensor([f]),
                           p3d_cameras=SimpleNamespace(K=torch.tensor([[[f, 0, 0, 0], [0, f, 0, 0], [0, 0, 0, 1],
                                                                        [0, 0, 1, 0]]])))
    return SimpleNamespace(device="cpu", training_cameras=cams)


def icosphere_like(seed, degenerate=False):
    """An icosahedron, jittered, with uint8 colours; `degenerate` welds two corners of face 0 into one point."""
    t = (1.0 + 5 ** 0.5) / 2.0
    v = np.array([[-1, t, 0], [1, t, 0], [-1, -t, 0], [1, -t, 0], [0, -1, t], [0, 1, t], [0, -1, -t], [0, 1, -t],
                  [t, 0, -1], [t, 0, 1], [-t, 0, -1], [-t, 0, 1]], np.float64)
    f = np.array([[0, 11, 5], [0, 5, 1], [0, 1, 7], [0, 7, 10], [0, 10, 11], [1, 5, 9], [5, 11, 4], [11, 10, 2],
                  [10, 7, 6], [7, 1, 8], [3, 9, 4], [3, 4, 2], [3, 2, 6], [3, 6, 8], [3, 8, 9], [4, 9, 5],
                  [2, 4, 11], [6, 2, 10], [8, 6, 7], [9, 8, 1]], np.int32)
    rng = np.random.default_rng(seed)
    v = v * 0.37 + 0.05 * rng.standard_normal(v.shape) + np.array([0.3, -0.2, 1.1])
    if degenerate:
        v[11] = v[0]             # face 0 = (0, 11, 5): a zero-length edge
    u8 = rng.integers(0, 256, size=(len(v), 3), dtype=np.uint8)
    return v, f, u8


def bound_model(sm, v, f, u8, n, extent):
    mesh = SimpleNamespace(vertices=v, triangles=f, vertex_colors=u8.astype(np.float64) / 255.0)
    pts = torch.tensor(v).float()
    return sm.SuGaR(nerfmodel=fake_nerfmodel(extent), points=pts, colors=torch.zeros_like(pts), initialize=True,
                    sh_levels=4, learnable_positions=True, triangle_scale=1.0, keep_track_of_knn=False,
                    knn_to_track=16, beta_mode="average", freeze_gaussians=False, surface_mesh_to_bind=mesh,
                    surface_mesh_thickness=None, learn_surface_mesh_positions=True, learn_surface_mesh_opacity=True,
                    learn_surface_mesh_scales=True, n_gaussians_per_surface_triangle=n)


def inputs(v, f, u8, extent):
    return {"verts": torch.tensor(v), "faces": torch.tensor(f), "vertex_colors_u8": torch.tensor(u8),
            "extent": extent}


def main():
    sm = import_reference_sugar()
    from sugar_scene.sugar_optimizer import OptimizationParams, SuGaROptimizer
    extent = 3.7
    for n in (1, 3, 4, 6):
        v, f, u8 = icosphere_like(n)
        model = bound_model(sm, v, f, u8, n, extent)
        torch.save({"inputs": inputs(v, f, u8, extent), "state_dict": model.state_dict()},
                   os.path.join(HERE, f"pipeline_bound_n{n}.pt"))
        print(f"n={n}", [(k, tuple(t.shape), str(t.dtype)) for k, t in model.state_dict().items()])
    v, f, u8 = icosphere_like(7, degenerate=True)
    model = bound_model(sm, v, f, u8, 4, extent)
    assert float(model._scales[0, 0].detach()) == float(np.log(np.float32(1e-7)))
    torch.save({"inputs": inputs(v, f, u8, extent), "state_dict": model.state_dict()},
               os.path.join(HERE, "pipeline_bound_degenerate_n4.pt"))

    # the coarse model: the 3DGS tensors copied into an unbound SuGaR
    g = torch.Generator().manual_seed(5)
    P = 40
    gs = {"xyz": torch.randn(P, 3, generator=g), "features_dc": torch.randn(P, 1, 3, generator=g),
          "features_rest": torch.randn(P, 15, 3, generator=g), "opacity": torch.randn(P, 1, generator=g),
          "scaling": torch.randn(P, 3, generator=g) - 3.0, "rotation": torch.randn(P, 4, generator=g)}
    model = sm.SuGaR(nerfmodel=fake_nerfmodel(extent), points=gs["xyz"].clone(),
                     colors=gs["features_dc"][:, 0] * 0.28209479177387814 + 0.5, initialize=False, sh_levels=4,
                     learnable_positions=True, triangle_scale=1.0, keep_track_of_knn=False, beta_mode="average",
                     surface_mesh_to_bind=None)
    with torch.no_grad():
        model._scales[...] = gs["scaling"]
        model._quaternions[...] = gs["rotation"]
        model.all_densities[...] = gs["opacity"]
        model._sh_coordinates_dc[...] = gs["features_dc"]
        model._sh_coordinates_rest[...] = gs["features_rest"]
    torch.save({"inputs": gs, "state_dict": model.state_dict()}, os.path.join(HERE, "pipeline_unbound.pt"))

    # save_model's file of a bound model, with a reference optimizer's state after two steps
    v, f, u8 = icosphere_like(3)
    model = bound_model(sm, v, f, u8, 3, extent)
    opt = SuGaROptimizer(model, OptimizationParams(iterations=100), spatial_lr_scale=0.8)
    for it in (1, 2):
        opt.update_learning_rate(it)
        for p in (model._points, model._sh_coordinates_dc, model._sh_coordinates_rest, model.all_densities,
                  model._scales, model._quaternions):
            p.grad = torch.randn(p.shape, generator=g)
        opt.step()
        opt.zero_grad(set_to_none=True)
    model.save_model(os.path.join(HERE, "pipeline_save_model_bound.pt"), train_losses=[0.25, 0.125], epoch=2,
                     iteration=2, optimizer_state_dict=opt.state_dict())


if __name__ == "__main__":
    main()
