"""The per-step ops check their tensors' shapes before the CUDA requirement, so a wrong shape raises ValueError
naming the argument instead of a kernel reading past a tensor (no GPU needed)."""
import pytest
import torch

from sugar_b200 import field, knn, meshbind


def _cloud(P=8, N=5, K=4):
    g = torch.Generator().manual_seed(0)
    return dict(x=torch.randn(N, 3, generator=g), idx=torch.randint(0, P, (N, K), generator=g),
                points=torch.randn(P, 3, generator=g), scaling=torch.rand(P, 3, generator=g) + 0.1,
                quaternions=torch.nn.functional.normalize(torch.randn(P, 4, generator=g), dim=-1),
                strengths=torch.rand(P, 1, generator=g), opac=torch.rand(N, K, generator=g))


def test_knn_points_checks_shapes():
    c = _cloud()
    with pytest.raises(ValueError, match="p1"):
        knn.knn_points(c["x"][:, :2], c["points"], 4)
    with pytest.raises(ValueError, match="p2"):
        knn.knn_points(c["x"], c["points"].reshape(-1), 4)
    with pytest.raises(ValueError, match="p2"):
        knn.knn_points(c["x"], torch.stack([c["points"], c["points"]]), 4)


@pytest.mark.parametrize("arg,bad", [("x", lambda t: t[:, :2]), ("points", lambda t: t[:, :2]),
                                     ("scaling", lambda t: t[1:]), ("quaternions", lambda t: t[:, :3]),
                                     ("strengths", lambda t: t[1:]), ("closest_gaussians_idx", lambda t: t[:, 0])])
def test_field_checks_shapes(arg, bad):
    c = _cloud()
    a = dict(x=c["x"], closest_gaussians_idx=c["idx"], points=c["points"], scaling=c["scaling"],
             quaternions=c["quaternions"], strengths=c["strengths"])
    a[arg] = bad(a[arg])
    with pytest.raises(ValueError, match=arg):
        field.field_values(**a)
    with pytest.raises(ValueError, match=arg):
        field.compute_density(**a)


@pytest.mark.parametrize("arg,bad", [("x", lambda t: t[:, :2]), ("gaussian_idx", lambda t: t[1:]),
                                     ("closest_gaussians_idx", lambda t: t[1:]), ("points", lambda t: t[:, :2]),
                                     ("scaling", lambda t: t[1:]), ("quaternions", lambda t: t[:, :3]),
                                     ("closest_gaussian_opacities", lambda t: t[:, 1:])])
def test_better_normal_loss_checks_shapes(arg, bad):
    c = _cloud()
    a = dict(x=c["x"], gaussian_idx=c["idx"][:, 0], closest_gaussians_idx=c["idx"], points=c["points"],
             scaling=c["scaling"], quaternions=c["quaternions"], closest_gaussian_opacities=c["opac"])
    a[arg] = bad(a[arg])
    with pytest.raises(ValueError, match=arg):
        field.better_normal_loss(**a)


@pytest.mark.parametrize("arg,bad", [("verts", lambda t: t[:, :2]), ("faces", lambda t: t.reshape(-1)),
                                     ("bary", lambda t: t[:, :2])])
def test_bind_to_mesh_checks_shapes(arg, bad):
    F, n = 2, 3
    a = dict(verts=torch.randn(4, 3), faces=torch.tensor([[0, 1, 2], [1, 2, 3]]), bary=meshbind.bary_coords(n),
             scales_raw=torch.zeros(F * n, 2), complex_raw=torch.zeros(F * n, 2), thickness=0.01)
    a[arg] = bad(a[arg])
    with pytest.raises(ValueError, match=arg):
        meshbind.bind_to_mesh(**a)


def test_valid_cpu_arguments_reach_the_cuda_requirement():
    c = _cloud()
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        knn.knn_points(c["x"], c["points"], 4)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        field.field_values(c["x"], c["idx"], c["points"], c["scaling"], c["quaternions"], c["strengths"])
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        field.better_normal_loss(c["x"], c["idx"][:, 0], c["idx"], c["points"], c["scaling"], c["quaternions"],
                                 c["opac"])
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        meshbind.bind_to_mesh(torch.randn(3, 3), torch.tensor([[0, 1, 2]]), meshbind.bary_coords(1)[:, :, None],
                              torch.zeros(1, 2), torch.zeros(1, 2), 0.01)
