"""The per-step ops reject arguments split across the CPU and a CUDA device with a ValueError naming the argument."""
import pytest
import torch

from sugar_b200 import field, knn, meshbind

pytestmark = pytest.mark.gpu


def _cloud(P=8, N=5, K=4):
    g = torch.Generator().manual_seed(0)
    c = dict(x=torch.randn(N, 3, generator=g), idx=torch.randint(0, P, (N, K), generator=g),
             points=torch.randn(P, 3, generator=g), scaling=torch.rand(P, 3, generator=g) + 0.1,
             quaternions=torch.nn.functional.normalize(torch.randn(P, 4, generator=g), dim=-1),
             strengths=torch.rand(P, 1, generator=g), opac=torch.rand(N, K, generator=g))
    return {k: v.cuda() for k, v in c.items()}


def test_knn_points_rejects_split_devices():
    c = _cloud()
    with pytest.raises(ValueError, match="p2"):
        knn.knn_points(c["x"], c["points"].cpu(), 4)


@pytest.mark.parametrize("arg", ["closest_gaussians_idx", "points", "scaling", "quaternions", "strengths"])
def test_field_rejects_split_devices(arg):
    c = _cloud()
    a = dict(x=c["x"], closest_gaussians_idx=c["idx"], points=c["points"], scaling=c["scaling"],
             quaternions=c["quaternions"], strengths=c["strengths"])
    a[arg] = a[arg].cpu()
    with pytest.raises(ValueError, match=arg):
        field.field_values(**a)
    with pytest.raises(ValueError, match=arg):
        field.compute_density(**a)


@pytest.mark.parametrize("arg", ["gaussian_idx", "closest_gaussians_idx", "points", "scaling", "quaternions",
                                 "closest_gaussian_opacities"])
def test_better_normal_loss_rejects_split_devices(arg):
    c = _cloud()
    a = dict(x=c["x"], gaussian_idx=c["idx"][:, 0], closest_gaussians_idx=c["idx"], points=c["points"],
             scaling=c["scaling"], quaternions=c["quaternions"], closest_gaussian_opacities=c["opac"])
    a[arg] = a[arg].cpu()
    with pytest.raises(ValueError, match=arg):
        field.better_normal_loss(**a)


@pytest.mark.parametrize("arg", ["faces", "bary", "scales_raw", "complex_raw"])
def test_bind_to_mesh_rejects_split_devices(arg):
    F, n = 2, 3
    a = dict(verts=torch.randn(4, 3, device="cuda"), faces=torch.tensor([[0, 1, 2], [1, 2, 3]], device="cuda"),
             bary=meshbind.bary_coords(n, "cuda"), scales_raw=torch.zeros(F * n, 2, device="cuda"),
             complex_raw=torch.zeros(F * n, 2, device="cuda"), thickness=0.01)
    a[arg] = a[arg].cpu()
    with pytest.raises(ValueError, match=arg):
        meshbind.bind_to_mesh(**a)
