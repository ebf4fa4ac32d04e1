"""CPU restatement of the coarse_density trainer's density estimation loss -- TEST INFRASTRUCTURE ONLY.

The trainer's projection-mode branch (sugar_trainers/coarse_density.py:642-656, 684-691; the trainer's settings
sdf_estimation_mode='density', use_projection_as_estimation=True, squared_sdf_estimation_loss=False, :121-156) in
PyTorch, on top of field_oracle.field_values_torch (get_field_values, sugar_model.py:1247-1316) and
field_oracle.smallest_axis (get_normals(estimate_from_points=False), :930-945).  Works in any float dtype.

tests/golden/densest_*.npz were produced by executing those trainer lines as they stand against a duck-typed SuGaR
(tests/golden/make_densest_golden.py); tests/test_density_estimation_cpu.py checks this file against them.
"""
import torch

from oracle.field_oracle import field_values_torch, smallest_axis


def density_estimation_loss_torch(x, gaussian_idx, nbr_idx, points, scaling, quaternions, strengths,
                                  density_factor=1.0, return_closest_gaussian_opacities=False):
    """Per-sample |rho - exp(-0.5 e^2 / beta^2)| [N]; tensors may require grad.  rho is fields['density'], the sum
    before the straight-through clamp (:1279), so rho >= 1 is not clamped here."""
    fields = field_values_torch(x, nbr_idx, points, scaling, quaternions, strengths, density_factor)
    normals = smallest_axis(scaling, quaternions)[gaussian_idx]                              # :655
    e = ((x - points[gaussian_idx]) * normals).sum(dim=-1)                                   # :656
    target = torch.exp(-0.5 * e.pow(2) / fields["beta"].pow(2))                              # :686
    loss = (fields["density"] - target).abs()                                                # :690
    if return_closest_gaussian_opacities:
        return loss, fields["closest_gaussian_opacities"].detach()
    return loss

