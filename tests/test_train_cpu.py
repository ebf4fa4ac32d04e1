"""sugar_b200.train's schedules without a GPU: the coarse trainers' per-iteration decisions and the refinement's SH
degree against the oracle's restatement of the reference's loops, at every iteration."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import optim_oracle as oo  # noqa: E402
from sugar_b200 import mcubes, train  # noqa: E402

SCALED = dict(regularize_from=10, entropy_window=(10, 20), prune_at=(20,), reset_neighbors_every=7, sdf_from=20)


def _oracle_kw(s):
    return dict(regularize_from=s["regularize_from"], start_entropy_regularization_from=s["entropy_window"][0],
                end_entropy_regularization_at=s["entropy_window"][1], prune_low_opacity_gaussians_at=s["prune_at"],
                reset_neighbors_every=s["reset_neighbors_every"], start_sdf_regularization_from=s["sdf_from"])


def as_events(names):
    """The oracle's ordered list as train's dict (a reset after the prune and one in the regularisation block are
    the same table, built once)."""
    ev = {"sh_degree": 3}
    ev.update({n: True for n in names})
    return ev


@pytest.mark.parametrize("sched,n", [({}, 15_000), (SCALED, 60)])
def test_coarse_phase_matches_the_oracle_at_every_iteration(sched, n):
    full = dict(regularize_from=7000, entropy_window=(7000, 9000), prune_at=(9000,), reset_neighbors_every=500,
                sdf_from=9000)
    full.update(sched)
    for it in range(1, n + 1):
        assert train.coarse_phase(it, **full) == as_events(oo.coarse_events(it, **_oracle_kw(full))), it


def test_coarse_phase_default_schedule():
    ev = {it: train.coarse_phase(it) for it in range(1, 15_001)}
    assert [it for it, e in ev.items() if "entropy" in e] == list(range(7001, 9000))
    assert [it for it, e in ev.items() if "prune" in e] == [9001]
    resets = [it for it, e in ev.items() if "reset_neighbors" in e]
    assert resets == sorted([7001, 9001] + list(range(7500, 15_001, 500)))
    assert [it for it, e in ev.items() if "sdf" in e] == list(range(9001, 15_001))
    assert all(e["sh_degree"] == 3 for e in ev.values())
    # the reference resets twice at an iteration that is both the prune's and a multiple of the period; here once
    assert oo.coarse_events(9001) == ["prune", "reset_neighbors", "sdf"]


def test_coarse_phase_scaled_schedule():
    ev = {it: train.coarse_phase(it, **SCALED) for it in range(1, 41)}
    assert [it for it, e in ev.items() if "entropy" in e] == list(range(11, 20))
    assert [it for it, e in ev.items() if "prune" in e] == [21]
    assert [it for it, e in ev.items() if "reset_neighbors" in e] == [11, 14, 21, 28, 35]
    assert [it for it, e in ev.items() if "sdf" in e] == list(range(21, 41))


@pytest.mark.parametrize("every,n", [(1000, 15_000), (3, 20)])
def test_refine_sh_degree_matches_the_oracle(every, n):
    want = oo.refine_sh_degrees(n, sh_warmup_every=every)
    assert [train.refine_sh_degree(it, every) for it in range(1, n + 1)] == want
    assert [train.refine_phase(it, every) for it in range(1, n + 1)] == [{"sh_degree": d} for d in want]
    if every == 1000:
        steps_at = [it for it in range(2, n + 1) if want[it - 1] != want[it - 2]]
        assert steps_at == [1001, 2001, 3001] and want[0] == 0 and want[-1] == 3


def test_refine_spatial_lr_scale():
    centres = torch.tensor([[0.0, 0.0, 0.0], [2.0, 0.0, 0.0], [0.0, 3.0, 1.0]])
    extent = mcubes.camera_spatial_extent(centres)
    n = 1_000_003
    # refine.py:459: the square root of an int64 tensor is a float32 tensor
    want = 10.0 * extent / float(torch.tensor(n, dtype=torch.float32).sqrt())
    assert train.refine_spatial_lr_scale(n, spatial_extent=extent) == want
    lo, hi = [-1.0, -2.0, 0.5], [3.0, 1.0, 2.0]
    r = float((torch.tensor(hi) - torch.tensor(lo)).norm() / 2.0)
    assert train.refine_spatial_lr_scale(n, fg_bbox=(lo, hi)) == 10.0 * r / float(torch.tensor(float(n)).sqrt())
    with pytest.raises(ValueError):
        train.refine_spatial_lr_scale(n)


def test_entropy_loss_is_the_masked_mean():
    o = torch.tensor([0.1, 0.5, 0.9, 0.999, 1e-6]).view(-1, 1)
    vis = torch.tensor([True, False, True, True, True])
    ov = o[vis]
    want = (-ov * torch.log(ov + 1e-10) - (1 - ov) * torch.log(1 - ov + 1e-10)).mean()
    assert torch.allclose(train.entropy_loss(o, vis), want, rtol=1e-6, atol=0)
    assert torch.isnan(train.entropy_loss(o, torch.zeros(5, dtype=torch.bool)))


@pytest.mark.parametrize("kw,match", [(dict(mode="l2"), "mode"), (dict(spatial_extent=None), "spatial_extent"),
                                      (dict(entropy_window=(10, 30), sdf_from=20, regularize_from=10),
                                       "entropy_window"), (dict(first_iteration=0), "first_iteration")])
def test_train_coarse_checks_arguments(kw, match):
    a = dict(mode="sdf", spatial_extent=1.0)
    a.update(kw)
    with pytest.raises(ValueError, match=match):
        train.train_coarse({}, [None], torch.zeros(4, 16, dtype=torch.int64), **a)
