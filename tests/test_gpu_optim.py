"""sugar_b200.optim.Adam (csrc/sgr_adam.cu) against torch.optim.Adam(foreach=True) on the same device, bit for bit: one
step over SuGaR's six groups with a misaligned view, a group without gradient and one at lr 0, at step 1 and 10 000;
200 steps interleaved with the Densifier; state moved between the two optimizers in both directions."""
import copy
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from sugar_b200 import densify, optim  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SHAPES = {"points": (3,), "sh_dc": (1, 3), "sh_rest": (15, 3), "densities": (1,), "scales": (3,), "quaternions": (4,)}
LRS = {"points": 1.6e-4 * 2.7, "sh_dc": 0.0025, "sh_rest": 0.0025 / 20, "densities": 0.05, "scales": 0.005,
       "quaternions": 0.001}


def bits(t):
    return t.detach().contiguous().view(torch.int32)


def same(a, b):
    return a.shape == b.shape and torch.equal(bits(a), bits(b))


def make_raw(P, seed, misaligned=()):
    g = torch.Generator(device=DEV).manual_seed(seed)
    raw = {}
    for k, s in SHAPES.items():
        n = P * int(torch.tensor(s).prod())
        if k in misaligned:   # a parameter that is a view one float into a larger buffer
            buf = torch.randn(n + 1, generator=g, device=DEV)
            raw[k] = torch.nn.Parameter(buf[1:].view((P,) + s))
            assert raw[k].data_ptr() % 16 == 4
        else:
            raw[k] = torch.nn.Parameter(torch.randn((P,) + s, generator=g, device=DEV))
    return raw


def clone_raw(raw):
    out = {}
    for k, v in raw.items():
        if v.data_ptr() % 16:   # keep the same misalignment
            buf = torch.empty(v.numel() + 1, device=DEV)
            buf[1:].copy_(v.detach().reshape(-1))
            out[k] = torch.nn.Parameter(buf[1:].view(v.shape))
        else:
            out[k] = torch.nn.Parameter(v.detach().clone())
    return out


def groups(raw, lrs):
    return [{"params": [raw[k]], "lr": lrs[k], "name": k} for k in SHAPES]


def set_grads(raws, seed, skip=(), scale=1e-3, misaligned=()):
    """The same gradients on every raw dict; for `misaligned` keys the first dict's gradient is a view one float into
    a larger buffer (the others get aligned copies)."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    for k in SHAPES:
        shape = raws[0][k].shape
        if k in skip:
            for r in raws:
                r[k].grad = None
            continue
        buf = torch.randn(shape.numel() + 1, generator=g, device=DEV) * scale
        grad = buf[1:].view(shape) if k in misaligned else buf[:-1].view(shape)
        grad[::7] = 0.0       # exact zeros, as invisible Gaussians have
        for i, r in enumerate(raws):
            r[k].grad = grad if i == 0 else grad.clone()


def compare(ours, ref, raw_a, raw_b, label):
    """Every parameter, moment and step count equal; a failure names the tensors that differ and in how many
    entries (exp_avg is the lerp, exp_avg_sq the mul and addcmul, the parameter the rest)."""
    bad = []
    for k in SHAPES:
        sa, sb = ours.state.get(raw_a[k], {}), ref.state.get(raw_b[k], {})
        assert set(sa) == set(sb), (label, k)
        pairs = [("param", raw_a[k], raw_b[k])]
        if sa:
            assert sa["step"].dtype == sb["step"].dtype == torch.float32 and not sa["step"].is_cuda
            assert float(sa["step"]) == float(sb["step"]), (label, k)
            pairs += [(m, sa[m], sb[m]) for m in ("exp_avg", "exp_avg_sq")]
        for name, a, b in pairs:
            assert a.shape == b.shape, (label, k, name)
            n = int((bits(a) != bits(b)).sum())
            if n:
                bad.append(f"{k}.{name}: {n} of {a.numel()} differ, max |diff| {float((a - b).abs().max()):.3g}")
    assert not bad, (label, bad)


@pytest.mark.parametrize("start_step,betas", [(0, (0.9, 0.999)), (9999, (0.9, 0.999)), (4, (0.3, 0.99))])
def test_one_step_bit_identical_to_torch_foreach(start_step, betas):
    """betas (0.3, 0.99): 1 - beta1 >= 0.5 takes ATen's other lerp branch, g - (g - m)(1 - w)."""
    P = 100_003
    mis = ("sh_rest",)
    lrs = dict(LRS, scales=0.0)                  # one group at lr 0
    raw_a = make_raw(P, 1, misaligned=mis)
    raw_b = clone_raw(raw_a)
    assert raw_b["sh_rest"].data_ptr() % 16 == 4
    ours = optim.Adam(groups(raw_a, lrs), lr=0.0, betas=betas, eps=1e-15)
    ref = torch.optim.Adam(groups(raw_b, lrs), lr=0.0, betas=betas, eps=1e-15, foreach=True)
    if start_step:
        # a state far into training: moments from a first step, then the counter moved on
        set_grads([raw_a, raw_b], 2, misaligned=mis)
        ours.step(), ref.step()
        compare(ours, ref, raw_a, raw_b, "first step")
        for k in SHAPES:
            g = torch.Generator(device=DEV).manual_seed(3)
            m = torch.randn(raw_a[k].shape, generator=g, device=DEV) * 1e-3
            v = torch.rand(raw_a[k].shape, generator=g, device=DEV) * 1e-6
            for opt, r in ((ours, raw_a), (ref, raw_b)):
                st = opt.state[r[k]]
                st["exp_avg"].copy_(m), st["exp_avg_sq"].copy_(v)
                st["step"].fill_(start_step)
    set_grads([raw_a, raw_b], 4, skip=("densities",), misaligned=mis)   # one group without a gradient
    before = raw_a["densities"].detach().clone()
    ours.step(), ref.step()
    compare(ours, ref, raw_a, raw_b, f"step {start_step + 1}")
    assert same(raw_a["densities"], before)
    if start_step == 0:
        assert raw_a["densities"] not in ours.state
    else:
        assert float(ours.state[raw_a["densities"]]["step"]) == start_step   # not advanced
        assert float(ours.state[raw_a["points"]]["step"]) == start_step + 1


def test_step_reads_nothing_back_and_is_one_launch():
    from sugar_b200 import _lib
    raw = make_raw(1000, 5)
    opt = optim.SugarOptimizer(raw, spatial_lr_scale=2.0)
    set_grads([raw], 6)
    opt.step()
    torch.cuda.synchronize()
    n0 = _lib.lib.sgr_launch_count()
    torch.cuda.set_sync_debug_mode("error")
    try:
        opt.update_learning_rate(10)
        opt.step()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert _lib.lib.sgr_launch_count() - n0 == 1
    assert [g["name"] for g in opt.param_groups] == ["points", "sh_coordinates_dc", "sh_coordinates_rest",
                                                     "all_densities", "scales", "quaternions"]
    assert opt.param_groups[0]["lr"] == optim.expon_lr(1.6e-4 * 2.0, 1.6e-6 * 2.0, max_steps=30_000)(10)


def test_rejects_bad_state_before_changing_any():
    raw = make_raw(10, 7)
    opt = optim.Adam([raw["points"]])
    raw["points"].grad = torch.ones_like(raw["points"])
    opt.step()
    opt.state[raw["points"]]["exp_avg"] = torch.zeros(5, 3, device=DEV)
    with pytest.raises(ValueError, match="exp_avg"):
        opt.step()
    assert float(opt.state[raw["points"]]["step"]) == 1.0   # nothing advanced by the refused step


def test_200_steps_with_the_densifier_bit_identical():
    P = 6000
    raw_a = make_raw(P, 11)
    with torch.no_grad():
        for r in (raw_a,):
            r["scales"].copy_(torch.log(torch.empty_like(r["scales"]).uniform_(0.004, 0.03)))
            r["densities"].add_(2.0)
    raw_b = clone_raw(raw_a)
    ours = optim.Adam(groups(raw_a, LRS), lr=0.0, eps=1e-15)
    ref = torch.optim.Adam(groups(raw_b, LRS), lr=0.0, eps=1e-15, foreach=True)
    da = densify.Densifier(raw_a, ours, scene_extent=1.0)
    db = densify.Densifier(raw_b, ref, scene_extent=1.0)
    events = []
    for it in range(1, 201):
        set_grads([raw_a, raw_b], 100 + it, skip=("sh_rest",) if it % 9 == 0 else ())
        ours.step(), ref.step()
        ours.zero_grad(set_to_none=True), ref.zero_grad(set_to_none=True)
        if it % 25 == 0:
            g = torch.Generator(device=DEV).manual_seed(it)
            n = raw_a["points"].shape[0]
            denom = torch.randint(1, 5, (n, 1), generator=g, device=DEV).float()
            accum = denom * torch.where(torch.rand(n, 1, generator=g, device=DEV) < 0.08, 4e-4, 1e-5)
            for d in (da, db):
                d.accum.copy_(accum), d.denom.copy_(denom)
                d.densify_and_prune(max_screen_size=20, generator=torch.Generator(device=DEV).manual_seed(it))
            events.append(("densify", it, raw_a["points"].shape[0]))
        if it in (60, 140):
            mask = torch.rand(raw_a["points"].shape[0], generator=torch.Generator(device=DEV).manual_seed(it),
                              device=DEV) < 0.1
            da.prune_points(mask), db.prune_points(mask)
            events.append(("prune", it, raw_a["points"].shape[0]))
        if it == 100:
            da.reset_opacity(), db.reset_opacity()
        compare(ours, ref, raw_a, raw_b, f"iteration {it}")
    print("events:", events)
    sizes = [n for _, _, n in events]
    assert len(set(sizes)) > 3, sizes   # the model grew and shrank


@pytest.mark.parametrize("direction", ["ours_to_torch", "torch_to_ours"])
def test_state_dict_interchange(direction):
    raw_a = make_raw(2049, 21)
    first = optim.Adam if direction == "ours_to_torch" else torch.optim.Adam
    second = torch.optim.Adam if direction == "ours_to_torch" else optim.Adam
    opt_a = first(groups(raw_a, LRS), lr=0.0, eps=1e-15)
    for i in range(3):
        set_grads([raw_a], 30 + i)
        opt_a.step()
    raw_b = clone_raw(raw_a)
    opt_b = second(groups(raw_b, LRS), lr=0.0, eps=1e-15)
    opt_b.load_state_dict(copy.deepcopy(opt_a.state_dict()))   # load_state_dict may share the tensors
    compare(opt_a, opt_b, raw_a, raw_b, "loaded")
    for i in range(3):
        set_grads([raw_a, raw_b], 40 + i)
        opt_a.step(), opt_b.step()
        compare(opt_a, opt_b, raw_a, raw_b, f"continued {i}")
