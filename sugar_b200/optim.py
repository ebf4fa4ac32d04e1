"""The trainers' optimizer: Adam as one CUDA launch over every parameter group (csrc/sgr_adam.cu), SuGaR's group table
and its position learning-rate schedule (sugar_scene/sugar_optimizer.py, sugar_utils/general_utils.py).

    opt = SugarOptimizer(raw, spatial_lr_scale=extent)       # the six groups over steps.py's raw dict
    opt.update_learning_rate(iteration)                       # the points group's exponential decay
    loss.backward(); opt.step(); opt.zero_grad(set_to_none=True)

`Adam` is a drop-in for torch.optim.Adam(params, lr, betas, eps) in its default (foreach) form: a step is bit-identical
to torch's, and its state uses torch's keys and types (`step` a CPU float32 scalar tensor, `exp_avg`, `exp_avg_sq`), so
`Densifier` re-keys it, `state_dict()` / `load_state_dict()` work, and state moves between the two optimizers in both
directions.  It reads and writes each element once (28 B per float32 parameter) where torch's foreach Adam runs seven
elementwise passes and allocates a temporary the size of every parameter.  Weight decay, AMSGrad, maximize and sparse
gradients are not supported (SuGaR uses none of them) and raise ValueError, as do parameters that are not contiguous
float32 CUDA tensors.
"""
import numpy as np
import torch

from ._lib import SGR_ADAM_MAX_SEGMENTS, SgrAdamSegment, check, lib, stream


def _check_param(p, name="params"):
    if not torch.is_tensor(p) or p.dtype != torch.float32:
        raise ValueError(f"{name} must be float32 tensors, got {p.dtype if torch.is_tensor(p) else type(p).__name__}")
    if not p.is_contiguous():
        raise ValueError(f"{name} must be contiguous (a parameter of shape {tuple(p.shape)} is not)")
    if not p.is_cuda:
        raise ValueError(f"{name} must be CUDA tensors, got one on {p.device} (sugar_b200 has no CPU path)")


def dense_grad(p):
    """-> p.grad as the kernel reads it (contiguous float32 of p's shape), or None.  Raises ValueError naming `grad` for
    a sparse gradient or one of another dtype or shape."""
    g = p.grad
    if g is None:
        return None
    if g.is_sparse:
        raise ValueError("grad: sparse gradients are not supported (Adam here is the dense update)")
    if g.dtype != torch.float32 or g.shape != p.shape or g.device != p.device:
        raise ValueError(f"grad must be float32 {tuple(p.shape)} on {p.device}, got {g.dtype} {tuple(g.shape)} on "
                         f"{g.device}")
    return g.contiguous()


class Adam(torch.optim.Optimizer):
    """torch.optim.Adam(params, lr, betas, eps) with one sgr_adam_step launch per step (see the module docstring)."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, amsgrad=False,
                 maximize=False):
        if not 0.0 <= lr:
            raise ValueError(f"lr must be >= 0, got {lr}")
        if not 0.0 <= eps:
            raise ValueError(f"eps must be >= 0, got {eps}")
        if len(betas) != 2 or not all(0.0 <= b < 1.0 for b in betas):
            raise ValueError(f"betas must be two values in [0, 1), got {betas}")
        defaults = dict(lr=lr, betas=tuple(betas), eps=eps, weight_decay=weight_decay, amsgrad=amsgrad,
                        maximize=maximize)
        self._check_options(defaults)
        super().__init__(params, defaults)

    @staticmethod
    def _check_options(group):
        if group.get("weight_decay", 0.0) != 0:
            raise ValueError(f"weight_decay must be 0, got {group['weight_decay']} (not supported)")
        if group.get("amsgrad", False):
            raise ValueError("amsgrad is not supported")
        if group.get("maximize", False):
            raise ValueError("maximize is not supported")

    def add_param_group(self, param_group):
        super().add_param_group(param_group)
        group = self.param_groups[-1]
        self._check_options(group)
        for p in group["params"]:
            _check_param(p)

    @torch.no_grad()
    def step(self, closure=None):
        """One Adam step of every parameter that has a gradient; parameters without one are skipped and their step
        count is not advanced.  One launch on the current stream (per 8 tensors); no host synchronisation."""
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        todo, dev = [], None
        for group in self.param_groups:   # every check before any state changes
            self._check_options(group)
            for p in group["params"]:
                g = dense_grad(p)
                if g is None:
                    continue
                _check_param(p)
                if dev is None:
                    dev = p.device
                elif p.device != dev:
                    raise ValueError(f"params must share one device, got {dev} and {p.device}")
                state = self.state[p]
                for name in ("exp_avg", "exp_avg_sq"):
                    t = state.get(name)
                    if t is not None and (t.shape != p.shape or t.dtype != torch.float32 or t.device != p.device or
                                          not t.is_contiguous()):
                        raise ValueError(f"state {name} must be contiguous float32 {tuple(p.shape)} on {p.device}")
                todo.append((group, p, g, state))
        segs = []
        for group, p, g, state in todo:
            if len(state) == 0:
                state["step"] = torch.tensor(0.0, dtype=torch.float32)
                state["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                state["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
            lr, (beta1, beta2), eps = group["lr"], group["betas"], group["eps"]
            if torch.is_tensor(lr):
                lr = lr.item()
            # torch's foreach Adam: the CPU step tensor advanced in float32, the corrections in float64 from its value
            state["step"] += 1
            t = state["step"].item()
            bc1 = 1 - beta1 ** t
            bc2 = 1 - beta2 ** t
            segs.append(SgrAdamSegment(p.data_ptr(), g.data_ptr(), state["exp_avg"].data_ptr(),
                                       state["exp_avg_sq"].data_ptr(), p.numel(), _f32(1 - beta1), _f32(beta2),
                                       _f32(1 - beta2), _f32(bc2 ** 0.5), _f32(eps), _f32((lr / bc1) * -1)))
        if segs:
            with torch.cuda.device(dev):
                st = stream(dev)
                for i in range(0, len(segs), SGR_ADAM_MAX_SEGMENTS):
                    chunk = segs[i:i + SGR_ADAM_MAX_SEGMENTS]
                    check(lib.sgr_adam_step(len(chunk), (SgrAdamSegment * len(chunk))(*chunk), st))
        return loss


def _f32(x):
    """A Python float rounded to float32, as torch's foreach kernels receive their scalar arguments."""
    return float(np.float32(x))


def expon_lr(lr_init, lr_final, lr_delay_steps=0, lr_delay_mult=1.0, max_steps=1_000_000):
    """get_expon_lr_func (sugar_utils/general_utils.py:23-58): a function of the step, lr_init at 0 and lr_final at
    max_steps, log-linear between, optionally eased in over lr_delay_steps.  Returns the same float64 values."""

    def helper(step):
        if step < 0 or (lr_init == 0.0 and lr_final == 0.0):
            return 0.0
        if lr_delay_steps > 0:
            eased = np.sin(0.5 * np.pi * np.clip(step / lr_delay_steps, 0, 1))   # a reverse cosine ease-in
            delay_rate = lr_delay_mult + (1 - lr_delay_mult) * eased
        else:
            delay_rate = 1.0
        t = np.clip(step / max_steps, 0, 1)
        return delay_rate * np.exp(np.log(lr_init) * (1 - t) + np.log(lr_final) * t)

    return helper


# (group name, key of the raw dict, learning-rate argument); sugar_optimizer.py:63-85 for a model that learns every
# parameter.  A bound model's "points" group holds the mesh vertices.
GROUPS = (("points", "points", "position_lr_init"), ("sh_coordinates_dc", "sh_dc", "feature_lr"),
          ("sh_coordinates_rest", "sh_rest", "feature_lr"), ("all_densities", "densities", "opacity_lr"),
          ("scales", "scales", "scaling_lr"), ("quaternions", "quaternions", "rotation_lr"))


def group_table(spatial_lr_scale, bound=False, position_lr_init=0.00016, feature_lr=0.0025, opacity_lr=0.05,
                scaling_lr=0.005, rotation_lr=0.001):
    """-> [(group name, raw key, initial lr)] of SuGaROptimizer: points at position_lr_init * spatial_lr_scale, SH rest
    at feature_lr / 20."""
    lrs = dict(position_lr_init=position_lr_init * spatial_lr_scale, feature_lr=feature_lr, opacity_lr=opacity_lr,
               scaling_lr=scaling_lr, rotation_lr=rotation_lr)
    out = []
    for name, key, arg in GROUPS:
        lr = lrs[arg] / 20.0 if name == "sh_coordinates_rest" else lrs[arg]
        out.append((name, "verts" if bound and key == "points" else key, lr))
    return out


class SugarOptimizer(Adam):
    """SuGaROptimizer over steps.py's raw dict: one group (one tensor) per parameter, Adam(lr=0.0, eps=1e-15).

    Unbound (`steps.activate`'s keys): points, sh_dc, sh_rest, densities, scales [P,3], quaternions [P,4].  Bound
    (`bound=True`, `steps.refine_step`'s keys): the points group is raw["verts"], and scales / quaternions are the
    [P,2] in-plane tensors.  The keyword arguments are OptimizationParams' defaults (sugar_optimizer.py:7-29)."""

    def __init__(self, raw, spatial_lr_scale, bound=False, position_lr_init=0.00016, position_lr_final=0.0000016,
                 position_lr_delay_mult=0.01, position_lr_max_steps=30_000, feature_lr=0.0025, opacity_lr=0.05,
                 scaling_lr=0.005, rotation_lr=0.001):
        self.spatial_lr_scale = spatial_lr_scale
        table = group_table(spatial_lr_scale, bound, position_lr_init, feature_lr, opacity_lr, scaling_lr,
                            rotation_lr)
        super().__init__([{"params": [raw[key]], "lr": lr, "name": name} for name, key, lr in table], lr=0.0,
                         eps=1e-15)
        # the reference passes no delay steps, so position_lr_delay_mult has no effect (as there)
        self.position_scheduler = expon_lr(position_lr_init * spatial_lr_scale, position_lr_final * spatial_lr_scale,
                                           lr_delay_mult=position_lr_delay_mult, max_steps=position_lr_max_steps)

    def update_learning_rate(self, iteration):
        """Set the points group's lr to the schedule's value at `iteration`; -> that value (0.0 without the group)."""
        lr = 0.0
        for group in self.param_groups:
            if group["name"] == "points":
                lr = self.position_scheduler(iteration)
                group["lr"] = lr
        return lr
