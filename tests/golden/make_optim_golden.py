"""Golden values of the position learning-rate schedule from the reference's OWN get_expon_lr_func.

Runs in the build container (needs /root/reference):  python tests/golden/make_optim_golden.py
sugar_utils/general_utils.py imports only numpy and torch, so the function is imported from the reference checkout
unchanged and evaluated at every iteration 0...30 000 for SuGaROptimizer's call (OptimizationParams' defaults, which
pass no delay steps) and for two delay settings, plus its disabled and negative-step cases.
Output: tests/golden/optim_expon_lr.npz with, per setting s, `s_args` float64 [lr_init, lr_final, lr_delay_steps,
lr_delay_mult, max_steps] and `s_lr` float64 [30 001] (the value at iteration i in row i).
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF = "/root/reference"

# (name, lr_init, lr_final, lr_delay_steps, lr_delay_mult, max_steps)
SETTINGS = (
    ("sugar", 0.00016 * 2.5, 0.0000016 * 2.5, 0, 0.01, 30_000),   # SuGaROptimizer at spatial_lr_scale 2.5
    ("delay500", 0.00016, 0.0000016, 500, 0.01, 30_000),
    ("delay2000", 1e-3, 1e-5, 2000, 0.5, 20_000),                  # clipped past max_steps
)


def main():
    sys.path.insert(0, REF)
    from sugar_utils.general_utils import get_expon_lr_func
    out = {}
    steps = np.arange(30_001)
    for name, lr_init, lr_final, delay_steps, delay_mult, max_steps in SETTINGS:
        f = get_expon_lr_func(lr_init, lr_final, lr_delay_steps=delay_steps, lr_delay_mult=delay_mult,
                              max_steps=max_steps)
        out[f"{name}_args"] = np.array([lr_init, lr_final, delay_steps, delay_mult, max_steps], np.float64)
        out[f"{name}_lr"] = np.array([float(f(int(i))) for i in steps], np.float64)
    f = get_expon_lr_func(0.0, 0.0)
    out["disabled_lr"] = np.array([float(f(i)) for i in (0, 1, 100)], np.float64)
    f = get_expon_lr_func(1e-3, 1e-5)
    out["negative_lr"] = np.array([float(f(-1))], np.float64)
    path = os.path.join(HERE, "optim_expon_lr.npz")
    np.savez_compressed(path, **out)
    print(path, {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
