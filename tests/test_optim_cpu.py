"""sugar_b200.optim without a GPU: the learning-rate schedule against the reference's own values, SuGaROptimizer's group
table against the oracle, and the argument checks of Adam and of the sgr_adam_step entry point."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import optim_oracle as oo  # noqa: E402
from sugar_b200 import optim  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "optim_expon_lr.npz")


@pytest.mark.parametrize("name", ["sugar", "delay500", "delay2000"])
def test_expon_lr_equals_the_reference_bit_for_bit(name):
    with np.load(GOLDEN) as z:
        lr_init, lr_final, delay_steps, delay_mult, max_steps = z[f"{name}_args"]
        want = z[f"{name}_lr"]
    f = optim.expon_lr(lr_init, lr_final, lr_delay_steps=int(delay_steps), lr_delay_mult=delay_mult,
                       max_steps=int(max_steps))
    got = np.array([f(i) for i in range(want.shape[0])], np.float64)
    assert np.array_equal(got.view(np.int64), want.view(np.int64))


def test_expon_lr_disabled_and_negative_steps():
    with np.load(GOLDEN) as z:
        disabled, negative = z["disabled_lr"], z["negative_lr"]
    f = optim.expon_lr(0.0, 0.0)
    assert [f(i) for i in (0, 1, 100)] == list(disabled) == [0.0] * 3
    assert optim.expon_lr(1e-3, 1e-5)(-1) == negative[0] == 0.0


@pytest.mark.parametrize("bound", [False, True])
@pytest.mark.parametrize("scale", [1.0, 3.7])
def test_group_table_matches_the_oracle(bound, scale):
    assert optim.group_table(scale, bound) == oo.optimizer_groups(scale, bound)
    names = [n for n, _, _ in optim.group_table(scale, bound)]
    assert names == ["points", "sh_coordinates_dc", "sh_coordinates_rest", "all_densities", "scales", "quaternions"]
    keys = [k for _, k, _ in optim.group_table(scale, bound)]
    assert keys == ["verts" if bound else "points", "sh_dc", "sh_rest", "densities", "scales", "quaternions"]
    lrs = dict((n, lr) for n, _, lr in optim.group_table(scale, bound))
    assert lrs["points"] == 0.00016 * scale and lrs["sh_coordinates_rest"] == 0.0025 / 20.0


def test_struct_layout_and_entry_point_validate_without_gpu():
    from sugar_b200 import _lib
    L = _lib.lib
    assert L.sgr_struct_bytes(7) == ctypes.sizeof(_lib.SgrAdamSegment) == 64
    S = _lib.SgrAdamSegment

    def call(segs, n=None):
        arr = (S * max(len(segs), 1))(*segs)
        return L.sgr_adam_step(len(segs) if n is None else n, arr, None)

    assert call([]) == 0                                      # nothing to do
    assert call([S(None, None, None, None, 0)]) == 0          # an empty segment may have null pointers
    assert call([S()] * 9) == -1 and b"n_segs=9" in L.sgr_last_error()
    assert call([], n=-1) == -1
    assert L.sgr_adam_step(1, None, None) == -1
    assert call([S(None, None, None, None, -1)]) == -1 and b"n=-1" in L.sgr_last_error()
    assert call([S(256, 256, 256, 256, 2 ** 31)]) == -1 and b"2^31" in L.sgr_last_error()
    assert call([S(256, None, 256, 256, 4)]) == -1 and b"null pointer" in L.sgr_last_error()
    assert b"segment 0" in L.sgr_last_error()


def _p(*shape, **kw):
    return torch.zeros(*shape, **kw)


@pytest.mark.parametrize("kw,arg", [(dict(weight_decay=0.01), "weight_decay"), (dict(amsgrad=True), "amsgrad"),
                                    (dict(maximize=True), "maximize"), (dict(lr=-1.0), "lr"), (dict(eps=-1.0), "eps"),
                                    (dict(betas=(0.9, 1.0)), "betas")])
def test_adam_rejects_unsupported_settings(kw, arg):
    with pytest.raises(ValueError, match=arg):
        optim.Adam([_p(4)], **kw)


@pytest.mark.parametrize("param,what", [(_p(4, dtype=torch.float64), "float32"), (_p(4, 3).t(), "contiguous"),
                                        (_p(4), "CUDA")])
def test_adam_rejects_unsupported_parameters(param, what):
    with pytest.raises(ValueError, match="params") as e:
        optim.Adam([param])
    assert what in str(e.value)
    with pytest.raises(ValueError, match="params"):
        optim.SugarOptimizer({k: param for k in ("points", "sh_dc", "sh_rest", "densities", "scales", "quaternions")},
                             1.0)


def test_adam_rejects_sparse_gradients():
    p = _p(5, 3)
    p.grad = torch.zeros(5, 3).to_sparse()
    with pytest.raises(ValueError, match="grad: sparse"):
        optim.dense_grad(p)
    p.grad = torch.arange(15.0).reshape(3, 5).t()   # a transposed gradient is legal: read from a contiguous copy
    g = optim.dense_grad(p)
    assert g.is_contiguous() and torch.equal(g, p.grad)
    p.grad = None
    assert optim.dense_grad(p) is None
