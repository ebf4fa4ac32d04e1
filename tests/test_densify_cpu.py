"""Densification and pruning without a GPU: the oracle (oracle/densify_oracle.py) on hand-built cases, the C ABI's
argument checks, and the view-parallel reduction of the statistics and the shared split draw over gloo."""
import ctypes
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import densify_oracle as do  # noqa: E402

# extent 1: clone / split at max scale 0.01, "big" at 0.1; max_grad 2e-4, min_opacity 0.005
ROWS = [  # (accum, denom, scale, density)
    (1e-3, 1.0, 0.005, 2.0),    # 0 clone
    (1e-3, 2.0, 0.05, 2.0),     # 1 split
    (1e-5, 1.0, 0.05, 2.0),     # 2 kept
    (1e-5, 1.0, 0.05, -9.0),    # 3 pruned: opacity 1.2e-4
    (0.0, 0.0, 0.005, 2.0),     # 4 grads 0/0 = NaN -> 0: kept, not cloned
    (1e-3, 1.0, 0.2, 2.0),      # 5 split; children at 0.125 > 0.1 are pruned when max_screen_size is truthy
]


def case(P=len(ROWS), moments=False):
    t = lambda v: torch.tensor(v, dtype=torch.float32)
    params = {"points": torch.arange(3 * P, dtype=torch.float32).reshape(P, 3),
              "densities": t([[r[3]] for r in ROWS]),
              "scales": torch.log(t([[r[2]] * 3 for r in ROWS])),
              "quaternions": t([[1.0, 0.1 * i, 0.0, 0.2] for i in range(P)]),
              "sh_dc": torch.arange(P, dtype=torch.float32).reshape(P, 1, 1).expand(P, 1, 3).contiguous(),
              "sh_rest": torch.randn(P, 15, 3, generator=torch.Generator().manual_seed(0))}
    stats = {"accum": t([[r[0]] for r in ROWS]), "denom": t([[r[1]] for r in ROWS]), "max_radii": torch.zeros(P)}
    mom = {}
    if moments:
        mom = {k: (v + 100.0, v + 200.0) for k, v in params.items()}
    return params, mom, stats


def run(max_screen_size, moments=False, **kw):
    params, mom, stats = case(moments=moments)
    args = dict(max_grad=2e-4, min_opacity=0.005, extent=1.0, max_screen_size=max_screen_size,
                generator=torch.Generator().manual_seed(3))
    args.update(kw)
    return do.densify_and_prune(params, mom, stats, **args)


def ids(params):
    return params["sh_dc"][:, 0, 0].long().tolist()


def test_output_order_originals_clones_children():
    p, m, s, info = run(None)
    assert ids(p) == [0, 2, 4, 0, 1, 5, 1, 5]
    assert info["split"].sum() == 2 and info["clone"].tolist() == [True] + [False] * 5
    # clones copy every raw field; children copy all but points and scales
    assert torch.equal(p["points"][3], p["points"][0]) and torch.equal(p["sh_rest"][3], p["sh_rest"][0])
    assert torch.equal(p["quaternions"][4], p["quaternions"][6]) and torch.equal(p["densities"][5], p["densities"][7])
    want = torch.log(torch.exp(case()[0]["scales"][1]) / 1.6)
    assert torch.equal(p["scales"][4], want) and torch.equal(p["scales"][6], want)
    assert not torch.equal(p["points"][4], p["points"][6])
    for v in s.values():                       # statistics are zeros of the new size
        assert v.shape[0] == 8 and not v.any()


def test_max_screen_size_none_and_zero_skip_the_size_clauses():
    assert ids(run(None)[0]) == ids(run(0)[0]) == [0, 2, 4, 0, 1, 5, 1, 5]
    assert ids(run(20)[0]) == [0, 2, 4, 0, 1, 1]      # children of 5 have max scale 0.125 > 0.1 * extent


def test_screen_clause_compares_the_reset_statistics():
    """max_radii2D is reset by each append, so a huge observed radius prunes nothing; a negative threshold (truthy)
    compares against the zeros and prunes everything."""
    params, mom, stats = case()
    stats["max_radii"][:] = 1e6
    p = do.densify_and_prune(params, mom, stats, 2e-4, 0.005, 1.0, 20, generator=torch.Generator().manual_seed(3))[0]
    assert ids(p) == [0, 2, 4, 0, 1, 1]
    assert run(-1)[0]["points"].shape[0] == 0


def test_nan_grads_count_as_zero():
    p, _, _, info = run(None)
    assert not info["clone"][4] and not info["split"][4] and 4 in ids(p)


def test_adam_moments_follow_rows_and_new_rows_start_at_zero():
    p, m, _, _ = run(None, moments=True)
    assert set(m) == set(do.KEYS)
    src = case()[0]
    for k, (a, b) in m.items():
        assert torch.equal(a[:3], src[k][[0, 2, 4]] + 100.0) and torch.equal(b[:3], src[k][[0, 2, 4]] + 200.0)
        assert not a[3:].any() and not b[3:].any()
    assert run(None)[1] == {}                   # no state before the first optimizer step


def test_no_split_rows():
    p, _, _, info = run(None, max_grad=1.0)
    assert info["split"].sum() == 0 and info["samples"].shape == (0, 3)
    assert ids(p) == [0, 1, 2, 4, 5]


def test_every_row_pruned():
    p, m, s, _ = run(None, moments=True, min_opacity=1.0)
    assert all(v.shape[0] == 0 for v in p.values()) and all(a.shape[0] == 0 for a, _ in m.values())


def test_prune_points_and_reset_opacity():
    params, mom, stats = case(moments=True)
    stats["accum"][:, 0] = torch.arange(6.0)
    mask = torch.tensor([False, True, False, True, True, False])
    p, m, s = do.prune_points(params, mom, stats, mask)
    assert ids(p) == [0, 2, 5] and s["accum"][:, 0].tolist() == [0.0, 2.0, 5.0]
    assert torch.equal(m["points"][0], params["points"][[0, 2, 5]] + 100.0)
    p2, m2 = do.reset_opacity(p, m)
    op = torch.sigmoid(p2["densities"])
    assert torch.allclose(op, torch.full_like(op, 0.01), rtol=1e-5)
    assert not m2["densities"][0].any() and torch.equal(m2["points"][0], m["points"][0])
    low = dict(p, densities=torch.full((3, 1), -9.0))          # below 0.01 already: unchanged up to logit(sigmoid)
    assert torch.allclose(do.reset_opacity(low, {})[0]["densities"], low["densities"], atol=1e-4)


def test_split_draw_is_randn_times_std():
    """The Densifier draws randn(2S, 3) and scales it in the kernel; the reference draws normal(0, std).  From the
    same generator state the two are the same numbers."""
    stds = torch.rand(14, 3, generator=torch.Generator().manual_seed(1)) + 0.01
    ref = torch.normal(mean=torch.zeros(14, 3), std=stds, generator=torch.Generator().manual_seed(9))
    z = torch.randn(14, 3, generator=torch.Generator().manual_seed(9))
    assert torch.equal(ref, z * stds)


def test_densify_entry_points_validate_arguments_without_gpu():
    from sugar_b200 import _lib
    L = _lib.lib
    assert L.sgr_densify_stats(-1, None, 3, *([None] * 6)) == -1
    assert L.sgr_densify_stats(10, None, 3, *([None] * 6)) == -1 and b"null pointer" in L.sgr_last_error()
    assert L.sgr_densify_stats(10, None, 1, *([None] * 6)) == -1                    # stride must hold gx, gy
    assert L.sgr_densify_stats(0, None, 3, *([None] * 6)) == 0                      # nothing to do
    g = _lib.SgrDensifyGates()
    assert L.sgr_densify_classify(-1, None, None, None, None, ctypes.byref(g), None, None) == -1
    assert L.sgr_densify_classify(10, None, None, None, None, ctypes.byref(g), None, None) == -1
    cols = (_lib.SgrDensifyColumn * 1)(_lib.SgrDensifyColumn(None, None, 0, 0))
    emit = lambda P, k, c, S, ch, n=1, cs=cols: L.sgr_densify_emit(P, k, c, S, ch, None, n, cs, None, None, None,
                                                                     None, 0.625, None, None)
    assert emit(-1, 0, 0, 0, 0) == -1
    assert emit(10, 5, 0, 11, 0) == -1 and b"counts disagree" in L.sgr_last_error()   # S > P
    assert emit(10, 5, 0, 2, 3) == -1                                                 # more children than splits
    assert emit(10, 9, 0, 2, 0) == -1                                                 # kept rows include split ones
    assert emit(10, 5, 0, 2, 2) == -1 and b"width" in L.sgr_last_error()             # width 0
    cols[0].width, cols[0].kind = 4, 2                                                # points must be 3 wide
    assert emit(10, 5, 0, 2, 2) == -1
    cols[0].width, cols[0].kind = 3, 0
    assert emit(10, 5, 0, 2, 2) == -1 and b"null pointer" in L.sgr_last_error()
    assert emit(10, 5, 0, 2, 2, n=25) == -1                                           # too many columns
    assert emit(0, 0, 0, 0, 0, n=0) == 0


def _worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from sugar_b200 import densify
    g = torch.Generator().manual_seed(10 + rank)
    accum, denom, radii = torch.rand(20, 1, generator=g), torch.rand(20, 1, generator=g), torch.rand(20, generator=g)
    local = [accum.clone(), denom.clone(), radii.clone()]
    densify.reduce_statistics(accum, denom, radii, dist.group.WORLD)
    z = densify.split_normals(5, "cpu", torch.Generator().manual_seed(77 + rank), dist.group.WORLD)
    q.put((rank, [t.numpy().copy() for t in local], [t.numpy().copy() for t in (accum, denom, radii)], z.numpy().copy()))
    dist.barrier()
    dist.destroy_process_group()
    q.close()
    q.join_thread()


def test_view_parallel_statistics_and_draw_gloo_world2():
    """Ranks with different statistics end with the summed accum / denom and the maximum max_radii2D, and with rank
    0's normals, so every rank makes the same densification decisions."""
    pytest.importorskip("sugar_b200._lib")
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = sorted((q.get(timeout=120) for _ in range(world)), key=lambda r: r[0])
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    (_, l0, r0, z0), (_, l1, r1, z1) = res
    assert not np.array_equal(l0[0], l1[0])
    np.testing.assert_array_equal(r0[0], l0[0] + l1[0])
    np.testing.assert_array_equal(r0[1], l0[1] + l1[1])
    np.testing.assert_array_equal(r0[2], np.maximum(l0[2], l1[2]))
    for a, b in zip(r0, r1):
        np.testing.assert_array_equal(a, b)
    np.testing.assert_array_equal(z0, z1)
    np.testing.assert_array_equal(z0, torch.randn(10, 3, generator=torch.Generator().manual_seed(77)).numpy())
