"""GPU: the fused mesh normal-consistency loss (sugar_b200/meshloss.py, csrc/sgr_meshloss.cu) against the float64
restatement of pytorch3d 0.7.4 (oracle/meshloss_oracle.py).

Tolerance rule: measured against the float64 oracle, the loss may be max(1e-5, 2 x the float32 oracle's own relative
error) off (relative), and dL/dverts max(1e-4, 2 x the float32 oracle's rel_err), rel_err = |a - b|_inf / |b|_inf.
Cases whose true value is 0 (flat sheets) are compared on the value only, to 1e-6 absolute."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import helpers as h
from oracle import meshloss_oracle as mlo
from sugar_b200 import scenes

pytestmark = pytest.mark.gpu


def fan(k):
    ang = np.linspace(0.3, 2 * np.pi - 0.2, k)
    v = np.concatenate([[[0, 0, 0], [1, 0, 0]], np.stack([np.linspace(0.2, 0.8, k), np.cos(ang), np.sin(ang)], 1)])
    return v.astype(np.float32), np.array([[0, 1, 2 + i] for i in range(k)], np.int64)


def cases():
    rng = np.random.default_rng(0)
    out = {"grid": scenes.height_field_mesh(60, 50, seed=1), "grid_permuted": scenes.height_field_mesh(60, 50, seed=2, permute=True),
           "icosphere": scenes.icosphere(4), "fan3": fan(3), "fan4": fan(4)}
    v, f = scenes.height_field_mesh(20, 20, seed=3, noise=1.0)
    out["duplicated_face"] = (v, np.concatenate([f, f[100:101]]))
    v, f = fan(2)
    v[3] = v[0]                      # the second face's opposite vertex on top of v0: its normal is exactly zero
    out["degenerate_pair"] = (v, f)
    v, f = scenes.icosphere(3)
    out["icosphere_noisy"] = ((v + 0.01 * rng.normal(size=v.shape)).astype(np.float32), f)
    return out


def ours(verts, faces, topology=None):
    from sugar_b200 import meshloss
    v = verts.detach().clone().requires_grad_(True)
    out = meshloss.mesh_normal_consistency(v, faces, topology)
    out.backward()
    return out.detach(), v.grad.detach()


def oracle(verts, faces, dtype):
    v = verts.detach().to(dtype).clone().requires_grad_(True)
    out = mlo.mesh_normal_consistency_torch(v, faces, "vectorised")
    out.sum().backward()
    return float(out.detach().sum()), v.grad.detach().double().cpu().numpy()


def check(verts, faces, what):
    loss, grad = ours(verts, faces)
    assert loss.shape == () and loss.dtype == torch.float32
    l64, g64 = oracle(verts, faces, torch.float64)
    l32, g32 = oracle(verts, faces, torch.float32)
    err = abs(float(loss) - l64) / abs(l64)
    allowed = max(1e-5, 2 * abs(l32 - l64) / abs(l64))
    assert err <= allowed, f"{what} loss: {err:.3e} > {allowed:.3e}"
    err = h.rel_err(grad.double().cpu().numpy(), g64)
    allowed = max(1e-4, 2 * h.rel_err(g32, g64))
    assert err <= allowed, f"{what} grad: {err:.3e} > {allowed:.3e}"


def as_cuda(v, f):
    return torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda()


@pytest.mark.parametrize("name", list(cases()))
def test_matches_float64_oracle(name):
    v, f = as_cuda(*cases()[name])
    check(v, f, name)


@pytest.mark.parametrize("name", ["grid_permuted", "icosphere", "fan4", "duplicated_face", "degenerate_pair"])
def test_topology_equals_oracle_pairs(name):
    from sugar_b200 import meshloss
    v, f = as_cuda(*cases()[name])
    topo = meshloss.mesh_topology(f, v.shape[0])
    want = mlo.pair_table(f, v.shape[0])
    key = lambda t: sorted((r[0], r[1], min(r[2], r[3]), max(r[2], r[3])) for r in t.tolist())
    assert topo.pairs.dtype == torch.int32 and topo.pairs.is_cuda
    assert key(topo.pairs) == key(want)
    assert torch.equal(topo.pairs.long(), want)          # and in pytorch3d's order
    ptr = topo.vert_ptr.long().cpu()
    assert int(ptr[-1]) == 4 * topo.num_pairs and bool((ptr[1:] >= ptr[:-1]).all())


def test_flat_sheets_give_zero():
    for permute in (False, True):
        v, f = as_cuda(*scenes.height_field_mesh(80, 70, amplitude=0.0, noise=0.0, permute=permute))
        loss, grad = ours(v, f)
        assert abs(float(loss)) <= 1e-6
        assert bool(torch.isfinite(grad).all())


def test_soup_gives_zero_and_zero_gradient():
    from sugar_b200 import _lib, meshloss
    v = torch.randn(300, 3, device="cuda")
    f = torch.arange(300, device="cuda").view(100, 3)
    topo = meshloss.mesh_topology(f, 300)
    assert topo.num_pairs == 0
    torch.cuda.synchronize()
    _lib.profile(True)
    try:
        loss, grad = ours(v, f, topo)
        torch.cuda.synchronize()
        prof = _lib.profile_read()
    finally:
        _lib.profile(False)
    assert loss.shape == () and float(loss) == 0.0
    assert grad.shape == v.shape and bool((grad == 0).all())
    assert not any(k.startswith("mesh_nc") for k in prof)   # a memset each way, no kernel


def test_large_permuted_grid():
    """The default refinement mesh's size: ~1M vertices, 2M faces, ids and face order shuffled."""
    v, f = as_cuda(*scenes.height_field_mesh(1001, 1001, seed=4, permute=True))
    assert f.shape[0] == 2_000_000
    check(v, f, "grid_2M_permuted")


def test_deterministic_and_cached_topology():
    from sugar_b200 import meshloss
    v, f = as_cuda(*scenes.height_field_mesh(300, 300, seed=5, permute=True))
    topo = meshloss.mesh_topology(f, v.shape[0])
    a, b, c = ours(v, f, topo), ours(v, f, topo), ours(v, f)
    for x, y in ((a, b), (a, c)):
        assert torch.equal(x[0], y[0]) and torch.equal(x[1], y[1])


def test_upstream_gradient_on_device_without_host_sync():
    from sugar_b200 import meshloss
    v, f = as_cuda(*scenes.height_field_mesh(50, 40, seed=6))
    topo = meshloss.mesh_topology(f, v.shape[0])
    ref = ours(v, f, topo)[1]
    p = v.clone().requires_grad_(True)
    up = torch.tensor(2.5, device="cuda")
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = meshloss.mesh_normal_consistency(p, topology=topo)
        out.backward(up)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    # the upstream factor enters each pair's gradient before its rounding to float, so entries that are sums of
    # cancelling pair terms move by float rounding of those terms, not of the entry
    assert h.rel_err(p.grad.cpu().numpy(), 2.5 * ref.cpu().numpy()) <= 1e-6


def test_errors():
    from sugar_b200 import meshloss
    v = torch.randn(10, 3, device="cuda")
    with pytest.raises(ValueError, match="outside"):
        meshloss.mesh_topology(torch.tensor([[0, 1, 10]], device="cuda"), 10)
    with pytest.raises(ValueError, match="outside"):
        meshloss.mesh_normal_consistency(v, torch.tensor([[0, -1, 2]], device="cuda"))
    topo = meshloss.mesh_topology(torch.tensor([[0, 1, 2], [2, 1, 3]], device="cuda"), 10)
    with pytest.raises(ValueError, match="built for"):
        meshloss.mesh_normal_consistency(v[:5], topology=topo)
    with pytest.raises(ValueError, match="float32"):
        meshloss.mesh_normal_consistency(v.double(), topology=topo)
    with pytest.raises(ValueError, match="faces"):
        meshloss.mesh_normal_consistency(v)


def refine_setup(verts_np, faces_np, W=320, H=240, n_per=6):
    from sugar_b200 import meshbind, meshloss, steps
    dev = torch.device("cuda")
    sc = scenes.make_scene(1000, W, H, seed=0)
    cam = steps.camera_from_scene(sc, dev)
    g = torch.Generator().manual_seed(0)
    v = torch.from_numpy(verts_np).clone()
    v[:, 0] = (v[:, 0] - 0.5) * 3.0
    v[:, 1] = (v[:, 1] - 0.5) * 2.0
    v[:, 2] = 4.0 + 3.0 * v[:, 2]
    F, P = faces_np.shape[0], faces_np.shape[0] * n_per
    faces = torch.from_numpy(faces_np).to(dev)
    mesh = SimpleNamespace(faces=faces, bary=meshbind.bary_coords(n_per, dev), thickness=1e-5,
                           topology=meshloss.mesh_topology(faces, v.shape[0]))
    base = dict(verts=v, sh_dc=0.5 * torch.randn(P, 1, 3, generator=g), sh_rest=0.1 * torch.randn(P, 15, 3, generator=g),
                densities=torch.randn(P, 1, generator=g) * 2, scales=torch.randn(P, 2, generator=g) * 0.4 - 4.0,
                quaternions=torch.randn(P, 2, generator=g))
    gt = torch.rand(3, H, W, generator=g).to(dev)
    return cam, mesh, {k: t.to(dev) for k, t in base.items()}, gt


def test_refine_step_adds_the_term_and_its_gradient():
    from sugar_b200 import _lib, meshloss, steps
    cam, mesh, base, gt = refine_setup(*scenes.height_field_mesh(40, 30, seed=7, noise=0.5))
    ops = steps.ours_ops()

    def run(fac):
        raw = {k: t.clone().requires_grad_(True) for k, t in base.items()}
        loss, _ = steps.refine_step(raw, mesh, cam, gt, ops, normal_consistency_factor=fac)
        return float(loss), raw["verts"].grad.detach().clone()
    run(0.0)
    torch.cuda.synchronize()
    _lib.profile(True)
    try:
        l0, g0 = run(0.0)
        torch.cuda.synchronize()
        prof0 = _lib.profile_read()
        l1, g1 = run(0.1)
        torch.cuda.synchronize()
        prof1 = _lib.profile_read()
    finally:
        _lib.profile(False)
    assert not any(k.startswith("mesh_nc") for k in prof0), prof0
    assert prof1.get("mesh_nc_forward", (0, 0))[1] == 2 and prof1.get("mesh_nc_backward", (0, 0))[1] == 2
    l0b, g0b = run(0.0)
    nc_loss, nc_grad = ours(base["verts"], mesh.faces, mesh.topology)
    assert float(nc_loss) > 0
    noise = abs(l0 - l0b)
    assert abs(l1 - (l0 + 0.1 * float(nc_loss))) <= 2 * noise + 1e-6 * abs(l1)
    want = g0 + 0.1 * nc_grad
    gnoise = float((g0 - g0b).abs().max())
    assert float((g1 - want).abs().max()) <= 2 * gnoise + 1e-6 * float(want.abs().max())
