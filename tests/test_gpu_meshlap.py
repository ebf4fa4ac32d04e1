"""GPU: the fused mesh Laplacian smoothing loss (sugar_b200/meshloss.py, csrc/sgr_meshlap.cu) against float64 autograd
on the restatement of pytorch3d 0.7.4 (oracle/meshlap_oracle.py), for each method.

Tolerance rules (tests/meshlap_cases.py defines the scales):
  * every case is built with each row |y_v| either exactly 0 or at least 1e-4 of the terms it sums (check_margin):
    y / |y| is undefined at 0;
  * well-conditioned meshes: the loss to 1e-5 relative, each gradient row to 1e-3 of (|row| + the terms it sums);
  * slivers, where Heron's formula in float32 is ill-conditioned in pytorch3d's own arithmetic: the kernel may be at
    most 25 % farther from float64 than the float32 restatement is, plus 1e-6, in the loss and in the gradient
    (|a - b|_inf / |b|_inf)."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import helpers as h
import meshlap_cases as mc
from oracle import meshlap_oracle as lo
from sugar_b200 import scenes

pytestmark = pytest.mark.gpu


def repeated_and_duplicated():
    v, f = mc.jittered_grid(20, seed=8, permute=False)
    rng = np.random.default_rng(8)
    extra = [[f[k, 0], f[k, 0], f[k, 2]] for k in rng.choice(len(f), 6, replace=False)]   # a repeated vertex
    return v, np.concatenate([f, extra, f[rng.choice(len(f), 10, replace=False)]])         # and duplicated faces


def cases():
    v, f = mc.jittered_grid(40, seed=2)
    return {"icosphere": scenes.icosphere(4), "grid_jittered_permuted": (v, f), "open_cap": mc.open_cap(4),
            "unused_vertices": mc.with_unused(v, f, 50, seed=3), "repeated_and_duplicated": repeated_and_duplicated()}


def as_cuda(v, f):
    return (torch.from_numpy(np.ascontiguousarray(v, np.float32)).cuda(),
            torch.from_numpy(np.ascontiguousarray(f, np.int64)).cuda())


def ours(verts, faces, method, topology=None):
    from sugar_b200 import meshloss
    v = verts.detach().clone().requires_grad_(True)
    out = meshloss.mesh_laplacian_smoothing(v, faces, method, topology)
    out.backward()
    return out.detach(), v.grad.detach()


def oracle(verts, faces, method, dtype):
    v = verts.detach().to(dtype).clone().requires_grad_(True)
    out = lo.mesh_laplacian_smoothing_torch(v, faces, method)
    out.backward()
    return float(out.detach()), v.grad.detach().double().cpu().numpy()


@pytest.mark.parametrize("method", mc.METHODS)
@pytest.mark.parametrize("name", list(cases()))
def test_matches_float64_oracle(name, method):
    v_np, f_np = cases()[name]
    mc.check_margin(v_np, f_np, method)
    v, f = as_cuda(v_np, f_np)
    loss, grad = ours(v, f, method)
    assert loss.shape == () and loss.dtype == torch.float32
    l64, g64 = oracle(v, f, method, torch.float64)
    assert abs(float(loss) - l64) <= 1e-5 * l64, (float(loss), l64)
    err = mc.row_errors(grad.double().cpu().numpy(), g64, mc.row_scale(v_np, f_np, method))
    assert err <= 1e-3, f"{name} {method}: row error {err:.3e}"


@pytest.mark.parametrize("method", mc.METHODS)
def test_slivers_within_float32_error(method):
    v_np, f_np = mc.slivers()
    mc.check_margin(v_np, f_np, method)
    v, f = as_cuda(v_np, f_np)
    loss, grad = ours(v, f, method)
    l64, g64 = oracle(v, f, method, torch.float64)
    l32, g32 = oracle(v, f, method, torch.float32)
    base = abs(l32 - l64) / l64
    assert abs(float(loss) - l64) / l64 <= 1.25 * base + 1e-6, (float(loss), l64, l32)
    err, base = h.rel_err(grad.double().cpu().numpy(), g64), h.rel_err(g32, g64)
    assert err <= 1.25 * base + 1e-6, (err, base)


def test_flat_union_jack_gives_exact_zero_rows():
    """uniform on a flat integer grid of degree-4 and -8 vertices: interior rows are exactly 0 in float64 and in the
    kernel, so every vertex two rings inside the border has a gradient of exactly 0 on both sides."""
    n = 33
    v_np, f_np = mc.union_jack(n)
    v, f = as_cuda(v_np, f_np)
    loss, grad = ours(v, f, "uniform")
    l64, g64 = oracle(v, f, "uniform", torch.float64)
    assert abs(float(loss) - l64) <= 1e-6 * l64
    zero64 = (g64 == 0).all(1)
    inner = (v_np[:, 0] >= 2) & (v_np[:, 0] <= n - 3) & (v_np[:, 1] >= 2) & (v_np[:, 1] <= n - 3)
    assert zero64[inner].all() and bool((grad.cpu().numpy()[zero64] == 0).all())
    assert mc.row_errors(grad.double().cpu().numpy(), g64, mc.row_scale(v_np, f_np, "uniform")) <= 1e-6


@pytest.mark.parametrize("method", mc.METHODS)
def test_large_mesh(method):
    """500k faces (BASELINE config 4's mesh size), ids and face order shuffled."""
    v_np, f_np = mc.jittered_grid(501, seed=4)
    assert f_np.shape[0] == 500_000
    mc.check_margin(v_np, f_np, method)
    v, f = as_cuda(v_np, f_np)
    loss, grad = ours(v, f, method)
    l64, g64 = oracle(v, f, method, torch.float64)
    assert abs(float(loss) - l64) <= 1e-5 * l64
    assert mc.row_errors(grad.double().cpu().numpy(), g64, mc.row_scale(v_np, f_np, method)) <= 1e-3


def test_topology_equals_cpu_program():
    from sugar_b200 import meshloss
    v_np, f_np = repeated_and_duplicated()
    v, f = as_cuda(v_np, f_np)
    gpu = meshloss.laplacian_topology(f, v.shape[0])
    cpu = meshloss._build_laplacian_topology(torch.from_numpy(f_np), len(v_np))
    for a, b in zip(gpu[:5], cpu[:5]):
        assert a.is_cuda and a.dtype == torch.int32 and torch.equal(a.cpu(), b)
    assert gpu.n_verts == cpu.n_verts and gpu.n_faces == cpu.n_faces


@pytest.mark.parametrize("method", mc.METHODS)
def test_deterministic_and_cached_topology(method):
    from sugar_b200 import meshloss
    v, f = as_cuda(*mc.jittered_grid(300, seed=5))
    topo = meshloss.laplacian_topology(f, v.shape[0])
    a, b, c = ours(v, f, method, topo), ours(v, f, method, topo), ours(v, f, method)
    for x, y in ((a, b), (a, c)):
        assert torch.equal(x[0], y[0]) and torch.equal(x[1], y[1])


@pytest.mark.parametrize("method", mc.METHODS)
def test_upstream_gradient_on_device_without_host_sync(method):
    from sugar_b200 import meshloss
    v, f = as_cuda(*mc.jittered_grid(50, seed=6))
    topo = meshloss.laplacian_topology(f, v.shape[0])
    ref = ours(v, f, method, topo)[1]
    p = v.clone().requires_grad_(True)
    up = torch.tensor(2.5, device="cuda")
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = meshloss.mesh_laplacian_smoothing(p, method=method, topology=topo)
        out.backward(up)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    assert h.rel_err(p.grad.cpu().numpy(), 2.5 * ref.cpu().numpy()) <= 1e-6


def test_errors():
    from sugar_b200 import meshloss
    v = torch.randn(10, 3, device="cuda")
    f = torch.tensor([[0, 1, 2], [2, 1, 3]], device="cuda")
    with pytest.raises(ValueError, match="method"):
        meshloss.mesh_laplacian_smoothing(v, f, method="cotangent")
    with pytest.raises(ValueError, match="outside"):
        meshloss.laplacian_topology(torch.tensor([[0, 1, 10]], device="cuda"), 10)
    with pytest.raises(ValueError, match="outside"):
        meshloss.mesh_laplacian_smoothing(v, torch.tensor([[0, -1, 2]], device="cuda"))
    with pytest.raises(ValueError, match="vertices"):
        meshloss.mesh_laplacian_smoothing(v, torch.zeros(0, 3, dtype=torch.int64, device="cuda"))
    with pytest.raises(ValueError, match=r"integer \[F,3\]"):
        meshloss.laplacian_topology(torch.zeros(4, 4, dtype=torch.int64, device="cuda"), 10)
    topo = meshloss.laplacian_topology(f, 10)
    with pytest.raises(ValueError, match="built for"):
        meshloss.mesh_laplacian_smoothing(v[:5], topology=topo)
    with pytest.raises(ValueError, match="float32"):
        meshloss.mesh_laplacian_smoothing(v.double(), topology=topo)
    with pytest.raises(ValueError, match=r"\[V,3\]"):
        meshloss.mesh_laplacian_smoothing(v[:, :2], topology=topo)
    with pytest.raises(ValueError, match="faces"):
        meshloss.mesh_laplacian_smoothing(v)
    cpu_topo = meshloss._build_laplacian_topology(f.cpu(), 10)
    with pytest.raises(ValueError, match="topology on"):
        meshloss.mesh_laplacian_smoothing(v, topology=cpu_topo)
    with pytest.raises(ValueError, match="faces on"):
        meshloss.mesh_laplacian_smoothing(v, f.cpu())


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
                           laplacian_topology=meshloss.laplacian_topology(faces, v.shape[0]))
    base = dict(verts=v, sh_dc=0.5 * torch.randn(P, 1, 3, generator=g), sh_rest=0.1 * torch.randn(P, 15, 3, generator=g),
                densities=torch.randn(P, 1, generator=g) * 2, scales=torch.randn(P, 2, generator=g) * 0.4 - 4.0,
                quaternions=torch.randn(P, 2, generator=g))
    gt = torch.rand(3, H, W, generator=g).to(dev)
    return cam, mesh, {k: t.to(dev) for k, t in base.items()}, gt


@pytest.mark.parametrize("method", mc.METHODS)
def test_refine_step_adds_the_term_and_its_gradient(method):
    """factor 5: the step's loss and verts.grad are the factor-0 step's plus 5 x the float64 oracle's term, within the
    step's own run-to-run noise plus the kernel's tolerance (1e-5 relative in the loss, 1e-3 of the row scale)."""
    from sugar_b200 import steps
    cam, mesh, base, gt = refine_setup(*scenes.height_field_mesh(40, 30, seed=7, noise=0.5))
    v_np, f_np = base["verts"].cpu().numpy(), mesh.faces.cpu().numpy()
    mc.check_margin(v_np, f_np, method)
    ops = steps.ours_ops()

    def run(fac):
        raw = {k: t.clone().requires_grad_(True) for k, t in base.items()}
        loss, _ = steps.refine_step(raw, mesh, cam, gt, ops, laplacian_smoothing_factor=fac,
                                    laplacian_smoothing_method=method)
        return float(loss), raw["verts"].grad.detach().clone()
    run(0.0)
    l0, g0 = run(0.0)
    l1, g1 = run(5.0)
    l0b, g0b = run(0.0)
    t64, tg64 = oracle(base["verts"], mesh.faces, method, torch.float64)
    assert t64 > 0
    noise = abs(l0 - l0b)
    assert abs(l1 - (l0 + 5.0 * t64)) <= 2 * noise + 1e-5 * abs(l1)
    gnoise = float((g0 - g0b).abs().max())
    term_grad = (g1.double() - g0.double()).cpu().numpy() / 5.0
    # float32 rounding of the sum g0 + 5 g_term: half an ulp of the larger of the two per entry
    rounding = (2 * gnoise + 1e-7 * float((g0.abs() + g1.abs()).max())) / 5.0
    assert mc.row_errors(term_grad, tg64, mc.row_scale(v_np, f_np, method) + rounding) <= 1e-3


@pytest.mark.parametrize("method", ["uniform", "cot"])
def test_train_refined_with_the_term(method):
    """Three train_refined iterations with laplacian_smoothing_factor 5 move verts as three hand-written iterations of
    the same loop do: refine_step, the bound SugarOptimizer, the same views."""
    from sugar_b200 import steps, train
    cam, mesh, base, gt = refine_setup(*scenes.height_field_mesh(30, 20, seed=9, noise=0.5))
    views = [(cam, gt)]
    raw_a = {k: t.clone().requires_grad_(True) for k, t in base.items()}
    losses = []
    train.train_refined(raw_a, mesh, views, spatial_lr_scale=1.0, num_iterations=3, dssim_factor=0.0,
                        normal_consistency_factor=0.0, laplacian_smoothing_factor=5.0,
                        laplacian_smoothing_method=method, on_iteration=lambda it, loss, ev: losses.append(float(loss)))
    raw_b = {k: t.clone().requires_grad_(True) for k, t in base.items()}
    opt = train._optimizer(None, raw_b, 1.0, bound=True)
    ops = steps.ours_ops()
    want = []
    for it in range(1, 4):
        opt.update_learning_rate(it)
        ev = train.refine_phase(it, 1000)
        loss, _ = steps.refine_step(raw_b, mesh, cam, gt, ops, dssim_factor=0.0, normal_consistency_factor=0.0,
                                    sh_deg=ev["sh_degree"], laplacian_smoothing_factor=5.0,
                                    laplacian_smoothing_method=method)
        want.append(float(loss))
        opt.step()
        opt.zero_grad(set_to_none=True)
    assert np.allclose(losses, want, rtol=1e-4, atol=1e-6), (losses, want)
    assert float((raw_a["verts"] - raw_b["verts"]).abs().max()) <= 1e-5
    assert float((raw_a["verts"] - base["verts"]).abs().max()) > 0
