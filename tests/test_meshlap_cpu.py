"""CPU checks of the mesh Laplacian smoothing loss: the pytorch3d restatement (oracle/meshlap_oracle.py) against an
independent float64 dense-matrix construction (tests/meshlap_cases.py) on hand cases, its invariances, the package's
topology program against the oracle's adjacency, the per-face and per-vertex kernel arithmetic compiled for the HOST
(sugar_b200/csrc/sgr_meshlap.cu, -DSGR_MESHLAP_HOST_TEST) against float64, the C entry points' validation without a
GPU, and refine_step's new term over the reference ops."""
import ctypes
import os
import shutil
import subprocess
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

import meshlap_cases as mc  # noqa: E402
from oracle import meshlap_oracle as lo  # noqa: E402
from sugar_b200 import scenes  # noqa: E402


def oracle64(verts, faces, method):
    v = torch.as_tensor(np.asarray(verts), dtype=torch.float64).requires_grad_(True)
    out = lo.mesh_laplacian_smoothing_torch(v, torch.as_tensor(faces), method)
    out.backward()
    return float(out.detach()), v.grad.numpy()


def hand_cases():
    tet = (np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0.2, 0.3, 1]]), np.array([[0, 2, 1], [0, 1, 3], [1, 2, 3], [0, 3, 2]]))
    ang = np.linspace(0.2, 2.6, 5)
    fan = (np.concatenate([[[0, 0, 0.1]], np.stack([np.cos(ang), np.sin(ang), 0.1 * ang], 1)]),
           np.array([[0, i, i + 1] for i in range(1, 5)]))
    v, f = fan
    unused = (np.concatenate([v, [[3.0, -1.0, 2.0], [0.5, 0.5, -2.0]]]), f)
    rep = (np.concatenate([v, [[0.4, -0.7, 0.3]]]), np.concatenate([f, [[2, 2, 6], [6, 3, 6]]]))   # repeated ids
    dup = (v, np.concatenate([f, f[1:2], f[2:3, ::-1]]))                                             # duplicated faces
    return {"tetrahedron": tet, "open_fan": fan, "unused_vertex": unused, "repeated_vertex": rep, "duplicated_face": dup}


@pytest.mark.parametrize("method", mc.METHODS)
@pytest.mark.parametrize("name", list(hand_cases()))
def test_oracle_equals_dense_construction(name, method):
    """To 1e-12 of the size of the terms summed: a degenerate face's clamped area makes its cotangents ~1e6."""
    v, f = hand_cases()[name]
    y = lo.laplacian_rows(torch.as_tensor(v, dtype=torch.float64), torch.as_tensor(f), method).numpy()
    Lp, s, d, want_y = mc.dense_parts(v, f, method)
    terms = 1.0 + np.abs(Lp).max() * np.abs(s).max() * np.abs(v).max() + np.abs(v).max()
    assert np.abs(y - want_y).max() <= 1e-12 * terms
    loss, grad = oracle64(v, f, method)
    want_l, want_g = mc.dense_loss_and_grad(v, f, method)
    assert abs(loss - want_l) <= 1e-12 * terms
    assert np.abs(grad - want_g).max() <= 1e-12 * (1.0 + mc.row_scale(v, f, method).max())


def test_oracle_quirks():
    """An unused vertex contributes |x| under uniform and cot, 0 under cotcurv; a self-loop counts 2 in the degree;
    an unknown method raises."""
    v, f = hand_cases()["unused_vertex"]
    for method in mc.METHODS:
        y = lo.laplacian_rows(torch.as_tensor(v, dtype=torch.float64), torch.as_tensor(f), method).numpy()
        want = np.zeros((2, 3)) if method == "cotcurv" else -v[-2:]
        assert np.abs(y[-2:] - want).max() == 0.0
    L = lo.laplacian(3, lo.edges_packed(torch.tensor([[0, 0, 1]]), 3), torch.float64, "cpu").to_dense()
    # edges (0, 1) twice as e12 / e20 -> one unique edge, and the self-loop (0, 0): deg 0 = 1 + 2
    assert torch.allclose(L, torch.tensor([[2 / 3 - 1, 1 / 3, 0], [1.0, -1, 0], [0, 0, -1]], dtype=torch.float64))
    with pytest.raises(ValueError, match="Method"):
        lo.mesh_laplacian_smoothing_torch(torch.zeros(3, 3), torch.tensor([[0, 1, 2]]), "cotan")


@pytest.mark.parametrize("method", mc.METHODS)
def test_invariant_under_face_order_and_vertex_ids(method):
    rng = np.random.default_rng(2)
    for v, f in (mc.jittered_grid(9, seed=3, permute=False), scenes.icosphere(2)):
        v = np.asarray(v, np.float64) + 0.02 * rng.normal(size=v.shape)
        base = float(lo.mesh_laplacian_smoothing_torch(torch.as_tensor(v), torch.as_tensor(f), method))
        perm = rng.permutation(len(v))
        inv = np.empty_like(perm)
        inv[perm] = np.arange(len(perm))
        f2 = np.roll(inv[f][rng.permutation(len(f))], 1, axis=1)     # and a cyclic rotation of every face's ids
        got = float(lo.mesh_laplacian_smoothing_torch(torch.as_tensor(v[perm]), torch.as_tensor(f2), method))
        assert abs(got - base) <= 1e-12 * max(1.0, abs(base))


def meshes_for_topology():
    rng = np.random.default_rng(6)
    v, f = mc.jittered_grid(8, seed=1)
    out = [scenes.height_field_mesh(20, 13, seed=7, permute=True), scenes.icosphere(1), mc.open_cap(1),
           (v, np.concatenate([f, f[:5], [[0, 1, 60], [1, 0, 61]]])), mc.with_unused(v, f, 5, seed=2),
           (np.zeros((5, 3)), np.array([[0, 1, 1], [1, 0, 2], [3, 3, 3]]))]   # repeated ids inside a face
    return out + [(np.zeros((9, 3)), rng.integers(0, 9, (30, 3)))]


def test_package_topology_equals_oracle_adjacency():
    """meshloss._build_laplacian_topology (the tensor program laplacian_topology runs on the GPU): its neighbour list is
    the oracle's uniform adjacency entry for entry (a self-loop twice), its corner list every face slot of each vertex
    in ascending order."""
    from sugar_b200 import meshloss
    for v, f in meshes_for_topology():
        V = len(v)
        topo = meshloss._build_laplacian_topology(torch.as_tensor(f), V)
        assert topo.n_verts == V and topo.n_faces == len(f) and topo.faces.dtype == torch.int32
        assert torch.equal(topo.faces.long(), torch.as_tensor(f))
        edges = lo.edges_packed(torch.as_tensor(f), V)
        A = torch.zeros(V, V, dtype=torch.int64)
        A.index_put_((edges[:, 0], edges[:, 1]), torch.ones(len(edges), dtype=torch.int64), accumulate=True)
        A.index_put_((edges[:, 1], edges[:, 0]), torch.ones(len(edges), dtype=torch.int64), accumulate=True)
        nptr, nidx = topo.nbr_ptr.long(), topo.nbr_idx.long()
        assert nptr.shape == (V + 1,) and int(nptr[0]) == 0 and int(nptr[-1]) == 2 * len(edges)
        assert torch.equal(topo.degree.long(), A.sum(1))
        cptr, cinc = topo.corner_ptr.long(), topo.corner_inc.long()
        assert int(cptr[-1]) == 3 * len(f)
        flat = torch.as_tensor(f).reshape(-1)
        for x in range(V):
            mine = nidx[nptr[x]:nptr[x + 1]]
            assert bool((mine[1:] >= mine[:-1]).all())
            assert torch.equal(torch.bincount(mine, minlength=V), A[x]), x
            assert torch.equal(cinc[cptr[x]:cptr[x + 1]], torch.nonzero(flat == x).reshape(-1)), x


def test_topology_rejects_bad_input():
    from sugar_b200 import meshloss
    with pytest.raises(ValueError, match="outside"):
        meshloss._build_laplacian_topology(torch.tensor([[0, 1, 2], [1, 2, 3]]), 3)
    with pytest.raises(ValueError, match="outside"):
        meshloss._build_laplacian_topology(torch.tensor([[0, -1, 2]]), 3)
    with pytest.raises(ValueError, match="vertices"):
        meshloss._build_laplacian_topology(torch.zeros(0, 3, dtype=torch.int64), 3)      # an empty mesh
    with pytest.raises(ValueError, match="vertices"):
        meshloss._build_laplacian_topology(torch.tensor([[0, 1, 2]]), 0)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        meshloss.laplacian_topology(torch.tensor([[0, 1, 2]]), 3)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        meshloss.mesh_laplacian_smoothing(torch.zeros(3, 3), torch.tensor([[0, 1, 2]]))
    with pytest.raises(ValueError, match="method"):
        meshloss.mesh_laplacian_smoothing(torch.zeros(3, 3), torch.tensor([[0, 1, 2]]), method="cotan")


def test_library_exports_the_new_entry_points():
    from sugar_b200 import _lib
    L = _lib.lib
    names = [L.sgr_kernel_name(k).decode() for k in range(L.sgr_num_kernel_kinds())]
    assert "misc" in names and names[-2:] == ["mesh_nc_forward", "mesh_nc_backward"]   # no kind was added
    for fn in ("sgr_mesh_lap_forward", "sgr_mesh_lap_backward"):
        assert fn in _lib.PROTOTYPES and hasattr(L, fn)
    assert (_lib.SGR_MESH_LAP_UNIFORM, _lib.SGR_MESH_LAP_COT, _lib.SGR_MESH_LAP_COTCURV) == (0, 1, 2)
    assert _lib.SGR_MESH_LAP_PARTIALS == 1024
    d = ctypes.c_void_p(256)
    assert L.sgr_mesh_lap_forward(3, 4, 2, *([d] * 8), None) == -1 and b"unknown method" in L.sgr_last_error()
    assert L.sgr_mesh_lap_forward(0, 0, 2, *([d] * 8), None) == -1 and b"bad sizes" in L.sgr_last_error()
    assert L.sgr_mesh_lap_forward(1, 4, 0, *([d] * 8), None) == -1 and b"bad sizes" in L.sgr_last_error()
    assert L.sgr_mesh_lap_forward(1, 4, 2 ** 30, *([d] * 8), None) == -1
    assert L.sgr_mesh_lap_backward(-1, 4, 2, *([d] * 7), None) == -1 and b"unknown method" in L.sgr_last_error()
    # every pointer is required except faces and face_w under uniform (those calls pass validation: not made here)
    for method in (0, 1, 2):
        for i in range(8):          # verts, faces, vert_ptr, vert_inc, face_w, vert_ys, partials, loss
            if method == 0 and i in (1, 4):
                continue
            ptrs = [d] * 8
            ptrs[i] = None
            assert L.sgr_mesh_lap_forward(method, 4, 2, *ptrs, None) == -1 and b"null pointer" in L.sgr_last_error()
        for i in range(7):          # faces, vert_ptr, vert_inc, face_w, vert_ys, g_loss, g_verts
            if method == 0 and i in (0, 3):
                continue
            ptrs = [d] * 7
            ptrs[i] = None
            assert L.sgr_mesh_lap_backward(method, 4, 2, *ptrs, None) == -1 and b"null pointer" in L.sgr_last_error()


@pytest.fixture(scope="module")
def host_lib(tmp_path_factory):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc) and not shutil.which("nvcc"):
        pytest.skip("nvcc not available: cannot compile the kernel arithmetic for the host")
    out = str(tmp_path_factory.mktemp("meshlap") / "libmeshlap_host.so")
    src = os.path.join(ROOT, "sugar_b200", "csrc", "sgr_meshlap.cu")
    subprocess.check_call([nvcc if os.path.exists(nvcc) else "nvcc", "-O1", "-std=c++17", "-DSGR_MESHLAP_HOST_TEST",
                           "-gencode", "arch=compute_90a,code=sm_90a", "--shared", "-Xcompiler", "-fPIC", src, "-o", out],
                          stderr=subprocess.DEVNULL)
    return ctypes.CDLL(out)


def host_rows(lib, verts, faces, method, g=1.0):
    """-> (|y_v| [V], dL/dx [V,3]) of the host-compiled kernel functions over the package's topology."""
    from sugar_b200 import meshloss
    topo = meshloss._build_laplacian_topology(torch.as_tensor(faces), len(verts))
    lists = (topo.nbr_ptr, topo.nbr_idx) if method == "uniform" else (topo.corner_ptr, topo.corner_inc)
    v = np.ascontiguousarray(verts, np.float32)
    f = np.ascontiguousarray(faces, np.int32)
    vp, vi = (np.ascontiguousarray(t.numpy(), np.int32) for t in lists)
    norms, grads = np.zeros(len(v)), np.zeros((len(v), 3))
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    code = {"uniform": 0, "cot": 1, "cotcurv": 2}[method]
    lib.mesh_lap_host(code, len(v), len(f), p(v), p(f), p(vp), p(vi), ctypes.c_double(g), p(norms), p(grads))
    return norms, grads


def arithmetic_cases():
    v, f = mc.jittered_grid(14, seed=4)
    hv, hf = hand_cases()["repeated_vertex"]
    out = {"grid_jittered": (v, f), "icosphere": scenes.icosphere(2), "open_cap": mc.open_cap(2),
           "unused": mc.with_unused(v, f, 7, seed=5), "repeated_and_duplicated": (hv, np.concatenate([hf, hf[:2]]))}
    return {k: (np.ascontiguousarray(v, np.float32), np.ascontiguousarray(f, np.int64)) for k, (v, f) in out.items()}


@pytest.mark.parametrize("method", mc.METHODS)
@pytest.mark.parametrize("name", list(arithmetic_cases()))
def test_kernel_arithmetic_on_host_matches_float64(host_lib, name, method):
    """Per vertex: |y_v| and the gradient row against float64 (the dense construction, from the same float32 inputs),
    relative to the size of the terms each sums.  uniform is double throughout; cot / cotcurv take pytorch3d's float32
    face values (a face with a repeated vertex has a clamped area and cotangents ~1e6); the backward reads y in
    float32."""
    v, f = arithmetic_cases()[name]
    n64 = mc.check_margin(v, f, method)
    _, g64 = mc.dense_loss_and_grad(v, f, method, g=1.5)
    norms, grads = host_rows(host_lib, v, f, method, g=1.5)
    tol = 1e-12 if method == "uniform" else 1e-6
    assert (np.abs(norms - n64) <= tol * mc.y_scale(v, f, method) + 1e-15 * np.abs(v).max()).all(), name
    assert mc.row_errors(grads, g64, mc.row_scale(v, f, method, g=1.5)) <= (1e-6 if method == "uniform" else 1e-4)
    ol, og = oracle64(v, f, method)
    assert abs(norms.sum() / len(v) - ol) <= (tol * mc.y_scale(v, f, method).sum() + 1e-15 * np.abs(v).max()) / len(v) * 2


def test_flat_union_jack_gives_exact_zero_rows(host_lib):
    v, f = mc.union_jack(9)
    norms, grads = host_rows(host_lib, v, f, "uniform")
    y = mc.dense_parts(v, f, "uniform")[3]
    interior = (v[:, 0] > 0) & (v[:, 0] < 8) & (v[:, 1] > 0) & (v[:, 1] < 8)
    assert (np.linalg.norm(y, axis=1)[interior] == 0).all() and (norms[interior] == 0).all()
    assert (norms[~interior] > 0.1).all()
    _, g64 = mc.dense_loss_and_grad(v, f, "uniform")
    assert mc.row_errors(grads, g64, mc.row_scale(v, f, "uniform")) <= 1e-6


class FakeRasterizer:
    """Differentiable stand-in for the rasterizer module: image = mean of the points' colour + 0 * geometry."""

    class GaussianRasterizationSettings:
        def __init__(self, **kw):
            self.__dict__.update(kw)

    class GaussianRasterizer:
        def __init__(self, st):
            self.st = st

        def __call__(self, means3D, means2D, opacities, scales, rotations, shs=None, colors_precomp=None):
            H, W = self.st.image_height, self.st.image_width
            c = colors_precomp if colors_precomp is not None else shs[:, 0]
            z = 0.01 * (means3D.mean() + opacities.mean() + scales.mean() + rotations.mean())
            return (c.mean(0)[:, None, None] + z).expand(3, H, W), torch.ones(means3D.shape[0], dtype=torch.int32)


@pytest.mark.parametrize("method", mc.METHODS)
def test_refine_step_laplacian_smoothing_over_reference_ops(method):
    """laplacian_smoothing_factor = 5 adds 5 x the oracle to the loss and its gradient to verts, before the normal
    consistency term; 0 never calls it."""
    import bench
    import bench_workloads as bw
    steps = bw._load_steps_without_package()
    sc = bench.load_scenes().make_scene(100, 24, 16, seed=1)
    cam = steps.camera_from_scene(sc, "cpu")
    ops = bw.reference_ops(torch, FakeRasterizer)
    calls = []
    lap, nc = ops.mesh_laplacian_smoothing, ops.mesh_normal_consistency
    ops.mesh_laplacian_smoothing = lambda v, f, m, t=None: calls.append(("lap", m)) or lap(v, f, m, t)
    ops.mesh_normal_consistency = lambda v, f, t=None: calls.append(("nc",)) or nc(v, f, t)
    v, f = scenes.height_field_mesh(6, 5, seed=2, noise=3.0)
    F = len(f)
    mesh = SimpleNamespace(faces=torch.from_numpy(f), bary=torch.tensor([[1 / 3, 1 / 3, 1 / 3]]), thickness=1e-5)
    gt = torch.rand(3, 16, 24, generator=torch.Generator().manual_seed(0))
    g = torch.Generator().manual_seed(1)
    base = dict(verts=torch.from_numpy(v) + torch.tensor([0.0, 0.0, 3.0]), sh_dc=0.5 * torch.randn(F, 1, 3, generator=g),
                sh_rest=0.1 * torch.randn(F, 15, 3, generator=g), densities=torch.randn(F, 1, generator=g),
                scales=torch.randn(F, 2, generator=g) - 3, quaternions=torch.randn(F, 2, generator=g))
    out = {}
    for fac in (0.0, 5.0):
        raw = {k: t.clone().requires_grad_(True) for k, t in base.items()}
        loss, _ = steps.refine_step(raw, mesh, cam, gt, ops, laplacian_smoothing_factor=fac,
                                    laplacian_smoothing_method=method, normal_consistency_factor=0.1)
        out[fac] = (float(loss), raw["verts"].grad.clone())
    assert calls == [("nc",), ("lap", method), ("nc",)]
    vv = base["verts"].clone().requires_grad_(True)
    term = lo.mesh_laplacian_smoothing_torch(vv, mesh.faces, method)
    term.backward()
    assert float(term.detach()) > 0
    assert abs(out[5.0][0] - out[0.0][0] - 5.0 * float(term.detach())) <= 1e-5
    assert torch.allclose(out[5.0][1], out[0.0][1] + 5.0 * vv.grad, atol=1e-6)
