"""CPU checks of the mesh normal-consistency loss: the pytorch3d restatement (oracle/meshloss_oracle.py) on hand cases
with known answers, its two pair builders against each other, the package's topology program against the oracle's
pair table, the per-pair kernel arithmetic compiled for the HOST (sugar_b200/csrc/sgr_meshloss.cu,
-DSGR_MESHLOSS_HOST_TEST) against the oracle's float64 autograd, the C entry points' validation without a GPU, and
refine_step's new term over the reference ops."""
import ctypes
import math
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

from oracle import meshloss_oracle as mlo  # noqa: E402
from sugar_b200 import scenes  # noqa: E402


def nc(verts, faces, builder="comprehension"):
    return mlo.mesh_normal_consistency_torch(torch.as_tensor(verts, dtype=torch.float64), torch.as_tensor(faces),
                                             builder)


def fan(k, seed=0):
    """k faces sharing the edge (0, 1), opposite vertices 2 .. k + 1 spread around it."""
    rng = np.random.default_rng(seed)
    ang = np.sort(rng.uniform(0, 2 * math.pi, k))
    verts = np.concatenate([[[0, 0, 0], [1, 0, 0]], np.stack([rng.uniform(0.2, 0.8, k), np.cos(ang), np.sin(ang)], 1)])
    faces = np.array([[0, 1, 2 + i] for i in range(k)])
    return verts, faces


def test_flat_sheet_gives_zero():
    v, f = scenes.height_field_mesh(9, 7, amplitude=0.0, noise=0.0)
    for builder in mlo.BUILDERS:
        val = nc(v, f, builder)
        assert val.dim() == 0 and abs(float(val)) <= 1e-15
    flipped = f.copy()
    flipped[::3] = flipped[::3, ::-1]          # the term does not depend on the winding
    assert abs(float(nc(v, flipped))) <= 1e-15


@pytest.mark.parametrize("theta", [0.0, 0.01, 0.3, 1.0, math.pi / 2, 2.5])
def test_hinge_gives_one_minus_cos(theta):
    """Two faces on the edge (0, 1), the second bent by theta out of the first's plane."""
    v = np.array([[0, 0, 0], [1, 0, 0], [0.3, 1, 0], [0.6, -math.cos(theta), math.sin(theta)]])
    f = np.array([[0, 1, 2], [1, 0, 3]])
    assert mlo.pair_table(torch.as_tensor(f), 4).shape[0] == 1
    assert abs(float(nc(v, f)) - (1 - math.cos(theta))) <= 1e-12


@pytest.mark.parametrize("k", [2, 3, 4, 5])
def test_fan_gives_all_pairs(k):
    v, f = fan(k, seed=k)
    for builder in mlo.BUILDERS:
        t = mlo.pair_table(torch.as_tensor(f), len(v), builder)
        assert t.shape == (k * (k - 1) // 2, 4)
        assert {tuple(r[:2]) for r in t.tolist()} == {(0, 1)}
        assert {frozenset(r[2:]) for r in t.tolist()} == {frozenset((2 + i, 2 + j)) for i in range(k) for j in range(i + 1, k)}
    assert np.isfinite(float(nc(v, f)))


def test_soup_and_boundary_only_give_no_pairs():
    soup = np.arange(12).reshape(4, 3)
    v = np.random.default_rng(0).normal(size=(12, 3))
    single = np.array([[0, 1, 2]])
    for verts, faces in ((v, soup), (v[:3], single)):
        out = nc(verts, faces)
        assert out.shape == (1,) and out.dtype == torch.float32 and float(out.detach()[0]) == 0.0
        assert mlo.pair_table(torch.as_tensor(faces), len(verts)).shape == (0, 4)


def test_duplicated_face_gives_two():
    v = np.random.default_rng(1).normal(size=(3, 3))
    out = nc(v, np.array([[0, 1, 2], [0, 1, 2]]))
    assert abs(float(out) - 2.0) <= 2e-7             # three pairs of 2, weighted by float32(1 / 3)
    out = nc(v, np.array([[0, 1, 2], [2, 1, 0]]))   # also with the opposite winding
    assert abs(float(out) - 2.0) <= 2e-7


def test_invariant_under_face_order_and_vertex_ids():
    rng = np.random.default_rng(2)
    for v, f in (scenes.height_field_mesh(12, 10, seed=3, noise=0.5), scenes.icosphere(2)):
        v = v + 0.02 * rng.normal(size=v.shape)
        base = float(nc(v, f))
        perm = rng.permutation(len(v))
        inv = np.empty_like(perm)
        inv[perm] = np.arange(len(perm))
        f2 = inv[f][rng.permutation(len(f))]
        f2 = np.roll(f2, 1, axis=1)                  # and a cyclic rotation of every face's ids
        assert abs(float(nc(v[perm], f2)) - base) <= 1e-12 * max(1.0, abs(base))


def test_pair_builders_agree():
    rng = np.random.default_rng(4)
    meshes = [scenes.height_field_mesh(15, 11, seed=5, permute=True), scenes.icosphere(2), fan(4), fan(6, seed=1)]
    v, f = scenes.height_field_mesh(8, 8)
    meshes.append((v, np.concatenate([f, f[rng.choice(len(f), 10)], [[0, 1, 60]]])))   # duplicates + a non-manifold edge
    for v, f in meshes:
        ft = torch.as_tensor(f)
        _, edge_idx, _ = mlo.sorted_entries(ft, len(v))
        E = int(edge_idx.max()) + 1
        a, b = mlo.pairs_comprehension(edge_idx, E), mlo.pairs_vectorised(edge_idx, E)
        assert torch.equal(a, b)
        assert float(nc(v, f, "comprehension")) == float(nc(v, f, "vectorised"))


def meshes_for_topology():
    rng = np.random.default_rng(6)
    v, f = scenes.height_field_mesh(8, 8)
    out = [scenes.height_field_mesh(20, 13, seed=7, permute=True), scenes.icosphere(1), fan(3), fan(4),
           (v, np.concatenate([f, f[:5], [[0, 1, 60], [1, 0, 61]]])), (np.zeros((12, 3)), np.arange(12).reshape(4, 3)),
           (np.zeros((5, 3)), np.array([[0, 1, 1], [1, 0, 2], [3, 3, 3]]))]   # repeated ids inside a face
    return out + [(np.zeros((9, 3)), rng.integers(0, 9, (30, 3)))]


def test_package_topology_equals_oracle_pair_table():
    """meshloss._build_topology (the tensor program mesh_topology runs on the GPU) gives the oracle's pairs in the
    oracle's order, and its CSR lists every (pair, slot) of each vertex in ascending order."""
    from sugar_b200 import meshloss
    for v, f in meshes_for_topology():
        V = len(v)
        topo = meshloss._build_topology(torch.as_tensor(f), V)
        want = mlo.pair_table(torch.as_tensor(f), V)
        assert topo.pairs.dtype == torch.int32 and torch.equal(topo.pairs.long(), want)
        assert topo.num_pairs == want.shape[0] and topo.n_verts == V and topo.n_faces == len(f)
        ptr, inc = topo.vert_ptr.long(), topo.vert_inc.long()
        assert ptr.shape == (V + 1,) and int(ptr[0]) == 0 and int(ptr[-1]) == 4 * want.shape[0]
        flat = want.reshape(-1)
        for x in range(V):
            mine = inc[ptr[x]:ptr[x + 1]]
            assert torch.equal(mine, torch.nonzero(flat == x).reshape(-1)), x


def test_topology_rejects_bad_ids():
    from sugar_b200 import meshloss
    with pytest.raises(ValueError, match="outside"):
        meshloss._build_topology(torch.tensor([[0, 1, 2], [1, 2, 3]]), 3)
    with pytest.raises(ValueError, match="outside"):
        meshloss._build_topology(torch.tensor([[0, -1, 2]]), 3)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        meshloss.mesh_topology(torch.tensor([[0, 1, 2]]), 3)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        meshloss.mesh_normal_consistency(torch.zeros(3, 3), torch.tensor([[0, 1, 2]]))


def test_scene_meshes():
    v, f = scenes.height_field_mesh(11, 6)
    assert v.shape == (66, 3) and f.shape == (100, 3) and v.dtype == np.float32 and f.dtype == np.int64
    vp, fp = scenes.height_field_mesh(11, 6, permute=True)
    assert sorted(map(tuple, np.round(v[f].reshape(-1, 9), 6))) == sorted(map(tuple, np.round(vp[fp].reshape(-1, 9), 6)))
    for s in (0, 1, 3):
        v, f = scenes.icosphere(s)
        assert v.shape == (10 * 4 ** s + 2, 3) and f.shape == (20 * 4 ** s, 3)
        assert np.allclose(np.linalg.norm(v, axis=1), 1.0, atol=1e-6)
        assert mlo.pair_table(torch.as_tensor(f), len(v)).shape[0] == 3 * len(f) // 2   # closed: every edge twice
        n = np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]])
        assert (np.einsum("ij,ij->i", n, v[f].mean(1)) > 0).all()                     # outward winding


def test_library_lists_the_new_kernels_and_prototypes():
    from sugar_b200 import _lib
    L = _lib.lib
    names = [L.sgr_kernel_name(k).decode() for k in range(L.sgr_num_kernel_kinds())]
    assert names[-2:] == ["mesh_nc_forward", "mesh_nc_backward"]
    assert names[:20][-2:] == ["loss_forward", "loss_backward"]          # earlier kinds keep their indices
    for fn in ("sgr_mesh_nc_forward", "sgr_mesh_nc_backward", "sgr_mesh_nc_forward_scratch_bytes",
               "sgr_mesh_nc_backward_scratch_bytes"):
        assert fn in _lib.PROTOTYPES and hasattr(L, fn)
    assert L.sgr_mesh_nc_forward_scratch_bytes(0) == 0 and L.sgr_mesh_nc_backward_scratch_bytes(0) == 0
    assert 0 < L.sgr_mesh_nc_forward_scratch_bytes(1000) <= L.sgr_mesh_nc_forward_scratch_bytes(3_000_000)
    assert L.sgr_mesh_nc_backward_scratch_bytes(1000) >= 48 * 1000
    dummy = ctypes.c_void_p(256)
    assert L.sgr_mesh_nc_forward(-1, 3, dummy, dummy, dummy, dummy, None) == -1 and b"bad sizes" in L.sgr_last_error()
    assert L.sgr_mesh_nc_forward(2 ** 30, 3, dummy, dummy, dummy, dummy, None) == -1
    assert L.sgr_mesh_nc_forward(5, 3, dummy, dummy, None, dummy, None) == -1 and b"null pointer" in L.sgr_last_error()
    for i in range(3):
        ptrs = [dummy] * 3
        ptrs[i] = None
        assert L.sgr_mesh_nc_forward(5, 3, ptrs[0], ptrs[1], dummy, ptrs[2], None) == -1
    for i in range(7):
        ptrs = [dummy] * 7
        ptrs[i] = None
        assert L.sgr_mesh_nc_backward(5, 3, *ptrs, None) == -1 and b"null pointer" in L.sgr_last_error()
    assert L.sgr_mesh_nc_backward(-2, 3, *([dummy] * 7), None) == -1


@pytest.fixture(scope="module")
def host_lib(tmp_path_factory):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc) and not shutil.which("nvcc"):
        pytest.skip("nvcc not available: cannot compile the kernel arithmetic for the host")
    out = str(tmp_path_factory.mktemp("meshloss") / "libmeshloss_host.so")
    src = os.path.join(ROOT, "sugar_b200", "csrc", "sgr_meshloss.cu")
    subprocess.check_call([nvcc if os.path.exists(nvcc) else "nvcc", "-O1", "-std=c++17", "-DSGR_MESHLOSS_HOST_TEST",
                           "-gencode", "arch=compute_90a,code=sm_90a", "--shared", "-Xcompiler", "-fPIC", src, "-o", out],
                          stderr=subprocess.DEVNULL)
    return ctypes.CDLL(out)


def host_loss_and_grad(lib, verts32, table, g=1.0):
    Q = table.shape[0]
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    pairs = np.ascontiguousarray(table, np.int32)
    terms, pg = np.zeros(Q), np.zeros((Q, 4, 3))
    w = float(np.float32(1.0 / Q))                   # pytorch3d's float32 weight, so that only the arithmetic differs
    lib.mesh_nc_host(ctypes.c_int(Q), p(verts32), p(pairs), ctypes.c_double(g * w), p(terms), p(pg))
    gv = np.zeros((len(verts32), 3))
    np.add.at(gv, pairs.reshape(-1), pg.reshape(-1, 3))
    return terms.sum() * w, gv


def oracle64(verts32, faces):
    v = torch.from_numpy(verts32.astype(np.float64)).requires_grad_(True)
    out = mlo.mesh_normal_consistency_torch(v, torch.as_tensor(faces), "vectorised")
    out.sum().backward()
    return float(out.detach().sum()), v.grad.numpy()


def cases_for_arithmetic():
    rng = np.random.default_rng(8)
    out = {"grid_permuted": scenes.height_field_mesh(30, 25, seed=9, permute=True),
           "icosphere": scenes.icosphere(3), "fan3": fan(3), "fan4": fan(4, seed=2)}
    v, f = scenes.height_field_mesh(10, 10, seed=1, noise=2.0)
    out["duplicated_face"] = (v, np.concatenate([f, f[17:18]]))
    v, f = fan(2, seed=3)
    v = v.astype(np.float32)
    v[3] = v[0]                                      # opposite vertex on top of v0: that normal is exactly zero
    out["zero_normal"] = (v, f)
    v2 = v.copy()
    v2[3] = v2[0] + np.float32(1e-5) * np.array([0, 0.3, 0.2], np.float32)  # |n| ~ 4e-6 * |e|: above eps
    v2[1] = v2[0] + np.float32(1e-4) * np.array([1, 0, 0], np.float32)      # |e| = 1e-4: |n| ~ 4e-10 < eps
    out["clamped_normal"] = (v2, f)
    # distinct ids inside each face: for a face like (a, a, b) torch's cross product leaves a 1e-16 residue where the
    # kernel's opposite-vertex form is exactly zero, and below eps that residue is divided by eps
    out["random"] = (rng.normal(size=(40, 3)), np.stack([rng.permutation(40)[:3] for _ in range(120)]))
    return {k: (np.ascontiguousarray(v, np.float32), np.ascontiguousarray(f, np.int64)) for k, (v, f) in out.items()}


@pytest.mark.parametrize("name", list(cases_for_arithmetic()))
def test_kernel_arithmetic_on_host_matches_oracle_float64(host_lib, name):
    v, f = cases_for_arithmetic()[name]
    table = mlo.pair_table(torch.as_tensor(f), len(v)).numpy()
    want_l, want_g = oracle64(v, f)
    got_l, got_g = host_loss_and_grad(host_lib, v, table)
    assert abs(got_l - want_l) <= 1e-12 * max(abs(want_l), 1e-3), (got_l, want_l)
    assert np.abs(got_g - want_g).max() <= 1e-9 * np.abs(want_g).max(), name


def test_small_angle_terms_keep_their_digits(host_lib):
    """Hinges bent by 1e-2 .. 1e-5 rad in float32 coordinates: the kernel's term matches 2 sin^2(theta / 2) of the
    angle between its own inputs' normals (atan2 in float64) to 1e-9 relative, where float32 1 - cos has no digits
    left (and float64 1 - cos only a few at 1e-5)."""
    for theta in (1e-2, 1e-3, 1e-4, 1e-5):
        v = np.array([[0, 0, 0], [1, 0, 0], [0.3, 1, 0], [0.6, -math.cos(theta), math.sin(theta)]], np.float32)
        f = np.array([[0, 1, 2], [1, 0, 3]])
        v64 = v.astype(np.float64)
        na, nb = np.cross(v64[1] - v64[0], v64[2] - v64[0]), -np.cross(v64[1] - v64[0], v64[3] - v64[0])
        ang = math.atan2(np.linalg.norm(np.cross(na, nb)), float(na @ nb))
        want = 2 * math.sin(ang / 2) ** 2
        got, _ = host_loss_and_grad(host_lib, v, mlo.pair_table(torch.as_tensor(f), 4).numpy())
        assert abs(got - want) <= 1e-9 * want, (theta, got, want)
        v32 = torch.from_numpy(v)
        f32 = float(mlo.mesh_normal_consistency_torch(v32, torch.as_tensor(f)))
        if theta <= 1e-4:
            assert abs(f32 - want) > 0.5 * want         # the float32 chain: cancellation


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


def test_refine_step_normal_consistency_over_reference_ops():
    """normal_consistency_factor = 0.1 adds 0.1 x the oracle to the loss and its gradient to verts; 0 never calls it."""
    import bench
    import bench_workloads as bw
    steps = bw._load_steps_without_package()
    sc = bench.load_scenes().make_scene(100, 24, 16, seed=1)
    cam = steps.camera_from_scene(sc, "cpu")
    ops = bw.reference_ops(torch, FakeRasterizer)
    calls = []
    inner = ops.mesh_normal_consistency
    ops.mesh_normal_consistency = lambda v, f, t=None: calls.append(1) or inner(v, f, t)
    v, f = scenes.height_field_mesh(6, 5, seed=2, noise=3.0)
    F, n = len(f), 1
    mesh = SimpleNamespace(faces=torch.from_numpy(f), bary=torch.tensor([[1 / 3, 1 / 3, 1 / 3]]), thickness=1e-5)
    gt = torch.rand(3, 16, 24, generator=torch.Generator().manual_seed(0))
    g = torch.Generator().manual_seed(1)
    base = dict(verts=torch.from_numpy(v) + torch.tensor([0.0, 0.0, 3.0]), sh_dc=0.5 * torch.randn(F * n, 1, 3, generator=g),
                sh_rest=0.1 * torch.randn(F * n, 15, 3, generator=g), densities=torch.randn(F * n, 1, generator=g),
                scales=torch.randn(F * n, 2, generator=g) - 3, quaternions=torch.randn(F * n, 2, generator=g))
    out = {}
    for fac in (0.0, 0.1):
        raw = {k: t.clone().requires_grad_(True) for k, t in base.items()}
        loss, _ = steps.refine_step(raw, mesh, cam, gt, ops, normal_consistency_factor=fac)
        out[fac] = (float(loss), raw["verts"].grad.clone())
    assert len(calls) == 1
    vv = base["verts"].clone().requires_grad_(True)
    nc_val = mlo.mesh_normal_consistency_torch(vv, mesh.faces)
    nc_val.backward()
    assert float(nc_val.detach()) > 0
    assert abs(out[0.1][0] - out[0.0][0] - 0.1 * float(nc_val.detach())) <= 1e-6
    assert torch.allclose(out[0.1][1], out[0.0][1] + 0.1 * vv.grad, atol=1e-7)
