"""Mesh-bound Gaussians (SURVEY 8f-4): (1) the PyTorch oracle against goldens produced by the reference's own
property code; (2) the arithmetic of the CUDA kernels -- forward and the hand-written adjoint -- compiled for the
HOST from the same source (sugar_b200/csrc/sgr_meshbind.cu, -DSGR_MESHBIND_HOST_TEST) against the oracle's
autograd.  No GPU needed; (2) is skipped where nvcc is absent."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from oracle import meshbind_oracle as mo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


@pytest.mark.parametrize("name", ["n6", "n1", "n3"])
def test_oracle_matches_reference_property_code(name):
    gold = np.load(os.path.join(GOLD, f"meshbind_{name}.npz"))
    F, V, n_per, seed = (int(v) for v in gold["cfg"])
    got = mo.values_and_grads(mo.make_case(F=F, V=V, n_per=n_per, seed=seed), seed)
    for k in ("points", "scaling", "quaternions"):
        assert rel(got[k], gold[k]) <= 1e-6, k
    for k in ("g_verts", "g_scales_raw", "g_complex_raw"):
        assert rel(got[k], gold[k]) <= 1e-5, k


def _host_lib(tmp_path_factory):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc) and not shutil.which("nvcc"):
        pytest.skip("nvcc not available: cannot compile the kernel arithmetic for the host")
    out = str(tmp_path_factory.mktemp("meshbind") / "libmeshbind_host.so")
    src = os.path.join(ROOT, "sugar_b200", "csrc", "sgr_meshbind.cu")
    subprocess.check_call([nvcc if os.path.exists(nvcc) else "nvcc", "-O1", "-std=c++17", "-DSGR_MESHBIND_HOST_TEST",
                           "-gencode", "arch=compute_90a,code=sm_90a", "--shared", "-Xcompiler", "-fPIC", src, "-o", out],
                          stderr=subprocess.DEVNULL)
    return C.CDLL(out)


@pytest.fixture(scope="module")
def host_lib(tmp_path_factory):
    return _host_lib(tmp_path_factory)


@pytest.mark.parametrize("n_per,seed", [(6, 0), (1, 1), (3, 2), (4, 3)])
def test_kernel_arithmetic_on_host_matches_oracle(host_lib, n_per, seed):
    case = mo.make_case(F=300, V=200, n_per=n_per, seed=seed)
    want = mo.values_and_grads({k: (v.double() if torch.is_tensor(v) and v.is_floating_point() else v)
                                for k, v in case.items()}, seed)
    F, P = case["faces"].shape[0], case["faces"].shape[0] * n_per
    f32 = lambda t: np.ascontiguousarray(t.numpy(), np.float32)
    verts, faces, bary = f32(case["verts"]), np.ascontiguousarray(case["faces"].numpy(), np.int64), f32(case["bary"])
    s_raw, c_raw = f32(case["scales_raw"]), f32(case["complex_raw"])
    pts, scl, qt = np.zeros((P, 3), np.float32), np.zeros((P, 3), np.float32), np.zeros((P, 4), np.float32)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    host_lib.meshbind_host_forward(C.c_int(F), C.c_int(n_per), p(verts), p(faces), p(bary), p(s_raw), p(c_raw),
                                   C.c_float(case["thickness"]), p(pts), p(scl), p(qt))
    assert rel(pts, want["points"]) <= 2e-6 and rel(scl, want["scaling"]) <= 2e-6 and rel(qt, want["quaternions"]) <= 2e-6
    wp, ws, wq = (f32(w) for w in mo.loss_weights(P, seed))
    gv, gs, gc = np.zeros_like(verts), np.zeros_like(s_raw), np.zeros_like(c_raw)
    host_lib.meshbind_host_backward(C.c_int(F), C.c_int(n_per), p(verts), p(faces), p(bary), p(s_raw), p(c_raw), p(wp),
                                    p(ws), p(wq), p(gv), p(gs), p(gc))
    assert rel(gs, want["g_scales_raw"]) <= 1e-5
    assert rel(gc, want["g_complex_raw"]) <= 1e-4
    assert rel(gv, want["g_verts"]) <= 1e-4
