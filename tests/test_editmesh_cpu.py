"""The editable mesh-bound model and the compositor without a GPU: (1) the oracle against goldens made by the
reference's own property code; (2) the edited-binding kernel's arithmetic (sugar_b200/csrc/sgr_meshbind.cu) compiled
for the HOST with -DSGR_MESHBIND_HOST_TEST, per Gaussian against the float64 oracle; (3) the argument checks of
meshbind.bind_to_edited_mesh and compose.Composition, which run before anything touches CUDA."""
import ctypes as C
import glob
import os

import numpy as np
import pytest
import torch

from oracle import editmesh_oracle as eo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
MESH_GOLDENS = sorted(os.path.basename(f)[9:-4] for f in glob.glob(os.path.join(GOLD, "editmesh_*.npz"))
                      if "shrot" not in f)
COLOR_GOLDENS = ["shrot_deg3", "shrot_deg1"]


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def load_case(name):
    g = np.load(os.path.join(GOLD, f"editmesh_{name}.npz"))
    case = {k: torch.from_numpy(g[k]) for k in ("verts", "reference_verts", "faces", "bary", "scales_raw", "complex_raw")}
    case["thickness"] = float(g["thickness"])
    return case, g


def test_goldens_cover_the_cases():
    assert {"identity_n6", "rigid_n1", "jitter_n3", "stretch_n4", "bent_n6"} <= set(MESH_GOLDENS)
    assert {int(load_case(n)[0]["bary"].shape[0]) for n in MESH_GOLDENS} == {1, 3, 4, 6}


@pytest.mark.parametrize("name", MESH_GOLDENS)
def test_oracle_matches_reference_property_code(name):
    case, gold = load_case(name)
    got = eo.edited_values(case)
    for k in ("points", "scaling", "quaternions"):
        assert rel(got[k], gold[k]) <= 1e-6, k


@pytest.mark.parametrize("name", COLOR_GOLDENS)
def test_oracle_rotated_colors_match_reference(name):
    g = np.load(os.path.join(GOLD, f"editmesh_{name}.npz"))
    got = eo.rotated_colors(*(torch.from_numpy(g[k]) for k in ("points", "sh", "campos", "rotation")), int(g["sh_degree"]))
    assert np.abs(got.numpy() - g["colors"]).max() <= 1e-6


def test_identity_edit_is_the_plain_binding():
    from oracle import meshbind_oracle as mo
    case = eo.make_case("identity", F=50, n_per=4, seed=9, dtype=torch.float64)
    got = eo.edited_values(case)
    p, s, q = mo.bind_to_mesh_torch(case["verts"], case["faces"], case["bary"], case["scales_raw"], case["complex_raw"],
                                    case["thickness"])
    assert rel(got["points"], p.numpy()) == 0 and rel(got["quaternions"], q.numpy()) <= 1e-14
    # the stretch is sum_k b_k * 1 here, and the float32 bary rows sum to 1 only within their own rounding
    assert rel(got["scaling"], s.numpy()) <= 1e-7


@pytest.fixture(scope="module")
def host_lib(tmp_path_factory):
    from test_meshbind_oracle import _host_lib
    return _host_lib(tmp_path_factory)


def host_edited(lib, case, out_rows=None, rows=None):
    f32 = lambda t: np.ascontiguousarray(t.numpy(), np.float32)
    F, n = case["faces"].shape[0], case["bary"].shape[0]
    N = F * n if rows is None else rows
    verts, ref, bary = f32(case["verts"]), f32(case["reference_verts"]), f32(case["bary"])
    faces = np.ascontiguousarray(case["faces"].numpy(), np.int64)
    s_raw, c_raw = f32(case["scales_raw"]), f32(case["complex_raw"])
    pts, scl, qt = np.full((N, 3), np.nan, np.float32), np.full((N, 3), np.nan, np.float32), np.full((N, 4), np.nan, np.float32)
    p = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)
    lib.meshbind_host_edited_forward(C.c_int(F), C.c_int(n), p(verts), p(ref), p(faces), p(bary), p(s_raw), p(c_raw),
                                     C.c_float(case["thickness"]), p(out_rows), p(pts), p(scl), p(qt))
    return dict(points=pts, scaling=scl, quaternions=qt)


# The float32 kernel against float64, as max |error| / max |value|.  The edited binding is not well conditioned in
# float32 even where every |<axis, base>| stays <= 0.999: arccos multiplies a dot product's rounding by up to
# 1 / sqrt(1 - 0.999^2) = 22, and the stretch of a skewed face turns the angle error into a scale error.  So the bound
# is the reference's own float32 arithmetic (the oracle in float32, bit-identical to the goldens): the kernel may be at
# most 25 % farther from float64 than it, plus 1e-7.  5e-6 caps both: the largest error the reference shows on these
# meshes is 4e-6 (scaling, jittered height field, largest dot 0.983).  points are a three-term sum: 5e-7.
@pytest.mark.parametrize("kind,n_per,mesh,seed", [("identity", 6, "soup", 0), ("rigid", 1, "soup", 1),
                                                  ("jitter", 6, "soup", 2), ("stretch", 4, "soup", 3),
                                                  ("bent", 3, "height", 4), ("jitter", 6, "height", 5)])
def test_kernel_arithmetic_on_host_matches_fp64_oracle(host_lib, kind, n_per, mesh, seed):
    case = eo.make_case(kind, F=3000, n_per=n_per, seed=seed, mesh=mesh)
    assert max(eo.max_axis_dot(case["verts"], case["faces"]), eo.max_axis_dot(case["reference_verts"], case["faces"])) <= 0.999
    got = host_edited(host_lib, case)
    want = eo.edited_values(case, torch.float64)
    ref32 = eo.edited_values(case)
    assert rel(got["points"], want["points"]) <= 5e-7
    for k in ("scaling", "quaternions"):
        err = rel(got[k], want[k])
        assert err <= 5e-6 and err <= 1.25 * rel(ref32[k], want[k]) + 1e-7, (k, err, rel(ref32[k], want[k]))
    assert np.all(got["scaling"][:, 0] == np.float32(case["thickness"]))


@pytest.mark.parametrize("name", MESH_GOLDENS)
def test_kernel_arithmetic_on_host_matches_goldens(host_lib, name):
    """Against the reference's own float32 values: 3.2e-7 measured, 1e-6 allowed."""
    case, gold = load_case(name)
    got = host_edited(host_lib, case)
    for k in ("points", "scaling", "quaternions"):
        assert rel(got[k], gold[k]) <= 1e-6, k


def test_kernel_on_host_writes_through_out_rows(host_lib):
    case = eo.make_case("jitter", F=40, n_per=3, seed=6)
    full = host_edited(host_lib, case)
    g = torch.Generator().manual_seed(0)
    idx = torch.randperm(120, generator=g)[:50]
    rows = np.full(120, -1, np.int64)
    rows[idx.numpy()] = 7 + np.arange(50)              # an offset into a larger buffer
    got = host_edited(host_lib, case, out_rows=rows, rows=60)
    for k in full:
        assert np.array_equal(got[k][7:57], full[k][idx.numpy()]), k
        assert np.isnan(got[k][:7]).all() and np.isnan(got[k][57:]).all(), k   # skipped Gaussians write nothing


# --- argument checks (CPU tensors: each must fail before the CUDA requirement is reached) ---

def _args(**over):
    case = eo.make_case("jitter", F=6, n_per=3, seed=0)
    a = dict(verts=case["verts"], reference_verts=case["reference_verts"], faces=case["faces"], bary=case["bary"],
             scales_raw=case["scales_raw"], complex_raw=case["complex_raw"], thickness=1e-5)
    a.update(over)
    return a


@pytest.mark.parametrize("bad,match", [
    (dict(verts=torch.zeros(18, 2)), "verts"),
    (dict(reference_verts=torch.zeros(17, 3)), "reference_verts"),
    (dict(reference_verts=torch.zeros(18, 3, dtype=torch.float64)), "reference_verts"),
    (dict(faces=torch.zeros(6, 3, dtype=torch.int32)), "faces"),
    (dict(bary=torch.zeros(3, 2)), "bary"),
    (dict(scales_raw=torch.zeros(17, 2)), "scales_raw"),
    (dict(complex_raw=torch.zeros(18, 3)), "complex_raw"),
    (dict(complex_raw=torch.zeros(18, 2, device="meta")), "complex_raw"),
])
def test_bind_to_edited_mesh_rejects_bad_arguments(bad, match):
    from sugar_b200 import meshbind
    with pytest.raises(ValueError, match=match):
        meshbind.bind_to_edited_mesh(**_args(**bad))


@pytest.mark.parametrize("which", ["verts", "reference_verts", "scales_raw", "complex_raw"])
def test_bind_to_edited_mesh_rejects_inputs_that_require_grad(which):
    from sugar_b200 import meshbind
    a = _args()
    a[which] = a[which].clone().requires_grad_(True)
    with pytest.raises(ValueError, match="forward only"):
        meshbind.bind_to_edited_mesh(**a)


def _bound_part(**over):
    a = _args()
    P = a["scales_raw"].shape[0]
    part = dict(verts=a["reference_verts"], faces=a["faces"], bary=a["bary"], scales_raw=a["scales_raw"],
                complex_raw=a["complex_raw"], thickness=1e-5, densities=torch.zeros(P, 1), sh=torch.zeros(P, 16, 3))
    part.update(over)
    return part


def _plain_part(P=10, **over):
    part = dict(points=torch.zeros(P, 3), scaling=torch.ones(P, 3), quaternions=torch.zeros(P, 4),
                opacities=torch.ones(P, 1), sh=torch.zeros(P, 16, 3))
    part.update(over)
    return part


@pytest.mark.parametrize("parts,match", [
    ([], "at least one"),
    ([_bound_part(idx=torch.tensor([0, 18]))], "idx"),
    ([_bound_part(idx=torch.tensor([-1, 3]))], "idx"),
    ([_bound_part(idx=torch.tensor([2, 2]))], "idx"),
    ([_plain_part(idx=torch.tensor([10]))], "idx"),
    ([_plain_part(idx=torch.tensor([[1]]))], "idx"),
    ([_bound_part(densities=torch.zeros(17, 1))], "densities"),
    ([_bound_part(sh=torch.zeros(18, 9, 2))], "sh"),
    ([_bound_part(), _plain_part(sh=torch.zeros(10, 9, 3))], "sh"),
    ([_plain_part(points=torch.zeros(10, 3, dtype=torch.float64))], "points"),
    ([_plain_part(quaternions=torch.zeros(9, 4))], "quaternions"),
    ([_plain_part(opacities=torch.zeros(10, 1, device="meta"))], "opacities"),
    ([_bound_part(faces=torch.zeros(6, 3))], "faces"),
    ([_bound_part(complex_raw=torch.zeros(18, 2, requires_grad=True))], "forward only"),
    ([_plain_part(points=torch.zeros(10, 3, requires_grad=True))], "forward only"),
])
def test_composition_rejects_bad_parts(parts, match):
    from sugar_b200 import compose
    with pytest.raises(ValueError, match=match):
        compose.Composition(parts)
