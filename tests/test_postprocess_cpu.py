"""CPU checks of the refined mesh's post-processing: the restatement (oracle/postprocess_oracle.py) against the
reference's own lines (tests/golden/postprocess_*.npz), its per-face rule at n = 6 against a direct count, the C entry
point's argument checks without a GPU and the Python entry points' argument checks."""
import glob
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import postprocess_oracle as ppo  # noqa: E402

GOLDEN = sorted(os.path.basename(p)[12:-4] for p in glob.glob(os.path.join(HERE, "golden", "postprocess_*.npz")))
OUTPUTS = ("faces", "scales", "quaternions", "densities", "sh_dc", "sh_rest")


def golden(name):
    return np.load(os.path.join(HERE, "golden", f"postprocess_{name}.npz"))


def golden_inputs(g):
    t = lambda k: torch.from_numpy(g[k])
    return dict(verts=t("verts"), faces=t("faces"), n=int(g["n"]), scales_raw=t("scales_raw"),
                complex_raw=t("complex_raw"), densities_raw=t("densities_raw"), sh_dc=t("sh_dc"), sh_rest=t("sh_rest"),
                thickness=float(g["thickness"]), density_threshold=float(g["density_threshold"]),
                iterations=int(g["iterations"]))


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32) if a.dtype == np.float32 else a


def test_golden_cases_are_present():
    assert set(GOLDEN) >= {"icosphere", "holes", "fan", "heightfield_it0", "heightfield_it1", "heightfield_it5",
                           "heightfield_it12", "nan"}


@pytest.mark.parametrize("name", GOLDEN)
def test_oracle_matches_the_reference_golden(name):
    g = golden(name)
    out = ppo.postprocess_mesh(**golden_inputs(g))
    assert np.array_equal(out.face_mask.numpy(), g["face_mask"])
    assert np.array_equal(out.eroded.numpy(), g["eroded"])
    for k in OUTPUTS:
        assert np.array_equal(bits(getattr(out, k).numpy()), bits(g[f"{k}_out"])), k
    assert np.array_equal(bits(out.eroded_density.numpy()), bits(g["eroded_density"]))
    assert not ppo.ambiguous(out, float(g["density_threshold"])).any()


def test_golden_cases_cover_the_issue():
    """Closed: nothing eroded; holes and height fields: some eroded faces come back and some do not; 12 rounds erode
    the whole height field; the fan's fin and the lone repeated-vertex face go in round 1."""
    g = {name: golden(name) for name in GOLDEN}
    assert len(g["icosphere"]["eroded"]) == 0 and g["icosphere"]["face_mask"].all()
    assert len(g["heightfield_it0"]["eroded"]) == 0
    for name in ("holes", "heightfield_it1", "heightfield_it5", "heightfield_it12", "nan", "fan"):
        back = g[name]["eroded_density"] > np.float32(0.1)
        assert back.any() and not back.all(), name
    assert len(g["heightfield_it12"]["eroded"]) == g["heightfield_it12"]["faces"].shape[0]
    counts = [len(g[f"heightfield_it{k}"]["eroded"]) for k in (0, 1, 5, 12)]
    assert counts == sorted(counts) and len(set(counts)) == 4
    nan = g["nan"]
    bad = np.nonzero(np.isnan(nan["densities_raw"][:, 0]))[0]
    assert len(bad) == 1 and bad[0] in nan["eroded"]
    assert len(g["fan"]["eroded"]) == 4


@pytest.mark.parametrize("name", GOLDEN)
def test_erosion_is_the_direct_count(name):
    g = golden(name)
    live = ~np.isnan(g["densities_raw"][:, 0])
    for it in range(0, 8):
        a = ppo.erode(torch.from_numpy(g["faces"]), it, torch.from_numpy(live)).numpy()
        assert np.array_equal(a, ppo.erode_by_counting(g["faces"], it, live)), it


def n6_case(seed=7):
    """A permuted, jittered height field with 6 Gaussians per face, strengths spread around 0.1 and a few faces with
    one NaN strength; the same seed serves the GPU test."""
    from sugar_b200 import scenes
    v, f = scenes.height_field_mesh(10, 9, seed=seed, permute=True)
    g = torch.Generator().manual_seed(seed)
    v = torch.from_numpy(v).clone()
    v[:, :2] += 0.1 / 9 * torch.randn(v.shape[0], 2, generator=g)
    F, n = f.shape[0], 6
    P = F * n
    d = torch.empty(P, 1).uniform_(np.log(0.005 / 0.995), np.log(0.06 / 0.94), generator=g)
    d[torch.randperm(P, generator=g)[:5]] = float("nan")
    return dict(verts=v, faces=torch.from_numpy(f), n=n, scales_raw=torch.randn(P, 2, generator=g) * 0.2 + np.log(0.02),
                complex_raw=torch.randn(P, 2, generator=g), densities_raw=d, sh_dc=torch.randn(P, 1, 3, generator=g),
                sh_rest=torch.randn(P, 15, 3, generator=g), thickness=1e-4, density_threshold=0.1, iterations=3)


def test_n6_rule_is_the_direct_per_face_restatement():
    from sugar_b200.meshbind import bary_coords
    from oracle import field_oracle as fo
    from oracle import meshbind_oracle as mbo
    c = n6_case()
    out = ppo.postprocess_mesh(**c)
    F, n = c["faces"].shape[0], 6
    live = ~torch.isnan(c["densities_raw"].view(F, n)).any(1)
    assert (~live).sum() >= 3
    eroded_mask = ppo.erode_by_counting(c["faces"].numpy(), c["iterations"], live.numpy())
    eroded = np.nonzero(~eroded_mask)[0]
    assert np.array_equal(out.eroded.numpy(), eroded)
    # the density at each eroded centre, Gaussian by Gaussian in float64 over its 16 nearest of all F n
    pts, sc, q = mbo.bind_to_mesh_torch(c["verts"].double(), c["faces"], bary_coords(n).double(),
                                        c["scales_raw"].double(), c["complex_raw"].double(), c["thickness"])
    x = c["verts"].double()[c["faces"][eroded]].mean(-2)
    idx = torch.cdist(x, pts).argsort(1)[:, :16]
    R = fo.quaternion_to_matrix(q)
    u = torch.einsum("rkji,rkj->rki", R[idx], x[:, None] - pts[idx]) / sc[idx]
    s = torch.sigmoid(c["densities_raw"].double().view(-1))[idx]
    rho = (s * torch.exp(-0.5 * (u * u).sum(-1))).sum(-1)
    assert torch.allclose(out.eroded_density.double(), rho, rtol=1e-4, atol=1e-7, equal_nan=True)
    back = rho > 0.1
    assert back.any() and not back.all()
    keep = eroded_mask.copy()
    keep[eroded] = back.numpy()
    assert np.array_equal(out.face_mask.numpy(), keep)
    rows = torch.from_numpy(np.repeat(keep, n))
    assert torch.equal(out.faces, c["faces"][torch.from_numpy(keep)])
    for k, src in (("scales", "scales_raw"), ("quaternions", "complex_raw"), ("densities", "densities_raw"),
                   ("sh_dc", "sh_dc"), ("sh_rest", "sh_rest")):
        assert torch.equal(getattr(out, k).view(torch.int32), c[src][rows].view(torch.int32)), k
    assert not ppo.ambiguous(out, 0.1).any()


def test_border_peel_rejects_bad_arguments_without_gpu():
    from sugar_b200 import _lib
    L = _lib.lib
    assert L.sgr_border_peel(-1, 1, None, None, None, None, None, None) == -1
    assert b"sgr_border_peel" in L.sgr_last_error()
    assert L.sgr_border_peel(2 ** 31 // 3 + 1, 1, None, None, None, None, None, None) == -1
    assert L.sgr_border_peel(4, -1, None, None, None, None, None, None) == -1
    assert L.sgr_border_peel(4, 2, None, None, None, None, None, None) == -1              # null tables
    assert L.sgr_border_peel(4, 2, 8, 8, 8, 16, 16, None) == -1                           # mask == mask_tmp
    assert L.sgr_border_peel(0, 5, None, None, None, None, None, None) == 0               # nothing to do
    assert L.sgr_border_peel(4, 0, None, None, None, None, None, None) == 0


def test_python_entry_points_check_their_arguments():
    from sugar_b200 import postprocess
    from sugar_b200._lib import SgrError
    faces = torch.tensor([[0, 1, 2]])
    with pytest.raises(ValueError, match="faces"):
        postprocess.erode_border_faces(faces.int(), 3)
    with pytest.raises(ValueError, match="vertices"):
        postprocess.erode_border_faces(faces, 0)
    with pytest.raises(ValueError, match="iterations"):
        postprocess.erode_border_faces(faces, 3, iterations=-1)
    with pytest.raises(ValueError, match="iterations"):
        postprocess.erode_border_faces(faces, 3, iterations=1.5)
    with pytest.raises(ValueError, match="face_mask"):
        postprocess.erode_border_faces(faces, 3, face_mask=torch.ones(2, dtype=torch.bool))
    with pytest.raises(SgrError, match="CUDA"):
        postprocess.erode_border_faces(faces, 3)
    c = n6_case()
    args = [c[k] for k in ("verts", "faces", "n", "scales_raw", "complex_raw", "densities_raw", "sh_dc", "sh_rest",
                           "thickness")]
    for i, bad, what in ((2, 5, "n must be"), (3, c["scales_raw"][1:], "scales_raw"),
                         (5, c["densities_raw"].view(-1), "densities_raw"), (6, c["sh_dc"].view(-1, 3), "sh_dc"),
                         (7, c["sh_rest"].double(), "sh_rest")):
        a = list(args)
        a[i] = bad
        with pytest.raises(ValueError, match=what):
            postprocess.postprocess_mesh(*a)
    small = [c["verts"], c["faces"][:2], 6] + [t[:12] for t in args[3:8]] + [1e-4]
    with pytest.raises(ValueError, match="at least 16"):
        postprocess.postprocess_mesh(*small)
    with pytest.raises(SgrError, match="CUDA"):
        postprocess.postprocess_mesh(*args)
