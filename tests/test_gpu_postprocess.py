"""GPU: the refined mesh's post-processing (sugar_b200/postprocess.py, csrc/sgr_postprocess.cu): the erosion against
its CPU restatement (oracle/postprocess_oracle.py) round by round, the whole post-process against the reference's own
lines (tests/golden/postprocess_*.npz) and, at n = 6, against the restatement; the output rebinds and textures."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from oracle import postprocess_oracle as ppo  # noqa: E402
import test_postprocess_cpu as pc  # noqa: E402

GOLDEN = pc.GOLDEN
OUTPUTS = pc.OUTPUTS
DENSITY_REL = 2e-5          # compute_density against its oracle (test_gpu_field.py)


def cuda_inputs(c):
    return {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in c.items()}


def assert_same_bits(a, b, what):
    a, b = a.cpu(), torch.as_tensor(b)
    assert a.shape == b.shape and a.dtype == b.dtype, what
    if a.dtype == torch.float32:
        a, b = a.view(torch.int32), b.view(torch.int32)
    assert torch.equal(a, b), what


def assert_density_close(a, b):
    a, b = a.cpu().double().numpy(), np.asarray(b, np.float64)
    assert a.shape == b.shape
    assert np.array_equal(np.isnan(a), np.isnan(b))
    ok = ~np.isnan(b)
    if ok.any():
        assert np.abs(a[ok] - b[ok]).max() <= DENSITY_REL * np.abs(b[ok]).max(), np.abs(a[ok] - b[ok]).max()


def fan(n_fan=100):
    """A closed icosphere with `n_fan` faces on one of its edges, two faces with a repeated vertex sharing their
    degenerate edge and one alone."""
    from sugar_b200 import scenes
    v, f = scenes.icosphere(1)
    a, b = f[0, 0], f[0, 1]
    c, d = next(g[:2] for g in f if a not in g and b not in g)
    tips = len(v) + np.arange(n_fan + 2)
    fin = np.stack([np.full(n_fan, a), np.full(n_fan, b), tips[:n_fan]], 1)
    deg = np.array([[c, c, d], [c, c, tips[n_fan]], [a, a, tips[n_fan + 1]]])
    return np.concatenate([f, fin, deg]).astype(np.int64), len(v) + n_fan + 2


@pytest.mark.parametrize("name", GOLDEN)
def test_erosion_is_the_oracles_round_by_round(name):
    from sugar_b200 import postprocess
    g = pc.golden(name)
    faces = torch.from_numpy(g["faces"])
    live = ~torch.isnan(torch.from_numpy(g["densities_raw"][:, 0]))
    counts = []
    for it in list(range(9)) + [12]:
        m = postprocess.erode_border_faces(faces.cuda(), g["verts"].shape[0], it, live.cuda())
        ref = ppo.erode(faces, it, live)
        assert m.dtype == torch.bool and m.is_cuda
        assert torch.equal(m.cpu(), ref), it
        counts.append(int(m.sum()))
    print(name, "live faces after each round:", counts)
    assert counts == sorted(counts, reverse=True)


def test_height_field_rings():
    """One ring of border faces per round until the mesh is gone, each round's count as the direct count's."""
    from sugar_b200 import postprocess, scenes
    v, f = scenes.height_field_mesh(20, 16, seed=3, permute=True)
    faces = torch.from_numpy(f)
    counts, ref = [], []
    for it in range(20):
        counts.append(int(postprocess.erode_border_faces(faces.cuda(), len(v), it).sum()))
        ref.append(int(ppo.erode_by_counting(f, it).sum()))
    print("live faces after each round:", counts)
    assert counts == ref
    assert counts[0] == len(f) and counts[-1] == 0 and all(a > b for a, b in zip(counts, counts[1:]) if a)


def test_hundred_face_fan_and_repeated_vertices():
    from sugar_b200 import postprocess
    f, V = fan(100)
    F = len(f)
    for it in (1, 2, 5):
        m = postprocess.erode_border_faces(torch.from_numpy(f).cuda(), V, it).cpu().numpy()
        assert np.array_equal(m, ppo.erode_by_counting(f, it)), it
        # the fan and the lone degenerate face go; the sphere and the two degenerate faces sharing (c, c) stay
        assert m[:F - 103].all() and not m[F - 103:F - 3].any() and m[F - 3:F - 1].all() and not m[F - 1]
    # with half of the fan dead from the start, the edge still has enough live entries
    live = torch.ones(F, dtype=torch.bool)
    live[F - 103:F - 53] = False
    m = postprocess.erode_border_faces(torch.from_numpy(f).cuda(), V, 3, live.cuda()).cpu().numpy()
    assert np.array_equal(m, ppo.erode_by_counting(f, 3, live.numpy()))


@pytest.mark.parametrize("name", GOLDEN)
def test_postprocess_is_the_reference_golden(name):
    from sugar_b200 import postprocess
    g = pc.golden(name)
    out = postprocess.postprocess_mesh(**cuda_inputs(pc.golden_inputs(g)))
    assert_same_bits(out.face_mask, torch.from_numpy(g["face_mask"]), "face_mask")
    assert_same_bits(out.eroded, torch.from_numpy(g["eroded"]), "eroded")
    for k in OUTPUTS:
        assert getattr(out, k).is_cuda
        assert_same_bits(getattr(out, k), torch.from_numpy(g[f"{k}_out"]), k)
    assert_density_close(out.eroded_density, g["eroded_density"])


def test_n6_is_the_oracle():
    from sugar_b200 import postprocess
    c = pc.n6_case()
    ref = ppo.postprocess_mesh(**c)
    out = postprocess.postprocess_mesh(**cuda_inputs(c))
    assert ref.eroded.numel() and not ref.face_mask.all()
    assert_same_bits(out.face_mask, ref.face_mask, "face_mask")
    for k in OUTPUTS:
        assert_same_bits(getattr(out, k), getattr(ref, k), k)
    assert_density_close(out.eroded_density, ref.eroded_density.numpy())


@pytest.mark.parametrize("n", [1, 6])
def test_output_rebinds_as_the_kept_rows_of_the_full_binding(n):
    from sugar_b200 import meshbind, postprocess
    c = cuda_inputs(pc.n6_case() if n == 6 else pc.golden_inputs(pc.golden("holes")))
    out = postprocess.postprocess_mesh(**c)
    bary = meshbind.bary_coords(n, "cuda")
    with torch.no_grad():
        full = meshbind.bind_to_mesh(c["verts"], c["faces"], bary, c["scales_raw"], c["complex_raw"], c["thickness"])
        new = meshbind.bind_to_mesh(c["verts"], out.faces, bary, out.scales, out.quaternions, c["thickness"])
    rows = out.face_mask.repeat_interleave(n)
    for k in ("points", "scaling", "quaternions"):
        assert torch.equal(getattr(new, k).view(torch.int32), getattr(full, k)[rows].view(torch.int32)), k


def test_postprocess_texture_save_load(tmp_path):
    from sugar_b200 import meshbind, objfile, postprocess, texture
    import test_gpu_texture as tg
    c = cuda_inputs(pc.golden_inputs(pc.golden("holes")))
    out = postprocess.postprocess_mesh(**c)
    with torch.no_grad():
        b = meshbind.bind_to_mesh(c["verts"], out.faces, meshbind.bary_coords(1, "cuda"), out.scales,
                                  out.quaternions, c["thickness"])
    cams = [tg.look_at((3.0, 1.0, 2.0), 192, 144), tg.look_at((-2.0, 3.0, 1.0), 192, 144)]
    verts_uv, faces_uv, tex = texture.extract_texture_image_and_uv_from_gaussians(
        c["verts"], out.faces, b.points, b.scaling, b.quaternions, torch.sigmoid(out.densities), out.sh_dc, cams)
    path = tmp_path / "postprocessed.obj"
    objfile.save_textured_mesh(path, c["verts"], out.faces, verts_uv, faces_uv, tex)
    v2, f2, uv2, fuv2, tex2 = objfile.load_textured_mesh(path, "cuda")
    assert v2.shape == c["verts"].shape and torch.equal(f2, out.faces) and torch.equal(fuv2, faces_uv)
    assert tex2.shape == tex.shape
    img = texture.render_textured_mesh(v2, f2, uv2, fuv2, tex2, cams[0])
    assert (img != 0).any()


def test_runs_are_identical_and_edge_cases():
    from sugar_b200 import postprocess
    c = cuda_inputs(pc.n6_case())
    a, b = postprocess.postprocess_mesh(**c), postprocess.postprocess_mesh(**c)
    for k in OUTPUTS + ("face_mask", "eroded", "eroded_density"):
        x, y = getattr(a, k), getattr(b, k)
        assert torch.equal(x.view(torch.int32) if x.is_floating_point() else x,
                           y.view(torch.int32) if y.is_floating_point() else y), k
    # iterations = 0 keeps every live face: only the faces with a NaN strength are eroded
    z = postprocess.postprocess_mesh(**dict(c, iterations=0))
    live = ~torch.isnan(c["densities_raw"].view(-1, 6)).any(1)
    assert torch.equal(z.eroded, torch.nonzero(~live)[:, 0])
    # F = 0: empty outputs
    e = postprocess.postprocess_mesh(c["verts"], c["faces"][:0], 6, *[t[:0] for t in (
        c["scales_raw"], c["complex_raw"], c["densities_raw"], c["sh_dc"], c["sh_rest"])], c["thickness"])
    assert e.faces.shape == (0, 3) and e.sh_rest.shape == (0, 15, 3) and e.face_mask.numel() == 0
    assert postprocess.erode_border_faces(c["faces"][:0], 10).shape == (0,)
    with pytest.raises(ValueError, match="face vertex ids"):
        postprocess.erode_border_faces(c["faces"], 3)
