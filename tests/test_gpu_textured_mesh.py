"""GPU: the textured mesh's render (texture.render_textured_mesh, csrc/sgr_texture.cu texture_render_kernel) against
its restatement (oracle/textured_mesh_oracle.render_view) and torch's grid_sample on the hand-made, icosphere and height-field
cases of test_gpu_texture.py; a one-view bake rendered back from its own camera; the far plane; and the textured mesh
through its files (sugar_b200/objfile.py)."""
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

from oracle import texture_oracle as to  # noqa: E402
from oracle import textured_mesh_oracle as tmo  # noqa: E402
import test_gpu_texture as tg  # noqa: E402

CASES = {"hand_made": (tg.hand_made, 200), "icosphere": (tg.icosphere_case, 10), "height_field": (tg.heightfield_case, 6)}


def setup(case, W=320, H=240):
    from sugar_b200 import splatmesh, texture
    make, s = CASES[case]
    sc, verts, faces = make(W, H)
    cam = tg.cam_of(sc)
    v, f = torch.from_numpy(verts).cuda(), torch.from_numpy(np.ascontiguousarray(faces, np.int64)).cuda()
    verts_uv, faces_uv, T = texture.uv_layout(f.shape[0], s, device="cuda")
    tex = torch.rand(T, T, 3, generator=torch.Generator().manual_seed(T)).cuda()
    zbuf, p2f = splatmesh.rasterize_mesh(v, f, cam)
    return sc, cam, v, f, verts_uv, faces_uv, tex, zbuf, p2f


def oracle_view(sc, v, f, verts_uv, faces_uv, tex, zbuf, p2f, mode, **kw):
    return tmo.render_view(v.cpu().double().numpy(), f.cpu().numpy(), verts_uv.cpu().numpy(), faces_uv.cpu().numpy(),
                          tex, sc.viewmatrix, sc.projmatrix, sc.width, sc.height, zbuf.cpu().numpy(),
                          p2f.cpu().numpy(), mode, **kw)


@pytest.mark.parametrize("case", list(CASES))
def test_nearest_sampling_is_the_oracles_texel_away_from_the_rounding_margins(case):
    from sugar_b200 import texture
    sc, cam, v, f, verts_uv, faces_uv, tex, zbuf, p2f = setup(case)
    bg = (0.25, 0.5, 0.75)
    img = texture.render_textured_mesh(v, f, verts_uv, faces_uv, tex, cam, sampling_mode="nearest", background=bg)
    ref = oracle_view(sc, v, f, verts_uv, faces_uv, tex.cpu(), zbuf, p2f, "nearest", background=bg)
    T = tex.shape[0]
    mask = ref["mask"]
    _, _, margin = to.texel_of_uv(ref["uv"][mask, 0], ref["uv"][mask, 1], T)
    clean = np.zeros_like(mask)
    clean[mask] = margin >= tg.MARGIN_PER_T * T
    got, want = img.cpu().numpy().reshape(3, -1), ref["image"].reshape(3, -1)
    print(f"{case}: T={T}, {int(mask.sum())} covered pixels, {int((mask & ~clean).sum())} at the margins")
    assert mask.sum() > 5000 and clean.sum() >= 0.99 * mask.sum()
    assert np.array_equal(got[:, clean].view(np.uint32), want[:, clean].view(np.uint32))
    assert (got[:, ~mask] == np.float32(bg)[:, None]).all()


@pytest.mark.parametrize("case", list(CASES))
def test_bilinear_sampling_is_grid_sample_at_the_oracles_uvs(case):
    from sugar_b200 import texture
    sc, cam, v, f, verts_uv, faces_uv, tex, zbuf, p2f = setup(case)
    img = texture.render_textured_mesh(v, f, verts_uv, faces_uv, tex, cam)      # bilinear, black background
    ref = oracle_view(sc, v, f, verts_uv, faces_uv, tex, zbuf, p2f, "bilinear")  # grid_sample on the GPU
    T = tex.shape[0]
    # the kernel's float32 UV is within MARGIN_PER_T T texels of the exact one on each axis (see test_gpu_texture),
    # so the bilinear value moves by at most that times the largest step between neighbouring texels, per axis
    step = max(float((tex[1:] - tex[:-1]).abs().max()), float((tex[:, 1:] - tex[:, :-1]).abs().max()))
    tol = 2 * tg.MARGIN_PER_T * T * step + 4e-7
    mask = ref["mask"]
    d = np.abs(img.cpu().numpy().reshape(3, -1) - ref["image"].reshape(3, -1))
    print(f"{case}: T={T}, max difference {d[:, mask].max():.3g}, tolerance {tol:.3g}, "
          f"{float((d[:, mask] == 0).mean()):.4f} of values equal")
    assert d[:, mask].max() <= tol
    assert (d[:, ~mask] == 0).all()


def gaussian_render(cam, points, scaling, quats, strengths, sh_dc):
    """The render extract_texture_image_and_uv_from_gaussians bakes: sh degree 0, black background."""
    from sugar_b200.diff_gaussian_rasterization import GaussianRasterizationSettings, GaussianRasterizer
    P = points.shape[0]
    st = GaussianRasterizationSettings(image_height=cam.height, image_width=cam.width, tanfovx=cam.tanfovx,
                                       tanfovy=cam.tanfovy, bg=torch.zeros(3, device="cuda"), scale_modifier=1.0,
                                       viewmatrix=cam.viewmatrix, projmatrix=cam.projmatrix, sh_degree=0,
                                       campos=cam.campos, prefiltered=False, debug=False)
    with torch.no_grad():
        return GaussianRasterizer(st)(means3D=points, means2D=torch.zeros_like(points), opacities=strengths.view(P, 1),
                                      shs=sh_dc.reshape(P, 1, 3), scales=scaling, rotations=quats)[0]


def test_one_view_bake_renders_back_from_its_camera():
    from sugar_b200 import splatmesh, texture
    verts, faces, points, scaling, quats, strengths, sh_dc, _ = tg.coloured_icosphere()
    W, H = 256, 192
    cam = tg.look_at((3.0, 1.0, 2.0), W, H)
    verts_uv, faces_uv, tex = texture.extract_texture_image_and_uv_from_gaussians(
        verts, faces, points, scaling, quats, strengths, sh_dc, [cam], square_size=10)
    T = tex.shape[0]
    assert T * T < 2 ** 24
    img = texture.render_textured_mesh(verts, faces, verts_uv, faces_uv, tex, cam, sampling_mode="nearest")
    # each pixel's texel, from the render itself: a map whose texels hold their own index
    ids = torch.arange(T * T, device="cuda", dtype=torch.float32).view(T, T, 1).expand(T, T, 3).contiguous()
    texel = texture.render_textured_mesh(verts, faces, verts_uv, faces_uv, ids, cam, sampling_mode="nearest")[0]
    zbuf, p2f = splatmesh.rasterize_mesh(verts, faces, cam)
    baked = ((p2f >= 0) & (zbuf > 0)).reshape(-1)
    texel = texel.reshape(-1).long()
    pix = torch.nonzero(baked)[:, 0]
    winner = torch.full((T * T,), -1, dtype=torch.long, device="cuda")
    winner.scatter_reduce_(0, texel[pix], pix, "amax")                         # the bake's rule: highest index
    won = winner[winner >= 0]
    colour = gaussian_render(cam, points, scaling, quats, strengths, sh_dc).clamp(0, 1).reshape(3, -1)
    flat = img.reshape(3, -1)
    print(f"{int(baked.sum())} baked pixels, {len(won)} winners")
    assert baked.sum() > 5000 and len(won) > 1000
    assert torch.equal(flat[:, won].view(torch.int32), colour[:, won].view(torch.int32))
    assert torch.equal(flat[:, pix].view(torch.int32), flat[:, winner[texel[pix]]].view(torch.int32))
    assert (flat[:, ~baked] == 0).all()


def test_far_plane_blend_matches_the_oracle_and_empty_pixels_are_the_background():
    from sugar_b200 import scenes, splatmesh, texture
    W, H = 320, 240
    sc = scenes.make_scene(10, W, H, seed=0)
    cam = tg.cam_of(sc)
    # a quad over pixels (20..300, 20..220) with corner depths 8, 11, 12, 9: every row crosses zfar = 10
    at = lambda px, py, z: [((2 * px + 1) / W - 1) * sc.tanfovx * z, ((2 * py + 1) / H - 1) * sc.tanfovy * z, z]
    v = torch.tensor([at(20, 20, 8.0), at(300, 20, 11.0), at(300, 220, 12.0), at(20, 220, 9.0)]).cuda()
    f = torch.tensor([[0, 1, 2], [0, 2, 3]]).cuda()
    verts_uv, faces_uv, T = texture.uv_layout(2, 10, device="cuda")
    colour, bg = (0.8, 0.3, 0.6), (0.1, 0.2, 0.9)
    tex = torch.tensor(colour).cuda().expand(T, T, 3).contiguous()
    kw = dict(background=bg, znear=0.01, zfar=10.0)
    img = texture.render_textured_mesh(v, f, verts_uv, faces_uv, tex, cam, sampling_mode="nearest", **kw)
    zbuf, p2f = splatmesh.rasterize_mesh(v, f, cam)
    ref = oracle_view(sc, v, f, verts_uv, faces_uv, tex.cpu(), zbuf, p2f, "nearest", **kw)
    got, want, mask = img.cpu().numpy().reshape(3, -1), ref["image"].reshape(3, -1), ref["mask"]
    z = zbuf.cpu().numpy().reshape(-1)
    c, b = np.float32(colour)[:, None], np.float32(bg)[:, None]
    mixed = mask & (np.abs(got - c).max(0) > 1e-3) & (np.abs(got - b).max(0) > 1e-3)
    print(f"{int(mask.sum())} covered pixels, {int((mask & (z > 10)).sum())} beyond zfar, {int(mixed.sum())} mixed; "
          f"max difference {np.abs(got - want).max():.3g}")
    assert (mask & (z < 9.9)).sum() > 1000 and (mask & (z > 10.1)).sum() > 1000 and mixed.sum() > 50
    assert np.abs(got - want).max() <= 4e-6                                   # expf against numpy's exp
    front = mask & (z < 9.9)
    assert np.array_equal(got[:, front], want[:, front])
    assert (np.abs(got[:, mask & (z > 10.1)] - b) <= 1e-6).all()
    assert (got[:, ~mask] == b).all()
    # no faces at all: the background everywhere
    empty = texture.render_textured_mesh(v, f[:0], verts_uv, faces_uv[:0], tex, cam, **kw)
    assert (empty.cpu().numpy().reshape(3, -1) == b).all()


def test_render_is_deterministic():
    from sugar_b200 import texture
    _, cam, v, f, verts_uv, faces_uv, tex, _, _ = setup("height_field", 640, 480)
    for mode in ("bilinear", "nearest"):
        a = texture.render_textured_mesh(v, f, verts_uv, faces_uv, tex, cam, sampling_mode=mode)
        b = texture.render_textured_mesh(v, f, verts_uv, faces_uv, tex, cam, sampling_mode=mode)
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))


def test_saved_and_loaded_mesh_renders_as_the_quantised_one(tmp_path):
    from sugar_b200 import objfile, texture
    verts, faces, points, scaling, quats, strengths, sh_dc, _ = tg.coloured_icosphere()
    W, H = 256, 192
    cams = [tg.look_at((3.0, 1.0, 2.0), W, H), tg.look_at((-2.0, 3.0, 1.0), W, H)]
    verts_uv, faces_uv, tex = texture.extract_texture_image_and_uv_from_gaussians(
        verts, faces, points, scaling, quats, strengths, sh_dc, cams, square_size=10)
    path = tmp_path / "textured.obj"
    objfile.save_textured_mesh(path, verts, faces, verts_uv, faces_uv, tex)
    v2, f2, uv2, fuv2, tex2 = objfile.load_textured_mesh(path, "cuda")
    q = lambda t: torch.tensor([float("%f" % x) for x in t.reshape(-1).tolist()], dtype=torch.float64).float() \
        .view(t.shape).cuda()
    qtex = (torch.trunc(tex.cpu().clamp(0, 1) * 255.0) / 255.0).cuda()    # the reader divides on the CPU
    for cam in cams:
        for mode in ("bilinear", "nearest"):
            a = texture.render_textured_mesh(v2, f2, uv2, fuv2, tex2, cam, sampling_mode=mode)
            b = texture.render_textured_mesh(q(verts), faces, q(verts_uv), faces_uv, qtex, cam, sampling_mode=mode)
            assert torch.equal(a.view(torch.int32), b.view(torch.int32))
            assert (a != 0).any()
