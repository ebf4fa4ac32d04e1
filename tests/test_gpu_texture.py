"""GPU: the UV texture extraction (sugar_b200/texture.py, csrc/sgr_texture.cu): the layout and the initial texels
against the reference's own lines (tests/golden/texture_*.npz), the per-view bake against its CPU restatement
(oracle/texture_oracle.py) on given z-buffers, and the whole extraction on a bound icosphere."""
import glob
import math
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import splatmesh_oracle as smo  # noqa: E402
from oracle import texture_oracle as to  # noqa: E402

GOLDEN = sorted(os.path.basename(p)[8:-4] for p in glob.glob(os.path.join(HERE, "golden", "texture_*.npz")))
# texel units, per unit of T: the float32 UV (barycentric and accumulator roundings, 2u - 1, + 1) is within about
# 5e-7 of the exact one, so u (T-1) within 5e-7 T plus the last product's rounding; 8e-7 T leaves a margin
MARGIN_PER_T = 8e-7


def golden(name):
    return np.load(os.path.join(HERE, "golden", f"texture_{name}.npz"))


@pytest.mark.parametrize("name", GOLDEN)
def test_uv_layout_is_the_reference_golden(name):
    from sugar_b200 import texture
    g = golden(name)
    verts_uv, faces_uv, T = texture.uv_layout(g["faces"].shape[0], int(g["square_size"]), device="cuda")
    assert verts_uv.is_cuda and T == g["texture"].shape[0]
    assert np.array_equal(verts_uv.cpu().numpy().view(np.uint32), g["verts_uv"].view(np.uint32))
    assert np.array_equal(faces_uv.cpu().numpy(), g["faces_uv"])


@pytest.mark.parametrize("name", GOLDEN)
def test_initial_texture_matches_the_reference_golden(name):
    from sugar_b200 import texture
    g = golden(name)
    c = lambda k: torch.from_numpy(g[k]).cuda()
    tex = texture.initial_texture(c("verts"), c("faces"), c("points"), c("scaling"), c("quaternions"), c("sh_dc"),
                                  square_size=int(g["square_size"])).cpu().numpy()
    ref = g["texture"]
    t = lambda k: torch.from_numpy(g[k])
    _, d2, owned = to.initial_texture(t("verts"), t("faces"), t("points"), t("scaling"), t("quaternions"),
                                      t("sh_dc"), int(g["square_size"]))
    d2, owned = d2.numpy(), owned.numpy()
    with np.errstate(invalid="ignore"):               # inf - inf with one Gaussian per face, NaN at square size 3
        tie = owned & (np.abs(d2[..., 1] - d2[..., 0]) <= 1e-4 * np.abs(d2[..., 0]))
    print(f"{name}: {int(tie.sum())} of {int(owned.sum())} owned texels excluded as argmax near-ties")
    assert tie.sum() <= 0.01 * owned.sum()
    assert tex.shape == ref.shape and tex.dtype == np.float32
    assert (np.abs(tex - ref)[~tie] <= 1e-6).all(), np.abs(tex - ref)[~tie].max()
    assert (tex[~owned] == 0.5).all()


def cam_of(sc):
    from sugar_b200 import steps
    return steps.camera_from_scene(sc, "cuda")


def hand_made(W, H):
    """Seeded triangles of all sizes and tilts in front of an identity camera, some overlapping, some crossing the
    image border."""
    from sugar_b200 import scenes
    sc = scenes.make_scene(10, W, H, seed=0)
    rng = np.random.default_rng(17)
    v = []
    for _ in range(60):
        z = rng.uniform(1.0, 8.0, 3)
        px, py = rng.uniform(-10, W + 10, 3), rng.uniform(-10, H + 10, 3)
        v += [[((2 * x + 1) / W - 1) * sc.tanfovx * zz, ((2 * y + 1) / H - 1) * sc.tanfovy * zz, zz]
              for x, y, zz in zip(px, py, z)]
    return sc, np.asarray(v, np.float32), np.arange(len(v)).reshape(-1, 3)


def icosphere_case(W, H):
    from sugar_b200 import scenes
    sc = scenes.make_scene(10, W, H, seed=0)
    v, f = scenes.icosphere(3, radius=1.2)
    return sc, (v + np.array([0.1, -0.2, 4.0], np.float32)).astype(np.float32), f


def heightfield_case(W, H):
    from sugar_b200 import scenes
    sc = scenes.make_scene(10, W, H, seed=5, camera="posed")
    v, f = scenes.height_field_mesh(60, 50, seed=3, amplitude=0.1, permute=True)
    # put the unit square 3 units in front of the posed camera, tilted
    Vt = sc.viewmatrix.astype(np.float64)
    inv = np.linalg.inv(Vt)
    view_pts = (v.astype(np.float64) - [0.5, 0.5, 0.0]) * [2.2, 1.8, 1.0] @ scenes._rot(np.array([1.0, 0.2, 0]), 0.5).T
    view_pts[:, 2] += 3.0
    return sc, (view_pts @ inv[:3, :3] + inv[3, :3]).astype(np.float32), f


def candidates(out, verts_uv, faces_uv, faces, verts, sc, r, T):
    """Texel ids a float32 UV may round to for the pixels within the margin of a half-integer: the oracle's texel and
    its neighbour across the near half."""
    MARGIN = MARGIN_PER_T * T
    near = (out["margin"] < MARGIN).reshape(-1)
    p2f = r["pix_to_face"].reshape(-1)
    b = to.pixel_barycentrics(verts.astype(np.float64), faces, sc.viewmatrix, sc.projmatrix, sc.width, sc.height,
                              np.where(near, p2f, -1))[near]
    uv = (b[:, :, None] * verts_uv.astype(np.float64)[faces_uv[p2f[near]]]).sum(1)
    x, y = np.clip(uv[:, 0] * (T - 1), 0, T - 1), np.clip(uv[:, 1] * (T - 1), 0, T - 1)
    other = lambda c: np.where(np.abs(np.abs(c - np.floor(c)) - 0.5) < MARGIN,
                               np.floor(c) + (np.rint(c) == np.floor(c)), np.rint(c))
    cols, rows = [np.rint(x), other(x)], [np.rint(y), other(y)]
    ids = [((T - 1 - rr) * T + cc).astype(np.int64) for rr in rows for cc in cols]
    return np.clip(np.concatenate(ids), 0, T * T - 1)


def compare_bake(sc, verts, faces, square_size, label, n_views=2):
    """Bake n_views views (the same z-buffer, different images) on the GPU and in the oracle; compare."""
    from sugar_b200 import texture
    W, H = sc.width, sc.height
    F = faces.shape[0]
    r = smo.rasterize(verts.astype(np.float64), faces, sc.viewmatrix, sc.projmatrix, W, H)
    verts_uv, faces_uv, T = texture.uv_layout(F, square_size, device="cuda")
    init = torch.rand(T, T, 3, generator=torch.Generator().manual_seed(3)).cuda()
    state = texture.new_bake_state(init)
    s_ref = np.zeros((T, T, 3), np.float32)
    c_ref = np.zeros((T, T), np.int64)
    dirty = np.zeros(T * T, bool)
    cam = cam_of(sc)
    v_t, f_t = torch.from_numpy(verts).cuda(), torch.from_numpy(np.ascontiguousarray(faces, np.int64)).cuda()
    rng = np.random.default_rng(11)
    for _ in range(n_views):
        image = rng.uniform(-0.2, 1.2, (3, H, W)).astype(np.float32)
        texture.bake_view(state, v_t, f_t, verts_uv, faces_uv, cam, torch.from_numpy(image).cuda(),
                          torch.from_numpy(r["zbuf"].astype(np.float32)).cuda(),
                          torch.from_numpy(r["pix_to_face"]).cuda())
        out = to.bake_view(s_ref, c_ref, verts.astype(np.float64), faces, verts_uv.cpu().numpy(),
                           faces_uv.cpu().numpy(), sc.viewmatrix, sc.projmatrix, image, r["zbuf"], r["pix_to_face"])
        # a pixel near a half-integer may land on the neighbouring texel: both candidates are excluded
        dirty[candidates(out, verts_uv.cpu().numpy(), faces_uv.cpu().numpy(), faces, verts, sc, r, T)] = True
    touched = c_ref.reshape(-1) > 0
    clean = touched & ~dirty
    print(f"{label}: T={T}, {int(touched.sum())} texels baked, {int((touched & dirty).sum())} excluded at margins")
    assert touched.sum() > 500
    assert clean.sum() >= 0.99 * touched.sum()
    s_gpu, c_gpu = state.sum.cpu().numpy().reshape(-1, 3), state.count.cpu().numpy().reshape(-1)
    assert np.array_equal(c_gpu[clean], c_ref.reshape(-1)[clean])
    assert np.array_equal(s_gpu[clean].view(np.uint32), s_ref.reshape(-1, 3)[clean].view(np.uint32))
    assert (c_gpu[~touched & ~dirty] == 0).all()
    assert (state.owner == -1).all()
    fin = texture.finish(state).cpu().numpy().reshape(-1, 3)
    ref = to.finish(s_ref, c_ref, init.cpu().numpy()).reshape(-1, 3)
    assert np.array_equal(fin[~dirty].view(np.uint32), ref[~dirty].view(np.uint32))
    return state


def test_bake_matches_oracle_hand_made_320x240():
    compare_bake(*hand_made(320, 240), square_size=200, label="hand-made 320x240")


def test_bake_matches_oracle_icosphere_320x240():
    compare_bake(*icosphere_case(320, 240), square_size=10, label="icosphere 320x240")


def test_bake_matches_oracle_height_field_320x240_and_is_deterministic():
    sc, verts, faces = heightfield_case(320, 240)
    a = compare_bake(sc, verts, faces, square_size=6, label="height field 320x240")
    b = compare_bake(sc, verts, faces, square_size=6, label="height field 320x240, again")
    assert torch.equal(a.count, b.count) and torch.equal(a.sum.view(torch.int32), b.sum.view(torch.int32))


def look_at(pos, W, H, fov_x=0.8, target=(0.0, 0.0, 0.0)):
    """steps.camera_from_scene-style namespace of a camera at `pos` looking at `target`."""
    from sugar_b200 import render
    p = torch.tensor(pos, dtype=torch.float32)
    z = p - torch.tensor(target, dtype=torch.float32)
    z = z / z.norm()                                            # OpenGL: the camera looks down -z
    up = torch.tensor([0.0, 0.0, 1.0]) if abs(float(z[2])) < 0.9 else torch.tensor([0.0, 1.0, 0.0])
    x = torch.linalg.cross(up, z)
    x = x / x.norm()
    y = torch.linalg.cross(z, x)
    c2w = torch.stack([x, y, z, p], 1).cuda()
    fov_y = 2 * math.atan(math.tan(fov_x / 2) * H / W)
    view, proj, center = render.camera_matrices(c2w, fov_x, fov_y)
    return SimpleNamespace(viewmatrix=view, projmatrix=proj, campos=center, width=W, height=H,
                           tanfovx=math.tan(fov_x / 2), tanfovy=math.tan(fov_y / 2))


def coloured_icosphere(n=6, scale=0.15):
    from sugar_b200 import meshbind, scenes
    v, f = scenes.icosphere(2)
    verts, faces = torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda()
    F = faces.shape[0]
    g = torch.Generator().manual_seed(9)
    colours = torch.rand(F, 3, generator=g).cuda()
    edge = float((verts[faces[:, 0]] - verts[faces[:, 1]]).norm(dim=-1).mean())
    scales_raw = torch.full((F * n, 2), math.log(scale * edge)).cuda()
    complex_raw = torch.tensor([1.0, 0.0]).repeat(F * n, 1).cuda()
    b = meshbind.bind_to_mesh(verts, faces, meshbind.bary_coords(n, "cuda"), scales_raw, complex_raw, 1e-3 * edge)
    sh_dc = ((colours - 0.5) / 0.28209479177387814).repeat_interleave(n, 0)
    strengths = torch.full((F * n,), 0.999, device="cuda")
    return verts, faces, b.points.detach(), b.scaling.detach(), b.quaternions.detach(), strengths, sh_dc, colours


def face_of_texel(F, s, T):
    owner = np.full((T, T), -1, np.int64)
    n_sq = T // s
    bottom, top = (t.numpy() for t in to.owned_texels(s))
    for f in range(F):
        k = f // 2
        loc = bottom if f % 2 == 0 else top
        i, j = (k // n_sq) * s + loc[:, 0], (k % n_sq) * s + loc[:, 1]
        owner[T - 1 - j, i] = f
    return owner


def test_extraction_bakes_visible_faces_with_their_colour():
    from sugar_b200 import splatmesh, texture
    verts, faces, points, scaling, quats, strengths, sh_dc, colours = coloured_icosphere()
    F, s = faces.shape[0], 10
    W, H = 256, 192
    # 8 cameras on a ring above the equator: the bottom cap is never seen
    cams = [look_at((3.5 * math.cos(a), 3.5 * math.sin(a), 2.5), W, H) for a in np.arange(8) * math.pi / 4]
    verts_uv, faces_uv, tex = texture.extract_texture_image_and_uv_from_gaussians(
        verts, faces, points, scaling, quats, strengths, sh_dc, cams, square_size=s)
    ref_uv, ref_fuv, T = texture.uv_layout(F, s, device="cuda")
    assert torch.equal(verts_uv, ref_uv) and torch.equal(faces_uv, ref_fuv) and tex.shape == (T, T, 3)
    init = texture.initial_texture(verts, faces, points, scaling, quats, sh_dc, square_size=s)
    seen = torch.zeros(F, dtype=torch.bool, device="cuda")
    for cam in cams:
        _, p2f = splatmesh.rasterize_mesh(verts, faces, cam)
        seen[p2f[p2f >= 0]] = True
    owner = torch.from_numpy(face_of_texel(F, s, T)).cuda()
    changed = (tex != init).any(-1)
    print(f"{int(seen.sum())} of {F} faces seen, {int(changed.sum())} texels baked")
    assert 0.3 * F < int(seen.sum()) < 0.95 * F
    # texels of faces never seen (nor their square's partner) keep the initial texture
    partner = (torch.arange(F, device="cuda") ^ 1).clamp(max=F - 1)
    unseen = ~seen & ~seen[partner]
    keep = (owner >= 0) & unseen[owner.clamp(min=0)]
    assert keep.sum() > 0 and torch.equal(tex[keep], init[keep])
    # baked texels of seen faces carry (about) their face's colour: the render blends each face's six Gaussians with
    # its neighbours', so the check is against the colour of an unrelated face as well as an absolute bound
    baked = changed & (owner >= 0) & seen[owner.clamp(min=0)]
    err = (tex[baked] - colours[owner[baked]]).abs().max(-1).values
    other = (tex[baked] - colours[(owner[baked] + F // 2) % F]).abs().max(-1).values
    print(f"colour error of {int(baked.sum())} baked texels: median {float(err.median()):.4f}, "
          f"90% {float(err.quantile(0.9)):.4f}; against another face's colour: median {float(other.median()):.4f}")
    assert baked.sum() > 0.2 * (owner >= 0).sum()
    assert float(err.median()) < 0.2 and float(err.median()) < 0.5 * float(other.median())
    # bit-identical from run to run; a view that sees nothing changes nothing
    away = look_at((0.0, 40.0, 0.0), W, H, target=(0.0, 80.0, 0.0))   # the sphere is behind it
    zb, p2f = splatmesh.rasterize_mesh(verts, faces, away)
    assert (p2f == -1).all()
    _, _, tex2 = texture.extract_texture_image_and_uv_from_gaussians(
        verts, faces, points, scaling, quats, strengths, sh_dc, cams[:4] + [away] + cams[4:], square_size=s)
    assert torch.equal(tex.view(torch.int32), tex2.view(torch.int32))


def test_empty_view_and_state_round_trip():
    from sugar_b200 import texture
    sc, verts, faces = icosphere_case(64, 48)
    verts_uv, faces_uv, T = texture.uv_layout(faces.shape[0], 10, device="cuda")
    init = torch.rand(T, T, 3, device="cuda")
    state = texture.new_bake_state(init)
    H, W = 48, 64
    texture.bake_view(state, torch.from_numpy(verts).cuda(), torch.from_numpy(faces).cuda(), verts_uv, faces_uv,
                      cam_of(sc), torch.rand(3, H, W, device="cuda"), torch.full((H, W), -1.0, device="cuda"),
                      torch.full((H, W), -1, dtype=torch.int64, device="cuda"))
    assert (state.count == 0).all() and (state.sum == 0).all() and (state.owner == -1).all()
    assert torch.equal(texture.finish(state), init)
