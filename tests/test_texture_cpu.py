"""CPU checks of the UV texture extraction: the restatement (oracle/texture_oracle.py) and sugar_b200.texture.uv_layout
against the reference's own layout and initial-texel lines (tests/golden/texture_*.npz), the per-view rule on
hand-made cases with known answers, the C entry points without a GPU and the Python entry points' argument checks."""
import ctypes
import glob
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import texture_oracle as to  # noqa: E402
from sugar_b200 import scenes  # noqa: E402

GOLDEN = sorted(os.path.basename(p)[8:-4] for p in glob.glob(os.path.join(HERE, "golden", "texture_*.npz")))


def golden(name):
    return np.load(os.path.join(HERE, "golden", f"texture_{name}.npz"))


def test_golden_cases_are_present():
    assert set(GOLDEN) >= {"f1_n1_s10", "f1_n6_s3", "f7_n6_s10", "f7_n1_s3", "heightfield_n6_s10", "heightfield_n1_s4"}


@pytest.mark.parametrize("name", GOLDEN)
def test_layout_matches_the_reference_golden(name):
    from sugar_b200 import texture
    g = golden(name)
    F, s = g["faces"].shape[0], int(g["square_size"])
    for verts_uv, faces_uv, T in (to.layout(F, s), texture.uv_layout(F, s)):
        assert T == g["texture"].shape[0] == texture.texture_size(F, s)
        assert verts_uv.dtype == torch.float32 and faces_uv.dtype == torch.int64
        assert np.array_equal(verts_uv.numpy().view(np.uint32), g["verts_uv"].view(np.uint32))
        assert np.array_equal(faces_uv.numpy(), g["faces_uv"])


@pytest.mark.parametrize("name", GOLDEN)
def test_oracle_initial_texture_matches_the_reference_golden(name):
    g = golden(name)
    t = lambda k: torch.from_numpy(g[k])
    tex, d2, owned = to.initial_texture(t("verts"), t("faces"), t("points"), t("scaling"), t("quaternions"), t("sh_dc"),
                                 int(g["square_size"]))
    assert np.array_equal(tex.numpy().view(np.uint32), g["texture"].view(np.uint32))
    owned = owned.numpy()
    F, s = g["faces"].shape[0], int(g["square_size"])
    assert owned.sum() == F * s * (s - 1) // 2
    assert (g["texture"][~owned] == 0.5).all()
    if int(g["n"]) > 1 and s > 3:
        # the argmax is not trivial: the texels do not all take the face's first Gaussian
        first = (g["sh_dc"].reshape(F, -1, 3)[:, 0] * to.SH_C0 + 0.5).astype(np.float32)
        picks_first = np.zeros(owned.shape, bool)
        for f in range(F):
            picks_first |= np.all(g["texture"] == first[f], -1)
        assert (owned & ~picks_first).mean() > 0.1 * owned.mean()


def test_layout_rejects_small_squares():
    from sugar_b200 import texture
    for fn in (to.layout, texture.uv_layout):
        with pytest.raises(ValueError, match="square_size must be >= 3"):
            fn(10, 2)


def test_texel_lookup_scales_by_t_minus_1_flips_y_and_rounds_half_to_even():
    T = 5
    row, col, _ = to.texel_of_uv(np.array([0.0, 1.0, 0.0, 1.0]), np.array([0.0, 0.0, 1.0, 1.0]), T)
    assert col.tolist() == [0, 4, 0, 4] and row.tolist() == [4, 4, 0, 0]
    # u (T-1) = 2.5 and 3.5 exactly: half to even; clamped outside [0, 1]
    row, col, margin = to.texel_of_uv(np.array([0.625, 0.875, -0.3, 1.7]), np.array([0.625, 0.875, -0.3, 1.7]), T)
    assert col.tolist() == [2, 4, 0, 4] and row.tolist() == [2, 0, 4, 0]
    assert margin[:2].tolist() == [0.0, 0.0] and margin[2:].tolist() == [0.5, 0.5]


def camera(W, H):
    return scenes.make_scene(10, W, H, seed=0)


def at_pixel(sc, px, py, z):
    ndc_x, ndc_y = (2.0 * px + 1.0) / sc.width - 1.0, (2.0 * py + 1.0) / sc.height - 1.0
    return [ndc_x * sc.tanfovx * (z + 1e-7), ndc_y * sc.tanfovy * (z + 1e-7), z]


def quad_case(W=40, H=30, s=10, z=3.0):
    """A camera-facing quad (faces 0 and 1 of square 0) over pixels (4.3 .. 35.6, 3.2 .. 26.7)."""
    sc = camera(W, H)
    x0, x1, y0, y1 = 4.3, 35.6, 3.2, 26.7
    verts = np.array([at_pixel(sc, x0, y0, z), at_pixel(sc, x1, y0, z), at_pixel(sc, x1, y1, z),
                      at_pixel(sc, x0, y1, z)], np.float64)
    faces = np.array([[0, 1, 2], [0, 2, 3]])
    verts_uv, faces_uv, T = to.layout(2, s)
    from oracle import splatmesh_oracle as smo
    r = smo.rasterize(verts, faces, sc.viewmatrix, sc.projmatrix, W, H)
    return sc, verts, faces, verts_uv.numpy(), faces_uv.numpy(), T, r


def test_camera_facing_quad_lands_on_the_affine_uv_texels():
    sc, verts, faces, verts_uv, faces_uv, T, r = quad_case()
    W, H = sc.width, sc.height
    rng = np.random.default_rng(0)
    image = rng.uniform(0, 1, (3, H, W)).astype(np.float32)
    s = np.zeros((T, T, 3), np.float32)
    c = np.zeros((T, T), np.int64)
    out = to.bake_view(s, c, verts, faces, verts_uv, faces_uv, sc.viewmatrix, sc.projmatrix, image, r["zbuf"],
                       r["pix_to_face"])
    x, y, _ = to.smo.project(verts, sc.viewmatrix, sc.projmatrix, W, H)
    jj, ii = np.mgrid[0:H, 0:W]
    cov = r["pix_to_face"] >= 0
    assert cov.sum() > 500 and (out["texel"][cov] >= 0).all() and (out["texel"][~cov] == -1).all()
    for f in (0, 1):
        # constant depth: the UV is the affine map of the pixel fixed by the three projected corners
        A = np.stack([x[faces[f]], y[faces[f]], np.ones(3)], 1)
        coef = np.linalg.solve(A, verts_uv[faces_uv[f]].astype(np.float64))
        sel = (r["pix_to_face"] == f) & (out["margin"] > 1e-6)
        uv = np.stack([ii[sel], jj[sel], np.ones(sel.sum())], 1) @ coef
        row, col, _ = to.texel_of_uv(uv[:, 0], uv[:, 1], T)
        assert sel.sum() > 100 and np.array_equal(out["texel"][sel], row * T + col)
        # the face's pixels stay on its own triangle's texels of square 0, well inside the T x T map
        assert (col[:, None] < T // 2 + 1).all() and (row >= T // 2 - 1).all()
    assert c.sum() == len(np.unique(out["texel"][cov]))


def test_several_pixels_on_one_texel_keep_the_highest_index_and_count_once():
    # square size 3: T = 6, so the quad's ~700 pixels crowd onto a few texels
    sc, verts, faces, verts_uv, faces_uv, T, r = quad_case(s=3)
    W, H = sc.width, sc.height
    image = (np.arange(3 * H * W, dtype=np.float32).reshape(3, H, W) / (3 * H * W))
    s = np.zeros((T, T, 3), np.float32)
    c = np.zeros((T, T), np.int64)
    out = to.bake_view(s, c, verts, faces, verts_uv, faces_uv, sc.viewmatrix, sc.projmatrix, image, r["zbuf"],
                       r["pix_to_face"])
    tx = out["texel"].reshape(-1)
    used = np.unique(tx[tx >= 0])
    assert 1 < len(used) < 0.05 * (tx >= 0).sum()
    for t in used:
        last = np.nonzero(tx == t)[0].max()
        assert np.array_equal(s.reshape(-1, 3)[t], image.reshape(3, -1)[:, last])
        assert c.reshape(-1)[t] == 1 and out["winner"].reshape(-1)[last]
    # a second view adds once more in float32
    s2 = s.copy()
    to.bake_view(s2, c, verts, faces, verts_uv, faces_uv, sc.viewmatrix, sc.projmatrix, image, r["zbuf"],
                 r["pix_to_face"])
    assert np.array_equal(s2.reshape(-1, 3)[used], s.reshape(-1, 3)[used] + s.reshape(-1, 3)[used])
    assert (c.reshape(-1)[used] == 2).all()


def test_unreached_texels_keep_their_initial_value_and_zbuf_zero_is_skipped():
    sc, verts, faces, verts_uv, faces_uv, T, r = quad_case()
    W, H = sc.width, sc.height
    init = np.random.default_rng(1).uniform(0, 1, (T, T, 3)).astype(np.float32)
    image = np.full((3, H, W), 2.0, np.float32)        # clamped to 1
    zbuf = r["zbuf"].copy()
    zbuf[:, : W // 2] = 0.0                            # zbuf > 0 only
    s = np.zeros((T, T, 3), np.float32)
    c = np.zeros((T, T), np.int64)
    out = to.bake_view(s, c, verts, faces, verts_uv, faces_uv, sc.viewmatrix, sc.projmatrix, image, zbuf,
                       r["pix_to_face"])
    assert (out["texel"][:, : W // 2] == -1).all() and (out["texel"][:, W // 2:] >= 0).any()
    tex = to.finish(s, c, init)
    reached = c > 0
    assert reached.sum() > 20 and (tex[reached] == 1.0).all() and np.array_equal(tex[~reached], init[~reached])


def test_library_lists_the_texture_entry_points():
    from sugar_b200 import _lib
    L = _lib.lib
    for fn in ("sgr_texture_init", "sgr_texture_bake_view"):
        assert fn in _lib.PROTOTYPES and hasattr(L, fn)
    names = [L.sgr_kernel_name(k).decode() for k in range(L.sgr_num_kernel_kinds())]
    assert "misc" in names and names[-2:] == ["mesh_nc_forward", "mesh_nc_backward"]   # no kind was added
    d = ctypes.c_void_p(256)
    # F = 10, s = 10: n_sq = int(sqrt(6) + 1) = 3, T = 30
    assert L.sgr_texture_init(10, 1, 30, 2, 30, *([d] * 7), None) == -1 and b"bad sizes" in L.sgr_last_error()
    assert L.sgr_texture_init(10, 0, 30, 10, 30, *([d] * 7), None) == -1 and b"bad sizes" in L.sgr_last_error()
    assert L.sgr_texture_init(-1, 1, 30, 10, 30, *([d] * 7), None) == -1
    assert L.sgr_texture_init(10, 1, 30, 10, 40, *([d] * 7), None) == -1 and b"texture size" in L.sgr_last_error()
    big = 2 * 46341 * 46341                            # T = 10 * n_sq > 46340
    assert L.sgr_texture_init(big // 100, 1, 30, 10, 10 * int((big // 200 + 1) ** 0.5 + 1), *([d] * 7), None) == -1
    assert L.sgr_texture_init(10, 1, 30, 10, 30, d, d, d, d, d, None, d, None) == -1
    assert b"null pointer" in L.sgr_last_error()
    assert L.sgr_texture_init(10, 1, 30, 10, 30, d, d, d, d, ctypes.c_void_p(264), d, d, None) == -1   # misaligned
    bake = lambda V, F, n_uv, T, W, H, ptrs: L.sgr_texture_bake_view(V, F, n_uv, T, *ptrs[:6], W, H, *ptrs[6:], None)
    assert bake(3, 1, 6, 46341, 8, 8, [d] * 13) == -1 and b"bad sizes" in L.sgr_last_error()
    assert bake(3, 1, 6, 20, 70000, 70000, [d] * 13) == -1 and b"bad sizes" in L.sgr_last_error()
    assert bake(3, -1, 6, 20, 8, 8, [d] * 13) == -1
    assert bake(3, 1, 6, 20, 8, 8, [d] * 12 + [None]) == -1 and b"null pointer" in L.sgr_last_error()
    assert bake(3, 1, 6, 20, 8, 8, [d, d, None] + [d] * 10) == -1 and b"null pointer" in L.sgr_last_error()
    assert bake(3, 1, 6, 20, 0, 8, [None] * 13) == 0                                       # no pixels


def test_python_entry_points_validate_arguments():
    from sugar_b200 import steps, texture
    cam = steps.camera_from_scene(camera(32, 24), "cpu")
    v, f = torch.zeros(6, 3), torch.tensor([[0, 1, 2], [3, 4, 5]])
    p, s = torch.zeros(4, 3), torch.ones(4, 3)
    q, sh = torch.tensor([[1.0, 0, 0, 0]]).repeat(4, 1), torch.zeros(4, 3)
    with pytest.raises(ValueError, match="square_size must be >= 3"):
        texture.initial_texture(v, f, p, s, q, sh, square_size=2)
    with pytest.raises(ValueError, match="faces must be int64"):
        texture.initial_texture(v, f.int(), p, s, q, sh)
    with pytest.raises(ValueError, match="verts must be float32"):
        texture.initial_texture(v.double(), f, p, s, q, sh)
    with pytest.raises(ValueError, match="quaternions"):
        texture.initial_texture(v, f, p, s, q[:, :3], sh)
    with pytest.raises(ValueError, match="sh_dc"):
        texture.initial_texture(v, f, p, s, q, sh[:, :2])
    with pytest.raises(ValueError, match="Gaussians on 2 faces"):
        texture.initial_texture(v, f, p[:3], s[:3], q[:3], sh[:3])
    with pytest.raises(ValueError, match="outside"):
        texture.initial_texture(v, torch.tensor([[0, 1, 6], [0, 1, 2]]), p, s, q, sh)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        texture.initial_texture(v, f, p, s, q, sh)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        texture.new_bake_state(torch.zeros(20, 20, 3))
    with pytest.raises(ValueError, match="init_texture"):
        texture.new_bake_state(torch.zeros(20, 19, 3))
    verts_uv, faces_uv, T = texture.uv_layout(2, 10)
    state = SimpleNamespace(sum=torch.zeros(T, T, 3), count=torch.zeros(T, T, dtype=torch.int32),
                            owner=torch.full((T, T), -1, dtype=torch.int32), init=torch.zeros(T, T, 3))
    img, z, p2f = torch.zeros(3, 24, 32), torch.zeros(24, 32), torch.full((24, 32), -1)
    call = lambda **kw: texture.bake_view(**{**dict(state=state, verts=v, faces=f, verts_uv=verts_uv,
                                                    faces_uv=faces_uv, cam=cam, image=img, zbuf=z,
                                                    pix_to_face=p2f), **kw})
    with pytest.raises(ValueError, match="image must be float32"):
        call(image=img[:, :-1])
    with pytest.raises(ValueError, match="zbuf must be float32"):
        call(zbuf=z.double())
    with pytest.raises(ValueError, match="pix_to_face must be int64"):
        call(pix_to_face=p2f.int())
    with pytest.raises(ValueError, match="faces_uv must be int64"):
        call(faces_uv=faces_uv[:1])
    with pytest.raises(ValueError, match="verts_uv must be float32"):
        call(verts_uv=verts_uv.double())
    with pytest.raises(ValueError, match="pix_to_face values outside"):
        call(pix_to_face=torch.full((24, 32), 2))
    with pytest.raises(ValueError, match="faces_uv ids outside"):
        call(faces_uv=faces_uv + 100)
    with pytest.raises(ValueError, match="face vertex ids outside"):
        call(faces=torch.tensor([[0, 1, 2], [3, 4, 9]]))
    with pytest.raises(ValueError, match="projmatrix"):
        call(cam=SimpleNamespace(**{**vars(cam), "projmatrix": cam.projmatrix.double()}))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        call()
    with pytest.raises(ValueError, match="strengths"):
        texture.extract_texture_image_and_uv_from_gaussians(v, f, p, s, q, torch.ones(5), sh, [cam])
