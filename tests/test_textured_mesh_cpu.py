"""CPU checks of the textured mesh's render and files: the C entry point's and render_textured_mesh's argument checks,
the render restatement (oracle/textured_mesh_oracle.py: sampling against torch's grid_sample, the K = 1 blend against
softmax_rgb_blend's formula), the .obj / .mtl / .png writer and reader (sugar_b200/objfile.py) and loss.psnr."""
import ctypes
import os
import struct
import sys
import zlib
from types import SimpleNamespace

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import textured_mesh_oracle as tmo  # noqa: E402
from sugar_b200 import objfile, scenes  # noqa: E402


def test_library_lists_the_render_entry_point_and_checks_its_arguments():
    from sugar_b200 import _lib
    L = _lib.lib
    assert "sgr_texture_render" in _lib.PROTOTYPES and hasattr(L, "sgr_texture_render")
    d = ctypes.c_void_p(256)

    def render(V=3, F=1, n_uv=3, Wt=8, Ht=4, W=8, H=8, mode=0, znear=1e-4, zfar=100.0, ptrs=None, uv=None):
        p = [d] * 10 if ptrs is None else ptrs
        if uv is not None:
            p = p[:2] + [uv] + p[3:]
        return L.sgr_texture_render(V, F, n_uv, Wt, Ht, *p[:7], W, H, p[7], p[8], mode, 0.0, 0.0, 0.0, znear, zfar,
                                    p[9], None)

    assert render(Wt=0) == -1 and b"bad sizes" in L.sgr_last_error()
    assert render(Ht=-1) == -1 and b"bad sizes" in L.sgr_last_error()
    assert render(Wt=65536, Ht=65536) == -1 and b"bad sizes" in L.sgr_last_error()
    assert render(W=70000, H=70000) == -1 and b"bad sizes" in L.sgr_last_error()
    assert render(F=-1) == -1 and b"bad sizes" in L.sgr_last_error()
    assert render(mode=2) == -1 and b"sampling_mode" in L.sgr_last_error()
    assert render(mode=-1) == -1 and b"sampling_mode" in L.sgr_last_error()
    assert render(znear=1.0, zfar=1.0) == -1 and b"znear < zfar" in L.sgr_last_error()
    assert render(zfar=float("inf")) == -1 and b"znear < zfar" in L.sgr_last_error()
    assert render(znear=float("nan")) == -1 and b"znear < zfar" in L.sgr_last_error()
    for k in range(10):                                  # every pointer is required when there are faces
        ptrs = [d] * 10
        ptrs[k] = None
        assert render(ptrs=ptrs) == -1 and b"null pointer" in L.sgr_last_error(), k
    # no faces: the mesh arrays may be null, the image, z-buffer, texture and matrices may not
    assert render(F=0, ptrs=[None] * 4 + [None] + [d] * 5) == -1 and b"null pointer" in L.sgr_last_error()
    assert render(uv=ctypes.c_void_p(260)) == -1 and b"8-byte aligned" in L.sgr_last_error()
    assert render(W=0, ptrs=[None] * 10) == 0                                   # no pixels


def cam_of(W=32, H=24, device="cpu"):
    from sugar_b200 import steps
    return steps.camera_from_scene(scenes.make_scene(10, W, H, seed=0), device)


def test_render_textured_mesh_validates_arguments():
    from sugar_b200 import texture
    cam = cam_of()
    v, f = torch.zeros(6, 3), torch.tensor([[0, 1, 2], [3, 4, 5]])
    verts_uv, faces_uv, T = texture.uv_layout(2, 10)
    tex = torch.zeros(T, T, 3)
    call = lambda **kw: texture.render_textured_mesh(**{**dict(verts=v, faces=f, verts_uv=verts_uv, faces_uv=faces_uv,
                                                               texture=tex, cam=cam), **kw})
    with pytest.raises(ValueError, match="sampling_mode"):
        call(sampling_mode="bicubic")
    with pytest.raises(ValueError, match="background must have 3"):
        call(background=(0.0, 0.0))
    with pytest.raises(ValueError, match="znear < zfar"):
        call(znear=5.0, zfar=5.0)
    with pytest.raises(ValueError, match="znear < zfar"):
        call(zfar=float("inf"))
    with pytest.raises(ValueError, match="texture must be float32"):
        call(texture=tex.double())
    with pytest.raises(ValueError, match="texture must be float32"):
        call(texture=tex[..., :2])
    with pytest.raises(ValueError, match="texture"):
        call(texture=torch.zeros(0, 4, 3))
    with pytest.raises(ValueError, match="verts_uv must be float32"):
        call(verts_uv=verts_uv.double())
    with pytest.raises(ValueError, match="faces_uv must be int64"):
        call(faces_uv=faces_uv[:1])
    with pytest.raises(ValueError, match="faces must be int64"):
        call(faces=f.int())
    with pytest.raises(ValueError, match="faces_uv ids outside"):
        call(faces_uv=faces_uv + 100)
    with pytest.raises(ValueError, match="projmatrix"):
        call(cam=SimpleNamespace(**{**vars(cam), "projmatrix": cam.projmatrix.double()}))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        call()


# ---------------------------------------------------------------------------------------------------------- sampling
def boundary_uvs(Wt, Ht, n=4000, seed=0):
    """Random UVs over [-0.3, 1.3], and UVs on texel centres (k / (size-1)), on half-texels and at the clip limits."""
    rng = np.random.default_rng(seed)
    rand = rng.uniform(-0.3, 1.3, (n, 2))
    ku, kv = rng.integers(0, Wt, n), rng.integers(0, Ht, n)
    centres = np.stack([ku / (Wt - 1), kv / (Ht - 1)], 1)
    halves = np.stack([(ku + 0.5) / (Wt - 1), (kv + 0.5) / (Ht - 1)], 1)
    edges = np.array([[0.0, 0.0], [1.0, 1.0], [0.0, 1.0], [1.0, 0.0], [-5.0, 7.0], [np.inf, -np.inf]])
    return torch.from_numpy(np.concatenate([rand, centres, halves, edges]).astype(np.float32))


@pytest.mark.parametrize("mode", ["bilinear", "nearest"])
@pytest.mark.parametrize("Wt,Ht", [(13, 13), (17, 6), (1, 5)])
def test_oracle_sampling_is_grid_sample_on_the_flipped_map(mode, Wt, Ht):
    tex = torch.rand(Ht, Wt, 3, generator=torch.Generator().manual_seed(Wt * Ht))
    uv = boundary_uvs(max(Wt, 2), max(Ht, 2))
    got = tmo.sample_texture(uv, tex, mode)
    # TexturesUV.sample_textures, written out: maps [N,C,H,W] flipped along H, grid uv * 2 - 1
    maps = torch.flip(tex.permute(2, 0, 1).unsqueeze(0), [2])
    want = torch.nn.functional.grid_sample(maps, (uv * 2.0 - 1.0)[None, None], mode=mode, align_corners=True,
                                           padding_mode="border")[0, :, 0].T
    assert got.dtype == torch.float32 and torch.equal(got.view(torch.int32), want.view(torch.int32))
    if mode == "nearest":
        # the bake's lookup (texel_of_uv for a square map) wherever the rounding is not at a half-texel
        finite = torch.isfinite(uv).all(1).numpy()
        u, v = uv[:, 0].double().numpy(), uv[:, 1].double().numpy()
        x = np.clip(u[finite] * (Wt - 1), 0, Wt - 1)
        y = np.clip(v[finite] * (Ht - 1), 0, Ht - 1)
        far = (np.abs(np.abs(x - np.floor(x)) - 0.5) > 1e-4) & (np.abs(np.abs(y - np.floor(y)) - 0.5) > 1e-4)
        cols, rows = np.rint(x).astype(int), (Ht - 1) - np.rint(y).astype(int)
        assert far.sum() > 1000
        assert torch.equal(got[finite][far], tex[rows[far], cols[far]])


def bilinear_restated(uv, tex):
    """grid_sampler_2d's bilinear arithmetic in float32 (numpy), products and sums rounded separately."""
    f32 = np.float32
    Ht, Wt = tex.shape[:2]
    t = tex.numpy()
    u, v = uv[:, 0].numpy(), uv[:, 1].numpy()
    with np.errstate(invalid="ignore"):
        ix = np.minimum(f32(Wt - 1), np.maximum(((u * f32(2) - f32(1)) + f32(1)) / f32(2) * f32(Wt - 1), f32(0)))
        iy = np.minimum(f32(Ht - 1), np.maximum(((v * f32(2) - f32(1)) + f32(1)) / f32(2) * f32(Ht - 1), f32(0)))
    ix, iy = np.nan_to_num(ix), np.nan_to_num(iy)
    x0, y0 = np.floor(ix).astype(int), np.floor(iy).astype(int)
    out = np.zeros((len(u), 3), f32)
    for dx, dy in ((0, 0), (1, 0), (0, 1), (1, 1)):
        x, y = x0 + dx, y0 + dy
        w = ((f32(1) - np.abs(ix - x.astype(f32))) * (f32(1) - np.abs(iy - y.astype(f32)))).astype(f32)
        ok = (x < Wt) & (y < Ht)
        out[ok] += t[Ht - 1 - y[ok], x[ok]] * w[ok, None]
    return out


def test_oracle_bilinear_is_torch_arithmetic_to_rounding():
    tex = torch.rand(11, 19, 3, generator=torch.Generator().manual_seed(4))
    uv = boundary_uvs(19, 11)
    got = tmo.sample_texture(uv, tex, "bilinear").numpy()
    want = bilinear_restated(uv, tex)
    assert np.abs(got - want).max() <= 4 * np.finfo(np.float32).eps


# ------------------------------------------------------------------------------------------------------------- blend
def softmax_rgb_blend_k1(colors, zbuf, mask, background, znear, zfar, sigma=1e-4, gamma=1e-4):
    """pytorch3d 0.7.4 softmax_rgb_blend for [P,K=1] fragments with prob = mask, in torch, line by line."""
    eps = 1e-10
    prob_map = mask.float()[:, None]
    z_inv = (zfar - zbuf[:, None]) / (zfar - znear) * mask[:, None]
    z_inv_max = torch.max(z_inv, dim=-1).values[..., None].clamp(min=eps)
    weights_num = prob_map * torch.exp((z_inv - z_inv_max) / gamma)
    delta = torch.exp((eps - z_inv_max) / gamma).clamp(min=eps)
    denom = weights_num.sum(dim=-1)[..., None] + delta
    weighted_colors = (weights_num[..., None] * colors[:, None]).sum(dim=-2)
    return (weighted_colors + delta * torch.tensor(background)) / denom


def test_blend_is_the_k1_formula_in_front_of_inside_and_beyond_the_far_band():
    znear, zfar, bg = 1e-4, 100.0, (0.1, 0.6, 0.9)
    rng = np.random.default_rng(2)
    band = zfar - 0.0025 * (zfar - znear)
    z = np.concatenate([rng.uniform(0.01, 90.0, 300), rng.uniform(band, zfar, 300), rng.uniform(zfar, 130.0, 300),
                        [zfar, band, 1e-4, -1.0]]).astype(np.float32)
    mask = np.ones(len(z), bool)
    mask[::7] = False
    c = rng.uniform(0, 1, (len(z), 3)).astype(np.float32)
    got = tmo.blend(c, z, mask, bg, znear, zfar)
    want = softmax_rgb_blend_k1(torch.from_numpy(np.where(mask[:, None], c, 0)), torch.from_numpy(z),
                                torch.from_numpy(mask), bg, znear, zfar).numpy()
    assert (got[~mask] == np.float32(bg)).all()
    front = mask & (z < 90.0)
    inside = mask & (z >= band) & (z < zfar)
    beyond = mask & (z > zfar + 0.5)                 # w = exp(z_inv / gamma) < e^-50
    # in front: delta is clamped to 1e-10, so (c + 1e-10 bg) / (1 + 1e-10) -- the texel up to 1e-10 bg
    assert np.array_equal(got[front], want[front].astype(np.float32))
    assert np.array_equal(got[front], ((c[front] + np.float32(1e-10) * np.float32(bg)) / np.float32(1.0 + 1e-10)))
    # inside the band the two colours mix; the division by gamma rounds differently (reciprocal vs quotient)
    mixed = inside & (np.abs(got - c).max(1) > 1e-3) & (np.abs(got - np.float32(bg)).max(1) > 1e-3)
    assert mixed.sum() > 50
    assert np.abs(got - want).max() < 1e-4
    # beyond: the background
    assert np.abs(got[beyond] - np.float32(bg)).max() <= 1e-6
    assert np.abs(got[beyond] - want[beyond]).max() <= 1e-6


# ------------------------------------------------------------------------------------------------------- obj / png I/O
def small_mesh():
    verts = torch.tensor([[0.0, 0.0, 0.0], [1.0, -2.5, 1e-7], [0.1234567, 3.0, -7.25], [12345.678, 0.5, 2.0]])
    faces = torch.tensor([[0, 1, 2], [2, 1, 3]])
    verts_uv = torch.tensor([[0.0, 0.0], [1.0, 0.5], [0.333333343, 0.9999999], [0.25, 1.0], [0.5, 0.5], [1.0, 1.0]])
    faces_uv = torch.tensor([[0, 1, 2], [3, 4, 5]])
    tex = torch.tensor([[[0.0, 0.5, 1.0], [1.5, -0.2, 0.999], [0.0039, 0.00393, 0.25]],
                        [[0.1, 0.2, 0.3], [float("nan"), 1.0, 0.0], [0.7, 0.8, 0.9]]])
    return verts, faces, verts_uv, faces_uv, tex


def test_obj_and_mtl_text_is_save_objs(tmp_path):
    verts, faces, verts_uv, faces_uv, tex = small_mesh()
    objfile.save_textured_mesh(tmp_path / "mesh.obj", verts, faces, verts_uv, faces_uv, tex)
    text = (tmp_path / "mesh.obj").read_text()
    want = "\nmtllib mesh.mtl\nusemtl mesh\n\n"
    want += "".join("v %f %f %f\n" % tuple(float(x) for x in r) for r in verts)
    want += "".join("vt %f %f\n" % tuple(float(x) for x in r) for r in verts_uv)
    want += "f 1/1 2/2 3/3\nf 3/4 2/5 4/6"
    assert text == want
    assert "v 12345.677734 0.500000 2.000000\n" in text and "v 1.000000 -2.500000 0.000000\n" in text
    assert (tmp_path / "mesh.mtl").read_text() == "newmtl mesh\nmap_Kd mesh.png\n"
    png = objfile.read_png(tmp_path / "mesh.png")
    assert png.dtype == np.uint8 and png.shape == (2, 3, 3)
    q = np.trunc(np.float32(255.0) * np.nan_to_num(np.clip(tex.numpy(), 0, 1)).astype(np.float32))
    assert np.array_equal(png, q.astype(np.uint8))
    assert png[0, 2].tolist() == [0, 1, 63]                                   # 0.99 and 1.002 truncate to 0 and 1


def test_save_load_round_trip_rounds_through_the_text_and_the_png(tmp_path):
    verts, faces, verts_uv, faces_uv, tex = small_mesh()
    rng = np.random.default_rng(5)
    verts = torch.cat([verts, torch.from_numpy(rng.normal(0, 30, (200, 3)).astype(np.float32))])
    verts_uv = torch.cat([verts_uv, torch.from_numpy(rng.uniform(0, 1, (200, 2)).astype(np.float32))])
    faces = torch.cat([faces, torch.from_numpy(rng.integers(0, 204, (150, 3)))])
    faces_uv = torch.cat([faces_uv, torch.from_numpy(rng.integers(0, 206, (150, 3)))])
    tex = torch.from_numpy(rng.uniform(-0.1, 1.1, (40, 30, 3)).astype(np.float32))
    path = str(tmp_path / "sub dir" / "model.obj")
    os.makedirs(os.path.dirname(path))
    objfile.save_textured_mesh(path, verts, faces, verts_uv, faces_uv, tex)
    v2, f2, uv2, fuv2, tex2 = objfile.load_textured_mesh(path)
    f32 = lambda t: torch.tensor([[float("%f" % float(x)) for x in r] for r in t], dtype=torch.float64).float()
    assert v2.dtype == torch.float32 and torch.equal(v2, f32(verts)) and torch.equal(uv2, f32(verts_uv))
    assert f2.dtype == torch.int64 and torch.equal(f2, faces) and torch.equal(fuv2, faces_uv)
    q = torch.trunc(tex.clamp(0, 1) * 255.0) / 255.0
    assert tex2.dtype == torch.float32 and tex2.shape == tex.shape and torch.equal(tex2, q)


def write_filtered_png(path, rgb, ftypes):
    """An independent PNG encoder for the tests: row r filtered with ftypes[r] (PNG spec, section 9)."""
    H, W, bpp = rgb.shape
    img = rgb.astype(np.int64)
    out = bytearray()
    for r in range(H):
        out.append(ftypes[r])
        for x in range(W):
            for ch in range(bpp):
                a = img[r, x - 1, ch] if x else 0
                b = img[r - 1, x, ch] if r else 0
                c = img[r - 1, x - 1, ch] if r and x else 0
                p = a + b - c
                pa, pb, pc = abs(p - a), abs(p - b), abs(p - c)
                paeth = a if pa <= pb and pa <= pc else (b if pb <= pc else c)
                pred = (0, a, b, (a + b) // 2, paeth)[ftypes[r]]
                out.append((img[r, x, ch] - pred) & 255)
    colour = 2 if bpp == 3 else 6
    chunk = lambda k, d: struct.pack(">I", len(d)) + k + d + struct.pack(">I", zlib.crc32(k + d) & 0xFFFFFFFF)
    with open(path, "wb") as f:
        f.write(objfile.PNG_SIGNATURE + chunk(b"IHDR", struct.pack(">IIBBBBB", W, H, 8, colour, 0, 0, 0)) +
                chunk(b"IDAT", zlib.compress(bytes(out))[:20]) + chunk(b"IDAT", zlib.compress(bytes(out))[20:]) +
                chunk(b"tEXt", b"k\x00v") + chunk(b"IEND", b""))


def png_filter_types(path):
    buf = open(path, "rb").read()
    pos, idat = 8, []
    while pos < len(buf):
        n, k = struct.unpack(">I4s", buf[pos:pos + 8])
        if k == b"IHDR":
            W, H, _, colour = struct.unpack(">IIBB", buf[pos + 8:pos + 18])
        if k == b"IDAT":
            idat.append(buf[pos + 8:pos + 8 + n])
        pos += 12 + n
    return set(np.frombuffer(zlib.decompress(b"".join(idat)), np.uint8).reshape(H, -1)[:, 0].tolist())


def test_png_codec_reads_every_filter_type_and_its_own_files(tmp_path):
    rng = np.random.default_rng(8)
    for bpp in (3, 4):
        img = rng.integers(0, 256, (23, 9, bpp)).astype(np.uint8)
        img[5:12] = np.cumsum(rng.integers(0, 9, (7, 9, bpp)), axis=1).astype(np.uint8)   # smooth rows
        types = [r % 5 for r in range(23)]
        write_filtered_png(tmp_path / f"f{bpp}.png", img, types)
        assert png_filter_types(tmp_path / f"f{bpp}.png") == {0, 1, 2, 3, 4}
        assert np.array_equal(objfile.read_png(tmp_path / f"f{bpp}.png"), img[..., :3])
        for t in range(5):                                                     # one filter type on every row
            write_filtered_png(tmp_path / "one.png", img, [t] * 23)
            assert np.array_equal(objfile.read_png(tmp_path / "one.png"), img[..., :3]), t
    img = rng.integers(0, 256, (31, 17, 3)).astype(np.uint8)
    objfile.write_png(tmp_path / "own.png", img)
    assert png_filter_types(tmp_path / "own.png") == {0}
    assert np.array_equal(objfile.read_png(tmp_path / "own.png"), img)


def test_png_codec_against_pillow(tmp_path):
    Image = pytest.importorskip("PIL.Image")
    rng = np.random.default_rng(9)
    H, W = 96, 64
    y, x = np.mgrid[0:H, 0:W]
    img = np.zeros((H, W, 3), np.uint8)
    img[:16] = rng.integers(0, 256, (16, W, 3))                               # noise
    img[16:32] = (x[16:32, :, None] * 4) % 256                                 # ramps along rows
    img[32:48] = img[31:32]                                                    # repeated rows
    img[48:96] = ((x[48:96] * 3 + y[48:96] * 5) % 256)[..., None] + rng.integers(0, 3, (48, W, 3)).astype(np.uint8)
    seen = set()
    for name, arr in (("rgb", img), ("rgba", np.dstack([img, 255 - img[..., :1]]))):
        Image.fromarray(arr).save(tmp_path / f"{name}.png")
        seen |= png_filter_types(tmp_path / f"{name}.png")
        assert np.array_equal(objfile.read_png(tmp_path / f"{name}.png"), img), name
    assert seen >= {1, 2, 4}, seen                                             # Pillow's adaptive choice
    # Pillow reads the codec's files and the test encoder's, every filter type
    objfile.write_png(tmp_path / "own.png", img)
    assert np.array_equal(np.asarray(Image.open(tmp_path / "own.png")), img)
    small = img[::8, ::8]
    write_filtered_png(tmp_path / "all.png", small, [r % 5 for r in range(small.shape[0])])
    assert np.array_equal(np.asarray(Image.open(tmp_path / "all.png").convert("RGB")), small)


def test_png_codec_rejects_what_it_cannot_read(tmp_path):
    img = np.zeros((4, 5, 3), np.uint8)
    objfile.write_png(tmp_path / "a.png", img)
    buf = bytearray(open(tmp_path / "a.png", "rb").read())
    for what, edit in (("not a PNG", lambda b: b"GIF89a" + b[6:]),
                       ("CRC", lambda b: b[:20] + bytes([b[20] ^ 1]) + b[21:]),
                       ("bit depth 16", lambda b: b[:24] + b"\x10" + b[25:]),
                       ("interlace 1", lambda b: b[:28] + b"\x01" + b[29:]),
                       ("colour type 3", lambda b: b[:25] + b"\x03" + b[26:]),
                       ("truncated", lambda b: b[:-12])):
        data = bytearray(edit(bytes(buf)))
        if what not in ("not a PNG", "CRC", "truncated"):                      # keep the edited IHDR's CRC valid
            data[29:33] = struct.pack(">I", zlib.crc32(bytes(data[12:29])) & 0xFFFFFFFF)
        open(tmp_path / "b.png", "wb").write(bytes(data))
        with pytest.raises(ValueError):
            objfile.read_png(tmp_path / "b.png")
    with pytest.raises(ValueError, match="uint8"):
        objfile.write_png(tmp_path / "c.png", img.astype(np.float32))


@pytest.mark.parametrize("line,match", [("f 1/1 2/2 3/3 1/1", "only triangles"), ("f 1/1/1 2/2/2 3/3/3", "only triangles"),
                                        ("f 1 2 3", "only triangles"), ("f 1//1 2//2 3//3", "only triangles"),
                                        ("vn 0 0 1", "unsupported line"), ("usemtl other", "second material"),
                                        ("f 1/1 2/2 9/3", "vertex indices outside"),
                                        ("f 1/1 2/2 3/-9", "UV vertex indices outside")])
def test_obj_reader_rejects_what_it_cannot_read(tmp_path, line, match):
    verts, faces, verts_uv, faces_uv, tex = small_mesh()
    objfile.save_textured_mesh(tmp_path / "m.obj", verts, faces, verts_uv, faces_uv, tex)
    text = (tmp_path / "m.obj").read_text()
    (tmp_path / "m.obj").write_text(text + "\n" + line + "\n")
    with pytest.raises(ValueError, match=match):
        objfile.load_textured_mesh(tmp_path / "m.obj")


def test_obj_reader_takes_negative_indices_comments_and_groups(tmp_path):
    verts, faces, verts_uv, faces_uv, tex = small_mesh()
    objfile.save_textured_mesh(tmp_path / "m.obj", verts, faces, verts_uv, faces_uv, tex)
    text = (tmp_path / "m.obj").read_text()
    (tmp_path / "m.obj").write_text("# written by hand\no part\ng grp\ns off\n" + text + "\nf -4/-6 -3/-5 -2/-4\n")
    _, f2, _, fuv2, _ = objfile.load_textured_mesh(tmp_path / "m.obj")
    assert f2.tolist() == faces.tolist() + [[0, 1, 2]] and fuv2.tolist() == faces_uv.tolist() + [[0, 1, 2]]
    (tmp_path / "n.obj").write_text(text.replace("mtllib m.mtl\n", ""))
    with pytest.raises(ValueError, match="mtllib"):
        objfile.load_textured_mesh(tmp_path / "n.obj")
    (tmp_path / "m.mtl").write_text("newmtl other\nmap_Kd m.png\n")
    with pytest.raises(ValueError, match="no map_Kd"):
        objfile.load_textured_mesh(tmp_path / "m.obj")


# -------------------------------------------------------------------------------------------------------------- psnr
def test_psnr_is_the_reference_formula():
    from sugar_b200 import loss
    g = torch.Generator().manual_seed(1)
    a, b = torch.rand(3, 3, 20, 30, generator=g), torch.rand(3, 3, 20, 30, generator=g)
    b[1] = a[1] + 0.01
    p = loss.psnr(a, b)
    mse = ((a.double() - b.double()) ** 2).reshape(3, -1).mean(1, keepdim=True)
    assert p.shape == (3, 1) and p.dtype == torch.float32
    assert torch.allclose(p.double(), 20 * torch.log10(1.0 / torch.sqrt(mse)), rtol=1e-5)
    assert abs(float(p[1]) - 40.0) < 1e-3
    assert torch.isinf(loss.psnr(a, a)).all()
