"""The textured mesh on disk: the .obj / .mtl / .png triple the reference writes at the end of
extract_refined_mesh_with_texture.py (sugar_extractors/refined_mesh.py:209-219) and reads back in metrics.py.

    save_textured_mesh(path, verts, faces, verts_uv, faces_uv, texture)     # pytorch3d.io.save_obj
    verts, faces, verts_uv, faces_uv, texture = load_textured_mesh(path)   # pytorch3d.io.load_objs_as_meshes
    image = texture.render_textured_mesh(verts, faces, verts_uv, faces_uv, texture, cam)

pytorch3d is not a dependency, so the lines below restate its published 0.7.4 source (pytorch3d/io/obj_io.py:
save_obj / _save, load_obj / _parse_obj / _format_faces_indices, and pytorch3d/io/mtl_io.py: _parse_mtl /
_load_texture_images with pytorch3d/io/utils.py: _read_image); nothing here was compared with pytorch3d itself.

Writing (save_obj with verts_uvs, faces_uvs and texture_map given, decimal_places None):
  <stem>.obj  "\\nmtllib <stem>.mtl\\nusemtl mesh\\n\\n", then one "v %f %f %f" line per vertex, one "vt %f %f" line per
              UV vertex and one "f a/ta b/tb c/tc" line per face (1-based), "\\n" after every line but the last
  <stem>.mtl  "newmtl mesh\\nmap_Kd <stem>.png\\n"
  <stem>.png  8-bit RGB of uint8(255 x) in float32: truncation, of the texture clamped to [0, 1] (NaN gives 0)
Reading (load_objs_as_meshes): "v" / "vt" numbers parsed to float64 and rounded to float32; face indices 1-based, or
negative counted from the end; the material's map_Kd image as float32 uint8 / 255, alpha dropped (convert("RGB")).
Accepted: triangles written "a/ta b/tb c/tc" under one material with a map_Kd image; "#" comments and "o" / "g" / "s"
lines are skipped.  Anything else (normals, other face forms, polygons, several materials) raises ValueError.

The PNG codec is the standard library's zlib and struct, so that this package depends on torch and numpy alone.  It
writes 8-bit RGB with filter type 0 on every row and reads 8-bit RGB and RGBA, not interlaced, with all five filter
types (Pillow, which writes the reference's PNGs, picks a filter per row).
"""
import os
import struct
import zlib

import numpy as np
import torch

PNG_SIGNATURE = b"\x89PNG\r\n\x1a\n"
MATERIAL = "mesh"


# ------------------------------------------------------------------------------------------------------------------ PNG
def _chunk(kind, data):
    return struct.pack(">I", len(data)) + kind + data + struct.pack(">I", zlib.crc32(kind + data) & 0xFFFFFFFF)


def write_png(path, rgb):
    """8-bit RGB PNG of `rgb` (uint8 [H,W,3] array), filter type 0 on every row."""
    rgb = np.ascontiguousarray(rgb)
    if rgb.dtype != np.uint8 or rgb.ndim != 3 or rgb.shape[2] != 3 or rgb.shape[0] < 1 or rgb.shape[1] < 1:
        raise ValueError(f"write_png takes a uint8 [H,W,3] array, got {rgb.dtype} {rgb.shape}")
    H, W = rgb.shape[:2]
    rows = np.zeros((H, 1 + 3 * W), np.uint8)          # column 0: the filter type byte
    rows[:, 1:] = rgb.reshape(H, 3 * W)
    with open(path, "wb") as f:
        f.write(PNG_SIGNATURE + _chunk(b"IHDR", struct.pack(">IIBBBBB", W, H, 8, 2, 0, 0, 0)) +
                _chunk(b"IDAT", zlib.compress(rows.tobytes(), 6)) + _chunk(b"IEND", b""))


def _unfilter(raw, H, W, bpp):
    """The filtered scanlines of the PNG spec (section 9) back to pixels: uint8 [H,W,bpp].  Sub, Average and Paeth
    depend on the pixel to the left and Up, Average and Paeth on the row above, so rows of mixed types are reconstructed
    along anti-diagonals, every pixel of one anti-diagonal at once."""
    rows = np.frombuffer(raw, np.uint8).reshape(H, 1 + W * bpp)
    ftype = rows[:, 0].astype(np.int64)
    if (ftype > 4).any():
        raise ValueError(f"PNG: filter type {int(ftype.max())} (0 to 4 exist)")
    data = rows[:, 1:].reshape(H, W, bpp).astype(np.int32)
    if not ftype.any():
        return data.astype(np.uint8)
    out = np.zeros((H + 1, W + 1, bpp), np.int32)       # a zero row above and a zero column to the left
    all_rows = np.arange(H)
    for d in range(H + W - 1):
        r = all_rows[max(0, d - W + 1):min(H, d + 1)]
        x = d - r
        a, b, c = out[r + 1, x], out[r, x + 1], out[r, x]   # left, up, up-left
        t = ftype[r][:, None]
        p = a + b - c
        pa, pb, pc = np.abs(p - a), np.abs(p - b), np.abs(p - c)
        paeth = np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, c))
        pred = np.select([t == 1, t == 2, t == 3, t == 4], [a, b, (a + b) >> 1, paeth], 0)
        out[r + 1, x + 1] = (data[r, x] + pred) & 255
    return out[1:, 1:].astype(np.uint8)


def read_png(path, keep_alpha=False):
    """-> uint8 [H,W,3]: an 8-bit RGB or RGBA (alpha dropped) PNG without interlacing.  With `keep_alpha` an RGBA
    PNG gives uint8 [H,W,4]."""
    with open(path, "rb") as f:
        buf = f.read()
    if buf[:8] != PNG_SIGNATURE:
        raise ValueError(f"{path}: not a PNG file")
    pos, ihdr, idat = 8, None, []
    while True:
        if pos + 8 > len(buf):
            raise ValueError(f"{path}: truncated PNG (no IEND chunk)")
        n, kind = struct.unpack(">I4s", buf[pos:pos + 8])
        data = buf[pos + 8:pos + 8 + n]
        if len(data) != n or pos + 12 + n > len(buf):
            raise ValueError(f"{path}: truncated PNG chunk {kind!r}")
        crc = struct.unpack(">I", buf[pos + 8 + n:pos + 12 + n])[0]
        if zlib.crc32(kind + data) & 0xFFFFFFFF != crc:
            raise ValueError(f"{path}: PNG chunk {kind!r} fails its CRC")
        pos += 12 + n
        if kind == b"IHDR":
            ihdr = struct.unpack(">IIBBBBB", data)
        elif kind == b"IDAT":
            idat.append(data)
        elif kind == b"IEND":
            break
        elif kind != b"PLTE" and not kind[0] & 0x20:     # PLTE is only a suggestion for truecolour images
            raise ValueError(f"{path}: unsupported critical PNG chunk {kind!r}")
    if ihdr is None or not idat:
        raise ValueError(f"{path}: PNG without IHDR or IDAT")
    W, H, depth, colour, compression, filt, interlace = ihdr
    if depth != 8 or colour not in (2, 6) or compression or filt or interlace or W < 1 or H < 1:
        raise ValueError(f"{path}: PNG of bit depth {depth}, colour type {colour}, interlace {interlace}: only 8-bit "
                         "RGB (2) and RGBA (6) without interlacing are read")
    bpp = 3 if colour == 2 else 4
    raw = zlib.decompress(b"".join(idat))
    if len(raw) != H * (1 + W * bpp):
        raise ValueError(f"{path}: PNG image data of {len(raw)} bytes, {H * (1 + W * bpp)} expected for {W}x{H}")
    px = _unfilter(raw, H, W, bpp)
    return np.ascontiguousarray(px if keep_alpha else px[..., :3])


# ------------------------------------------------------------------------------------------------------------- .obj I/O
def _stem_paths(path):
    base, _ = os.path.splitext(os.fspath(path))
    return base + ".mtl", base + ".png", os.path.basename(base)


def _rows(t, name, dtype, width):
    if not torch.is_tensor(t) or t.dtype != dtype or t.dim() != 2 or t.shape[1] != width:
        got = f"{t.dtype} {tuple(t.shape)}" if torch.is_tensor(t) else type(t).__name__
        raise ValueError(f"{name} must be {str(dtype).replace('torch.', '')} [N,{width}], got {got}")
    return t.detach().cpu()


def save_textured_mesh(path, verts, faces, verts_uv, faces_uv, texture):
    """Write `path` (.obj), and beside it <stem>.mtl and <stem>.png, as the reference's save_obj call does.

    verts float32 [V,3], faces int64 [F,3], verts_uv float32 [n_uv,2], faces_uv int64 [F,3], texture float32 [H,W,3]
    (as texture.extract_texture_image_and_uv_from_gaussians returns them; any device)."""
    verts = _rows(verts, "verts", torch.float32, 3)
    faces = _rows(faces, "faces", torch.int64, 3)
    verts_uv = _rows(verts_uv, "verts_uv", torch.float32, 2)
    faces_uv = _rows(faces_uv, "faces_uv", torch.int64, 3)
    if faces_uv.shape[0] != faces.shape[0]:
        raise ValueError(f"faces_uv has {faces_uv.shape[0]} rows, faces {faces.shape[0]}")
    if not torch.is_tensor(texture) or texture.dtype != torch.float32 or texture.dim() != 3 or texture.shape[2] != 3:
        raise ValueError("texture must be float32 [H,W,3]")
    mtl_path, png_path, stem = _stem_paths(path)
    lines = f"\nmtllib {stem}.mtl\nusemtl {MATERIAL}\n\n"
    if len(verts) or len(faces):
        V, n_uv, F = verts.shape[0], verts_uv.shape[0], faces.shape[0]
        body = ("v %f %f %f\n" * V) % tuple(verts.reshape(-1).tolist())
        body += ("vt %f %f\n" * n_uv) % tuple(verts_uv.reshape(-1).tolist())
        ids = torch.stack([faces + 1, faces_uv + 1], -1).reshape(-1).tolist()
        body += ("f %d/%d %d/%d %d/%d\n" * F) % tuple(ids)
        lines += body[:-1] if F else body                      # no newline after the last face
    with open(path, "w") as f:
        f.write(lines)
    # (texture_map.clamp(0, 1) * 255.0).astype(uint8): float32 product, truncated
    q = (texture.detach().cpu().clamp(0.0, 1.0) * 255.0).nan_to_num(0.0).numpy().astype(np.uint8)
    write_png(png_path, q)
    with open(mtl_path, "w") as f:
        f.write(f"newmtl {MATERIAL}\nmap_Kd {stem}.png\n")


def _parse_mtl(path):
    """-> {material name: map_Kd file name}."""
    maps, name = {}, None
    with open(path) as f:
        for line in f:
            tokens = line.strip().split()
            if not tokens:
                continue
            if tokens[0] == "newmtl":
                name = tokens[1] if len(tokens) > 1 else ""
            elif tokens[0] == "map_Kd" and name is not None:
                maps[name] = line.strip()[len("map_Kd"):].strip()
    return maps


def _face_ids(ids, n, what, path):
    """1-based or negative (from the end) obj indices -> 0-based int64, checked against [0, n)."""
    ids = np.asarray(ids, np.int64).reshape(-1, 3)
    ids = np.where(ids > 0, ids - 1, ids + n)
    bad = (ids < 0) | (ids >= n)
    if bad.any():
        raise ValueError(f"{path}: {int(bad.sum())} face {what} indices outside the {n} {what}s")
    return torch.from_numpy(ids)


def load_textured_mesh(path, device="cpu"):
    """Read an .obj written by save_textured_mesh (or any triangle .obj in that form) as load_objs_as_meshes does.
    -> (verts float32 [V,3], faces int64 [F,3], verts_uv float32 [n_uv,2], faces_uv int64 [F,3],
    texture float32 [H,W,3]) on `device`, ready for texture.render_textured_mesh."""
    path = os.fspath(path)
    v, vt, fv, ft = [], [], [], []
    mtllib, material = None, None
    with open(path) as f:
        for no, line in enumerate(f, 1):
            tokens = line.split()
            if not tokens or tokens[0].startswith("#") or tokens[0] in ("o", "g", "s"):
                continue
            key = tokens[0]
            if key == "v" and len(tokens) >= 4:
                v.extend(tokens[1:4])
            elif key == "vt" and len(tokens) >= 3:
                vt.extend(tokens[1:3])
            elif key == "f":
                corners = [c.split("/") for c in tokens[1:]]
                if len(corners) != 3 or any(len(c) != 2 or not c[0] or not c[1] for c in corners):
                    raise ValueError(f"{path}:{no}: only triangles written 'f a/ta b/tb c/tc' are read, got "
                                     f"{line.strip()!r}")
                if material is None:
                    raise ValueError(f"{path}:{no}: a face before any 'usemtl' line")
                for c in corners:
                    fv.append(c[0])
                    ft.append(c[1])
            elif key == "mtllib" and len(tokens) >= 2:
                if mtllib is not None:
                    raise ValueError(f"{path}:{no}: a second 'mtllib' line (one material is read)")
                mtllib = line.strip()[len("mtllib"):].strip()
            elif key == "usemtl" and len(tokens) >= 2:
                if material is not None and tokens[1] != material:
                    raise ValueError(f"{path}:{no}: a second material {tokens[1]!r} (one material is read)")
                material = tokens[1]
            else:
                raise ValueError(f"{path}:{no}: unsupported line {line.strip()!r}")
    if mtllib is None or material is None:
        raise ValueError(f"{path}: no 'mtllib' / 'usemtl' line: the texture cannot be found")
    data_dir = os.path.dirname(path)
    maps = _parse_mtl(os.path.join(data_dir, mtllib))
    if material not in maps:
        raise ValueError(f"{path}: material {material!r} has no map_Kd image in {mtllib}")
    verts = torch.from_numpy(np.fromiter(map(float, v), np.float64, len(v)).reshape(-1, 3).astype(np.float32))
    verts_uv = torch.from_numpy(np.fromiter(map(float, vt), np.float64, len(vt)).reshape(-1, 2).astype(np.float32))
    faces = _face_ids([int(x) for x in fv], verts.shape[0], "vertex", path)
    faces_uv = _face_ids([int(x) for x in ft], verts_uv.shape[0], "UV vertex", path)
    # _read_image(format="RGB") as float32, then / 255.0
    texture = torch.from_numpy(read_png(os.path.join(data_dir, maps[material])).astype(np.float32)) / 255.0
    return tuple(t.to(device) for t in (verts, faces, verts_uv, faces_uv, texture))
