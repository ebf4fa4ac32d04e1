"""Seeded datasets on disk for the reader tests: a small COLMAP model (.bin or .txt) with PNG images, and a small
NeRF-synthetic scene with RGBA PNGs.  The writers restate COLMAP's model formats (the layout colmap_loader.py reads)
and an 8-bit PNG encoder, so that the fixtures need nothing but numpy and the standard library."""
import json
import math
import os
import struct
import zlib

import numpy as np

PNG_SIGNATURE = b"\x89PNG\r\n\x1a\n"


def write_png(path, px):
    """uint8 [H,W,3|4] -> an 8-bit RGB or RGBA PNG (filter type 0 on every row)."""
    px = np.ascontiguousarray(px, np.uint8)
    H, W, C = px.shape
    chunk = lambda kind, data: (struct.pack(">I", len(data)) + kind + data +  # noqa: E731
                                struct.pack(">I", zlib.crc32(kind + data) & 0xFFFFFFFF))
    raw = b"".join(b"\x00" + px[y].tobytes() for y in range(H))
    with open(path, "wb") as f:
        f.write(PNG_SIGNATURE + chunk(b"IHDR", struct.pack(">IIBBBBB", W, H, 8, 2 if C == 3 else 6, 0, 0, 0)) +
                chunk(b"IDAT", zlib.compress(raw, 6)) + chunk(b"IEND", b""))


def rotmat2qvec(R):
    """colmap's rotmat2qvec (the quaternion of largest eigenvalue, w >= 0)."""
    Rxx, Ryx, Rzx, Rxy, Ryy, Rzy, Rxz, Ryz, Rzz = np.asarray(R, np.float64).flat
    K = np.array([[Rxx - Ryy - Rzz, 0, 0, 0], [Ryx + Rxy, Ryy - Rxx - Rzz, 0, 0],
                  [Rzx + Rxz, Rzy + Ryz, Rzz - Rxx - Ryy, 0], [Ryz - Rzy, Rzx - Rxz, Rxy - Ryx, Rxx + Ryy + Rzz]]) / 3.0
    vals, vecs = np.linalg.eigh(K)
    q = vecs[[3, 0, 1, 2], np.argmax(vals)]
    return -q if q[0] < 0 else q


def look_at(centre, target, up=(0.0, 1.0, 0.0)):
    """World -> camera rotation of a COLMAP camera (x right, y down, z forward) at `centre` looking at `target`."""
    z = np.asarray(target, np.float64) - centre
    z /= np.linalg.norm(z)
    x = np.cross(z, -np.asarray(up, np.float64))
    x /= np.linalg.norm(x)
    y = np.cross(z, x)
    return np.stack([x, y, z])


def ring_poses(n, radius=4.0, height=1.0, seed=0):
    """n seeded world -> camera (R_wc, t_wc) poses on a ring around the origin, looking at it."""
    rng = np.random.Generator(np.random.PCG64(seed))
    poses = []
    for i in range(n):
        a = 2 * math.pi * i / n + rng.uniform(-0.2, 0.2)
        c = np.array([radius * math.cos(a), height + rng.uniform(-0.3, 0.3), radius * math.sin(a)])
        R = look_at(c, rng.normal(0, 0.1, 3))
        poses.append((R, -R @ c))
    return poses


def write_colmap(sparse_dir, cameras, images, points, binary=True):
    """cameras: [(id, model name, width, height, params)]; images: [(id, qvec, tvec, camera id, name)];
    points: (xyz [N,3], rgb uint8 [N,3]).  Writes cameras / images / points3D as .bin or .txt."""
    ids = {"SIMPLE_PINHOLE": 0, "PINHOLE": 1, "SIMPLE_RADIAL": 2, "OPENCV": 4}
    os.makedirs(sparse_dir, exist_ok=True)
    xyz, rgb = points
    if binary:
        with open(os.path.join(sparse_dir, "cameras.bin"), "wb") as f:
            f.write(struct.pack("<Q", len(cameras)))
            for cid, model, w, h, params in cameras:
                f.write(struct.pack("<iiQQ", cid, ids[model], w, h) + struct.pack("<" + "d" * len(params), *params))
        with open(os.path.join(sparse_dir, "images.bin"), "wb") as f:
            f.write(struct.pack("<Q", len(images)))
            for iid, q, t, cid, name in images:
                f.write(struct.pack("<idddddddi", iid, *q, *t, cid) + name.encode() + b"\x00")
                f.write(struct.pack("<Q", 2) + struct.pack("<ddqddq", 1.5, 2.5, -1, 3.0, 4.0, 0))
        with open(os.path.join(sparse_dir, "points3D.bin"), "wb") as f:
            f.write(struct.pack("<Q", len(xyz)))
            for i in range(len(xyz)):
                f.write(struct.pack("<QdddBBBd", i + 1, *xyz[i], *(int(c) for c in rgb[i]), 0.5))
                f.write(struct.pack("<Q", 1) + struct.pack("<ii", 1, 0))
        return
    with open(os.path.join(sparse_dir, "cameras.txt"), "w") as f:
        f.write("# Camera list\n")
        for cid, model, w, h, params in cameras:
            f.write(f"{cid} {model} {w} {h} " + " ".join(repr(float(p)) for p in params) + "\n")
    with open(os.path.join(sparse_dir, "images.txt"), "w") as f:
        f.write("# Image list\n")
        for iid, q, t, cid, name in images:
            f.write(f"{iid} " + " ".join(repr(float(v)) for v in (*q, *t)) + f" {cid} {name}\n")
            f.write("1.5 2.5 -1 3.0 4.0 1\n")
    with open(os.path.join(sparse_dir, "points3D.txt"), "w") as f:
        f.write("# 3D point list\n")
        for i in range(len(xyz)):
            f.write(f"{i + 1} " + " ".join(repr(float(v)) for v in xyz[i]) + " " +
                    " ".join(str(int(c)) for c in rgb[i]) + " 0.5 1 0\n")


def colmap_case(root, binary=True, n=10, seed=0, sizes=((45, 31), (40, 30)), rgba_every=3, simple=True):
    """A seeded COLMAP dataset under `root`: n views over two cameras (PINHOLE, and SIMPLE_PINHOLE when `simple`),
    noise PNG images (every `rgba_every`-th RGBA, partial alpha), names listed out of order, 200 points.  -> root."""
    rng = np.random.Generator(np.random.PCG64(seed))
    (w0, h0), (w1, h1) = sizes
    second = (2, "SIMPLE_PINHOLE", w1, h1, [37.0, w1 / 2, h1 / 2]) if simple else \
        (2, "PINHOLE", w1, h1, [37.0, 36.0, w1 / 2, h1 / 2])
    cameras = [(1, "PINHOLE", w0, h0, [40.0, 42.5, w0 / 2, h0 / 2]), second]
    images = []
    os.makedirs(os.path.join(root, "images"), exist_ok=True)
    for i, (R, t) in enumerate(ring_poses(n, seed=seed)):
        cid = 1 + i % 2
        w, h = (w0, h0) if cid == 1 else (w1, h1)
        name = f"frame_{(7 * i) % n:03d}.png"
        C = 4 if i % rgba_every == 0 else 3
        px = rng.integers(0, 256, (h, w, C), dtype=np.uint8)
        if C == 4:
            px[..., 3] = rng.choice(np.array([0, 64, 128, 200, 255], np.uint8), (h, w))
        write_png(os.path.join(root, "images", name), px)
        images.append((i + 1, rotmat2qvec(R), t, cid, name))
    xyz = rng.normal(0, 1, (200, 3))
    rgb = rng.integers(0, 256, (200, 3), dtype=np.uint8)
    write_colmap(os.path.join(root, "sparse", "0"), cameras, images[::-1], (xyz, rgb), binary=binary)
    return root


def nerf_case(root, n_train=4, n_test=2, size=(24, 20), seed=0):
    """A seeded NeRF-synthetic scene under `root`: RGBA PNG frames (alpha 0 / partial / 255) with Blender
    camera-to-world matrices.  -> root."""
    rng = np.random.Generator(np.random.PCG64(seed))
    W, H = size
    for split, n in (("train", n_train), ("test", n_test)):
        frames = []
        os.makedirs(os.path.join(root, split), exist_ok=True)
        for i, (R, t) in enumerate(ring_poses(n, seed=seed + (split == "test"))):
            px = rng.integers(0, 256, (H, W, 4), dtype=np.uint8)
            px[..., 3] = rng.choice(np.array([0, 1, 128, 254, 255], np.uint8), (H, W))
            write_png(os.path.join(root, split, f"r_{i}.png"), px)
            c2w = np.eye(4)
            c2w[:3, :3] = R.T
            c2w[:3, 3] = -R.T @ t
            c2w[:3, 1:3] *= -1      # COLMAP axes to Blender's
            frames.append({"file_path": f"./{split}/r_{i}", "transform_matrix": c2w.tolist()})
        with open(os.path.join(root, f"transforms_{split}.json"), "w") as f:
            json.dump({"camera_angle_x": 0.69111120, "frames": frames}, f)
    return root
