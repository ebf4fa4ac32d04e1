"""Real scenes: COLMAP and NeRF-synthetic readers, cameras.json both ways, and the ground-truth images as the
reference prepares them.

    scene = load_colmap_scene("data/garden", resolution=-1)                    # 3DGS: readColmapSceneInfo + loadCam
    raw = train.init_from_points(torch.from_numpy(scene.points).cuda(), scene.colors)
    train.train_3dgs(raw, scene.train, scene.nerf_radius, rng=rng)
    write_cameras_json("out/cameras.json", scene.camera_list)                  # Scene.__init__'s cameras.json
    gsply.save_gaussians_ply("out/point_cloud/iteration_7000/point_cloud.ply", raw)
    train_views, test_views = load_gs_cameras("data/garden", "out")            # SuGaR: load_gs_cameras

Each view is `(cam, gt)`: `cam` the namespace the steps take (viewmatrix, projmatrix, campos, width, height, tanfovx,
tanfovy) plus the camera's metadata (name, uid, colmap_id, R, T, FoVx, FoVy, orig_width, orig_height); `gt` the
float32 [3,H,W] image on the device.  The matrices are gaussian_splatting/scene/cameras.py:37-59's: the float32
getWorld2View2(R, T) transposed, getProjectionMatrix(0.01, 100, FoVx, FoVy) transposed (scenes.projection_matrix),
their float32 product on the device and the camera centre from the inverse.  R is stored transposed (the
world-to-camera rotation is R^T), as the reference stores it.

Images are decoded on the host (PNG: objfile.read_png; JPEG: Pillow, imported only when a JPEG is met) and prepared on
the GPU by one sm_90a kernel per pass (csrc/sgr_image.cu), byte for byte as the reference's Pillow and numpy lines
(oracle/imageprep_oracle.py restates them): the float64 alpha composite where the reference composites, Pillow's
antialiased bicubic Image.resize (an RGBA image through premultiplied RGBa), then uint8 / 255.  The alpha channel is
never applied as a mask: loadCam's test `resized_image_rgb.shape[1] == 4` compares the image height with 4
(camera_utils.py:47-50), so the reference drops it for every image taller than 4 px, and so does this module.

Deliberate differences from the reference:
  - SuGaR's load_gs_cameras takes the image extension of `os.listdir(images)[0]`, which depends on directory order;
    here each camera resolves `<img_name>.{jpg,png,JPG,PNG}` and raises if there is none or more than one.
  - Nothing is written into the dataset: without points3D.ply the COLMAP points are converted in memory, rounded as
    storePly -> fetchPly would round them (float32 xyz, uint8 colours / 255); the NeRF-synthetic random cloud
    likewise.
  - COLMAP's text cameras.txt may hold SIMPLE_PINHOLE cameras (the reference's text reader asserts PINHOLE).
  - load_gs_cameras reads `<gs_output_path>/cameras.json` (the reference concatenates the two strings).
  - A NeRF-synthetic frame's image is `<path>/<file_path><extension>`.  The reference joins `path` onto that path a
    second time (dataset_readers.py:188, 200), which finds the file only because its argument parser makes the
    source path absolute; here a relative `path` works too.
Only PINHOLE and SIMPLE_PINHOLE cameras, resolution scale 1.0 and device-resident images are supported.
"""
import functools
import json
import math
import os
import struct
from types import SimpleNamespace

import numpy as np
import torch

from . import mcubes, objfile, scenes
from ._lib import SGR_IMAGE_COMPOSITE, SGR_IMAGE_PLAIN, SGR_IMAGE_PREMULTIPLY, check, lib, ptr, stream, tensor

ZNEAR, ZFAR = 0.01, 100.0
IMAGE_EXTENSIONS = (".jpg", ".png", ".JPG", ".PNG")


# ------------------------------------------------------------------------------------------------- image preparation
PRECISION_BITS = 22


def _bicubic(x):
    """Pillow's bicubic_filter (a = -0.5) in its own evaluation order."""
    x = np.abs(x)
    return np.where(x < 1.0, ((-0.5 + 2.0) * x - (-0.5 + 3.0)) * x * x + 1,
                    np.where(x < 2.0, (((x - 5) * x + 8) * x - 4) * -0.5, 0.0))


def resample_coeffs(in_size: int, out_size: int):
    """Pillow's bicubic Image.resize table for one axis (libImaging/Resample.c precompute_coeffs and
    normalize_coeffs_8bpc, in float64 as the C code evaluates it) -> (bounds int32 [out,2] = (first tap, taps),
    coeffs int32 [out, ksize] in 22-bit fixed point, ksize).  The weights of a row are divided by their sum taken left
    to right; taps past a row's count are 0."""
    if in_size < 1 or out_size < 1:
        raise ValueError(f"resample sizes must be >= 1, got {in_size} -> {out_size}")
    scale = float(in_size) / out_size
    filterscale = max(scale, 1.0)
    support = 2.0 * filterscale
    ksize = int(math.ceil(support)) * 2 + 1
    center = (np.arange(out_size, dtype=np.float64) + 0.5) * scale
    xmin = np.maximum(np.trunc(center - support + 0.5), 0).astype(np.int64)
    count = np.minimum(np.trunc(center + support + 0.5), in_size).astype(np.int64) - xmin
    k = np.zeros((out_size, ksize))
    total = np.zeros(out_size)
    for x in range(ksize):
        w = np.where(x < count, _bicubic(((x + xmin) - center + 0.5) * (1.0 / filterscale)), 0.0)
        k[:, x] = w
        total = total + w
    k = np.where(total[:, None] != 0.0, k / np.where(total == 0.0, 1.0, total)[:, None], k)
    k = k * float(1 << PRECISION_BITS)
    fixed = np.trunc(np.where(k < 0, -0.5 + k, 0.5 + k)).astype(np.int32)
    fixed[np.arange(ksize)[None, :] >= count[:, None]] = 0
    bounds = np.ascontiguousarray(np.stack([xmin, count], 1), dtype=np.int32)
    return bounds, fixed, ksize


@functools.lru_cache(maxsize=64)
def _tables(in_size, out_size, dev):
    """resample_coeffs' tables on `dev`, built once per (in, out, device) among the 64 most recently used."""
    b, c, k = resample_coeffs(in_size, out_size)
    return torch.from_numpy(b).to(dev), torch.from_numpy(c).to(dev), k


def prepare_image(image, width: int, height: int, background=None, device="cuda"):
    """A decoded uint8 [H,W,C] image (C = 3 or 4; numpy or torch) -> the float32 [3, height, width] ground truth on
    `device`, as the reference prepares it (see the module docstring).  `background`: None, or "white" / "black" to
    composite an RGBA image over it first (an RGB image is composited as opaque).  An RGBA image without a composite
    is resized through premultiplied RGBa, or copied when the size does not change; its alpha is dropped."""
    if background not in (None, "white", "black"):
        raise ValueError(f"background must be None, 'white' or 'black', got {background!r}")
    dev = torch.device(device)
    if dev.type != "cuda":
        raise ValueError(f"prepare_image runs on a CUDA device, got {dev}")
    img = torch.as_tensor(image)
    if img.dim() != 3 or img.shape[2] not in (3, 4):
        raise ValueError(f"image must be uint8 [H,W,3|4], got {tuple(img.shape)}")
    img = tensor(img.to(dev, non_blocking=False), "image", torch.uint8, ("H", "W", img.shape[2]))
    H, W, C = img.shape
    width, height = int(width), int(height)
    if width < 1 or height < 1:
        raise ValueError(f"output size must be >= 1, got {width}x{height}")
    if background is not None and C == 3:       # image.convert("RGBA") of an RGB image: alpha 255
        img = torch.cat([img, torch.full((H, W, 1), 255, dtype=torch.uint8, device=dev)], 2)
        C = 4
    resized = (width, height) != (W, H)
    mode = SGR_IMAGE_COMPOSITE if background is not None else \
        SGR_IMAGE_PREMULTIPLY if C == 4 and resized else SGR_IMAGE_PLAIN
    xb = xc = yb = yc = None
    kx = ky = 0
    if width != W:
        xb, xc, kx = _tables(W, width, dev)
    if height != H:
        yb, yc, ky = _tables(H, height, dev)
    tmp = torch.empty((H, width, 4), dtype=torch.uint8, device=dev) if width != W and height != H else None
    out = torch.empty((3, height, width), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        check(lib.sgr_image_prepare(H, W, C, mode, int(background == "white"), width, kx, ptr(xb), ptr(xc), height,
                                    ky, ptr(yb), ptr(yc), img.data_ptr(), ptr(tmp), out.data_ptr(), stream(dev)))
    return out


def read_image(path):
    """-> uint8 [H,W,3|4] of a PNG (objfile.read_png) or a JPEG (Pillow, imported here only)."""
    ext = os.path.splitext(path)[1].lower()
    if ext == ".png":
        return objfile.read_png(path, keep_alpha=True)
    if ext in (".jpg", ".jpeg"):
        try:
            from PIL import Image
        except ImportError as e:
            raise ImportError(f"{path}: reading JPEG images needs the 'PIL' module (Pillow); PNG scenes need only "
                              "torch and numpy") from e
        with Image.open(path) as im:
            if im.mode not in ("RGB", "RGBA"):
                raise ValueError(f"{path}: JPEG of mode {im.mode}, only RGB is read")
            return np.asarray(im).copy()
    raise ValueError(f"{path}: unsupported image type {ext!r} (PNG or JPEG)")


# ------------------------------------------------------------------------------------------------- resolution rules
def gs_resolution(orig_w: int, orig_h: int, resolution: int = -1):
    """loadCam's size rule (gaussian_splatting/utils/camera_utils.py:20-40) at resolution scale 1.0: r in {1, 2, 4, 8}
    gives (round(w / r), round(h / r)) (half to even); -1 brings an image wider than 1600 px to 1600 wide with
    int(w / scale); any other value is a target width."""
    if resolution in (1, 2, 4, 8):
        return round(orig_w / (1.0 * resolution)), round(orig_h / (1.0 * resolution))
    if resolution == -1:
        global_down = orig_w / 1600 if orig_w > 1600 else 1
    else:
        global_down = orig_w / resolution
    scale = float(global_down) * 1.0
    return int(orig_w / scale), int(orig_h / scale)


def sugar_resolution(orig_w: int, orig_h: int, image_resolution: int = 1, max_img_size: int = 1920):
    """load_gs_cameras' size rule (sugar_scene/cameras.py:109-117): the factor r in {1, 2, 4, 8} (else 1), times
    max(w, h) / max_img_size when the ORIGINAL long side exceeds max_img_size, then round() of each side."""
    factor = image_resolution if image_resolution in (1, 2, 4, 8) else 1
    if max(orig_h, orig_w) > max_img_size:
        factor = (max(orig_h, orig_w) / max_img_size) * factor
    return round(orig_w / factor), round(orig_h / factor)


# ------------------------------------------------------------------------------------------------------- cameras
def focal2fov(focal, pixels):
    return 2 * math.atan(pixels / (2 * focal))


def fov2focal(fov, pixels):
    return pixels / (2 * math.tan(fov / 2))


def qvec2rotmat(q):
    return np.array([
        [1 - 2 * q[2] ** 2 - 2 * q[3] ** 2, 2 * q[1] * q[2] - 2 * q[0] * q[3], 2 * q[3] * q[1] + 2 * q[0] * q[2]],
        [2 * q[1] * q[2] + 2 * q[0] * q[3], 1 - 2 * q[1] ** 2 - 2 * q[3] ** 2, 2 * q[2] * q[3] - 2 * q[0] * q[1]],
        [2 * q[3] * q[1] - 2 * q[0] * q[2], 2 * q[2] * q[3] + 2 * q[0] * q[1], 1 - 2 * q[1] ** 2 - 2 * q[2] ** 2]])


def world_to_view(R, T):
    """getWorld2View2(R, T) with no translate or scale: float32 [4,4] world -> camera."""
    Rt = np.zeros((4, 4))
    Rt[:3, :3] = np.asarray(R).transpose()
    Rt[:3, 3] = T
    Rt[3, 3] = 1.0
    return np.float32(np.linalg.inv(np.linalg.inv(Rt)))   # through C2W, as getWorld2View2 goes


def camera_center(R, T):
    """The camera centre as getNerfppNorm takes it: inv(getWorld2View2(R, T))[:3, 3] (float32)."""
    return np.linalg.inv(world_to_view(R, T))[:3, 3]


def make_camera(R, T, FoVx, FoVy, width, height, device="cuda", **meta):
    """The steps' camera namespace for the posed pinhole (R, T, FoVx, FoVy) at width x height, as Camera / GSCamera
    build it, with `meta` (name, uid, ...) and R, T, FoVx, FoVy attached."""
    dev = torch.device(device)
    viewmatrix = torch.tensor(world_to_view(R, T)).transpose(0, 1).to(dev)
    proj = torch.from_numpy(scenes.projection_matrix(ZNEAR, ZFAR, math.tan(FoVx / 2), math.tan(FoVy / 2))
                            .astype(np.float32)).transpose(0, 1).to(dev)
    projmatrix = viewmatrix.unsqueeze(0).bmm(proj.unsqueeze(0)).squeeze(0)
    campos = viewmatrix.inverse()[3, :3]
    return SimpleNamespace(viewmatrix=viewmatrix.contiguous(), projmatrix=projmatrix.contiguous(),
                           campos=campos.contiguous(), width=int(width), height=int(height),
                           tanfovx=math.tan(FoVx * 0.5), tanfovy=math.tan(FoVy * 0.5), R=np.asarray(R),
                           T=np.asarray(T), FoVx=FoVx, FoVy=FoVy, **meta)


# ------------------------------------------------------------------------------------------------------- COLMAP
CAMERA_MODELS = {0: ("SIMPLE_PINHOLE", 3), 1: ("PINHOLE", 4), 2: ("SIMPLE_RADIAL", 4), 3: ("RADIAL", 5),
                 4: ("OPENCV", 8), 5: ("OPENCV_FISHEYE", 8), 6: ("FULL_OPENCV", 12), 7: ("FOV", 5),
                 8: ("SIMPLE_RADIAL_FISHEYE", 4), 9: ("RADIAL_FISHEYE", 5), 10: ("THIN_PRISM_FISHEYE", 12)}
SUPPORTED_MODELS = ("SIMPLE_PINHOLE", "PINHOLE")


def _read(f, fmt):
    n = struct.calcsize("<" + fmt)
    data = f.read(n)
    if len(data) != n:
        raise ValueError(f"{f.name}: truncated COLMAP file")
    return struct.unpack("<" + fmt, data)


def _data_lines(path):
    with open(path) as f:
        lines = [ln.strip() for ln in f]
    return [ln for ln in lines if ln and ln[0] != "#"]


def _read_cameras(sparse_dir):
    cams = {}
    p = os.path.join(sparse_dir, "cameras.bin")
    if os.path.exists(p):
        with open(p, "rb") as f:
            for _ in range(_read(f, "Q")[0]):
                cid, model_id, w, h = _read(f, "iiQQ")
                if model_id not in CAMERA_MODELS:
                    raise ValueError(f"{p}: unknown COLMAP camera model id {model_id}")
                name, n = CAMERA_MODELS[model_id]
                cams[cid] = SimpleNamespace(id=cid, model=name, width=w, height=h, params=np.array(_read(f, "d" * n)))
        return cams
    p = os.path.join(sparse_dir, "cameras.txt")
    for ln in _data_lines(p):
        e = ln.split()
        cams[int(e[0])] = SimpleNamespace(id=int(e[0]), model=e[1], width=int(e[2]), height=int(e[3]),
                                          params=np.array(tuple(map(float, e[4:]))))
    return cams


def _read_images(sparse_dir):
    imgs = {}
    p = os.path.join(sparse_dir, "images.bin")
    if os.path.exists(p):
        with open(p, "rb") as f:
            for _ in range(_read(f, "Q")[0]):
                props = _read(f, "idddddddi")
                name = b""
                while True:
                    c = f.read(1)
                    if c in (b"", b"\x00"):
                        break
                    name += c
                n2d = _read(f, "Q")[0]
                f.seek(24 * n2d, os.SEEK_CUR)
                imgs[props[0]] = SimpleNamespace(id=props[0], qvec=np.array(props[1:5]), tvec=np.array(props[5:8]),
                                                 camera_id=props[8], name=name.decode("utf-8"))
        return imgs
    p = os.path.join(sparse_dir, "images.txt")
    with open(p) as f:
        while True:
            ln = f.readline()
            if not ln:
                break
            ln = ln.strip()
            if ln and ln[0] != "#":
                e = ln.split()
                imgs[int(e[0])] = SimpleNamespace(id=int(e[0]), qvec=np.array(tuple(map(float, e[1:5]))),
                                                  tvec=np.array(tuple(map(float, e[5:8]))), camera_id=int(e[8]),
                                                  name=e[9])
                f.readline()   # the image's 2D points
    return imgs


def _read_points(sparse_dir):
    p = os.path.join(sparse_dir, "points3D.bin")
    if os.path.exists(p):
        with open(p, "rb") as f:
            n = _read(f, "Q")[0]
            xyz, rgb = np.empty((n, 3)), np.empty((n, 3))
            for i in range(n):
                props = _read(f, "QdddBBBd")
                xyz[i], rgb[i] = props[1:4], props[4:7]
                f.seek(8 * _read(f, "Q")[0], os.SEEK_CUR)
        return xyz, rgb
    p = os.path.join(sparse_dir, "points3D.txt")
    if not os.path.exists(p):
        return None
    lines = _data_lines(p)
    xyz, rgb = np.empty((len(lines), 3)), np.empty((len(lines), 3))
    for i, ln in enumerate(lines):
        e = ln.split()
        xyz[i] = tuple(map(float, e[1:4]))
        rgb[i] = tuple(map(int, e[4:7]))
    return xyz, rgb


def read_colmap_model(sparse_dir):
    """COLMAP's cameras, images and points3D from `sparse_dir`, each in .bin or else .txt (colmap_loader.py) ->
    namespace(cameras {id: (id, model, width, height, params)}, images {id: (id, qvec, tvec, camera_id, name)},
    points (xyz float64 [N,3], rgb float64 [N,3]) or None).  Raises ValueError for a camera model other than PINHOLE
    or SIMPLE_PINHOLE, as the reference's assert does."""
    cams = _read_cameras(sparse_dir)
    for c in cams.values():
        if c.model not in SUPPORTED_MODELS:
            raise ValueError(f"{sparse_dir}: camera {c.id} is {c.model}: only undistorted datasets (PINHOLE or "
                             "SIMPLE_PINHOLE cameras) are supported")
    return SimpleNamespace(cameras=cams, images=_read_images(sparse_dir), points=_read_points(sparse_dir))


def stored_points(xyz, rgb):
    """storePly -> fetchPly of (xyz, rgb 0..255): (float32 xyz, uint8 rgb / 255 as float64)."""
    return np.asarray(xyz).astype(np.float32), np.asarray(rgb).astype(np.uint8) / 255.0


def _info(colmap_id, R, T, FoVx, FoVy, image_path, name, width, height, background):
    """CameraInfo: the camera and its image before loading, under the names the cams carry."""
    return SimpleNamespace(colmap_id=colmap_id, R=R, T=T, FoVx=FoVx, FoVy=FoVy, image_path=image_path, name=name,
                           orig_width=width, orig_height=height, background=background)


def _ply_points(ply_path):
    from .gsply import read_sfm_points
    return read_sfm_points(ply_path)


def _scene_info(train, test, points, colors):
    return SimpleNamespace(train=train, test=test, camera_list=test + train, points=points, colors=colors,
                           nerf_radius=mcubes.nerfpp_radius(np.stack([camera_center(c.R, c.T) for c in train])))


def read_colmap_scene_info(source_path, images="images", eval=False, llffhold=8):
    """readColmapSceneInfo (dataset_readers.py:68-177) without the images -> namespace(train, test: CameraInfo
    namespaces (colmap_id = the COLMAP camera id, R, T, FoVx, FoVy, image_path, name, orig_width / orig_height = the
    COLMAP camera's size); camera_list: test + train, cameras.json's order; points float32 [N,3], colors float64
    [N,3] (gsply.read_sfm_points' arrays); nerf_radius: getNerfppNorm's radius of the train cameras).  Sorted by
    image name; with `eval` every `llffhold`-th camera is a test camera."""
    sparse = os.path.join(source_path, "sparse", "0")
    model = read_colmap_model(sparse)
    infos = []
    for extr in model.images.values():
        intr = model.cameras[extr.camera_id]
        fx = intr.params[0]
        fy = fx if intr.model == "SIMPLE_PINHOLE" else intr.params[1]
        image_path = os.path.join(source_path, images or "images", os.path.basename(extr.name))
        infos.append(_info(intr.id, np.transpose(qvec2rotmat(extr.qvec)), np.array(extr.tvec),
                           focal2fov(fx, intr.width), focal2fov(fy, intr.height), image_path,
                           os.path.basename(image_path).split(".")[0], intr.width, intr.height, None))
    infos.sort(key=lambda c: c.name)
    ply = os.path.join(sparse, "points3D.ply")
    if os.path.exists(ply):
        points, colors = _ply_points(ply)
    elif model.points is not None:
        points, colors = stored_points(*model.points)
    else:
        raise FileNotFoundError(f"{sparse}: no points3D.ply, points3D.bin or points3D.txt")
    return _scene_info([c for i, c in enumerate(infos) if not eval or i % llffhold != 0],
                       [c for i, c in enumerate(infos) if eval and i % llffhold == 0], points, colors)


def _transforms_infos(path, transforms, white_background, extension):
    with open(os.path.join(path, transforms)) as f:
        contents = json.load(f)
    fovx = contents["camera_angle_x"]
    infos = []
    for idx, frame in enumerate(contents["frames"]):
        image_path = os.path.join(path, frame["file_path"] + extension)
        c2w = np.array(frame["transform_matrix"])
        c2w[:3, 1:3] *= -1                       # OpenGL / Blender axes (Y up, Z back) to COLMAP's (Y down, Z forward)
        w2c = np.linalg.inv(c2w)
        image = read_image(image_path)           # FoVy and CameraInfo's size need the image size
        h, w = image.shape[:2]
        info = _info(idx, np.transpose(w2c[:3, :3]), w2c[:3, 3], fovx, focal2fov(fov2focal(fovx, w), h), image_path,
                     os.path.splitext(os.path.basename(image_path))[0], w, h, "white" if white_background else "black")
        info.image = image
        infos.append(info)
    return infos


def random_points(rng, num_pts=100_000):
    """readNerfSyntheticInfo's random cloud from `rng` (a numpy RandomState), as storePly -> fetchPly rounds it."""
    xyz = rng.random_sample((num_pts, 3)) * 2.6 - 1.3
    shs = rng.random_sample((num_pts, 3)) / 255.0
    return stored_points(xyz, (shs * 0.28209479177387814 + 0.5) * 255)


def read_nerf_synthetic_info(path, white_background=False, eval=False, extension=".png", points_rng=None):
    """readNerfSyntheticInfo (dataset_readers.py:179-259) -> the namespace of read_colmap_scene_info (colmap_id = the
    frame index; each info also holds its decoded `image`).  The OpenGL camera axes are flipped to COLMAP's; FoVy
    comes from FoVx and the image size; without `eval` the test views join the train views.  The points are
    `points3d.ply` when it exists, else readNerfSyntheticInfo's 100k random points drawn from `points_rng` (a numpy
    RandomState; required then)."""
    train = _transforms_infos(path, "transforms_train.json", white_background, extension)
    test = _transforms_infos(path, "transforms_test.json", white_background, extension)
    if not eval:
        train, test = train + test, []
    ply = os.path.join(path, "points3d.ply")
    if os.path.exists(ply):
        points, colors = _ply_points(ply)
    elif points_rng is None:
        raise ValueError(f"{path} has no points3d.ply: pass points_rng (a numpy RandomState) for the random cloud")
    else:
        points, colors = random_points(points_rng)
    return _scene_info(train, test, points, colors)


def load_views(infos, resolution=-1, device="cuda"):
    """loadCam of each CameraInfo (camera_utils.py:20-56) at resolution scale 1.0 -> [(cam, gt)], uid = the index:
    the image decoded, composited over the info's background (NeRF-synthetic), resized to gs_resolution's size and
    divided by 255 on the GPU."""
    views = []
    for i, info in enumerate(infos):
        img = getattr(info, "image", None)
        img = read_image(info.image_path) if img is None else img
        w, h = gs_resolution(img.shape[1], img.shape[0], resolution)
        gt = prepare_image(img, w, h, background=info.background, device=device)
        cam = make_camera(info.R, info.T, info.FoVx, info.FoVy, w, h, device=device, name=info.name, uid=i,
                          colmap_id=info.colmap_id, orig_width=info.orig_width, orig_height=info.orig_height)
        views.append((cam, gt))
    return views


def _load_scene(info, resolution, device, shuffle_rng):
    train, test = list(info.train), list(info.test)
    if shuffle_rng is not None:       # Scene.__init__ shuffles the infos before loadCam numbers them (uid)
        shuffle_rng.shuffle(train)
        shuffle_rng.shuffle(test)
    train, test = load_views(train, resolution, device), load_views(test, resolution, device)
    return SimpleNamespace(train=train, test=test, camera_list=info.camera_list, points=info.points,
                           colors=info.colors, nerf_radius=info.nerf_radius)


def load_colmap_scene(source_path, images="images", eval=False, llffhold=8, resolution=-1, device="cuda",
                      shuffle_rng=None):
    """3DGS's Scene over a COLMAP dataset (read_colmap_scene_info + load_views) -> namespace(train, test: lists of
    (cam, gt); camera_list, points, colors, nerf_radius as read_colmap_scene_info gives them).  `shuffle_rng`: a
    random.Random that shuffles train and then test, as Scene.__init__ does (after safe_state's random.seed(0))."""
    return _load_scene(read_colmap_scene_info(source_path, images, eval, llffhold), resolution, device, shuffle_rng)


def load_nerf_synthetic_scene(path, white_background=False, eval=False, extension=".png", resolution=-1,
                              device="cuda", points_rng=None, shuffle_rng=None):
    """3DGS's Scene over a NeRF-synthetic (Blender) dataset (read_nerf_synthetic_info + load_views) -> the namespace
    of load_colmap_scene.  Every image is composited over white or black in float64 before any resize."""
    info = read_nerf_synthetic_info(path, white_background, eval, extension, points_rng)
    return _load_scene(info, resolution, device, shuffle_rng)


# ------------------------------------------------------------------------------------------------- cameras.json
def camera_to_json(id, cam):
    """camera_to_JSON (camera_utils.py:62-82) of a CameraInfo or a view's cam: its original width and height."""
    Rt = np.zeros((4, 4))
    Rt[:3, :3] = cam.R.transpose()
    Rt[:3, 3] = cam.T
    Rt[3, 3] = 1.0
    W2C = np.linalg.inv(Rt)
    return {"id": id, "img_name": cam.name, "width": cam.orig_width, "height": cam.orig_height,
            "position": W2C[:3, 3].tolist(), "rotation": [x.tolist() for x in W2C[:3, :3]],
            "fy": fov2focal(cam.FoVy, cam.orig_height), "fx": fov2focal(cam.FoVx, cam.orig_width)}


def write_cameras_json(path, cams):
    """Scene.__init__'s cameras.json: camera_to_JSON of each CameraInfo or cam, id = its index.  Pass a scene's
    `camera_list` (test then train, in reader order, before any shuffle) to write the reference's file."""
    with open(path, "w") as f:
        json.dump([camera_to_json(i, c) for i, c in enumerate(cams)], f)


def _find_image(image_dir, name):
    found = [os.path.join(image_dir, name + e) for e in IMAGE_EXTENSIONS
             if os.path.isfile(os.path.join(image_dir, name + e))]
    if len(found) != 1:
        raise FileNotFoundError(f"{image_dir}: {'no' if not found else 'more than one'} image {name}"
                                f"{{{','.join(IMAGE_EXTENSIONS)}}}" + (f": {found}" if found else ""))
    return found[0]


def gs_camera_entries(entries, remove_indices=()):
    """load_gs_cameras' choice of cameras.json entries (sugar_scene/cameras.py:36-62): the entries at
    `remove_indices` dropped, the last entry of each repeated img_name kept, sorted by img_name."""
    remove = set(remove_indices)
    by_name = {}
    for i, e in enumerate(entries):
        if i not in remove:
            by_name[e["img_name"]] = e
    return sorted(by_name.values(), key=lambda e: e["img_name"])


def load_gs_cameras(source_path, gs_output_path, image_resolution=1, max_img_size=1920, white_background=False,
                    remove_indices=(), eval_split=False, eval_split_interval=8, device="cuda"):
    """SuGaR's load_gs_cameras (sugar_scene/cameras.py:15-139) with GaussianSplattingWrapper's split
    (gs_model.py:125-146) -> (train views, test views).  Reads `<gs_output_path>/cameras.json`; drops the entries at
    `remove_indices`; keeps the last entry of a repeated img_name; sorts by name (gs_camera_entries); loads
    `<source_path>/images/<img_name>.<ext>` (see the module docstring), composited over white with
    `white_background`, at sugar_resolution's size.  With `eval_split` every `eval_split_interval`-th view (i %
    interval == 0) is a test view; otherwise the test list is empty."""
    with open(os.path.join(gs_output_path, "cameras.json")) as f:
        entries = gs_camera_entries(json.load(f), remove_indices)
    image_dir = os.path.join(source_path, "images")
    views = []
    for e in entries:
        W2C = np.zeros((4, 4))
        W2C[:3, :3] = np.array(e["rotation"])
        W2C[:3, 3] = np.array(e["position"])
        W2C[3, 3] = 1
        Rt = np.linalg.inv(W2C)
        T = Rt[:3, 3]
        R = Rt[:3, :3].transpose()
        fov_y, fov_x = focal2fov(e["fy"], e["height"]), focal2fov(e["fx"], e["width"])
        img = read_image(_find_image(image_dir, e["img_name"]))
        orig_h, orig_w = img.shape[:2]
        w, h = sugar_resolution(orig_w, orig_h, image_resolution, max_img_size)
        gt = prepare_image(img, w, h, background="white" if white_background else None, device=device)
        cam = make_camera(R, T, fov_x, fov_y, w, h, device=device, name=e["img_name"], uid=e["id"],
                          colmap_id=e["id"], orig_width=e["width"], orig_height=e["height"])
        views.append((cam, gt))
    if not eval_split:
        return views, []
    return ([v for i, v in enumerate(views) if i % eval_split_interval != 0],
            [v for i, v in enumerate(views) if i % eval_split_interval == 0])
