"""Golden values of the reference's dataset loading, from Pillow and the reference's OWN reader lines.

Runs in the build container (needs /root/reference and Pillow):  python tests/golden/make_dataset_golden.py

dataset_pil.npz: Pillow's Image.resize (default filter) of seeded images and the reference's float64 composite, case
by case (`<case>_in` uint8 [H,W,C], `<case>_out` uint8 [h,w,3] = the bytes PILtoTorch divides by 255), and the
Pillow version that made them.  The composite line `Image.fromarray(np.array(arr*255.0, dtype=np.byte), "RGB")`
relies on Pillow 10 reinterpreting int8 as RGB bytes; Pillow 12 refuses int8 arrays, so the same bytes are taken by
viewing the int8 array as uint8.

dataset_readers.npz: tests/dataset_cases.py's seeded datasets loaded by the reference's modules, imported from the
checkout unchanged: gaussian_splatting/scene/colmap_loader.py, dataset_readers.py (readColmapSceneInfo,
readNerfSyntheticInfo), utils/camera_utils.py (loadCam, camera_to_JSON) and sugar_scene/cameras.py (load_gs_cameras).
Their heavy imports are stood in for: plyfile by an in-memory store (storePly -> fetchPly round trips through the
same structured dtype; nothing is written into the dataset), gaussian_model by BasicPointCloud, pytorch3d by empty
modules, and Camera / GSCamera by recorders of their arguments.  Per case `<case>_*`: each view's name, colmap id,
R, T, FoVx, FoVy, CameraInfo width and height, and its prepared bytes (uint8 of round(255 image)), the point cloud,
the nerf radius, and the cameras.json text.  Of the 100k-point random cloud only the first 100 rows and a sha256 of
all of it are kept.
"""
import hashlib
import json
import os
import shutil
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
REF = "/root/reference"

import dataset_cases as dc  # noqa: E402


# ----------------------------------------------------------------------------------------------------- Pillow cases
def pil_cases():
    from PIL import Image
    rng = np.random.Generator(np.random.PCG64(7))
    u8 = lambda *s: rng.integers(0, 256, s, dtype=np.uint8)  # noqa: E731

    def rgba(h, w):
        px = u8(h, w, 4)
        px[..., 3] = np.where(rng.random((h, w)) < 0.3, rng.choice(np.array([0, 255], np.uint8), (h, w)), px[..., 3])
        return px

    resize = {   # name: (image, (w, h))
        "down_nonint": (u8(37, 53, 3), (20, 14)),
        "down_x2": (u8(32, 48, 3), (24, 16)),
        "down_x4": (u8(32, 48, 3), (12, 8)),
        "down_x8": (u8(64, 96, 3), (12, 8)),
        "width_only": (u8(21, 50, 3), (17, 21)),
        "height_only": (u8(50, 21, 3), (21, 13)),
        "up": (u8(9, 13, 3), (31, 22)),
        "same": (u8(11, 7, 3), (7, 11)),
        "one_px_wide": (u8(40, 1, 3), (1, 15)),
        "to_one_px": (u8(16, 30, 3), (1, 5)),
        "rgba_premul": (rgba(36, 60), (24, 15)),
        "rgba_premul_width": (rgba(20, 33), (12, 20)),
        "rgba_same": (rgba(9, 8), (8, 9)),
        "big_down": (u8(131, 217, 3), (67, 41)),
    }
    out = {"pillow_version": np.array(Image.__version__)}
    for name, (img, size) in resize.items():
        mode = "RGB" if img.shape[2] == 3 else "RGBA"
        out[f"{name}_in"] = img
        out[f"{name}_out"] = np.ascontiguousarray(np.array(Image.fromarray(img, mode).resize(size))[..., :3])
    for bg in ("white", "black"):
        for name, (img, size) in (("composite", (rgba(23, 29), (29, 23))),
                                  ("composite_down", (rgba(40, 44), (21, 20)))):
            norm_data = img / 255.0
            b = np.array([1, 1, 1]) if bg == "white" else np.array([0, 0, 0])
            arr = norm_data[:, :, :3] * norm_data[:, :, 3:4] + b * (1 - norm_data[:, :, 3:4])
            comp = Image.fromarray(np.array(arr * 255.0, dtype=np.byte).view(np.uint8), "RGB")
            out[f"{name}_{bg}_in"] = img
            out[f"{name}_{bg}_out"] = np.ascontiguousarray(np.array(comp.resize(size)))
    return out


# ------------------------------------------------------------------------------------------- the reference's readers
_PLY = {}


def _stand_ins():
    """Modules the readers import but this container lacks or must not run."""
    def package(name, path):
        m = types.ModuleType(name)
        m.__path__ = [path]
        sys.modules[name] = m

    package("scene", os.path.join(REF, "gaussian_splatting", "scene"))   # without scene/__init__.py's model imports
    package("utils", os.path.join(REF, "gaussian_splatting", "utils"))
    from typing import NamedTuple

    class BasicPointCloud(NamedTuple):
        points: np.ndarray
        colors: np.ndarray
        normals: np.ndarray
    gm = types.ModuleType("scene.gaussian_model")
    gm.BasicPointCloud = BasicPointCloud
    sys.modules["scene.gaussian_model"] = gm

    class PlyElement:
        @staticmethod
        def describe(elements, name):
            return elements

    class PlyData:
        def __init__(self, elements):
            self.elements = elements

        def write(self, path):
            _PLY[path] = self.elements[0].copy()

        @staticmethod
        def read(path):
            return {"vertex": _PLY[path]}
    ply = types.ModuleType("plyfile")
    ply.PlyData, ply.PlyElement = PlyData, PlyElement
    sys.modules["plyfile"] = ply
    for name in ("pytorch3d", "pytorch3d.renderer", "pytorch3d.renderer.cameras"):
        sys.modules[name] = types.ModuleType(name)
    sys.modules["pytorch3d.renderer"].FoVPerspectiveCameras = None
    sys.modules["pytorch3d.renderer.cameras"]._get_sfm_calibration_matrix = None
    # os.path.exists of the .ply the readers would write: only what storePly put in the store
    import scene.dataset_readers as dr
    real_exists = os.path.exists
    dr.os = types.SimpleNamespace(path=types.SimpleNamespace(
        join=os.path.join, basename=os.path.basename, exists=lambda p: p in _PLY or (real_exists(p) and not
                                                                                     p.endswith(".ply"))))


def _record(**kw):
    return types.SimpleNamespace(**kw)


def _views(prefix, cams, out):
    out[f"{prefix}_names"] = np.array([c.image_name for c in cams])
    out[f"{prefix}_colmap_id"] = np.array([c.colmap_id for c in cams], np.int64)
    out[f"{prefix}_R"] = np.stack([c.R for c in cams])
    out[f"{prefix}_T"] = np.stack([c.T for c in cams])
    out[f"{prefix}_fov"] = np.array([[c.FoVx, c.FoVy] for c in cams], np.float64)
    for i, c in enumerate(cams):
        img = c.image.numpy()
        u8 = np.round(img * 255.0).astype(np.uint8)
        assert np.array_equal(u8.astype(np.float32) / np.float32(255.0), img)
        out[f"{prefix}_img{i}"] = np.ascontiguousarray(u8.transpose(1, 2, 0))


def reader_cases(tmp):
    sys.path.insert(0, os.path.join(REF, "gaussian_splatting"))
    _stand_ins()
    import scene.dataset_readers as dr
    import utils.camera_utils as cu
    from PIL import Image
    cu.Camera = _record
    real_fromarray = Image.fromarray
    Image.fromarray = lambda a, mode=None: real_fromarray(a.view(np.uint8) if a.dtype == np.int8 else a, mode)
    out = {}

    def scene_case(name, info, resolution):
        args = types.SimpleNamespace(resolution=resolution, data_device="cpu")
        camlist = list(info.test_cameras) + list(info.train_cameras)
        out[f"{name}_json"] = np.array(json.dumps([cu.camera_to_JSON(i, c) for i, c in enumerate(camlist)]))
        out[f"{name}_info_size"] = np.array([[c.width, c.height] for c in camlist], np.int64)
        out[f"{name}_n_test"] = np.array(len(info.test_cameras))
        cams = [cu.loadCam(args, i, c, 1.0) for i, c in enumerate(camlist)]
        _views(name, cams, out)
        pts, cols = info.point_cloud.points, info.point_cloud.colors
        if len(pts) > 1000:   # the random cloud: its first rows and the digest of all of it
            out[f"{name}_digest"] = np.array(hashlib.sha256(pts.tobytes() + cols.tobytes()).hexdigest())
            pts, cols = pts[:100], cols[:100]
        out[f"{name}_points"] = pts
        out[f"{name}_colors"] = cols
        out[f"{name}_radius"] = np.array(info.nerf_normalization["radius"], np.float64)

    colmap_bin = dc.colmap_case(os.path.join(tmp, "colmap_bin"), binary=True)
    scene_case("colmap_bin", dr.readColmapSceneInfo(colmap_bin, "images", True), 2)
    colmap_txt = dc.colmap_case(os.path.join(tmp, "colmap_txt"), binary=False, simple=False, seed=1)
    scene_case("colmap_txt", dr.readColmapSceneInfo(colmap_txt, "images", False), -1)
    nerf = dc.nerf_case(os.path.join(tmp, "nerf"))
    for white in (True, False):
        np.random.seed(3)
        scene_case(f"nerf_{'white' if white else 'black'}", dr.readNerfSyntheticInfo(nerf, white, True), 2)

    # SuGaR's load_gs_cameras on the binary case's cameras.json, with a removed entry and a repeated name
    sys.path.insert(0, REF)
    import sugar_scene.cameras as sc
    sc.GSCamera = _record
    entries = json.loads(str(out["colmap_bin_json"]))
    dup = dict(entries[4], id=99, position=[p + 0.25 for p in entries[4]["position"]])
    entries.append(dup)
    gs_json = json.dumps(entries)
    out["gs_cameras_json"] = np.array(gs_json)
    gs_out = os.path.join(tmp, "gs_out") + os.sep
    os.makedirs(gs_out)
    with open(gs_out + "cameras.json", "w") as f:
        f.write(gs_json)
    for name, kw in (("gs_plain", dict(image_resolution=2, max_img_size=20, remove_indices=[1])),
                     ("gs_white", dict(image_resolution=1, white_background=True))):
        cams = sc.load_gs_cameras(colmap_bin, gs_out, **kw)
        out[f"{name}_uid"] = np.array([c.uid for c in cams], np.int64)
        _views(name, cams, out)
    Image.fromarray = real_fromarray
    return out


def main():
    pil = pil_cases()
    path = os.path.join(HERE, "dataset_pil.npz")
    np.savez_compressed(path, **pil)
    print(path, len(pil))
    tmp = tempfile.mkdtemp()
    try:
        readers = reader_cases(tmp)
    finally:
        shutil.rmtree(tmp)
    readers["pillow_version"] = pil["pillow_version"]
    path = os.path.join(HERE, "dataset_readers.npz")
    np.savez_compressed(path, **readers)
    print(path, len(readers))


if __name__ == "__main__":
    main()
