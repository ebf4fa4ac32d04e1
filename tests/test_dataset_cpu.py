"""CPU checks of the dataset path: the image-preparation oracle against Pillow and its goldens, the package's resample
tables, the premultiply / composite rules on every input, the readers and cameras.json against the reference's own
reader lines (tests/golden/make_dataset_golden.py), and the size rules at their rounding boundaries."""
import json
import os
from types import SimpleNamespace

import numpy as np
import pytest

import dataset_cases as dc
from oracle import imageprep_oracle as o
from sugar_b200 import dataset

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _golden(name):
    return np.load(os.path.join(GOLDEN, name))


def _pil():
    return pytest.importorskip("PIL.Image")


def _all_pairs():
    v, a = np.meshgrid(np.arange(256), np.arange(256))
    return np.stack([v, v, v, a], -1).astype(np.uint8)     # [256 alphas, 256 values, 4]


# ---------------------------------------------------------------------------------------------------- image rules
def test_oracle_matches_pil_on_random_sizes():
    Image = _pil()
    rng = np.random.Generator(np.random.PCG64(11))
    for t in range(200):
        H, W = (int(x) for x in rng.integers(1, 70, 2))
        h = H if t % 5 == 0 else int(rng.integers(1, 70))
        w = W if t % 7 == 0 else int(rng.integers(1, 70))
        C = 4 if t % 2 else 3
        img = rng.integers(0, 256, (H, W, C), dtype=np.uint8)
        ref = np.array(Image.fromarray(img, "RGBA" if C == 4 else "RGB").resize((w, h)))[..., :3]
        assert np.array_equal(o.prepare_bytes(img, w, h), ref), (H, W, C, h, w)


def test_oracle_matches_goldens():
    g = _golden("dataset_pil.npz")
    cases = sorted(k[:-3] for k in g.files if k.endswith("_in"))
    assert len(cases) == 18
    for name in cases:
        img, ref = g[name + "_in"], g[name + "_out"]
        bg = "white" if name.endswith("_white") else "black" if name.endswith("_black") else None
        got = o.prepare_bytes(img, ref.shape[1], ref.shape[0], background=bg)
        assert np.array_equal(got, ref), name
    assert str(g["pillow_version"]).split(".")[0] in ("10", "11", "12")


@pytest.mark.parametrize("sizes", [(5187, 1600), (3361, 1037), (4946, 1600), (3286, 1063), (1, 7), (7, 1), (9, 31),
                                   (31, 9), (800, 800), (1000, 999), (1920, 1919), (3, 2)])
def test_package_tables_equal_oracle_tables(sizes):
    b0, c0, k0 = o.resample_coeffs(*sizes)
    b1, c1, k1 = dataset.resample_coeffs(*sizes)
    assert k0 == k1 and np.array_equal(b0, b1) and np.array_equal(c0, c1)
    assert b1.dtype == np.int32 and c1.dtype == np.int32
    assert (b1[:, 0] >= 0).all() and (b1[:, 0] + b1[:, 1] <= sizes[0]).all() and (b1[:, 1] >= 1).all()


def test_premultiply_and_unpremultiply_on_every_pair():
    Image = _pil()
    px = _all_pairs()
    assert np.array_equal(o.premultiply(px), np.array(Image.fromarray(px, "RGBA").convert("RGBa")))
    assert np.array_equal(o.unpremultiply(px), np.array(Image.fromarray(px, "RGBa").convert("RGBA")))


@pytest.mark.parametrize("white", [True, False])
def test_composite_on_every_triple(white):
    px = _all_pairs()
    norm_data = px / 255.0
    bg = np.array([1, 1, 1]) if white else np.array([0, 0, 0])
    arr = norm_data[:, :, :3] * norm_data[:, :, 3:4] + bg * (1 - norm_data[:, :, 3:4])
    with np.errstate(invalid="ignore"):
        ref = np.array(arr * 255.0, dtype=np.byte).view(np.uint8)   # the bytes Pillow 10 reads from the int8 array
    got = o.composite(px, white)
    assert np.array_equal(got, ref)
    assert np.array_equal(got[255, :, 0], np.arange(256))            # opaque pixels keep their value
    rounded = np.round(arr[128, :, 0] * 255.0)
    assert (got[128, :, 0] != rounded).sum() > 100                   # truncation, not rounding, at alpha 128


# ------------------------------------------------------------------------------------------------------ size rules
@pytest.mark.parametrize("w,h,r,want", [
    (45, 31, 2, (22, 16)),            # 22.5 -> 22, 15.5 -> 16: half to even
    (47, 33, 2, (24, 16)),            # 23.5 -> 24, 16.5 -> 16
    (10, 6, 4, (2, 2)),               # 2.5 -> 2, 1.5 -> 2
    (100, 60, 8, (12, 8)),            # 12.5 -> 12, 7.5 -> 8
    (1600, 1063, -1, (1600, 1063)),   # exactly 1600 wide: unchanged
    (1601, 1000, -1, (1599, 999)),    # int(1601 / (1601 / 1600)) = int(1599.99...): the reference loses a pixel
    (4946, 3286, -1, (1600, 1063)),
    (5187, 3361, -1, (1600, 1036)),   # int(3361 / 3.241875) = int(1036.74...)
    (800, 800, -1, (800, 800)),
    (1000, 500, 400, (400, 200)),     # any other value is a target width
    (1000, 500, 3, (3, 1)),           # 3 is a target width too: int(500 / 333.33)
])
def test_gs_resolution(w, h, r, want):
    assert dataset.gs_resolution(w, h, r) == want


@pytest.mark.parametrize("w,h,r,m,want", [
    (1920, 1080, 1, 1920, (1920, 1080)),    # exactly the cap: unchanged
    (1921, 1080, 1, 1920, (1920, 1079)),    # round(1080 / (1921 / 1920)) = round(1079.44)
    (1080, 1921, 1, 1920, (1079, 1920)),
    (4000, 3000, 2, 1920, (960, 720)),      # the cap uses the ORIGINAL long side: factor 2 * 4000 / 1920
    (45, 31, 2, 1920, (22, 16)),
    (45, 31, 3, 1920, (45, 31)),            # not in {1, 2, 4, 8}: factor 1
    (45, 31, 2, 20, (10, 7)),               # 2 * 45 / 20 = 4.5: round(10.0), round(6.89)
])
def test_sugar_resolution(w, h, r, m, want):
    assert dataset.sugar_resolution(w, h, r, m) == want


# ----------------------------------------------------------------------------------------------------- the readers
def _check_infos(g, name, infos):
    assert [c.name for c in infos] == list(g[f"{name}_names"])
    assert [c.colmap_id for c in infos] == list(g[f"{name}_colmap_id"])
    np.testing.assert_array_equal(np.stack([c.R for c in infos]), g[f"{name}_R"])
    np.testing.assert_array_equal(np.stack([c.T for c in infos]), g[f"{name}_T"])
    np.testing.assert_array_equal(np.array([[c.FoVx, c.FoVy] for c in infos]), g[f"{name}_fov"])


def _check_scene(g, name, info, tmp_path):
    assert len(info.test) == int(g[f"{name}_n_test"])
    cams = info.camera_list
    assert [(c.orig_width, c.orig_height) for c in cams] == [tuple(s) for s in g[f"{name}_info_size"]]
    _check_infos(g, name, cams)
    path = tmp_path / f"{name}_cameras.json"
    dataset.write_cameras_json(path, cams)
    assert path.read_text() == str(g[f"{name}_json"])     # json.dump of equal values: equal bytes
    # mcubes.nerfpp_radius reduces in float64; the reference reduces its float32 centres in float32
    assert info.nerf_radius == pytest.approx(float(g[f"{name}_radius"]), rel=1e-6)
    n = len(g[f"{name}_points"])
    np.testing.assert_array_equal(info.points[:n], g[f"{name}_points"])
    np.testing.assert_array_equal(info.colors[:n], g[f"{name}_colors"])
    assert info.points.dtype == np.float32 and info.colors.dtype == np.float64


@pytest.mark.parametrize("binary", [True, False])
def test_colmap_reader_matches_reference(tmp_path, binary):
    g = _golden("dataset_readers.npz")
    name = "colmap_bin" if binary else "colmap_txt"
    root = dc.colmap_case(str(tmp_path / name), binary=binary, simple=binary, seed=0 if binary else 1)
    before = sorted(os.listdir(os.path.join(root, "sparse", "0")))
    info = dataset.read_colmap_scene_info(root, eval=binary)
    _check_scene(g, name, info, tmp_path)
    assert sorted(os.listdir(os.path.join(root, "sparse", "0"))) == before    # nothing written into the dataset


@pytest.mark.parametrize("white", [True, False])
def test_nerf_synthetic_reader_matches_reference(tmp_path, white):
    import hashlib
    g = _golden("dataset_readers.npz")
    name = f"nerf_{'white' if white else 'black'}"
    root = dc.nerf_case(str(tmp_path / "nerf"))
    info = dataset.read_nerf_synthetic_info(root, white, eval=True, points_rng=np.random.RandomState(3))
    _check_scene(g, name, info, tmp_path)
    digest = hashlib.sha256(info.points.tobytes() + info.colors.tobytes()).hexdigest()
    assert digest == str(g[f"{name}_digest"])
    assert not os.path.exists(os.path.join(root, "points3d.ply"))


def test_colmap_model_rejects_distorted_cameras(tmp_path):
    sparse = str(tmp_path / "sparse" / "0")
    dc.write_colmap(sparse, [(1, "OPENCV", 10, 8, [5.0, 5.0, 5.0, 4.0, 0.1, 0.0, 0.0, 0.0])],
                    [(1, np.array([1.0, 0, 0, 0]), np.zeros(3), 1, "a.png")], (np.zeros((1, 3)), np.zeros((1, 3))))
    with pytest.raises(ValueError, match="OPENCV.*PINHOLE or SIMPLE_PINHOLE"):
        dataset.read_colmap_model(sparse)


def test_colmap_points_ply_is_read_when_present(tmp_path):
    root = dc.colmap_case(str(tmp_path / "c"), n=3)
    rng = np.random.Generator(np.random.PCG64(2))
    xyz = rng.normal(size=(5, 3)).astype(np.float32)
    rgb = rng.integers(0, 256, (5, 3), dtype=np.uint8)
    header = ("ply\nformat binary_little_endian 1.0\nelement vertex 5\n" + "".join(
        f"property float {p}\n" for p in ("x", "y", "z", "nx", "ny", "nz")) +
        "property uchar red\nproperty uchar green\nproperty uchar blue\nend_header\n").encode()
    rows = np.zeros(5, [("xyz", "<f4", 3), ("n", "<f4", 3), ("rgb", "u1", 3)])
    rows["xyz"], rows["rgb"] = xyz, rgb
    with open(os.path.join(root, "sparse", "0", "points3D.ply"), "wb") as f:
        f.write(header + rows.tobytes())
    info = dataset.read_colmap_scene_info(root)
    np.testing.assert_array_equal(info.points, xyz)
    np.testing.assert_array_equal(info.colors, rgb / 255.0)


@pytest.mark.parametrize("name,remove", [("gs_plain", [1]), ("gs_white", [])])
def test_gs_camera_entries_match_reference(name, remove):
    """load_gs_cameras' removal, repeated-name and sort rules against the reference's own choice (the images are
    checked on the GPU)."""
    g = _golden("dataset_readers.npz")
    entries = json.loads(str(g["gs_cameras_json"]))
    assert entries[-1]["img_name"] == entries[4]["img_name"]     # a repeated name: the reference keeps the last
    chosen = dataset.gs_camera_entries(entries, remove)
    assert [e["id"] for e in chosen] == list(g[f"{name}_uid"])
    assert [e["img_name"] for e in chosen] == list(g[f"{name}_names"])


@pytest.mark.parametrize("kind", ["nerf", "colmap"])
def test_readers_take_relative_paths(tmp_path, monkeypatch, kind):
    if kind == "nerf":
        dc.nerf_case(str(tmp_path / "data" / "lego"))
        read = lambda p: dataset.read_nerf_synthetic_info(p, True, points_rng=np.random.RandomState(0))  # noqa: E731
    else:
        dc.colmap_case(str(tmp_path / "data" / "lego"), n=3)
        read = dataset.read_colmap_scene_info  # noqa: E731
    absolute = read(str(tmp_path / "data" / "lego"))
    monkeypatch.chdir(tmp_path)
    relative = read(os.path.join("data", "lego"))
    assert [c.name for c in relative.camera_list] == [c.name for c in absolute.camera_list]
    for c in relative.camera_list:
        assert os.path.isfile(c.image_path) and not os.path.isabs(c.image_path)
    if kind == "nerf":
        assert all(np.array_equal(r.image, a.image) for r, a in zip(relative.camera_list, absolute.camera_list))


def test_shuffle_numbers_views_after_shuffling(tmp_path, monkeypatch):
    """Scene.__init__ shuffles the CameraInfos, then loadCam numbers them: uid is the index after the shuffle."""
    import random
    root = dc.colmap_case(str(tmp_path / "c"), n=6)
    order = list(range(6))
    random.Random(4).shuffle(order)
    names = [c.name for c in dataset.read_colmap_scene_info(root).train]
    monkeypatch.setattr(dataset, "prepare_image", lambda img, w, h, background=None, device="cuda": None)
    monkeypatch.setattr(dataset, "make_camera", lambda *a, device=None, **meta: SimpleNamespace(**meta))
    scene = dataset.load_colmap_scene(root, device="cpu", shuffle_rng=random.Random(4))
    assert [c.name for c, _ in scene.train] == [names[i] for i in order]
    assert [c.uid for c, _ in scene.train] == list(range(6))
    assert [c.name for c in scene.camera_list] == names


def test_image_lookup_is_unambiguous(tmp_path):
    d = tmp_path / "images"
    d.mkdir()
    (d / "a.png").write_bytes(b"")
    (d / "b.png").write_bytes(b"")
    (d / "b.jpg").write_bytes(b"")
    assert dataset._find_image(str(d), "a") == str(d / "a.png")
    with pytest.raises(FileNotFoundError, match="more than one"):
        dataset._find_image(str(d), "b")
    with pytest.raises(FileNotFoundError, match="no image"):
        dataset._find_image(str(d), "c")


def test_read_png_keeps_alpha_only_when_asked(tmp_path):
    from sugar_b200 import objfile
    px = np.random.Generator(np.random.PCG64(0)).integers(0, 256, (5, 7, 4), dtype=np.uint8)
    dc.write_png(str(tmp_path / "x.png"), px)
    assert np.array_equal(objfile.read_png(str(tmp_path / "x.png")), px[..., :3])
    assert np.array_equal(objfile.read_png(str(tmp_path / "x.png"), keep_alpha=True), px)
