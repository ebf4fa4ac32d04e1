"""The dataset path on the GPU: the sgr_image kernels byte for byte against Pillow's goldens and the numpy oracle
(oracle/imageprep_oracle.py), the readers' images against the reference's own loading lines
(tests/golden/make_dataset_golden.py), a render -> PNG + COLMAP -> load -> render round trip, and pre-training, the
cameras.json hand-off and the coarse trainer on a loaded scene."""
import json
import math
import os
import random
import sys
import zlib

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import dataset_cases as dc  # noqa: E402
from oracle import imageprep_oracle as o  # noqa: E402
from sugar_b200 import dataset, gsply, knn, mcubes, steps, train  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _golden(name):
    return np.load(os.path.join(HERE, "golden", name))


def _expect(gt, u8):
    """gt float32 [3,H,W] on the device must be u / 255 of the uint8 [H,W,3] bytes, bit for bit."""
    got = gt.cpu().numpy()
    want = o.to_float(u8)
    assert got.shape == want.shape and got.dtype == np.float32
    bad = np.argwhere(got.view(np.int32) != want.view(np.int32))
    assert bad.size == 0, (len(bad), bad[:5])


# ------------------------------------------------------------------------------------------------------- the kernels
def test_kernel_equals_pillow_goldens():
    g = _golden("dataset_pil.npz")
    for name in sorted(k[:-3] for k in g.files if k.endswith("_in")):
        img, ref = g[name + "_in"], g[name + "_out"]
        bg = "white" if name.endswith("_white") else "black" if name.endswith("_black") else None
        _expect(dataset.prepare_image(img, ref.shape[1], ref.shape[0], background=bg, device=DEV), ref)


@pytest.mark.parametrize("case", [
    ("rgb_mipnerf", (3361, 5187, 3), (1600, 1037), None),
    ("rgba_premultiplied", (1501, 2003, 4), (977, 640), None),
    ("rgba_height_only", (700, 300, 4), (300, 451), None),
    ("rgba_same_size", (301, 203, 4), (203, 301), None),
    ("composite_white_down", (1100, 1700, 4), (800, 518), "white"),
    ("composite_black_same", (300, 400, 4), (400, 300), "black"),
    ("composite_rgb_white", (200, 300, 3), (150, 100), "white"),
    ("upscale", (97, 131, 3), (400, 301), None),
    ("one_px", (1, 1, 3), (3, 2), None),
])
def test_kernel_equals_oracle(case):
    name, shape, (w, h), bg = case
    rng = np.random.Generator(np.random.PCG64(zlib.crc32(name.encode())))
    img = rng.integers(0, 256, shape, dtype=np.uint8)
    if shape[2] == 4:   # a third of the alphas at 0 or 255, as on object borders and backgrounds
        img[..., 3] = np.where(rng.random(shape[:2]) < 0.33, rng.choice(np.array([0, 255], np.uint8), shape[:2]),
                               img[..., 3])
    oracle_img = img if shape[2] == 4 or bg is None else \
        np.concatenate([img, np.full(shape[:2] + (1,), 255, np.uint8)], 2)    # convert("RGBA")
    want = o.prepare_bytes(oracle_img, w, h, background=bg)
    got = dataset.prepare_image(img, w, h, background=bg, device=DEV)
    _expect(got, want)
    torch.cuda.synchronize()
    assert torch.equal(got, dataset.prepare_image(torch.from_numpy(img).to(DEV), w, h, background=bg, device=DEV))


def test_prepare_image_rejects_bad_input():
    with pytest.raises(ValueError, match="uint8"):
        dataset.prepare_image(np.zeros((4, 4, 2), np.uint8), 2, 2, device=DEV)
    with pytest.raises(ValueError, match="uint8"):
        dataset.prepare_image(np.zeros((4, 4, 3), np.float32), 2, 2, device=DEV)
    with pytest.raises(ValueError, match="background"):
        dataset.prepare_image(np.zeros((4, 4, 4), np.uint8), 2, 2, background="grey", device=DEV)
    with pytest.raises(ValueError, match=">= 1"):
        dataset.prepare_image(np.zeros((4, 4, 3), np.uint8), 0, 2, device=DEV)


# ----------------------------------------------------------------------------------------- the readers' images
def _check_views(g, name, views):
    assert [c.name for c, _ in views] == list(g[f"{name}_names"])
    np.testing.assert_array_equal(np.stack([c.R for c, _ in views]), g[f"{name}_R"])
    np.testing.assert_array_equal(np.stack([c.T for c, _ in views]), g[f"{name}_T"])
    for i, (cam, gt) in enumerate(views):
        ref = g[f"{name}_img{i}"]
        assert (cam.height, cam.width) == ref.shape[:2]
        _expect(gt, ref)


def test_colmap_images_equal_reference(tmp_path):
    g = _golden("dataset_readers.npz")
    root = dc.colmap_case(str(tmp_path / "bin"), binary=True)
    scene = dataset.load_colmap_scene(root, eval=True, resolution=2, device=DEV)
    _check_views(g, "colmap_bin", scene.test + scene.train)
    root = dc.colmap_case(str(tmp_path / "txt"), binary=False, simple=False, seed=1)
    scene = dataset.load_colmap_scene(root, eval=False, resolution=-1, device=DEV)
    _check_views(g, "colmap_txt", scene.test + scene.train)


@pytest.mark.parametrize("white", [True, False])
def test_nerf_synthetic_images_equal_reference(tmp_path, white):
    g = _golden("dataset_readers.npz")
    root = dc.nerf_case(str(tmp_path / "nerf"))
    scene = dataset.load_nerf_synthetic_scene(root, white, eval=True, resolution=2, device=DEV,
                                              points_rng=np.random.RandomState(3))
    _check_views(g, f"nerf_{'white' if white else 'black'}", scene.test + scene.train)


def test_load_gs_cameras_equals_reference(tmp_path):
    g = _golden("dataset_readers.npz")
    root = dc.colmap_case(str(tmp_path / "bin"), binary=True)
    out = tmp_path / "gs_out"
    out.mkdir()
    (out / "cameras.json").write_text(str(g["gs_cameras_json"]))
    for name, kw in (("gs_plain", dict(image_resolution=2, max_img_size=20, remove_indices=[1])),
                     ("gs_white", dict(image_resolution=1, white_background=True))):
        views, test = dataset.load_gs_cameras(root, str(out), device=DEV, **kw)
        assert test == []
        assert [c.uid for c, _ in views] == list(g[f"{name}_uid"])
        np.testing.assert_array_equal(np.array([[c.FoVx, c.FoVy] for c, _ in views]), g[f"{name}_fov"])
        _check_views(g, name, views)
    train_v, test_v = dataset.load_gs_cameras(root, str(out), eval_split=True, eval_split_interval=4, device=DEV)
    assert [c.name for c, _ in test_v] == list(g["gs_white_names"][::4])
    assert len(train_v) + len(test_v) == len(g["gs_white_names"])


# ------------------------------------------------------------------------------------------------ end to end
def hidden_cloud(P=6000, seed=31):
    """A seeded cloud of Gaussians in a ball of radius 1 about the origin, the raw dict of steps.activate."""
    gen = torch.Generator().manual_seed(seed)
    d = torch.randn(P, 3, generator=gen)
    pts = d / d.norm(dim=1, keepdim=True) * torch.rand(P, 1, generator=gen).pow(1 / 3)
    raw = dict(points=pts, sh_dc=0.8 * torch.randn(P, 1, 3, generator=gen), sh_rest=torch.zeros(P, 15, 3),
               densities=torch.full((P, 1), 1.5), scales=torch.full((P, 3), math.log(0.03)) +
               0.2 * torch.randn(P, 3, generator=gen), quaternions=torch.randn(P, 4, generator=gen))
    return {k: v.to(DEV) for k, v in raw.items()}


def render(raw, cam):
    with torch.no_grad():
        return steps.render(steps.ours_ops(), steps.activate(raw), cam, torch.zeros(3, device=DEV), sh_deg=0)[0]


def write_rendered_colmap(root, raw, n=12, W=160, H=120, fx=150.0, fy=152.0):
    """Renders of `raw` from n ring cameras saved as PNG, with the COLMAP model of those cameras and the cloud's
    jittered centres as its points."""
    os.makedirs(os.path.join(root, "images"), exist_ok=True)
    images, cams = [], {}
    for i, (Rwc, t) in enumerate(dc.ring_poses(n, seed=4)):
        name = f"view_{i:02d}.png"
        cam = dataset.make_camera(Rwc.T, t, dataset.focal2fov(fx, W), dataset.focal2fov(fy, H), W, H, device=DEV)
        img = render(raw, cam).clamp(0, 1)
        px = (img * 255.0).round().to(torch.uint8).permute(1, 2, 0).cpu().numpy()
        dc.write_png(os.path.join(root, "images", name), px)
        images.append((i + 1, dc.rotmat2qvec(Rwc), t, 1, name))
        cams[name.split(".")[0]] = cam
    gen = torch.Generator().manual_seed(3)
    xyz = raw["points"].cpu()[::3] + 0.03 * torch.randn(raw["points"][::3].shape, generator=gen)
    rgb = ((raw["sh_dc"][::3, 0].cpu() * 0.28209479177387814 + 0.5).clamp(0, 1) * 255).to(torch.uint8)
    dc.write_colmap(os.path.join(root, "sparse", "0"), [(1, "PINHOLE", W, H, [fx, fy, W / 2, H / 2])], images,
                    (xyz.double().numpy(), rgb.numpy()))
    return cams


def test_render_round_trip_and_training_on_a_loaded_scene(tmp_path):
    raw_hidden = hidden_cloud()
    root = str(tmp_path / "scene")
    cams = write_rendered_colmap(root, raw_hidden)
    scene = dataset.load_colmap_scene(root, resolution=1, device=DEV, shuffle_rng=random.Random(0))
    assert len(scene.train) == 12 and scene.test == []
    worst = 0.0
    for cam, gt in scene.train:
        ref = cams[cam.name]
        for k in ("viewmatrix", "projmatrix", "campos"):
            torch.testing.assert_close(getattr(cam, k), getattr(ref, k), rtol=0, atol=2e-6)
        assert (cam.width, cam.height, cam.tanfovx, cam.tanfovy) == (ref.width, ref.height, ref.tanfovx, ref.tanfovy)
        d = (render(raw_hidden, cam).clamp(0, 1) - gt).abs()
        worst = max(worst, float(d.max()))
        # the PNG holds the render rounded to bytes: the same conventions give it back within half a step
        assert float(torch.quantile(d.flatten(), 0.999)) <= 0.5 / 255 + 1e-4, cam.name
    print(f"round trip: largest |render - png| {worst * 255:.3f} / 255")
    assert worst <= 2.0 / 255

    # pre-training from the scene's SfM points: the loss falls
    raw = train.init_from_points(torch.from_numpy(scene.points).to(DEV), scene.colors)
    losses = []
    train.train_3dgs(raw, scene.train, scene.nerf_radius, num_iterations=300, densify_from_iter=100,
                     densify_until_iter=250, densification_interval=50, opacity_reset_interval=3000, sh_every=100,
                     rng=random.Random(1), on_iteration=lambda it, l, ev: losses.append(l))
    lv = torch.stack(losses).cpu().numpy()
    print(f"train_3dgs on the loaded scene: loss {lv[:20].mean():.4f} -> {lv[-20:].mean():.4f}")
    assert np.all(np.isfinite(lv)) and lv[-20:].mean() < 0.7 * lv[:20].mean()

    # the hand-off: cameras.json and the .ply, then SuGaR's loader and the coarse trainer
    out = tmp_path / "gs_out"
    out.mkdir()
    dataset.write_cameras_json(str(out / "cameras.json"), scene.camera_list)
    entries = json.loads((out / "cameras.json").read_text())
    assert [e["id"] for e in entries] == list(range(12)) and entries[0]["img_name"] == "view_00"
    ply = str(out / "point_cloud" / "iteration_300" / "point_cloud.ply")
    gsply.save_gaussians_ply(ply, raw)
    views, test = dataset.load_gs_cameras(root, str(out), device=DEV)
    assert test == [] and [c.name for c, _ in views] == sorted(cams)
    by_name = {c.name: (c, gt) for c, gt in scene.train}
    for cam, gt in views:
        ref, ref_gt = by_name[cam.name]
        for k in ("viewmatrix", "projmatrix", "campos"):
            torch.testing.assert_close(getattr(cam, k), getattr(ref, k), rtol=0, atol=2e-6)
        assert cam.tanfovx == pytest.approx(ref.tanfovx, rel=1e-12) and cam.tanfovy == pytest.approx(ref.tanfovy,
                                                                                                      rel=1e-12)
        assert torch.equal(gt, ref_gt)
    back = gsply.load_gaussians_ply(ply, sh_degree=3, device=DEV)
    knn_idx = knn.reset_neighbors(back["points"].detach(), 16)[1]
    extent = mcubes.camera_spatial_extent(torch.stack([c.campos.cpu() for c, _ in views]))
    seen = []
    train.train_coarse(back, views, knn_idx, mode="density", spatial_extent=extent, num_iterations=7003,
                       first_iteration=7000, n_samples=10_000, on_iteration=lambda it, l, ev: seen.append(float(l)))
    assert len(seen) == 4 and all(math.isfinite(x) for x in seen)
