#!/usr/bin/env python
"""Time the UV texture extraction (sugar_b200/texture.py): the initial texels, the per-view ops and the whole call.

    python scripts/bench_texture.py [--cases 400k_n6 2m_n1] [--views 50] [--iters 10] [--repeats 3]

Workloads: scenes.height_field_mesh of ~400k faces with 6 bound Gaussians per face and ~2M faces with 1 (meshbind,
in-plane scales 0.3 grid steps), square size 10, 1920x1080, `views` cameras orbiting above the mesh.  Arms, CUDA events
around `iters` calls, `repeats` rounds alternating the arms in one process:
    initial_texture   texture.initial_texture
    render            one view's rasterizer call (sh degree 0, black background), the mean over the views
    rasterize_mesh    splatmesh.rasterize_mesh of one view (includes its one host read of the face-id check)
    bake              one view's two bake kernels (texture._bake: no argument checks), the mean over the views
    extraction        the whole extract_texture_image_and_uv_from_gaussians over all views (one call per round)
    ref_init_torch    the reference's initial-texel lines restated in PyTorch (oracle/texture_oracle.initial_texture)
                      on the GPU: the only reference-side arm, pytorch3d being unavailable
    mesh_render       texture.render_textured_mesh of one view (bilinear): rasterize_mesh, its argument checks and
                      the shading kernel, the mean over the views
    shade             the shading kernel alone over a view's z-buffer (texture._shade), bilinear
    shade_nearest     the same with sampling_mode='nearest'
    shade_torch       the same pass in PyTorch from the perspective-correct barycentrics pytorch3d's rasterizer hands
                      its shader (computed outside the timing): gathers for the UV interpolation, F.grid_sample on the
                      flipped map, the K = 1 blend
Byte model: texture_init_kernel 12 B per texel written + per face 24 B ids + 36 B vertices + n x 52 B Gaussians;
per view texture_claim_kernel + texture_add_kernel 36 B per pixel (12 B image, 4 B zbuf, 8 B face id, 8 B texel scratch
written and read, 4 B owner) + 108 B per baked pixel (face ids, vertices, UV ids and UVs, before cache reuse) + 32 B per
winning texel (sum and count read and written); texture_render_kernel 24 B per pixel (zbuf, face id, the RGB written)
+ 156 B per covered pixel (face and UV ids, vertices, UVs, four texels; before cache reuse).  HBM shares are against the H100 SXM data sheet's 3.35 TB/s.  Every
line carries the card's name, power limit and max SM clock, read in the same run.
"""
import argparse
import json
import math
import os
import sys
from types import SimpleNamespace

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_meshloss import card, median  # noqa: E402

PEAK_GBS = 3350.0
CASES = {"400k_n6": (448, 448, 6), "2m_n1": (1001, 1001, 1)}
W, H, S = 1920, 1080, 10


def time_ms(torch, fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def orbit(torch, n):
    """n cameras on a circle of radius 1.1 at height 0.9 around the unit square's centre, looking at it."""
    from sugar_b200 import render
    cams = []
    fov_x = 1.0
    fov_y = 2 * math.atan(math.tan(fov_x / 2) * H / W)
    for a in range(n):
        t = 2 * math.pi * a / n
        p = torch.tensor([0.5 + 1.1 * math.cos(t), 0.5 + 1.1 * math.sin(t), 0.9])
        z = p - torch.tensor([0.5, 0.5, 0.0])
        z = z / z.norm()
        x = torch.linalg.cross(torch.tensor([0.0, 0.0, 1.0]), z)
        x = x / x.norm()
        c2w = torch.stack([x, torch.linalg.cross(z, x), z, p], 1).cuda()
        view, proj, center = render.camera_matrices(c2w, fov_x, fov_y)
        cams.append(SimpleNamespace(viewmatrix=view, projmatrix=proj, campos=center, width=W, height=H,
                                    tanfovx=math.tan(fov_x / 2), tanfovy=math.tan(fov_y / 2)))
    return cams


def profile_kernels(torch, fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    kern = {}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
        if t > 0 and "texture" in ev.key:
            name = ev.key.split("(")[0].split("::")[-1].split("<")[0]
            kern[name] = round(kern.get(name, 0.0) + t / 1e3, 4)
    return kern


def torch_barycentrics(torch, verts, faces, cam, p2f):
    """float32 [H,W,3] perspective-correct barycentrics of each pixel's face (0 where none), in float64 on the GPU
    through the z-buffer's projection: what pytorch3d's rasterizer returns beside pix_to_face."""
    v = torch.cat([verts.double(), torch.ones(verts.shape[0], 1, device=verts.device, dtype=torch.float64)], 1)
    z = (v @ cam.viewmatrix.double())[:, 2]
    h = v @ cam.projmatrix.double()
    ndc = h[:, :2] / (h[:, 3:4] + 1e-7)
    x, y = ((ndc[:, 0] + 1.0) * W - 1.0) * 0.5, ((ndc[:, 1] + 1.0) * H - 1.0) * 0.5
    pix = torch.nonzero(p2f.reshape(-1) >= 0)[:, 0]
    f = faces[p2f.reshape(-1)[pix]]
    X, Y, Z = x[f], y[f], z[f]
    sx, sy = (pix % W).double(), (pix // W).double()
    area = (X[:, 2] - X[:, 0]) * (Y[:, 1] - Y[:, 0]) - (Y[:, 2] - Y[:, 0]) * (X[:, 1] - X[:, 0])
    b = torch.stack([((sx - X[:, (e + 1) % 3]) * (Y[:, (e + 2) % 3] - Y[:, (e + 1) % 3]) -
                      (sy - Y[:, (e + 1) % 3]) * (X[:, (e + 2) % 3] - X[:, (e + 1) % 3])) / area for e in range(3)], 1)
    w = b * torch.stack([Z[:, 1] * Z[:, 2], Z[:, 0] * Z[:, 2], Z[:, 0] * Z[:, 1]], 1)
    out = torch.zeros(H * W, 3, device=verts.device)
    out[pix] = (w / w.sum(1, keepdim=True).clamp(min=1e-8)).float()
    return out.view(H, W, 3)


def shade_torch_pass(torch, faces_uv, verts_uv, tex, zbuf, p2f, bary, znear=1e-4, zfar=100.0):
    """interpolate_face_attributes, TexturesUV.sample_textures (bilinear) and softmax_rgb_blend (K = 1, prob = 1,
    black background) in PyTorch.  -> [3,H,W]"""
    mask = p2f >= 0
    uv = (bary[..., None] * verts_uv[faces_uv[p2f.clamp(min=0)]]).sum(-2) * mask[..., None]       # [H,W,2]
    maps = torch.flip(tex.permute(2, 0, 1)[None], [2])
    c = torch.nn.functional.grid_sample(maps, (uv * 2.0 - 1.0)[None], mode="bilinear", align_corners=True,
                                        padding_mode="border")[0]                                  # [3,H,W]
    eps = 1e-10
    z_inv = (zfar - zbuf) / (zfar - znear) * mask
    z_max = z_inv.clamp(min=eps)
    w = mask * torch.exp((z_inv - z_max) / 1e-4)
    delta = torch.exp((eps - z_max) / 1e-4).clamp(min=eps)
    return (w * c) / (w + delta)


def case_line(args, name, info):
    import torch
    from oracle import texture_oracle as to
    from sugar_b200 import meshbind, scenes, splatmesh, texture
    from sugar_b200.diff_gaussian_rasterization import GaussianRasterizationSettings, GaussianRasterizer
    nx, ny, n = CASES[name]
    v, f = scenes.height_field_mesh(nx, ny, seed=0, permute=True)
    verts, faces = torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda()
    F, P = faces.shape[0], faces.shape[0] * n
    h = 1.0 / (nx - 1)
    g = torch.Generator(device="cuda").manual_seed(0)
    b = meshbind.bind_to_mesh(verts, faces, meshbind.bary_coords(n, "cuda"),
                              torch.full((P, 2), math.log(0.3 * h), device="cuda"),
                              torch.randn(P, 2, device="cuda", generator=g), 1e-3 * h)
    pts, scaling, quats = b.points.detach(), b.scaling.detach(), b.quaternions.detach()
    sh_dc = torch.randn(P, 3, device="cuda", generator=g) * 0.5
    strengths = torch.full((P,), 0.9, device="cuda")
    cams = orbit(torch, args.views)
    verts_uv, faces_uv, T = texture.uv_layout(F, S, device="cuda")
    init = texture.initial_texture(verts, faces, pts, scaling, quats, sh_dc, S)
    bg = torch.zeros(3, device="cuda")

    def render(cam):
        st = GaussianRasterizationSettings(image_height=H, image_width=W, tanfovx=cam.tanfovx, tanfovy=cam.tanfovy,
                                           bg=bg, scale_modifier=1.0, viewmatrix=cam.viewmatrix,
                                           projmatrix=cam.projmatrix, sh_degree=0, campos=cam.campos,
                                           prefiltered=False, debug=False)
        return GaussianRasterizer(st)(means3D=pts, means2D=torch.zeros_like(pts), opacities=strengths.view(-1, 1),
                                      shs=sh_dc.view(-1, 1, 3), scales=scaling, rotations=quats)[0]

    with torch.no_grad():
        images = [render(c) for c in cams]
        zbufs = [splatmesh.rasterize_mesh(verts, faces, c) for c in cams]
    state = texture.new_bake_state(init)
    it = iter(range(10 ** 9))
    last = [0]

    def pick():
        last[0] = next(it) % len(cams)
        return last[0]

    it_k = lambda: last[0]            # the view pick() just chose (the shade arms' z-buffer for their camera)

    def bake_one():
        k = pick()
        texture._bake(state, verts, faces, verts_uv, faces_uv, cams[k], images[k], *zbufs[k])

    def render_one():
        with torch.no_grad():
            render(cams[pick()])

    arms = {"initial_texture": lambda: texture.initial_texture(verts, faces, pts, scaling, quats, sh_dc, S),
            "render": render_one,
            "rasterize_mesh": lambda: splatmesh.rasterize_mesh(verts, faces, cams[pick()]),
            "bake": bake_one,
            "extraction": lambda: texture.extract_texture_image_and_uv_from_gaussians(
                verts, faces, pts, scaling, quats, strengths, sh_dc, cams, square_size=S),
            "ref_init_torch": lambda: to.initial_texture(verts, faces, pts, scaling, quats, sh_dc, S, margins=False)}
    bary = [torch_barycentrics(torch, verts, faces, c, p2f) for c, (_, p2f) in zip(cams, zbufs)]

    def shade_torch(k):
        zbuf, p2f = zbufs[k]
        return shade_torch_pass(torch, faces_uv, verts_uv, init, zbuf, p2f, bary[k])

    arms.update({
        "mesh_render": lambda: texture.render_textured_mesh(verts, faces, verts_uv, faces_uv, init, cams[pick()]),
        "shade": lambda: texture._shade(verts, faces, verts_uv, faces_uv, init, cams[pick()], *zbufs[it_k()]),
        "shade_nearest": lambda: texture._shade(verts, faces, verts_uv, faces_uv, init, cams[pick()], *zbufs[it_k()],
                                                sampling_mode="nearest"),
        "shade_torch": lambda: shade_torch(pick())})
    iters = {k: (1 if k == "extraction" else args.iters) for k in arms}
    for fn in arms.values():
        fn()
    ms = {k: [] for k in arms}
    for _ in range(args.repeats):
        for k, fn in arms.items():
            ms[k].append(round(time_ms(torch, fn, iters[k]), 4))
    # agreement of the two init arms, determinism of the whole call
    ref = to.initial_texture(verts, faces, pts, scaling, quats, sh_dc, S, margins=False)[0]
    init_diff = float((ref != init).any(-1).float().mean())
    t1 = texture.extract_texture_image_and_uv_from_gaussians(verts, faces, pts, scaling, quats, strengths, sh_dc,
                                                             cams, square_size=S)[2]
    t2 = texture.extract_texture_image_and_uv_from_gaussians(verts, faces, pts, scaling, quats, strengths, sh_dc,
                                                             cams, square_size=S)[2]
    # the shading kernel against the torch pass at view 0 (bilinear; the UVs differ by their float32 rounding)
    shade_max_diff = float((texture._shade(verts, faces, verts_uv, faces_uv, init, cams[0], *zbufs[0]) -
                            shade_torch(0)).abs().max())
    # per-view stats for the byte model
    baked = sum(int(((p2f >= 0) & (z > 0)).sum()) for z, p2f in zbufs) / len(zbufs)
    st = texture.new_bake_state(init)
    texture._bake(st, verts, faces, verts_uv, faces_uv, cams[0], images[0], *zbufs[0])
    winners = int((st.count > 0).sum())
    kern_init = profile_kernels(torch, arms["initial_texture"])
    kern_shade = profile_kernels(torch, lambda: texture._shade(verts, faces, verts_uv, faces_uv, init, cams[0],
                                                               *zbufs[0]))
    kern_bake = profile_kernels(torch, lambda: texture._bake(st, verts, faces, verts_uv, faces_uv, cams[0],
                                                             images[0], *zbufs[0]))
    kern = {**kern_init, **kern_bake, **kern_shade}
    npix = W * H
    model = {"texture_init_kernel": 12 * T * T + F * (60 + 52 * n),
             "bake (claim + add)": 36 * npix + 108 * int((zbufs[0][1] >= 0).sum()) + 32 * winners,
             "texture_render_kernel": 24 * npix + 156 * int((zbufs[0][1] >= 0).sum())}
    bake_ms = kern.get("texture_claim_kernel", 0.0) + kern.get("texture_add_kernel", 0.0)
    times = {"texture_init_kernel": kern.get("texture_init_kernel"), "bake (claim + add)": bake_ms or None,
             "texture_render_kernel": kern.get("texture_render_kernel")}
    gbs = {k: round(model[k] / (times[k] * 1e-3) / 1e9, 1) for k in model if times.get(k)}
    print(json.dumps({
        "what": "UV texture extraction", "case": name, "faces": F, "gaussians_per_face": n, "texture_size": T,
        "image": f"{W}x{H}", "views": len(cams), "iters": iters, "repeats": args.repeats, "ms": ms,
        "median_ms": {k: median(v) for k, v in ms.items()},
        "mean_baked_pixels_per_view": round(baked), "winning_texels_view0": winners,
        "init_texels_differing_from_torch_restatement": init_diff,
        "deterministic": bool(torch.equal(t1, t2)), "shade_vs_torch_max_abs_diff": shade_max_diff, "kernels_ms": kern, "model_bytes": model, "achieved_gbs": gbs,
        "hbm_frac_of_3350_gbs": {k: round(x / PEAK_GBS, 3) for k, x in gbs.items()}, "card": info}), flush=True)
    del images, zbufs, state, st
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", nargs="+", default=list(CASES))
    ap.add_argument("--views", type=int, default=50)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    info = card()
    for name in args.cases:
        case_line(args, name, info)
    return 0


if __name__ == "__main__":
    sys.exit(main())
