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
Byte model: texture_init_kernel 12 B per texel written + per face 24 B ids + 36 B vertices + n x 52 B Gaussians;
per view texture_claim_kernel + texture_add_kernel 36 B per pixel (12 B image, 4 B zbuf, 8 B face id, 8 B texel scratch
written and read, 4 B owner) + 108 B per baked pixel (face ids, vertices, UV ids and UVs, before cache reuse) + 32 B per
winning texel (sum and count read and written).  HBM shares are against the H100 SXM data sheet's 3.35 TB/s.  Every
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
    pick = lambda: next(it) % len(cams)

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
    # per-view stats for the byte model
    baked = sum(int(((p2f >= 0) & (z > 0)).sum()) for z, p2f in zbufs) / len(zbufs)
    st = texture.new_bake_state(init)
    texture._bake(st, verts, faces, verts_uv, faces_uv, cams[0], images[0], *zbufs[0])
    winners = int((st.count > 0).sum())
    kern_init = profile_kernels(torch, arms["initial_texture"])
    kern_bake = profile_kernels(torch, lambda: texture._bake(st, verts, faces, verts_uv, faces_uv, cams[0],
                                                             images[0], *zbufs[0]))
    kern = {**kern_init, **kern_bake}
    npix = W * H
    model = {"texture_init_kernel": 12 * T * T + F * (60 + 52 * n),
             "bake (claim + add)": 36 * npix + 108 * int((zbufs[0][1] >= 0).sum()) + 32 * winners}
    bake_ms = kern.get("texture_claim_kernel", 0.0) + kern.get("texture_add_kernel", 0.0)
    times = {"texture_init_kernel": kern.get("texture_init_kernel"), "bake (claim + add)": bake_ms or None}
    gbs = {k: round(model[k] / (times[k] * 1e-3) / 1e9, 1) for k in model if times.get(k)}
    print(json.dumps({
        "what": "UV texture extraction", "case": name, "faces": F, "gaussians_per_face": n, "texture_size": T,
        "image": f"{W}x{H}", "views": len(cams), "iters": iters, "repeats": args.repeats, "ms": ms,
        "median_ms": {k: median(v) for k, v in ms.items()},
        "mean_baked_pixels_per_view": round(baked), "winning_texels_view0": winners,
        "init_texels_differing_from_torch_restatement": init_diff,
        "deterministic": bool(torch.equal(t1, t2)), "kernels_ms": kern, "model_bytes": model, "achieved_gbs": gbs,
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
