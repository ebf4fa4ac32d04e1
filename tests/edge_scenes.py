"""Scenes at the projection's edges: the 1.3 tan(fov) guard band, the near plane, centres far off screen and
scale_modifier != 1.

TEST INFRASTRUCTURE ONLY.  `scenes.make_scene` keeps every mean at |x/z| <= 1.1 tan(fov), so the per-Gaussian
projection's clamp, its backward gates, the near-plane cull at depth == 0.2f, the overflow of denom^2 in the
cov2D backward, the saturating (int)ceilf of the radius and the footprint masks of centres far outside the image
are never reached there.  Each builder here places seeded (PCG64) Gaussians at one of those edges and returns
(Scene, {class name: bool [P]}), the classes decided by the fp32 values the kernels compute (`fp32_view`, `gates`,
project64.denom_overflows), and the CPU tests assert that every class keeps visible, contributing rows.

CASES: name -> dict(build, use_sh, sh_degree, scale_modifier, bg).  All images are 160 x 96 (tanfovx = tan 30 deg).
"""
import math

import numpy as np

W, H = 160, 96
F32_MAX = float(np.finfo(np.float32).max)
INT32_MAX = 2 ** 31 - 1


def _base(P, seed, camera):
    from sugar_b200 import scenes
    return scenes.make_scene(P, W, H, seed=seed, camera=camera, frac_behind=0.0)


def _to_world(sc, cam):
    """Camera-space points -> world points for `sc`'s camera (x_cam = R x_world + t)."""
    V = sc.viewmatrix.astype(np.float64).T
    return np.ascontiguousarray((np.asarray(cam, np.float64) - V[:3, 3]) @ V[:3, :3], np.float32)


def _f32(x):
    return np.asarray(x, np.float64).astype(np.float32)


def _xf_row(m, r, p):
    """xf_row of the kernels and the oracle, in fp32: fadd(fma(z, m8, fma(x, m0, y * m4)), m12).  The fmas are
    formed as the exact double product plus one double sum, then rounded to fp32."""
    x, y, z = (p[:, k].astype(np.float64) for k in range(3))
    t = _f32(y * np.float64(m[4 + r]))
    t = _f32(x * np.float64(m[r]) + t.astype(np.float64))
    t = _f32(z * np.float64(m[8 + r]) + t.astype(np.float64))
    return _f32(t.astype(np.float64) + np.float64(m[12 + r]))


def fp32_view(sc):
    """The view-space position (tx, ty, tz) and txtz, tytz, limx, limy as the kernels compute them in fp32."""
    m = np.asarray(sc.viewmatrix, np.float32).reshape(-1)
    tx, ty, tz = (_xf_row(m, r, sc.means3D) for r in range(3))
    limx = np.float32(np.float32(sc.tanfovx) * np.float32(1.3))
    limy = np.float32(np.float32(sc.tanfovy) * np.float32(1.3))
    with np.errstate(divide="ignore", invalid="ignore"):
        return dict(tx=tx, ty=ty, tz=tz, txtz=tx / tz, tytz=ty / tz, limx=limx, limy=limy)


def gates(sc):
    """The backward's x_grad_mul / y_grad_mul decisions (1 inside [-lim, lim], 0 outside), fp32."""
    v = fp32_view(sc)
    gx = ~((v["txtz"] < -v["limx"]) | (v["txtz"] > v["limx"]))
    gy = ~((v["tytz"] < -v["limy"]) | (v["tytz"] > v["limy"]))
    return gx, gy


# ---------------------------------------------------------------------------------------------------------------------
# builders
def guard_band(seed=101, camera="posed", P=320):
    """Means at |x/z| and / or |y/z| in (1.3, 3] tan(fov): x only, y only, both, with both signs; scales large
    enough that the footprints reach into the image (the projected sigma is at least f s / z, which is set to
    0.5-1.2x the centre's distance from the image)."""
    sc = _base(P, seed, camera)
    rng = np.random.Generator(np.random.PCG64(seed + 1))
    tfx, tfy = float(np.float32(sc.tanfovx)), float(np.float32(sc.tanfovy))
    focal = W / (2 * tfx)
    kinds = np.array(["x", "y", "xy"])[np.arange(P) % 3]
    z = rng.uniform(2.0, 8.0, P)
    sx = np.where(rng.uniform(size=P) < 0.5, -1.0, 1.0)
    sy = np.where(rng.uniform(size=P) < 0.5, -1.0, 1.0)
    out_x = np.isin(kinds, ["x", "xy"])
    out_y = np.isin(kinds, ["y", "xy"])
    rx = np.where(out_x, sx * rng.uniform(1.32, 3.0, P), rng.uniform(-0.9, 0.9, P))
    ry = np.where(out_y, sy * rng.uniform(1.32, 3.0, P), rng.uniform(-0.9, 0.9, P))
    cam = np.stack([rx * tfx * z, ry * tfy * z, z], 1)
    # pixels between the centre and the image, per axis
    dx = np.maximum(np.abs(rx) - 1.0, 0.0) * W / 2
    dy = np.maximum(np.abs(ry) - 1.0, 0.0) * H / 2
    dist = np.maximum(np.hypot(dx, dy), 4.0)
    s = rng.uniform(0.5, 1.2, P) * dist * z / focal
    scales = s[:, None] * np.exp(rng.normal(0.0, 0.25, (P, 3)))
    opac = rng.uniform(0.05, 0.4, (P, 1))
    sc = sc._replace(means3D=_to_world(sc, cam), scales=_f32(scales), opacities=_f32(opac))
    v = fp32_view(sc)
    ox = (np.abs(v["txtz"]) > v["limx"])
    oy = (np.abs(v["tytz"]) > v["limy"])
    cls = {"x_only": ox & ~oy, "y_only": oy & ~ox, "both": ox & oy}
    for name, o, t in (("x", ox, v["txtz"]), ("y", oy, v["tytz"])):
        cls[f"{name}_pos"], cls[f"{name}_neg"] = o & (t > 0), o & (t < 0)
    return sc, cls


def guard_edge_rows():
    """(axis, sign, k, other) of the guard_edge rows: k ulps of x (or y) past 2 fl32(1.3 tanfov) (k < 0: inside)."""
    return [(axis, sign, k, other) for axis in ("x", "y") for sign in (1, -1) for k in (-2, -1, 0, 1, 2)
            for other in (-0.5, 0.0, 0.5)]


def guard_edge(seed=202):
    """Identity camera, every mean at z = 2, so that x / z is exact in fp32: x = 2 fl32(1.3 tanfovx) and +-1, +-2
    ulps (likewise y), both signs.  At txtz == limx the gate is 1 and the clamp a no-op; one ulp past, the gate is
    0 and t.x is clamped."""
    rows = guard_edge_rows()
    P = len(rows)
    sc = _base(P, seed, "identity")
    rng = np.random.Generator(np.random.PCG64(seed + 1))
    tf = {"x": np.float32(sc.tanfovx), "y": np.float32(sc.tanfovy)}
    lim = {k: np.float32(v * np.float32(1.3)) for k, v in tf.items()}
    m = np.zeros((P, 3), np.float32)
    m[:, 2] = 2.0
    for i, (axis, sign, k, other) in enumerate(rows):
        e = np.float32(2) * lim[axis]                   # exact: a power-of-two multiple
        for _ in range(abs(k)):
            e = np.nextafter(e, np.float32(np.inf) if k > 0 else np.float32(0))
        a, o = (0, 1) if axis == "x" else (1, 0)
        m[i, a] = sign * e
        m[i, o] = np.float32(other * 2.0 * float(tf["y" if axis == "x" else "x"]))
    # the footprint reaches ~0.15 W (0.15 H) over the edge: projected sigma f s / z ~ 30 px
    scales = 0.45 * np.exp(rng.normal(0.0, 0.15, (P, 3)))
    opac = rng.uniform(0.15, 0.45, (P, 1))
    sc = sc._replace(means3D=m, scales=_f32(scales), opacities=_f32(opac))
    k = np.array([r[2] for r in rows])
    return sc, {"inside": k < 0, "at_edge": k == 0, "past_edge": k > 0}


NEAR = np.float32(0.2)


def near_plane(seed=303):
    """Identity camera (depth == z exactly): z = 0.2f (culled), 0.2f + 1 and + 2 ulps, 0.2001, 0.21, 0.25 (kept)
    with ordinary scales; huge splats just past the plane whose denom^2 overflows (denom2inv == 0) and whose
    3 sqrt(lmax) exceeds 2^31 (the radius saturates at INT32_MAX); and points behind the camera."""
    z1 = np.nextafter(NEAR, np.float32(1))
    z2 = np.nextafter(z1, np.float32(1))
    depths = [("at_plane", NEAR)] * 6 + [("ulp1", z1)] * 6 + [("ulp2", z2)] * 6 + \
             [("kept", np.float32(v)) for v in (0.2001, 0.21, 0.25) for _ in range(6)] + \
             [("overflow", np.float32(0.21))] * 4 + [("saturated", np.float32(0.205))] * 3 + \
             [("behind", np.float32(v)) for v in (-0.5, 0.0, 0.1)]
    P = len(depths)
    sc = _base(P, seed, "identity")
    rng = np.random.Generator(np.random.PCG64(seed + 1))
    kind = np.array([d[0] for d in depths])
    z = np.array([d[1] for d in depths], np.float32)
    tfx, tfy = float(np.float32(sc.tanfovx)), float(np.float32(sc.tanfovy))
    m = np.stack([_f32(z * tfx * rng.uniform(-0.8, 0.8, P)), _f32(z * tfy * rng.uniform(-0.8, 0.8, P)), z], 1)
    # ordinary: 3-20 px sigma at f / z ~ 690 px per unit
    s = np.exp(rng.uniform(math.log(0.005), math.log(0.03), P))
    s = np.where(kind == "overflow", rng.uniform(150.0, 400.0, P), s)     # sigma ~ 1e5 px: denom ~ 1e20
    scales = s[:, None] * np.exp(rng.normal(0.0, 0.1, (P, 3)))
    # saturated: an axis-aligned needle, sigma_x ~ 1.3e9 px (3 sigma > 2^31) and sigma_y ~ 10 px, so that
    # a c stays far below FLT_MAX and det, conic and lmax stay finite
    sat = kind == "saturated"
    scales[sat] = np.stack([rng.uniform(1.9e6, 2.4e6, P), np.full(P, 0.015), np.full(P, 0.015)], 1)[sat]
    rots = sc.rotations.copy()
    rots[sat] = (1.0, 0.0, 0.0, 0.0)
    opac = np.where(np.isin(kind, ["overflow", "saturated"]), 0.03, rng.uniform(0.3, 0.8, P))[:, None]
    sc = sc._replace(means3D=m, scales=_f32(scales), rotations=_f32(rots), opacities=_f32(opac))
    return sc, {k: kind == k for k in ("at_plane", "ulp1", "ulp2", "kept", "overflow", "saturated", "behind")}


def offscreen_centres(seed=404, P=72):
    """Centres 1 to 50 image widths (heights) outside the image, left, right, above or below, with footprints that
    still reach in (projected sigma >= 0.5x the distance); and a few whose ellipse half-extent exceeds 1e6 px
    (the footprint masks' `all` path)."""
    sc = _base(P, seed, "identity")
    rng = np.random.Generator(np.random.PCG64(seed + 1))
    tfx, tfy = float(np.float32(sc.tanfovx)), float(np.float32(sc.tanfovy))
    focal = W / (2 * tfx)
    huge = np.arange(P) >= P - 6
    D = np.exp(rng.uniform(0.0, math.log(50.0), P))                 # image sizes outside
    D = np.where(huge, rng.uniform(1.0, 3.0, P), D)
    side = np.arange(P) % 4
    z = rng.uniform(3.0, 8.0, P)
    along = rng.uniform(-0.8, 0.8, P)
    # ndc of the centre: 1 + 2 D past the edge (pixel W - 1/2 + D W)
    out = np.where(side % 2 == 0, 1.0, -1.0) * (1.0 + 2.0 * D)
    rx = np.where(side < 2, out, along)
    ry = np.where(side < 2, along, out)
    cam = np.stack([rx * tfx * z, ry * tfy * z, z], 1)
    dist = D * np.where(side < 2, W, H)
    s = rng.uniform(0.6, 1.0, P) * dist * z / focal
    s = np.where(huge, rng.uniform(2e6, 4e6, P) * z / focal, s)
    scales = s[:, None] * np.exp(rng.normal(0.0, 0.2, (P, 3)))
    opac = rng.uniform(0.03, 0.15, (P, 1))
    sc = sc._replace(means3D=_f32(cam), scales=_f32(scales), opacities=_f32(opac))
    return sc, {"near": ~huge & (D < 5), "far": ~huge & (D >= 5), "e_all": huge}


def ordinary(seed=505):
    """An ordinary posed scene (make_scene), for scale_modifier."""
    from sugar_b200 import scenes
    sc = scenes.make_scene(2500, W, H, seed=seed, camera="posed")
    return sc, {"all": np.ones(sc.means3D.shape[0], bool)}


CASES = {
    "guard_band_posed_sh3": dict(build=lambda: guard_band(101, "posed"), use_sh=True, sh_degree=3,
                                 scale_modifier=1.0, bg=(0.0, 0.0, 0.0)),
    "guard_band_posed_colors": dict(build=lambda: guard_band(111, "posed"), use_sh=False, sh_degree=0,
                                    scale_modifier=1.0, bg=(0.1, 0.2, 0.3)),
    # seed 121 put one pair's fp32 alpha within 4 ulps of 1/255 behind 80 splats, which blend64 would exclude
    "guard_band_identity_colors": dict(build=lambda: guard_band(122, "identity"), use_sh=False, sh_degree=0,
                                       scale_modifier=1.0, bg=(0.25, 0.5, 1.0)),
    "guard_band_identity_sh3": dict(build=lambda: guard_band(131, "identity"), use_sh=True, sh_degree=3,
                                    scale_modifier=1.0, bg=(0.0, 0.0, 0.0)),
    "guard_edge": dict(build=guard_edge, use_sh=False, sh_degree=0, scale_modifier=1.0, bg=(0.1, 0.2, 0.3)),
    "near_plane": dict(build=near_plane, use_sh=False, sh_degree=0, scale_modifier=1.0, bg=(0.1, 0.2, 0.3)),
    "offscreen_centres": dict(build=offscreen_centres, use_sh=False, sh_degree=0, scale_modifier=1.0,
                              bg=(0.1, 0.2, 0.3)),
    "scale_mod_0.5_posed_sh3": dict(build=ordinary, use_sh=True, sh_degree=3, scale_modifier=0.5,
                                    bg=(0.0, 0.0, 0.0)),
    "scale_mod_1.7_posed_sh3": dict(build=ordinary, use_sh=True, sh_degree=3, scale_modifier=1.7,
                                    bg=(0.0, 0.0, 0.0)),
    "scale_mod_0.5_guard_band": dict(build=lambda: guard_band(111, "posed"), use_sh=False, sh_degree=0,
                                     scale_modifier=0.5, bg=(0.1, 0.2, 0.3)),
    "scale_mod_1.7_guard_band": dict(build=lambda: guard_band(111, "posed"), use_sh=False, sh_degree=0,
                                     scale_modifier=1.7, bg=(0.1, 0.2, 0.3)),
}


def opts(name):
    c = CASES[name]
    return dict(use_sh=c["use_sh"], sh_degree=c["sh_degree"], scale_modifier=c["scale_modifier"])


def upstream(name):
    from sugar_b200 import scenes
    return scenes.upstream_grad(W, H, seed=7 + sorted(CASES).index(name))
