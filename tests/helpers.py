"""Shared test plumbing: run the same seeded scene through (a) the sugar_b200 CUDA path,
(b) the CPU oracle, (c) the unmodified reference CUDA build in oracle/_ref (when present), whose results
the GPU tests read from tests/golden/refbuild_*.npz (tests/golden/make_refbuild_golden.py)."""
import hashlib
import importlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIR = os.path.join(ROOT, "oracle", "_ref")
GOLDEN_DIR = os.path.join(ROOT, "tests", "golden")

# what a golden keeps of a gradient tensor: its shape, |g|_inf, N_STRIDED evenly spaced entries and the N_TOP
# largest -- or the whole tensor, for cases whose gradients hold at most WHOLE_MAX entries in all
N_STRIDED, N_TOP, WHOLE_MAX = 256, 32, 40_000


def _np(x):
    return x.detach().cpu().numpy() if hasattr(x, "detach") else np.asarray(x)


def digest(x):
    """SHA-256 of an array's values (not of its dtype or shape): integers as int64, floats by their fp32 bits.
    Two arrays with equal digests are bit-identical, which is what the reference comparisons require."""
    a = _np(x).reshape(-1)
    a = a.astype(np.float32).view(np.uint32).astype(np.int64) if a.dtype.kind == "f" else a.astype(np.int64)
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), np.uint8)


def strided_idx(n):
    return np.unique(np.arange(N_STRIDED, dtype=np.int64) * n // N_STRIDED) if n else np.zeros(0, np.int64)


def grad_summary(prefix, g, whole=False):
    """{prefix_*: ...} of one gradient for a golden file (g: torch tensor on any device)."""
    import torch
    f = g.detach().reshape(-1).float()
    k = min(N_TOP, f.numel())
    top = torch.topk(f.abs(), k).indices.cpu().numpy().astype(np.int64) if k else np.zeros(0, np.int64)
    a = f.cpu().numpy()
    d = {prefix + "_shape": np.asarray(g.shape, np.int64), prefix + "_inf": np.float64(np.abs(a).max() if a.size else 0.0),
         prefix + "_top_idx": top, prefix + "_top": a[top], prefix + "_strided": a[strided_idx(a.size)]}
    if whole:
        d[prefix + "_whole"] = a
    return d


def golden_rel_err(g, gold, prefix):
    """rel_err of a gradient against the reference's: over the whole tensor where the golden keeps it, else over the
    entries it keeps (grad_summary).  The shapes must match."""
    a = _np(g)
    assert tuple(a.shape) == tuple(gold[prefix + "_shape"]), f"{prefix}: shape {a.shape} vs {gold[prefix + '_shape']}"
    a = a.astype(np.float64).reshape(-1)
    if prefix + "_whole" in gold:
        return rel_err(a, gold[prefix + "_whole"])
    d = max(np.abs(a[gold[prefix + "_top_idx"]] - gold[prefix + "_top"]).max(initial=0.0),
            np.abs(a[strided_idx(a.size)] - gold[prefix + "_strided"]).max(initial=0.0))
    return d / max(float(gold[prefix + "_inf"]), 1e-30)


def load_golden(name):
    """tests/golden/refbuild_<name>.npz as a dict (what the reference build computed on the same inputs)."""
    with np.load(os.path.join(GOLDEN_DIR, f"refbuild_{name}.npz")) as z:
        return {k: z[k] for k in z.files}


def assert_digests(gold, got):
    """Every digest_<field> of `gold` must match the array got[field]."""
    for k in gold:
        if k.startswith("digest_"):
            field = k[len("digest_"):]
            assert np.array_equal(digest(got[field]), gold[k]), f"{field} not bit-identical to the reference build"


def scene_kwargs(sc, use_sh=True, use_cov_precomp=False, sh_degree=3, cov3D=None, scale_modifier=1.0):
    kw = dict(means3D=sc.means3D, opacities=sc.opacities, viewmatrix=sc.viewmatrix, projmatrix=sc.projmatrix,
              campos=sc.campos, W=sc.width, H=sc.height, tanfovx=sc.tanfovx, tanfovy=sc.tanfovy, sh_degree=sh_degree,
              scale_modifier=scale_modifier)
    if use_sh:
        kw["shs"] = sc.shs
    else:
        kw["colors_precomp"] = sc.colors_precomp
    if use_cov_precomp:
        kw["cov3D_precomp"] = cov3D
    else:
        kw["scales"] = sc.scales
        kw["rotations"] = sc.rotations
    return kw


ALPHA_MIN = np.float32(1) / np.float32(255)   # the blend's threshold 1.0f / 255.0f: the one o with o * 255 == 1 in fp32
EDGE_OPACITIES = [0.3, ALPHA_MIN, np.nextafter(ALPHA_MIN, np.float32(0)), np.nextafter(ALPHA_MIN, np.float32(1)), 0.05,
                  ALPHA_MIN, 0.7, np.nextafter(ALPHA_MIN, np.float32(0)), ALPHA_MIN]


def opacity_edge_scene():
    """Gaussians on the optical axis of an identity camera, 33x33 pixels: every mean projects to pixel (16, 16) exactly,
    where power == 0 and alpha == min(0.99, opacity).  Opacities 1/255 (drawn there: alpha < 1/255 is false), one ulp
    below it (never drawn), one ulp above, and ordinary values, front to back in EDGE_OPACITIES order; the farthest is
    1/255, so it decides n_contrib at the centre."""
    from sugar_b200 import scenes
    P = len(EDGE_OPACITIES)
    sc = scenes.make_scene(P, 33, 33, seed=255, camera="identity", frac_behind=0.0)
    m = np.zeros((P, 3), np.float32)
    m[:, 2] = 2.0 + 0.5 * np.arange(P)
    return sc._replace(means3D=m, opacities=np.asarray(EDGE_OPACITIES, np.float32).reshape(P, 1))


def sh_basis(d, deg):
    """Real SH basis [P,16] in float64 for unit directions d [P,3], in the reference's order and sign convention
    (forward.cu:20-71 / backward.cu:20-139); zero beyond degree `deg`."""
    C0, C1 = 0.28209479177387814, 0.4886025119029199
    C2 = (1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396)
    C3 = (-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658,
          1.445305721320277, -0.5900435899266435)
    x, y, z = d[:, 0], d[:, 1], d[:, 2]
    b = np.zeros((d.shape[0], 16))
    b[:, 0] = C0
    if deg > 0:
        b[:, 1], b[:, 2], b[:, 3] = -C1 * y, C1 * z, -C1 * x
    if deg > 1:
        xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
        b[:, 4], b[:, 5], b[:, 6] = C2[0] * xy, C2[1] * yz, C2[2] * (2 * zz - xx - yy)
        b[:, 7], b[:, 8] = C2[3] * xz, C2[4] * (xx - yy)
    if deg > 2:
        b[:, 9], b[:, 10] = C3[0] * y * (3 * xx - yy), C3[1] * xy * z
        b[:, 11], b[:, 12] = C3[2] * y * (4 * zz - xx - yy), C3[3] * z * (2 * zz - 3 * xx - 3 * yy)
        b[:, 13], b[:, 14] = C3[4] * x * (4 * zz - xx - yy), C3[5] * z * (xx - yy)
        b[:, 15] = C3[6] * x * (xx - 3 * yy)
    return b


def run_oracle(sc, bg, dL=None, **opts):
    from oracle import raster_oracle as ro
    kw = scene_kwargs(sc, **opts)
    fw = ro.forward(bg=bg, **kw)
    bw = ro.backward(fw, dL) if dL is not None else None
    return fw, bw


def have_ref():
    return os.path.exists(os.path.join(REF_DIR, "diff_gaussian_rasterization", "_C.so"))


def load_ref_module():
    """Import the reference build under its own name without shadowing ours."""
    if "diff_gaussian_rasterization_ref" in sys.modules:
        return sys.modules["diff_gaussian_rasterization_ref"]
    import torch  # noqa: F401  (the extension links libtorch)
    spec = importlib.util.spec_from_file_location(
        "diff_gaussian_rasterization_ref", os.path.join(REF_DIR, "diff_gaussian_rasterization", "__init__.py"),
        submodule_search_locations=[os.path.join(REF_DIR, "diff_gaussian_rasterization")])
    mod = importlib.util.module_from_spec(spec)
    sys.modules["diff_gaussian_rasterization_ref"] = mod
    spec.loader.exec_module(mod)
    return mod


def to_torch(sc, device="cuda"):
    import torch
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(device)
    return {k: t(getattr(sc, k)) for k in ("means3D", "scales", "rotations", "opacities", "shs", "colors_precomp",
                                           "viewmatrix", "projmatrix", "campos")}


PACKED_MAX_P = 1 << 24   # SGR_PACKED_MAX_P (sgr_internal.cuh): the instance lists of P >= 2^24 Gaussians hold plain ids


def pad_culled(t, names, pad_to=PACKED_MAX_P):
    """The per-Gaussian tensors t[name] (names as in to_torch) with culled Gaussians appended up to pad_to rows, built
    on their device.  The padding's means sit at the camera centre, at view depth 0, so preprocess culls them at the
    near plane; they have finite scales, identity rotations, opacity and colour 0.5 and zero SH rows."""
    import torch
    P = t["means3D"].shape[0]
    fill = dict(means3D=t["campos"].reshape(3), scales=0.01, rotations=torch.tensor([1.0, 0.0, 0.0, 0.0]),
                opacities=0.5, colors_precomp=0.5, shs=0.0)
    out = {}
    for k in names:
        row = torch.as_tensor(fill[k], dtype=t[k].dtype).to(t[k].device)
        out[k] = torch.cat([t[k], row.expand((pad_to - P,) + t[k].shape[1:])])
    return out


def run_module(mod, sc, bg, dL=None, use_sh=True, use_cov_precomp=False, sh_degree=3, cov3D=None, device="cuda",
               debug=False, pad_to=None, scale_modifier=1.0):
    """Run GaussianRasterizer of `mod` (ours or the reference build).  Returns dict with image, radii, grads and
    the saved opaque buffers.  pad_to: the Gaussians of `sc` followed by culled ones up to pad_to (pad_culled)."""
    import torch
    t = to_torch(sc, device)
    if pad_to:
        t.update(pad_culled(t, ["means3D", "opacities", "shs" if use_sh else "colors_precomp", "scales", "rotations"],
                            pad_to))
    leaf = lambda x: x.detach().requires_grad_(True)   # to_torch and pad_culled made fresh tensors
    means3D = leaf(t["means3D"]); opac = leaf(t["opacities"])
    means2D = torch.zeros_like(means3D, requires_grad=True)
    settings = mod.GaussianRasterizationSettings(
        image_height=sc.height, image_width=sc.width, tanfovx=sc.tanfovx, tanfovy=sc.tanfovy,
        bg=torch.from_numpy(np.asarray(bg, np.float32)).to(device), scale_modifier=scale_modifier,
        viewmatrix=t["viewmatrix"], projmatrix=t["projmatrix"], sh_degree=sh_degree, campos=t["campos"],
        prefiltered=False, debug=debug)
    rast = mod.GaussianRasterizer(raster_settings=settings)
    kw = {}
    leaves = dict(means3D=means3D, means2D=means2D, opacities=opac)
    if use_sh:
        leaves["shs"] = kw["shs"] = leaf(t["shs"])
    else:
        leaves["colors_precomp"] = kw["colors_precomp"] = leaf(t["colors_precomp"])
    if use_cov_precomp:
        leaves["cov3D_precomp"] = kw["cov3D_precomp"] = leaf(torch.from_numpy(cov3D).to(device))
    else:
        leaves["scales"] = kw["scales"] = leaf(t["scales"])
        leaves["rotations"] = kw["rotations"] = leaf(t["rotations"])
    color, radii = rast(means3D=means3D, means2D=means2D, opacities=opac, **kw)
    out = dict(color=color.detach(), radii=radii.detach())
    fn = color.grad_fn
    saved = fn.saved_tensors if fn is not None else None
    if saved is not None:
        out["geom"], out["binning"], out["img"] = saved[7], saved[8], saved[9]
        out["num_rendered"] = fn.num_rendered
    if dL is not None:
        (color * torch.from_numpy(dL).to(device)).sum().backward()
        out["grads"] = {k: v.grad.detach() for k, v in leaves.items() if v.grad is not None}
    return out


PER_GAUSSIAN = ("radii", "depths", "means2D", "conic_opacity", "rgb", "clamped", "tiles_touched")


def run_state(sc, bg, dL=None, plain_ids=False, pad_to=PACKED_MAX_P, **opts):
    """`sc` through ours, as numpy arrays: the forward state (_C.inspect_state), num_rendered, radii and color of a
    forward-only run, and with an upstream gradient dL the image (color_bw) and gradients (grad_<name>) of a
    forward + backward run.  plain_ids: culled Gaussians are appended up to pad_to (pad_culled), so that the library
    lists plain ids, as it does for any cloud that large.  The padded rows must have radius 0, no tiles and zero
    gradients; every per-Gaussian array is returned for the Gaussians of `sc` alone (the visible ids, and so the
    lists, do not change)."""
    import torch
    from sugar_b200 import _C, diff_gaussian_rasterization as ours
    P, W, H = sc.means3D.shape[0], sc.width, sc.height
    pad = pad_to if plain_ids else None

    def rows(k, v):
        if plain_ids and (k in ("radii", "tiles_touched") or k.startswith("grad_")):
            assert not v[P:].any(), f"{k}: a padded Gaussian is not culled"
        return (v[:P] if k in PER_GAUSSIAN or k.startswith("grad_") else v).cpu().numpy()
    a = run_module(ours, sc, bg, None, pad_to=pad, **opts)
    st = _C.inspect_state(pad or P, W, H, a["num_rendered"], a["geom"], a["binning"], a["img"])
    out = {k: rows(k, v) for k, v in dict(st, radii=a["radii"], color=a["color"]).items()}
    out["num_rendered"] = np.int64(a["num_rendered"])
    del a, st
    if dL is not None:
        b = run_module(ours, sc, bg, dL, pad_to=pad, **opts)
        out.update({"grad_" + k: rows("grad_" + k, v) for k, v in b["grads"].items()})
        out["color_bw"] = b["color"].cpu().numpy()
        del b
    if plain_ids:
        torch.cuda.empty_cache()
    return out


def decode_ref_state(out, P, W, H):
    """Decode the reference's GeometryState / BinningState / ImageState chunks
    (rasterizer_impl.cu:155-194: 128-byte aligned bump allocation, in this order)."""
    import torch
    R = out["num_rendered"]

    def carve(buf, specs):
        base = buf.data_ptr()
        off = 0
        res = {}
        for name, dtype, count in specs:
            addr = (base + off + 127) & ~127
            off = addr - base
            nbytes = count * torch.empty((), dtype=dtype).element_size()
            res[name] = buf[off:off + nbytes].view(dtype)
            off += nbytes
        return res
    g = carve(out["geom"], [("depths", torch.float32, P), ("clamped", torch.uint8, 3 * P),
                            ("internal_radii", torch.int32, P), ("means2D", torch.float32, 2 * P),
                            ("cov3D", torch.float32, 6 * P), ("conic_opacity", torch.float32, 4 * P),
                            ("rgb", torch.float32, 3 * P), ("tiles_touched", torch.int32, P)])
    b = carve(out["binning"], [("point_list", torch.int32, R), ("point_list_unsorted", torch.int32, R),
                               ("keys", torch.int64, R)])
    i = carve(out["img"], [("final_T", torch.float32, W * H), ("n_contrib", torch.int32, W * H),
                           ("ranges", torch.int32, 2 * W * H)])
    T = ((W + 15) // 16) * ((H + 15) // 16)
    return dict(depths=g["depths"], clamped=g["clamped"].view(P, 3), means2D=g["means2D"].view(P, 2),
                cov3D=g["cov3D"].view(P, 6), conic_opacity=g["conic_opacity"].view(P, 4), rgb=g["rgb"].view(P, 3),
                tiles_touched=g["tiles_touched"], point_list=b["point_list"], keys=b["keys"],
                final_T=i["final_T"].view(H, W), n_contrib=i["n_contrib"].view(H, W),
                ranges=i["ranges"][:2 * T].view(T, 2))


def rel_err(a, b):
    """|a-b|_inf / |b|_inf (per-tensor relative error, SURVEY section 7 'hard parts')."""
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    d = np.abs(a - b).max() if a.size else 0.0
    return d / max(np.abs(b).max() if b.size else 0.0, 1e-30)


def row_errors(got, want, bound, rows=None):
    """Row-wise comparison of [P, C] arrays (one row per Gaussian): per row the largest |got - want| / bound over its
    components (a nonzero difference against a zero bound, and any non-finite `got` or difference, count as
    infinite, so a NaN fails the check).  rows: bool [P], the rows compared (default all).  Returns
    dict(ratio_rows [P] (0 outside `rows`), ratio (the largest), worst_row, worst_col, n_over (rows with ratio > 1)).
    Unlike rel_err, a row far below the tensor's largest is held to its own bound."""
    got = np.asarray(got, np.float64).reshape(len(got), -1)
    want = np.asarray(want, np.float64).reshape(got.shape)
    bound = np.asarray(bound, np.float64).reshape(got.shape)
    d = np.abs(got - want)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(d == 0, 0.0, d / bound)
    r[~np.isfinite(got) | ~np.isfinite(r)] = np.inf
    if rows is not None:
        r[~np.asarray(rows, bool)] = 0.0
    per_row = r.max(1) if r.size else np.zeros(len(got))
    worst = int(np.argmax(per_row)) if per_row.size else 0
    return dict(ratio_rows=per_row, ratio=float(per_row[worst]) if per_row.size else 0.0, worst_row=worst,
                worst_col=int(np.argmax(r[worst])) if r.size else 0, n_over=int((per_row > 1.0).sum()))


def grad_sensitivity(sc, bg, dL, eps=1e-6, **opts):
    """Conditioning probe for the per-Gaussian backward chain (CPU oracle): relative change (|.|_inf / |g|_inf)
    of each returned gradient when the blend accumulators dL_dmeans2D / dL_dconic are perturbed by `eps`
    relative noise, i.e. by what fp32 summation order alone does to them.  For surface-aligned Gaussians
    with a 1e-6 axis, eps = 1e-6 moves dL_drotations by ~1e-4: there a fixed 1e-4 bar measures the
    conditioning of the reference's formula, not the implementation."""
    import ctypes as C
    from oracle import raster_oracle as ro
    fw, bw = run_oracle(sc, np.asarray(bg, np.float32), dL, **opts)
    L, i, _p = ro.lib(), fw["_in"], ro._p
    P, W, H, M, D = fw["P"], fw["W"], fw["H"], fw["M"], fw["D"]
    cov3Ds = i["cov3D_precomp"] if i["cov3D_precomp"] is not None else fw["cov3D"]

    def chain(dm2d, dconic):
        g = dict(means3D=np.zeros((P, 3), np.float32), cov3D_precomp=np.zeros((P, 6), np.float32),
                 shs=np.zeros((P, max(M, 1), 3), np.float32), scales=np.zeros((P, 3), np.float32),
                 rotations=np.zeros((P, 4), np.float32))
        L.oracle_preprocess_backward(
            C.c_int(P), C.c_int(D), C.c_int(M), _p(i["means3D"]), _p(fw["radii"]), _p(i["shs"]), _p(fw["clamped"]),
            _p(i["scales"]), _p(i["rotations"]), C.c_float(i["scale_modifier"]), _p(cov3Ds), _p(i["viewmatrix"]),
            _p(i["projmatrix"]), C.c_int(W), C.c_int(H), C.c_float(i["tanfovx"]), C.c_float(i["tanfovy"]),
            _p(i["campos"]), _p(dm2d), _p(dconic), _p(bw["dL_dcolors"].copy()), _p(g["means3D"]), _p(g["cov3D_precomp"]),
            _p(g["shs"]), _p(g["scales"]), _p(g["rotations"]))
        return g
    base = chain(bw["dL_dmeans2D"].copy(), bw["dL_dconic"].copy())
    rng = np.random.default_rng(0)
    noisy = lambda a: (a * (1 + eps * rng.standard_normal(a.shape))).astype(np.float32)
    pert = chain(noisy(bw["dL_dmeans2D"]), noisy(bw["dL_dconic"]))
    return {k: float(np.abs(pert[k] - base[k]).max() / max(np.abs(base[k]).max(), 1e-30)) for k in base}


def check_linear_properties(run, W, H, tol_img=1e-5, tol_grad=1e-4):
    """Size-independent invariants of the rasterizer, for any implementation behind
    run(bg, dL) -> (color f32[3,H,W], radii, {name: grad} or None), all numpy:
      * the background enters as  image(bg) = image(0) + final_T * bg  with one final_T for the three channels
        (forward.cu:361-367), and radii do not depend on it;
      * the backward is linear in the upstream image gradient.
    The CPU suite runs it on the oracle (small), the GPU suite on the CUDA path at the headline size."""
    from sugar_b200 import scenes
    c0, r0, _ = run((0.0, 0.0, 0.0), None)
    c1, r1, _ = run((1.0, 1.0, 1.0), None)
    T = c1 - c0
    assert np.abs(T[0] - T[1]).max() <= tol_img and np.abs(T[0] - T[2]).max() <= tol_img
    assert T.min() >= -tol_img and T.max() <= 1.0 + tol_img
    bg2 = np.array([0.25, 0.5, 1.0], np.float32)
    c2, r2, _ = run(tuple(float(v) for v in bg2), None)
    assert np.abs(c2 - (c0 + T[0][None] * bg2[:, None, None])).max() <= 2 * tol_img
    assert np.array_equal(r0, r1) and np.array_equal(r0, r2)
    d1, d2 = scenes.upstream_grad(W, H, seed=1), scenes.upstream_grad(W, H, seed=2)
    a, b = 0.75, -1.5
    g1, g2 = run((0.0, 0.0, 0.0), d1)[2], run((0.0, 0.0, 0.0), d2)[2]
    g12 = run((0.0, 0.0, 0.0), (a * d1 + b * d2).astype(np.float32))[2]
    assert set(g1) == set(g12) and len(g12) >= 5
    for k in g12:
        err = rel_err(g12[k], a * g1[k] + b * g2[k])
        assert err <= tol_grad, f"backward not linear in dL for {k}: {err:.2e}"
