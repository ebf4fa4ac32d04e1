"""Poisson mesh of the coarse model's level-set points (csrc/sgr_poisson.cu).

The reference's default extraction branch (sugar_extractors/coarse_mesh.py:228-490) collects level-set points with
normals and colours over the training views, splits them into a foreground and a background box, removes statistical
outliers with open3d, runs open3d's `create_from_point_cloud_poisson(pcd, depth=10)` on each part, drops the vertices
below the 0.1 quantile of Poisson density, then decimates, cleans and merges.  Here, without open3d:

    cloud = surface_point_cloud(points, scaling, quaternions, strengths, sh_dc, cameras)      # composition only
    mesh = extract_mesh_poisson(cloud["points"], cloud["colors"], cloud["normals"], spatial_extent)
    mcubes.write_ply(path, **mesh["combined"])

The discrete problem (oracle/poisson_oracle.py restates it in float64; the kernels follow it):
  * Domain: the samples' bounding box, largest side B; the cube of side L = 1.1 B centred on the box's centre
    (open3d's scale 1.1, width 0).  N = 2^depth nodes per axis at cell centres, x_i = o + (i + 0.5) h, h = L / N,
    depth in [5, 10].  A sample's grid coordinates are g = (p - o) * inv_h - 0.5 in float32 (o and inv_h = N / L
    rounded to float32, each operation rounded once).
  * Basis: phi_i, the trilinear hat of node i, in grid units.
  * Area per sample: a = (number of occupied cells) / n for every sample, a cell being the cube between eight nodes
    that holds the sample's hat support (a uniform-density stand-in for the density-based sample weights of SPR).
  * System: sum_{j in N6(i)} (u_i - u_j) + q_i u_i = b_i with b_i = -a sum_s n_s . grad phi_i(p_s) (the weak divergence
    of the splatted normal field) and q_i = alpha a sum_s phi_i(p_s) (the screening term lumped to the diagonal),
    missing neighbours at the cube's faces dropped (zero flux).  u grows towards the inside: it approximates the
    inside indicator up to the screening's shift.  alpha = point_weight = 4 is the point weight of the Screened Poisson
    paper and PoissonRecon's documented default; what open3d passes was not checked.
  * Iso-value: the mean over the samples of the trilinear interpolation of u; the surface is
    mcubes.marching_cubes(u, iso) (inside where u > iso, normals pointing out), mapped to world by o + (v + 0.5) h.
  * Vertex density (open3d's second return value, used only for the trim): sum_s phi_i(p_s) splatted on the grid of
    depth - 2, interpolated trilinearly at the vertex, plus 2^-20 / (1 + (d / h)^2) with d the vertex's distance to
    its nearest sample (knn.knn_points, K = 1).  The splat alone is 0 at every vertex farther than the depth - 2 hats
    reach (4 h per axis) from the samples, and on an open surface the part Poisson closes beyond that holds more than a
    tenth of the vertices, so the 0.1 quantile would be 0 and `densities < quantile` would remove nothing; the distance
    term keeps the density positive and falling with the distance, so the trim removes the farthest vertices first, as
    it does with open3d's densities.  Near the samples the splat (at least about one sample's worth) dominates.
    Because the grid is dense, the closing surface is meshed at full resolution (open3d's octree meshes it coarsely,
    with few vertices), so on an open surface the 0.1 quantile removes its farthest part, not all of it.
  * Vertex colour: sum_s phi_i(p_s) c_s and sum_s phi_i(p_s) splatted at full depth, each interpolated at the vertex,
    then divided; where the denominator is 0, the nearest sample's colour (knn.knn_points, K = 1).

Deliberate differences from open3d (PoissonRecon):
  * a dense regular grid instead of an adaptive octree: the same finest resolution, at the cost of memory, not of
    accuracy near the samples;
  * degree-1 hats and a 7-point stiffness instead of PoissonRecon's B-splines;
  * uniform sample areas;
  * lumped screening;
  * density and colour as defined above.
Away from the samples the surface therefore differs from open3d's; that is the region the density trim removes.  The
output was not compared with open3d's.

Solver: geometric multigrid V(2,2) cycles with red-black Gauss-Seidel down to a 4^3 grid, until
|b - A u|_2 / |b|_2 <= 1e-5, at most 30 cycles; otherwise RuntimeError.  One host read per cycle.  Every grid is
computed without float atomics, so a reconstruction is bit-identical from run to run.

Memory (bytes, G = 4 N^3 for one float32 grid): the bin starts (G), b, q and u (3 G), the multigrid levels below the
finest (3 G / 7) and 16 n of binned samples, so about 4.43 G + 16 n at the solve (18 GiB at depth 10 with 10M
samples), plus 28 n bytes of sort scratch while the binning runs; b, q and the levels are freed before marching
cubes, and the density and colour grids are splatted one at a time into one grid after u is freed.
"""
import ctypes as C

import numpy as np
import torch

from ._lib import check, lib, require_cuda, stream, tensor

RED_BLOCKS = 1024          # partial sums of the library's fixed-order reductions
TOLERANCE = 1e-5
MAX_CYCLES = 30
SYSTEM, WEIGHT, ATTRIBUTE = 0, 1, 2
DENSITY_FALLOFF = 2.0 ** -20   # the vertex density's distance term at a sample (in hat weights, i.e. samples)


def domain(points, depth):
    """-> (o float64[3], h, o32 float32[3], inv_h32): the grid's origin corner and spacing for `points` [n,3]."""
    lo = points.min(dim=0).values.double().cpu().numpy()
    hi = points.max(dim=0).values.double().cpu().numpy()
    B = float((hi - lo).max())
    if not B > 0.0 or not np.isfinite(B):
        raise ValueError(f"the samples' bounding box must have a positive finite largest side, got {B}")
    N = 1 << depth
    L = 1.1 * B
    o = 0.5 * (lo + hi) - 0.5 * L
    return o, L / N, o.astype(np.float32), np.float32(N / L)


def _bin(points, depth, o32, inv_h32):
    """-> (starts int32 [N^3], binned float32 [n,4], occupied bins): the samples sorted by bin, each bin in sample
    order (sgr_poisson_bin)."""
    n, N = points.shape[0], 1 << depth
    dev = points.device
    starts = torch.empty(N ** 3, dtype=torch.int32, device=dev)
    binned = torch.empty((n, 4), dtype=torch.float32, device=dev)
    keys = torch.empty(2 * n, dtype=torch.int32, device=dev)
    records = torch.empty((n, 4), dtype=torch.float32, device=dev)
    tiles = (n + 255) // 256
    hist = torch.empty(256 * tiles, dtype=torch.int32, device=dev)
    sums = torch.empty((max(N ** 3, 256 * tiles) + 4095) // 4096 + 1, dtype=torch.int32, device=dev)
    occ = C.c_int64(0)
    check(lib.sgr_poisson_bin(n, points.data_ptr(), N, float(o32[0]), float(o32[1]), float(o32[2]), float(inv_h32),
                              starts.data_ptr(), binned.data_ptr(), keys.data_ptr(), records.data_ptr(),
                              hist.data_ptr(), sums.data_ptr(), C.byref(occ), stream(dev)))
    return starts, binned, int(occ.value)


def _splat(N, starts, binned, mode, attr=None, channel=0, area=0.0, alpha=0.0):
    dev = starts.device
    out0 = torch.empty((N, N, N), dtype=torch.float32, device=dev)
    out1 = torch.empty((N, N, N), dtype=torch.float32, device=dev) if mode == SYSTEM else None
    check(lib.sgr_poisson_splat(N, binned.shape[0], starts.data_ptr(), binned.data_ptr(), mode,
                                None if attr is None else attr.data_ptr(), channel, float(area), float(alpha),
                                out0.data_ptr(), None if out1 is None else out1.data_ptr(), stream(dev)))
    return out0 if out1 is None else (out0, out1)


def _interpolate(grid, pts, stride, scale=1.0, offset=0.0, values=True, want_sum=False):
    dev = grid.device
    m = pts.shape[0]
    if m == 0 and not want_sum:
        return torch.zeros(0, dtype=torch.float32, device=dev), 0.0
    vals = torch.empty(m, dtype=torch.float32, device=dev) if values else None
    partial = torch.empty(RED_BLOCKS, dtype=torch.float64, device=dev)
    s = C.c_double(0.0)
    check(lib.sgr_poisson_interpolate(grid.shape[0], grid.data_ptr(), m, pts.data_ptr() if m else None, stride,
                                      float(scale), float(offset), None if vals is None else vals.data_ptr(),
                                      partial.data_ptr(), C.byref(s) if want_sum else None, stream(dev)))
    return vals, s.value


def _check_samples(points, normals, colors):
    require_cuda("poisson", points, normals, colors)
    points = tensor(points, "points", torch.float32, ("n", 3))
    n = points.shape[0]
    if n == 0:
        raise ValueError("points is empty: nothing to reconstruct")
    if n >= 2 ** 31:
        raise ValueError(f"{n} samples: at most 2^31 - 1")
    dev = points.device
    normals = tensor(normals, "normals", torch.float32, (n, 3), dev, "points")
    if colors is not None:
        colors = tensor(colors, "colors", torch.float32, (n, 3), dev, "points")
    return points, normals, colors


class _Timer:
    """CUDA events around named stages on the current stream (scripts/bench_poisson.py); inert when not enabled."""

    def __init__(self, enabled):
        self.enabled, self.marks = enabled, []

    def mark(self, name):
        if self.enabled:
            e = torch.cuda.Event(enable_timing=True)
            e.record()
            self.marks.append((name, e))

    def stages(self):
        torch.cuda.synchronize()
        return [(self.marks[i][0], self.marks[i - 1][1].elapsed_time(self.marks[i][1]))
                for i in range(1, len(self.marks))]


def solve(points, normals, depth=10, point_weight=4.0, _timer=None):
    """The screened system of `points` / `normals` (float32 CUDA [n,3]) at `depth` and its solution:
    -> {"u" [N,N,N], "b", "q", "iso", "cycles", "residual", "area", "o", "h", "o32", "inv_h32", "binned", "starts"}.
    b and q are returned for tests; extract_mesh_poisson drops them before marching cubes."""
    t = _timer or _Timer(False)
    if not isinstance(depth, int) or not 5 <= depth <= 10:
        raise ValueError(f"depth must be an int in [5, 10], got {depth!r}")
    points, normals, _ = _check_samples(points, normals, None)
    dev = points.device
    with torch.cuda.device(dev):
        if not bool(torch.isfinite(normals).all()) or bool((normals.abs().amax(dim=1) == 0).any()):
            raise ValueError("normals must be finite and non-zero")
        o, h, o32, inv_h32 = domain(points, depth)
        N, n = 1 << depth, points.shape[0]
        t.mark("start")
        starts, binned, occupied = _bin(points, depth, o32, inv_h32)
        t.mark("binning")
        area = occupied / n
        b, q = _splat(N, starts, binned, SYSTEM, normals, area=area, alpha=point_weight)
        t.mark("splat")
        levels = depth - 1
        us = [torch.zeros((N, N, N), dtype=torch.float32, device=dev)]
        bs, qs = [b], [q]
        for l in range(1, levels):
            M = N >> l
            us.append(torch.empty((M, M, M), dtype=torch.float32, device=dev))
            bs.append(torch.empty((M, M, M), dtype=torch.float32, device=dev))
            qs.append(torch.empty((M, M, M), dtype=torch.float32, device=dev))
            check(lib.sgr_poisson_coarsen(M * 2, qs[l - 1].data_ptr(), qs[l].data_ptr(), stream(dev)))
        partial = torch.empty(RED_BLOCKS, dtype=torch.float64, device=dev)
        bnorm = C.c_double(0.0)
        check(lib.sgr_poisson_residual_norm(N, 1.0, None, b.data_ptr(), q.data_ptr(), partial.data_ptr(),
                                            C.byref(bnorm), stream(dev)))
        if not bnorm.value > 0.0:
            raise ValueError("the normals' splatted divergence is zero everywhere: no surface to reconstruct")
        t.mark("pyramid")
        arr = lambda ts: (C.c_void_p * levels)(*[x.data_ptr() for x in ts])
        ua, ba, qa = arr(us), arr(bs), arr(qs)
        rnorm = C.c_double(0.0)
        ratio, cycles = 1.0, 0
        while cycles < MAX_CYCLES and ratio > TOLERANCE:
            check(lib.sgr_poisson_vcycle(depth, ua, ba, qa, partial.data_ptr(), C.byref(rnorm), stream(dev)))
            cycles += 1
            ratio = rnorm.value / bnorm.value
            t.mark(f"vcycle {cycles}")
        if not ratio <= TOLERANCE:
            raise RuntimeError(f"poisson: |b - Au| / |b| = {ratio:.3e} after {cycles} V-cycles (tolerance "
                               f"{TOLERANCE:g})")
        u = us[0]
        del us, bs, qs, ua, ba, qa
        _, total = _interpolate(u, binned, 4, values=False, want_sum=True)
        t.mark("iso-value")
    return {"u": u, "b": b, "q": q, "iso": total / n, "cycles": cycles, "residual": ratio, "area": area, "o": o,
            "h": h, "o32": o32, "inv_h32": inv_h32, "binned": binned, "starts": starts}


def poisson_reconstruction(points, normals, depth=10, colors=None, point_weight=4.0, _timer=None):
    """open3d's create_from_point_cloud_poisson(pcd, depth) on the discrete problem of this module's docstring.
    points / normals (unit, pointing out of the surface) / colors: float32 CUDA [n,3].
    -> {"verts" float32 [V,3] (world), "faces" int64 [F,3], "colors" float32 [V,3] or None, "densities" float32 [V],
    "cycles" (V-cycles run), "residual" (the final |b - Au| / |b|)}.
    ValueError on a depth outside [5, 10], mismatched shapes, zero normals, n = 0 or a flat bounding box."""
    from .mcubes import marching_cubes
    t = _timer or _Timer(False)
    points, normals, colors = _check_samples(points, normals, colors)
    s = solve(points, normals, depth, point_weight, t)
    dev = points.device
    N, o, h = 1 << depth, s["o"], s["h"]
    with torch.cuda.device(dev):
        del s["b"], s["q"]
        vi, faces = marching_cubes(s.pop("u"), s["iso"])
        t.mark("marching cubes")
        verts = (torch.from_numpy(o).to(dev) + (vi.double() + 0.5) * h).float()
        # density on the grid of depth - 2: its node I sits at fine index 4 I + 1.5
        o2, inv_h2 = s["o32"], np.float32((N >> 2) / (N * h))
        starts2, binned2, _ = _bin(points, depth - 2, o2, inv_h2)
        dens_grid = _splat(N >> 2, starts2, binned2, WEIGHT)
        del starts2, binned2
        densities = _interpolate(dens_grid, vi, 3, 0.25, -0.375)[0]
        del dens_grid
        t.mark("density grid")
        V = verts.shape[0]
        if V:
            from .knn import knn_points
            d2, nearest = knn_points(verts, points, 1)
            d2, nearest = d2[:, 0], nearest[:, 0]
            densities += DENSITY_FALLOFF / (1.0 + d2 / np.float32(h * h))
        t.mark("nearest sample")
        out_colors = None
        if colors is not None:
            grid = _splat(N, s["starts"], s["binned"], WEIGHT)
            den = _interpolate(grid, vi, 3)[0]
            num = []
            for ch in range(3):
                check(lib.sgr_poisson_splat(N, points.shape[0], s["starts"].data_ptr(), s["binned"].data_ptr(),
                                            ATTRIBUTE, colors.data_ptr(), ch, 0.0, 0.0, grid.data_ptr(), None,
                                            stream(dev)))
                num.append(_interpolate(grid, vi, 3)[0])
            del grid
            out_colors = torch.stack(num, dim=1) / den[:, None]
            empty = den == 0
            out_colors[empty] = colors[nearest[empty]]
        t.mark("colour")
    return {"verts": verts, "faces": faces, "colors": out_colors, "densities": densities, "cycles": s["cycles"],
            "residual": s["residual"]}


def remove_statistical_outlier(points, nb_neighbors=20, std_ratio=20.0):
    """open3d's PointCloud.remove_statistical_outlier(nb_neighbors, std_ratio) -> kept indices, int64, ascending.
    Restated from open3d 0.17's published source (not checked against open3d itself): each point's value is the mean
    Euclidean distance over its K = nb_neighbors nearest points (itself included, as neighbour 0); the mean and the
    sample standard deviation (n - 1) are taken over the points whose value is > 0; a point is kept when its value is
    > 0 and strictly below mean + std_ratio * std.  With fewer than two points of value > 0, those points are kept."""
    from .knn import knn_points
    require_cuda("poisson", points)
    points = tensor(points, "points", torch.float32, ("n", 3))
    n = points.shape[0]
    if nb_neighbors < 1 or std_ratio <= 0:
        raise ValueError(f"need nb_neighbors >= 1 and std_ratio > 0, got {nb_neighbors}, {std_ratio}")
    if n == 0:
        return torch.zeros(0, dtype=torch.int64, device=points.device)
    K = min(int(nb_neighbors), n)
    d2 = knn_points(points, points, K)[0]
    avg = d2.double().sqrt().mean(dim=1)
    pos = avg > 0
    valid = avg[pos]
    if valid.numel() < 2:
        return pos.nonzero()[:, 0]
    bound = valid.mean() + std_ratio * valid.std(unbiased=True)
    return (pos & (avg < bound)).nonzero()[:, 0]


def quantile_index(V, q):
    """numpy.quantile's default (linear) method for V sorted values: -> (lo, hi, gamma) with the quantile
    s[lo] + gamma (s[hi] - s[lo]) (computed as numpy does, from the nearer end when gamma >= 0.5)."""
    virtual = q * (V - 1)
    lo = int(np.floor(virtual))
    lo = min(max(lo, 0), V - 1)
    return lo, min(lo + 1, V - 1), virtual - lo


def quantile(values, q):
    """np.quantile(values, q) (linear interpolation over all V values) by a sort, for any V (torch.quantile refuses
    more than 2^24 values).  -> a Python float, computed in float64."""
    V = values.numel()
    if V == 0:
        raise ValueError("quantile of an empty tensor")
    s = values.reshape(-1).double().sort().values
    lo, hi, g = quantile_index(V, float(q))
    a, b = float(s[lo]), float(s[hi])
    return b - (b - a) * (1.0 - g) if g >= 0.5 else a + (b - a) * g


def remove_vertices_by_mask(verts, faces, mask, colors=None, normals=None):
    """open3d's TriangleMesh.remove_vertices_by_mask: drop the masked vertices and every face that references one,
    re-index the rest in order; vertices left unreferenced stay.  -> {"verts", "faces", "colors", "normals"} (None
    where not given)."""
    V = verts.shape[0]
    mask = torch.as_tensor(mask, device=verts.device)
    if mask.dtype != torch.bool or mask.shape != (V,):
        raise ValueError(f"mask must be bool [{V}], got {mask.dtype} {tuple(mask.shape)}")
    keep = ~mask
    new_id = torch.cumsum(keep.long(), 0) - 1
    fkeep = keep[faces].all(dim=1) if faces.numel() else torch.zeros(0, dtype=torch.bool, device=verts.device)
    return {"verts": verts[keep], "faces": new_id[faces[fkeep]],
            "colors": None if colors is None else colors[keep], "normals": None if normals is None else normals[keep]}


def _part_mesh(points, colors, normals, depth, density_quantile):
    from .mcubes import vertex_normals
    keep = remove_statistical_outlier(points, nb_neighbors=20, std_ratio=20.0)
    p, c, nr = points[keep], colors[keep], normals[keep]
    m = poisson_reconstruction(p, nr, depth=depth, colors=c)
    if density_quantile > 0.0 and m["verts"].shape[0]:
        thr = quantile(m["densities"], density_quantile)
        m = remove_vertices_by_mask(m["verts"], m["faces"], m["densities"].double() < thr, m["colors"])
    return {"verts": m["verts"], "faces": m["faces"], "colors": m["colors"],
            "normals": vertex_normals(m["verts"], m["faces"])}


def extract_mesh_poisson(points, colors, normals, spatial_extent, center=None, fg_bbox_factor=1.0,
                         bg_bbox_factor=4.0, poisson_depth=10, vertices_density_quantile=0.1, decimation_target=None):
    """The reference's Poisson extraction (coarse_mesh.py:329-489) for level-set points / colours / normals (float32
    CUDA [n,3]).  `spatial_extent` is mcubes.camera_spatial_extent of the training cameras and `center` their mean
    position when the box is centred (center_bbox), else None.  The foreground holds the points strictly inside
    center +- fg_bbox_factor * extent, the background the others strictly inside center +- bg_bbox_factor * extent.
    Each non-empty part: outlier removal (20 neighbours, std ratio 20), poisson_reconstruction at `poisson_depth`,
    removal of the vertices whose density is below the `vertices_density_quantile` quantile (when > 0), then with
    `decimation_target` the quadric decimation and clean-up of mcubes.extract_mesh_marching_cubes.
    -> {"foreground", "background", "combined"} meshes (verts, faces, colors, normals); an empty part is an empty
    mesh.  ValueError when both parts are empty."""
    from .mcubes import _decimated
    require_cuda("poisson", points, colors, normals)
    points = tensor(points, "points", torch.float32, ("n", 3))
    n, dev = points.shape[0], points.device
    colors = tensor(colors, "colors", torch.float32, (n, 3), dev, "points")
    normals = tensor(normals, "normals", torch.float32, (n, 3), dev, "points")
    e = float(spatial_extent)
    c = torch.zeros(1, 3, device=dev) if center is None else torch.as_tensor(center, dtype=torch.float32,
                                                                                device=dev).reshape(1, 3)
    lo, hi = c - fg_bbox_factor * e, c + fg_bbox_factor * e
    fg = (points > lo).all(dim=-1) & (points < hi).all(dim=-1)
    bg = ((points - c).abs().max(dim=-1).values < bg_bbox_factor * e) & ~fg
    empty = lambda: {"verts": torch.zeros((0, 3), device=dev), "faces": torch.zeros((0, 3), dtype=torch.int64,
                                                                                      device=dev),
                     "colors": torch.zeros((0, 3), device=dev), "normals": torch.zeros((0, 3), device=dev)}
    if not bool(fg.any()) and not bool(bg.any()):
        raise ValueError("Both foreground and background meshes are empty: no point lies in either box")
    with torch.no_grad():
        parts = []
        for m in (fg, bg):
            if not bool(m.any()):
                parts.append(empty())
                continue
            mesh = _part_mesh(points[m], colors[m], normals[m], poisson_depth, vertices_density_quantile)
            parts.append(_decimated(mesh, decimation_target) if decimation_target is not None else mesh)
        fg_mesh, bg_mesh = parts
        comb = {k: torch.cat([fg_mesh[k], bg_mesh[k] + (fg_mesh["verts"].shape[0] if k == "faces" else 0)])
                for k in fg_mesh}
    return {"foreground": fg_mesh, "background": bg_mesh, "combined": comb}


def surface_point_cloud(points, scaling, quaternions, strengths, sh_dc, cameras, surface_level=0.3,
                        n_total_points=10_000_000, generator=None):
    """The level-set point collection of coarse_mesh.py:243-327 for one surface level: per camera (a namespace as
    levelset.level_surface_points_from_camera takes), an SH-degree-0 render clamped to [0, 1], the level-set points on
    the splatted-mesh depth (use_gaussian_depth=False, the K = 16 neighbour table built once, triangle_scale 2,
    2 n_per_frame rays), their colours from the render at their pixels, and a seeded random subset of
    n_per_frame = n_total_points // len(cameras) + 1 of them.  sh_dc [P,3] or [P,1,3]; `generator`, when given, is a
    torch.Generator on the points' device.
    -> {"points", "colors", "normals"}, float32 [m,3]."""
    from .diff_gaussian_rasterization import GaussianRasterizationSettings, GaussianRasterizer
    from .knn import reset_neighbors
    from .levelset import level_surface_points_from_camera
    dev = points.device
    n_per_frame = int(n_total_points // len(cameras)) + 1
    shs = sh_dc.reshape(-1, 1, 3).float().contiguous()
    out = {"points": [], "colors": [], "normals": []}
    knn_idx = reset_neighbors(points, K=16)[1]
    for cam in cameras:
        with torch.no_grad():
            st = GaussianRasterizationSettings(image_height=int(cam.height), image_width=int(cam.width),
                                               tanfovx=cam.tanfovx, tanfovy=cam.tanfovy, bg=torch.zeros(3, device=dev),
                                               scale_modifier=1.0, viewmatrix=cam.viewmatrix,
                                               projmatrix=cam.projmatrix, sh_degree=0, campos=cam.campos,
                                               prefiltered=False, debug=False)
            rgb = GaussianRasterizer(st)(means3D=points, means2D=torch.zeros_like(points),
                                         opacities=strengths.reshape(-1, 1), shs=shs, scales=scaling,
                                         rotations=quaternions)[0]
            rgb = rgb.clamp(min=0.0, max=1.0).permute(1, 2, 0).contiguous()
        # the normals are d density / d x by autograd: outside no_grad
        res = level_surface_points_from_camera(points, scaling, quaternions, strengths, cam,
                                               surface_levels=(surface_level,), n_surface_points=2 * n_per_frame,
                                               return_normals=True, return_pixel_idx=True, generator=generator,
                                               use_gaussian_depth=False, knn_idx=knn_idx, triangle_scale=2.0)
        r = res[surface_level]
        with torch.no_grad():
            pts = r["intersection_points"]
            idx = torch.randperm(pts.shape[0], device=dev, generator=generator)[:n_per_frame]
            out["points"].append(pts[idx])
            out["colors"].append(rgb.view(-1, 3)[r["pixel_idx"]][idx])
            out["normals"].append(r["normals"][idx].detach())
    return {k: torch.cat(v).float() if v else torch.zeros((0, 3), device=dev) for k, v in out.items()}
