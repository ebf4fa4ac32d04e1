"""The backward blend's accumulators, Gaussian by Gaussian, against the float64 blend reference (tests/blend64.py).

The suite's other gradient checks hold a tensor to |a - b|_inf / |b|_inf, which only sees the Gaussians whose gradient
is near the tensor's largest; most rows of a deep tile could be zero and pass.  Here every visible Gaussian's every
accumulator component is held to the bound E of its own: the rounding a correct fp32 kernel can make for it.

* Accumulators.  The backward runs through sgr_rasterize_backward_staged (sgr_rasterize_backward_feature with the
  feature channel) on the forward's own buffers, with a scratch buffer the test owns, so that the blend's 8-float
  record per Gaussian (dmean2D x y, conic a b c, opacity; chunk_flush in sgr_backward.cu) -- dL/dconic included, which
  no public output exposes -- can be read next to dL_dcolors (and dL_dvalues).  |gpu - ref64| <= E for every visible,
  non-excluded Gaussian and component; the rows of Gaussians without a contributing pair must be exactly zero.  A
  failure names the worst Gaussian, its ratio, its tiles with their size classes, and where it sits in each tile's walk
  (list position, walk slot, 64-record batch, 8x4 blocks, rank among the block's members and whether that falls in
  the warp's last, partial chunk of 16).
* Per-Gaussian chain.  The GPU's own accumulators and dL_dcolors go through the CPU oracle's preprocess backward, and
  the GPU's means3D / cov3D / scales / rotations / SH gradients are compared row by row with its result: both start
  from identical fp32 inputs, so what is left is the per-Gaussian arithmetic.  The bar of a row is
  max(CHAIN_RTOL |row|_inf, 5 x the row's sensitivity to 1e-6 relative noise on the accumulators), which keeps the
  1e-6 scale axis of mesh_bound honest without loosening the other rows.
* Scenes.  Every test_gpu_parity.CASES scene (packed ids), every test_gpu_blend_backward_overlap scene and the walk
  boundaries below (both id formats: packed ids with masks, and plain ids, P padded to 2^24 with culled Gaussians),
  the feature channel, and the C2 configuration (100k Gaussians, 800x800, SH degree 2) whole.
"""
import ctypes as C

import numpy as np
import pytest

import blend64 as b64
import helpers as h
import test_gpu_blend_backward_overlap as ov
import test_gpu_parity as tp

pytestmark = pytest.mark.gpu

BWD_B, CH = 64, 16     # records per batch and splats per chunk of the backward blend (sgr_backward.cu)
# per-row bar of the chain comparison (module docstring).  Largest |gpu - oracle chain| / |row| measured on an H100
# over every scene here: means3D 1.1e-5, cov3D 3.7e-5, sh 6e-7; scales 4.4e-4 and rotations 7.1e-5 (mesh_bound,
# coplanar: the scale / rotation chain cancels, beyond what 1e-6 noise on the accumulators shows); raw-parameter mode:
# densities 1.4e-4 (held by its sensitivity), scales 5.5e-5, rotations 6.0e-5, sh_rest 6e-7
CHAIN_RTOL = dict(means3D=1e-4, cov3D=1e-4, sh=1e-4, scales=1e-3, rotations=1e-3, opacity=1e-4, sh_rest=1e-4)
MAX_EXCLUDED = 0.01    # at most this fraction of the visible Gaussians may be excluded as ambiguous (and 3)


# ---------------------------------------------------------------------------------------------------------------------
# running the op with the test's own buffers
def _forward(sc, bg, use_sh=False, sh_degree=0, use_cov_precomp=False, cov3D=None, pad_to=None, values=None,
             feat_bg=None):
    import torch
    from sugar_b200 import _C
    t = h.to_torch(sc)
    names = ["means3D", "opacities", "shs" if use_sh else "colors_precomp", "scales", "rotations"]
    if pad_to:
        t.update(h.pad_culled(t, names, pad_to))
    Pt = t["means3D"].shape[0]
    if use_cov_precomp:
        t["cov3D_precomp"] = torch.from_numpy(cov3D).cuda()
    vals = None
    if values is not None:
        vals = torch.zeros(Pt, dtype=torch.float32, device="cuda")
        vals[:len(values)] = torch.from_numpy(np.asarray(values, np.float32)).cuda()
    bgt = torch.tensor(bg, dtype=torch.float32, device="cuda")
    fbg = None if feat_bg is None else torch.tensor([feat_bg], dtype=torch.float32, device="cuda")
    e = torch.empty(0, device="cuda")
    sh = t["shs"] if use_sh else e
    colors = e if use_sh else t["colors_precomp"]
    scales, rots = (e, e) if use_cov_precomp else (t["scales"], t["rotations"])
    cov = t["cov3D_precomp"] if use_cov_precomp else e
    args = (bgt, t["means3D"], colors, t["opacities"], scales, rots, 1.0, cov, t["viewmatrix"], t["projmatrix"],
            sc.tanfovx, sc.tanfovy, sc.height, sc.width, sh, sh_degree, t["campos"], False, False)
    out = _C.rasterize_gaussians(*args, values=vals, feature_bg=fbg)
    R, color, radii, geom, binning, img = out[:6]
    st = _C.inspect_state(Pt, sc.width, sc.height, R, geom, binning, img)
    return dict(t=t, R=R, radii=radii, geom=geom, binning=binning, img=img, args=args, vals=vals, fbg=fbg,
                st={k: v.cpu().numpy() for k, v in st.items()}, Pt=Pt, M=sh.size(1) if use_sh else 0,
                sh_degree=sh_degree)


def scratch_accumulators(b, P):
    """The blend accumulators [P, 8] in the scratch of _C._alloc_backward's buffers `b`, after a backward."""
    base = b["scratch"].data_ptr()
    off = ((base + 255) // 256 * 256 - base) // 4           # launch_backward: gacc = align_up(scratch, SGR_ALIGN)
    return b["scratch"][off:off + 8 * P].view(P, 8)


def _backward(f, dL, dD=None, sh_rest=None):
    """The backward on f's forward buffers, through the C entry point, with the test's scratch: (grads, gacc [P,8]).
    sh_rest: raw-parameter mode (sugar_b200/fused.py), the plan carries the second SH gradient array."""
    import torch
    from sugar_b200 import _C, _lib
    (bgt, means3D, colors, _o, scales, rots, smod, cov, vm, pm, tfx, tfy, H, W, sh, deg, campos, _p, _d) = f["args"]
    Pt, M = f["Pt"], f["M"]
    raw = sh_rest is not None
    b = _C._alloc_backward(Pt, M, means3D.device, with_records=False, split_sh=raw)
    dLt = torch.from_numpy(np.ascontiguousarray(dL, np.float32)).cuda()
    view = _C._view_struct(bgt, smod, vm, pm, tfx, tfy, H, W, deg, campos, False, False)
    g = _C._gauss_struct(Pt, M, means3D, None, sh, colors, scales, rots, cov, sh_rest)
    inputs = (C.byref(view), C.byref(g), f["radii"].data_ptr(), f["geom"].data_ptr(), f["binning"].data_ptr(),
              f["img"].data_ptr(), int(f["R"]), dLt.data_ptr())
    grads = (b["means2D"].data_ptr(), b["colors"].data_ptr(), b["opacity"].data_ptr(), b["means3D"].data_ptr(),
             b["cov3D"].data_ptr(), b["sh"].data_ptr() if M else None, b["scales"].data_ptr(),
             b["rotations"].data_ptr())
    stream = torch.cuda.current_stream().cuda_stream
    dval = None
    if dD is not None:
        dval = torch.empty(Pt, dtype=torch.float32, device="cuda")
        dDt = torch.from_numpy(np.ascontiguousarray(dD, np.float32)).cuda()
        _lib.check(_lib.lib.sgr_rasterize_backward_feature(*inputs, f["vals"].data_ptr(), f["fbg"].data_ptr(),
                                                           dDt.data_ptr(), *grads, dval.data_ptr(),
                                                           b["scratch"].data_ptr(), stream))
    else:
        plan = _lib.SgrBackwardPlan(num_chunks=1, dL_dsh_rest=b["sh_rest"].data_ptr() if M > 1 else None) \
            if raw else None
        _lib.check(_lib.lib.sgr_rasterize_backward_staged(*inputs, *grads, b["scratch"].data_ptr(), stream,
                                                          None if plan is None else C.byref(plan)))
    torch.cuda.synchronize()
    gacc = scratch_accumulators(b, Pt)
    out = {k: b[k].cpu().numpy() for k in ("means2D", "colors", "opacity", "means3D", "cov3D", "scales", "rotations")}
    if M:
        out["sh"] = b["sh"].cpu().numpy()
    if raw:
        out["sh_rest"] = b["sh_rest"].cpu().numpy()
    if dval is not None:
        out["values"] = dval.cpu().numpy()
    return out, gacc.cpu().numpy()


# ---------------------------------------------------------------------------------------------------------------------
# where a Gaussian sits in the walk, for failure messages
def _size_class(c):
    return "<=512" if c <= 512 else "<=2048" if c <= 2048 else "<=8192" if c <= 8192 else ">8192"


def locate(st, gid):
    """Human-readable place of Gaussian gid in every tile walk it is part of."""
    H, W = st["final_T"].shape
    gx = (W + 15) // 16
    pl = st["point_list"].view(np.uint32).astype(np.int64)
    keys = st["keys"].view(np.uint64)
    rng = st["ranges"].view(np.uint32).astype(np.int64)
    nc = st["n_contrib"].view(np.uint32).astype(np.int64)
    fp = st["footprint"]
    out = []
    for k in np.flatnonzero(pl == gid)[:4]:
        t = int(keys[k] >> np.uint64(32))
        lo, hi = rng[t]
        ty, tx = divmod(t, gx)
        tile_nc = nc[16 * ty:16 * ty + 16, 16 * tx:16 * tx + 16]
        n_full = int(tile_nc.max())
        live = fp[lo:hi] != 0
        pos, lpos, n_live = int(k - lo), int(live[:k - lo].sum()), int(live[:n_full].sum())
        slot = n_live - 1 - lpos
        s = (f"tile {t} ({tx},{ty}) of {hi - lo} instances [{_size_class(hi - lo)}]: list position {pos} "
             f"(live {lpos} of {n_live} walked), walk slot {slot}, batch {slot // BWD_B}")
        blocks = []
        tp = b64.tile_pairs(st, t)
        blk_of = (b64.LY // 4) * 2 + b64.LX // 8
        for blk in range(8):
            if not (int(fp[k]) >> blk) & 1:
                continue
            # the members that take a chunk slot: those with a contributing pair in the block, in walk order (back to
            # front); a member without one is skipped by the warp
            contrib = tp["V"][blk_of == blk].any(0) if tp is not None else np.zeros(0, bool)
            mem = [p for p in range(len(contrib) - 1, -1, -1) if contrib[p]]
            if pos in mem:
                r, total = mem.index(pos), len(mem)
                blocks.append(f"block {blk}: contributing member {r} of {total} (chunk {r // CH}"
                              f"{', the last, partial one' if total % CH and r >= total - total % CH else ''})")
            else:
                blocks.append(f"block {blk}: member without a contributing pair")
        out.append(s + "; " + "; ".join(blocks))
    return " | ".join(out)


# ---------------------------------------------------------------------------------------------------------------------
# the checks
def check_accumulators(label, st, got, r):
    """|got - ref64| <= E per Gaussian and component (got: [P, C] as blend64.gpu_accumulators); returns the report."""
    ok = r["touched"] & ~r["excluded"]
    nvis = int(r["touched"].sum())
    nex = int(r["excluded"].sum())
    assert nex <= max(3, MAX_EXCLUDED * nvis), f"{label}: {nex} of {nvis} Gaussians excluded as ambiguous"
    idle = ~r["touched"] & ~r["excluded"]
    bad_idle = np.flatnonzero((got[idle] != 0).any(1))
    assert bad_idle.size == 0, (f"{label}: {bad_idle.size} Gaussians without a contributing pair have nonzero "
                                f"accumulators, e.g. {np.flatnonzero(idle)[bad_idle[0]]}")
    err = h.row_errors(got, r["ref"], r["bound"], rows=ok)
    ratio, g, k = err["ratio"], err["worst_row"], err["worst_col"]
    if ratio > 1.0:
        pytest.fail(f"{label}: Gaussian {g} component {b64.NAMES[k]}: gpu {got[g, k]:.9g} ref64 {r['ref'][g, k]:.9g} "
                    f"|d| / E = {ratio:.3g} (E {r['bound'][g, k]:.3g}); {err['n_over']} Gaussians over; "
                    f"{locate(st, g)}")
    return dict(ratio=float(ratio), excluded=nex, visible=nvis, ambiguous_pairs=int(r["n_ambiguous"]))


def _check_record_copies(label, gacc, grads, P, opacity_factor=None):
    """The public dL_dmeans2D and dL_dopacity are the blend record's values, copied (raw mode: dL_dopacity times
    o (1 - o) in fp32, the activated opacity o as the forward stored it)."""
    m2d = grads["means2D"][:P]
    assert np.array_equal(m2d[:, :2], gacc[:, :2]) and not m2d[:, 2].any(), f"{label}: dL_dmeans2D != the record's"
    want = gacc[:, 5] if opacity_factor is None else gacc[:, 5] * opacity_factor
    assert np.array_equal(grads["opacity"][:P, 0], want), f"{label}: dL_dopacity != the record's"


def _oracle_chain(fw, dm2d, dconic, dcol):
    from oracle import raster_oracle as ro
    L, i, _p = ro.lib(), fw["_in"], ro._p
    P, W, H, M, D = fw["P"], fw["W"], fw["H"], fw["M"], fw["D"]
    cov3Ds = i["cov3D_precomp"] if i["cov3D_precomp"] is not None else fw["cov3D"]
    g = dict(means3D=np.zeros((P, 3), np.float32), cov3D=np.zeros((P, 6), np.float32),
             sh=np.zeros((P, max(M, 1), 3), np.float32), scales=np.zeros((P, 3), np.float32),
             rotations=np.zeros((P, 4), np.float32))
    L.oracle_preprocess_backward(
        C.c_int(P), C.c_int(D), C.c_int(M), _p(i["means3D"]), _p(fw["radii"]), _p(i["shs"]), _p(fw["clamped"]),
        _p(i["scales"]), _p(i["rotations"]), C.c_float(i["scale_modifier"]), _p(cov3Ds), _p(i["viewmatrix"]),
        _p(i["projmatrix"]), C.c_int(W), C.c_int(H), C.c_float(i["tanfovx"]), C.c_float(i["tanfovy"]),
        _p(i["campos"]), _p(np.ascontiguousarray(dm2d, np.float32)), _p(np.ascontiguousarray(dconic, np.float32)),
        _p(np.ascontiguousarray(dcol, np.float32)), _p(g["means3D"]), _p(g["cov3D"]), _p(g["sh"]), _p(g["scales"]),
        _p(g["rotations"]))
    return g


def _accumulator_inputs(gacc, P):
    """The record's dmean2D / dconic in the oracle's layouts ([P,3], and [P,2,2] as raster_oracle.backward passes)."""
    dm2d = np.zeros((P, 3), np.float32)
    dm2d[:, :2] = gacc[:P, :2]
    dconic = np.zeros((P, 4), np.float32)
    dconic[:, [0, 1, 3]] = gacc[:P, 2:5]
    return dm2d, dconic


def _noisy(*arrays):
    """The arrays with 1e-6 relative noise (what fp32 summation order does to the accumulators)."""
    rng = np.random.default_rng(0)
    return [(a * (1 + 1e-6 * rng.standard_normal(a.shape))).astype(np.float32) for a in arrays]


def compare_rows(label, want, pert, got, rows=None):
    """Row by row: |got - want| <= max(CHAIN_RTOL |row|_inf, 5 x the row's sensitivity |pert - want|_inf), for every
    name of `want` (dicts of [P, ...] arrays).  Returns {name: (largest |d| / bar, largest |d| / |row|)}."""
    rep, bad = {}, []
    for k in want:
        w = want[k].reshape(len(want[k]), -1).astype(np.float64)
        gk = got[k].reshape(w.shape).astype(np.float64)
        sens = np.abs(pert[k].reshape(w.shape) - w).max(1)
        bar = np.maximum(CHAIN_RTOL[k] * np.abs(w).max(1), 5.0 * sens)[:, None] * np.ones_like(w)
        err = h.row_errors(gk, w, bar, rows=rows)
        rel = np.abs(gk - w).max(1) / np.maximum(np.abs(w).max(1), 1e-30)
        if rows is not None:
            rel = rel[rows]
        rep[k] = (float(err["ratio"]), float(rel.max(initial=0.0)))
        if err["ratio"] > 1.0:
            g = err["worst_row"]
            bad.append(f"{k}: Gaussian {g} |d|/bar {err['ratio']:.3g} (|d| {np.abs(gk[g] - w[g]).max():.3g}, "
                       f"|row| {np.abs(w[g]).max():.3g}, sensitivity {sens[g]:.3g}); {err['n_over']} rows over")
    assert not bad, f"{label} chain: " + "; ".join(bad)
    return rep


def check_chain(label, fw, gacc, grads, use_sh, covpre):
    """The GPU's per-Gaussian gradients against the oracle's chain fed with the GPU's own accumulators, row by row."""
    P = fw["P"]
    dm2d, dconic = _accumulator_inputs(gacc, P)
    dcol = grads["colors"][:P]
    base = _oracle_chain(fw, dm2d, dconic, dcol)
    pert = _oracle_chain(fw, *_noisy(dm2d, dconic), dcol)
    names = ["means3D", "cov3D"] + (["sh"] if use_sh else []) + ([] if covpre else ["scales", "rotations"])
    return compare_rows(label, {k: base[k] for k in names}, {k: pert[k] for k in names},
                        {k: grads[k][:P] for k in names})


def run_scene(label, sc, bg, plain_ids=False, use_sh=False, sh_degree=0, use_cov_precomp=False, cov3D=None,
              values=None, feat_bg=None, dD=None, chain=True, shape_check=None):
    from sugar_b200 import scenes
    P, W, H = sc.means3D.shape[0], sc.width, sc.height
    dL = scenes.upstream_grad(W, H)
    opts = dict(use_sh=use_sh, sh_degree=sh_degree, use_cov_precomp=use_cov_precomp, cov3D=cov3D)
    f = _forward(sc, bg, pad_to=h.PACKED_MAX_P if plain_ids else None, values=values, feat_bg=feat_bg, **opts)
    grads, gacc = _backward(f, dL, dD)
    st = dict(f["st"])
    for k in h.PER_GAUSSIAN:                                # the scene's Gaussians (padding is culled)
        if k in st:
            st[k] = st[k][:P]
    if plain_ids:
        assert not f["radii"][P:].any() and not gacc[P:].any() and not grads["colors"][P:].any()
    if shape_check is not None and not plain_ids:
        shape_check(st)
    colors = st["rgb"] if use_sh else sc.colors_precomp
    r = b64.blend_backward64(st, bg, dL, colors, clamped=st["clamped"] if use_sh else None, values=values,
                             feat_bg=feat_bg or 0.0, dL_dfeat=dD)
    _check_record_copies(label, gacc[:P], grads, P)
    got = b64.gpu_accumulators(gacc[:P], grads["colors"][:P], None if dD is None else grads["values"][:P])
    rep = check_accumulators(label, st, got, r)
    if chain and dD is None:
        fw, _ = h.run_oracle(sc, np.asarray(bg, np.float32), None, **opts)
        assert np.array_equal(fw["radii"], f["radii"][:P].cpu().numpy())
        rep["chain"] = check_chain(label, fw, gacc, grads, use_sh, use_cov_precomp)
    print(f"\n[grad_rows] {label}: {rep}")
    return rep


# ---------------------------------------------------------------------------------------------------------------------
# walk boundaries that no other scene pins (identity camera, axis-aligned splats; test_gpu_blend_backward_overlap)
def _splats_in_block0(n, seed, op, dz=0.01, spread=(1.5, 0.5)):
    rng = np.random.Generator(np.random.PCG64(seed))
    return [(3.5 + rng.uniform(-spread[0], spread[0]), 1.5 + rng.uniform(-spread[1], spread[1]), 2.0 + dz * i, 0.6,
             0.6, op) for i in range(n)]


def _block_members(st, tile, blk):
    """Gaussians with a contributing pair in 8x4 block `blk` of `tile`, and the tile's pair decisions."""
    tp = b64.tile_pairs(st, tile)
    inblk = (b64.LY // 4) * 2 + b64.LX // 8 == blk
    return tp["ids"][tp["V"][inblk].any(0)], tp


def _shape_members(n):
    def check(st):
        ids, _ = _block_members(st, 0, 0)
        assert len(ids) == n, (len(ids), n)
    return check


def _shape_walk(n):
    def check(st):
        nc = st["n_contrib"].view(np.uint32)
        assert int(nc[0:4, 0:8].max()) == n and int(nc[:16, :16].max()) == n
        lo = int(st["ranges"].view(np.uint32)[0, 0])
        assert np.all(st["footprint"][lo:lo + n] & 1), "the walked records are block-0 members"
    return check


def _shape_lone_warp(st):
    lo, hi = (int(x) for x in st["ranges"].view(np.uint32)[0])
    assert hi - lo > CH and np.all(st["footprint"][lo:hi] == 1 << 5), st["footprint"][lo:hi]


def _shape_second_half(st):
    _, tp = _block_members(st, 0, 0)
    g = int(np.flatnonzero(tp["ids"] == 19)[0])             # the probe, the farthest splat
    blk0 = (b64.LY // 4) * 2 + b64.LX // 8 == 0
    vrows = set(b64.LY[blk0][tp["V"][blk0][:, g]].tolist())
    assert vrows == {2, 3}, vrows


def _shape_far(st):
    ids, tp = _block_members(st, 0, 0)
    m = st["means2D"][ids]
    assert (np.abs(m[:, 0] - 3.5) > 64).any(), m


def _shape_edge(st):
    H, W = st["final_T"].shape
    assert W % 16 and H % 16
    gx, gy = (W + 15) // 16, (H + 15) // 16
    tp = b64.tile_pairs(st, gx * gy - 1)
    assert tp is not None and tp["V"][tp["inside"]].any() and (tp["px"][tp["V"].any(1)] == W - 1).any()


def _shape_early_stop(st):
    tp = b64.tile_pairs(st, 0)
    n = len(tp["ids"])
    nc, fT = tp["nc"], st["final_T"][tp["pyc"], tp["pxc"]]
    # pixels that stopped because the next contributing splat would take T below 1e-4, in the middle of a batch
    stop = []
    for p in np.flatnonzero(tp["inside"] & (nc < n)):
        nxt = np.flatnonzero((tp["p32"][p, nc[p]:] <= 0) & (tp["alpha32"][p, nc[p]:] >= b64.ALPHA_MIN))
        if nxt.size and fT[p] * (1 - tp["alpha32"][p, nc[p] + nxt[0]]) < 1e-4 and (n - nc[p]) % BWD_B:
            stop.append(p)
    assert stop, "no pixel terminates early inside a batch"


def _shape_threshold(st):
    tp = b64.tile_pairs(st, 0)
    near = tp["V"] & ~tp["amb"] & (np.abs(tp["alpha32"] - b64.ALPHA_MIN) < 1e-5 * b64.ALPHA_MIN) & (tp["p32"] != 0)
    assert near.sum() >= 2, int(near.sum())


def _threshold_scene():
    """Splats whose fp32 alpha at the pixel right of their centre is 1/255 x (1 + d), |d| <= 8e-6 (so the backward's
    exact-expf fix-up decides them), at power != 0; opacities tuned on the CPU oracle's forward (bit-identical)."""
    splats = [(2.5 + 3 * (i % 2), 1.5 + (i // 2) * 0.0, 2.0 + 0.1 * i, 0.7, 0.7, 0.5) for i in range(4)]
    sc = ov._scene(16, 16, splats, seed=11)
    fw, _ = h.run_oracle(sc, np.zeros(3, np.float32), None, use_sh=False)
    op = sc.opacities.copy()
    for i, d in enumerate((3e-6, -3e-6, 6e-6, 8e-6)):
        mx, my = fw["means2D"][i].astype(np.float64)
        a, b, c = fw["conic_opacity"][i, :3].astype(np.float64)
        dx, dy = mx - (np.floor(mx + 0.5) + 1), my - np.floor(my + 0.5)
        pw = -0.5 * (a * dx * dx + c * dy * dy) - b * dx * dy
        op[i, 0] = np.float32(float(h.ALPHA_MIN) * (1 + d) / np.exp(pw))
    return sc._replace(opacities=op)


def _early_stop_splats():
    sp = _splats_in_block0(150, 21, 0.03)
    for i in range(40, 45):                                 # opaque, narrow, on pixel (2, 1): T < 1e-4 there at ~43
        sp[i] = (2.0, 1.0, sp[i][2], 0.7, 0.7, 0.97)
    return sp


BOUNDARY = {
    # contributing members of block 0: a full chunk, a full chunk plus one, a partial chunk only
    "members_16": (lambda: ov._scene(16, 16, _splats_in_block0(16, 1, 0.2), 16), _shape_members(16)),
    "members_17": (lambda: ov._scene(16, 16, _splats_in_block0(17, 2, 0.2), 17), _shape_members(17)),
    "members_15": (lambda: ov._scene(16, 16, _splats_in_block0(15, 3, 0.2), 15), _shape_members(15)),
    # a block walk of exactly 256 records (four full stages) and of 257 (the pipeline wraps)
    "walk_256": (lambda: ov._scene(16, 16, _splats_in_block0(256, 4, 0.02), 256), _shape_walk(256)),
    "walk_257": (lambda: ov._scene(16, 16, _splats_in_block0(257, 5, 0.02), 257), _shape_walk(257)),
    # only warp 5 (pixels 8-15 x 8-11) has members; its seven siblings idle through the whole pipeline
    "lone_warp": (lambda: ov._scene(16, 16, [(11.5, 9.5, 2.0 + 0.01 * i, 0.3, 0.3, 0.3) for i in range(40)], 40),
                  _shape_lone_warp),
    # the farthest splat contributes to rows 2-3 of block 0 only: the second half's moment shift alone
    "second_half": (lambda: ov._scene(16, 16, _splats_in_block0(20, 6, 0.2, spread=(1.5, 0.2))[:-1]
                                      + [(4.3, 3.0, 3.0, 0.55, 0.3, 0.3)], 20), _shape_second_half),
    # a wide splat centred ~7 tiles right of block 0 contributes there: |ax| ~ 115 in the moment shift
    "far_centre": (lambda: ov._scene(128, 16, [(2.0, 1.5, 2.0, 0.6, 0.6, 0.3), (118.5, 1.7, 3.0, 40.0, 0.8, 0.99),
                                               (5.0, 2.0, 4.0, 0.6, 0.6, 0.4)], 3), _shape_far),
    # tiles on the right / bottom edge of a 37x21 image
    "edge_tiles": (lambda: ov._scene(37, 21, [(36.0, 20.0, 2.0, 1.5, 1.5, 0.6), (33.5, 18.0, 2.5, 2.0, 1.0, 0.5),
                                              (30.0, 20.5, 3.0, 3.0, 3.0, 0.4), (36.5, 10.0, 3.5, 1.0, 4.0, 0.5)], 4),
                   _shape_edge),
    # pixels that reach T < 1e-4 in the middle of a 64-record batch, next to pixels that walk on
    "early_stop": (lambda: ov._scene(16, 16, _early_stop_splats(), 150), _shape_early_stop),
    # fp32 alpha within 1e-5 of 1/255 at power != 0: the exact-expf fix-up decides
    "alpha_threshold": (_threshold_scene, _shape_threshold),
}
BG = (0.25, 0.5, 1.0)


@pytest.mark.parametrize("unpacked", [False, True], ids=["packed_ids", "unpacked_ids"])
@pytest.mark.parametrize("name", list(BOUNDARY))
def test_walk_boundaries(name, unpacked):
    make, shape = BOUNDARY[name]
    run_scene(f"{name}/{'plain' if unpacked else 'packed'}", make(), BG, plain_ids=unpacked, shape_check=shape)


@pytest.mark.parametrize("unpacked", [False, True], ids=["packed_ids", "unpacked_ids"])
@pytest.mark.parametrize("name", list(ov.SCENES))
def test_overlap_scenes(name, unpacked):
    run_scene(f"{name}/{'plain' if unpacked else 'packed'}", ov._make(name), BG, plain_ids=unpacked,
              shape_check=lambda st: ov._check_shape(name, st))


@pytest.mark.parametrize("case", tp.CASES, ids=[c[0] for c in tp.CASES])
def test_parity_scenes(case):
    name, P, W, H, camera, use_sh, deg, covpre, bg = case
    sc = tp._scene(name, P, W, H, camera)
    cov3D = tp._cov_from_oracle(sc) if covpre else None
    run_scene(name, sc, bg, use_sh=use_sh, sh_degree=deg, use_cov_precomp=covpre, cov3D=cov3D)


@pytest.mark.parametrize("use_sh", [False, True], ids=["colors", "sh3"])
def test_feature_channel(use_sh):
    """The colour + depth blend (depth.rasterize_with_depth's entry point): dL/dvalues and the four-channel sums."""
    from sugar_b200 import scenes
    P, W, H = 4000, 200, 120
    sc = scenes.make_scene(P, W, H, seed=31, camera="posed")
    z = (sc.means3D @ sc.viewmatrix[:3, :3] + sc.viewmatrix[3, :3])[:, 2].astype(np.float32)
    dD = scenes.upstream_grad(W, H, seed=5)[0]
    run_scene(f"feature/{'sh3' if use_sh else 'colors'}", sc, (0.1, 0.2, 0.3), use_sh=use_sh,
              sh_degree=3 if use_sh else 0, values=z, feat_bg=float(z.max()), dD=dD)


def test_c2_config():
    """C2 (100k Gaussians, 800x800, SH degree 2): every Gaussian."""
    case = tp.ORACLE_CASES[-1]
    name, P, W, H, camera, use_sh, deg, covpre, bg = case
    run_scene(name, tp._scene(name, P, W, H, camera), bg, use_sh=use_sh, sh_degree=deg)


def _dnormvdv(v, dv):
    """d normalize(v) / dv applied to dv (auxiliary.h's dnormvdv, float64): (I - v v^T / |v|^2) dv / |v|."""
    n2 = (v * v).sum(1, keepdims=True)
    return (n2 * dv - (v * dv).sum(1, keepdims=True) * v) / n2 ** 1.5


def test_raw_parameter_mode():
    """Raw-parameter mode (fused.py: logit opacities, log scales, un-normalised quaternions, SH in (dc, rest) arrays):
    the same blend accumulators against ref64, and the raw chain's rows against the activated chain (the oracle's,
    fed with the GPU's accumulators, on the activations evaluated in float64) taken through the activations'
    derivatives in float64: d sigmoid = o (1 - o), d exp = scale, normalisation as dnormvdv."""
    from sugar_b200 import scenes
    W, H = 200, 120
    run_raw_mode("raw", scenes.make_scene(4000, W, H, seed=12, camera="posed"), (0.1, 0.2, 0.3),
                 scenes.upstream_grad(W, H, seed=3))


def run_raw_mode(label, sc, bg, dL, deg=3):
    """test_raw_parameter_mode's checks on the scene `sc` (SH of degree `deg`, 16 coefficients)."""
    import torch
    from sugar_b200 import _C
    P, W, H, M = sc.means3D.shape[0], sc.width, sc.height, 16
    t = h.to_torch(sc)
    dens = torch.logit(t["opacities"].clamp(1e-4, 1 - 1e-4)).contiguous()
    s_raw = t["scales"].log().contiguous()
    q_raw = (t["rotations"] * 1.7).contiguous()
    sh_dc, sh_rest = t["shs"][:, :1].contiguous(), t["shs"][:, 1:].contiguous()
    e = torch.empty(0, device="cuda")
    args = (torch.tensor(bg, dtype=torch.float32, device="cuda"), t["means3D"], e, dens, s_raw, q_raw, 1.0, e,
            t["viewmatrix"], t["projmatrix"], sc.tanfovx, sc.tanfovy, H, W, sh_dc, deg, t["campos"], False, False)
    R, _color, radii, geom, binning, img = _C.rasterize_gaussians(*args, sh_rest=sh_rest)
    st = {k: v.cpu().numpy() for k, v in _C.inspect_state(P, W, H, R, geom, binning, img).items()}
    f = dict(args=args, Pt=P, M=M, R=R, radii=radii, geom=geom, binning=binning, img=img)
    grads, gacc = _backward(f, dL, sh_rest=sh_rest)
    o32 = st["conic_opacity"][:, 3]
    _check_record_copies(label, gacc, grads, P, opacity_factor=o32 * (np.float32(1) - o32))
    r = b64.blend_backward64(st, bg, dL, st["rgb"], clamped=st["clamped"])
    rep = check_accumulators(label, st, b64.gpu_accumulators(gacc, grads["colors"]), r)

    # the activated counterpart, in float64, as the oracle's inputs
    d64, s64, q64 = (x.double().cpu().numpy() for x in (dens, s_raw, q_raw))
    op64, sc64 = 1.0 / (1.0 + np.exp(-d64)), np.exp(s64)
    qn64 = q64 / np.linalg.norm(q64, axis=1, keepdims=True)
    act = sc._replace(opacities=op64.astype(np.float32), scales=sc64.astype(np.float32), rotations=qn64.astype(np.float32))
    fw, _ = h.run_oracle(act, np.asarray(bg, np.float32), None, use_sh=True, sh_degree=deg)
    rad = radii.cpu().numpy()
    same = fw["radii"] == rad                               # a last-ulp activation can move a radius across an integer
    assert same.mean() > 0.999, same.mean()
    fw["clamped"] = st["clamped"].astype(np.uint8)          # the SH clamp bits of the GPU's colours
    dm2d, dconic = _accumulator_inputs(gacc, P)

    def raw_chain(dm2d, dconic, dopa, op):
        a = _oracle_chain(fw, dm2d, dconic, grads["colors"])
        return dict(means3D=a["means3D"].astype(np.float64), opacity=(dopa * op[:, 0] * (1 - op[:, 0]))[:, None],
                    scales=a["scales"] * sc64, rotations=_dnormvdv(q64, a["rotations"].astype(np.float64)),
                    sh=a["sh"][:, :1], sh_rest=a["sh"][:, 1:])
    want = raw_chain(dm2d, dconic, gacc[:, 5].astype(np.float64), op64)
    # the sensitivity also moves the activated opacity by one fp32 ulp, as the kernel's fp32 sigmoid may: near o = 1,
    # o (1 - o) is ill-conditioned (1 - o loses the digits of o)
    nm, nc, no = _noisy(dm2d, dconic, gacc[:, 5])
    pert = raw_chain(nm, nc, no.astype(np.float64), op64 * (1 + 2.0 ** -23))
    rows = same & (rad > 0)
    rep["chain"] = compare_rows(label, want, pert, {k: grads[k] for k in want}, rows=rows)
    assert not any(grads[k][rad == 0].any() for k in want), "a culled Gaussian has raw gradients"
    print(f"\n[grad_rows] {label}: {rep}")
    return rep
