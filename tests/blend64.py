"""Float64 pair-level reference of the blend backward, with an error bound per Gaussian and component.

TEST INFRASTRUCTURE ONLY.  `oracle/raster_oracle.c` restates the reference's fp32 arithmetic in the reference's order;
this module restates the same operation in float64 and says, for every Gaussian and accumulator component, how far a
correct fp32 kernel may land from it.  The tests then hold each Gaussian to a bound of its own instead of holding a
whole tensor to a fraction of its largest entry, which hides every row far below the largest one.

Inputs are the forward's fp32 state (bit-identical between ours, the oracle and the reference): means2D,
conic_opacity, colours, point_list, ranges, n_contrib, final_T, plus bg and the upstream image gradient.  The discrete
decisions come from that state and are not re-decided in float64: a pair counts when its list position is below the
pixel's n_contrib, its fp32 power is <= 0 and its fp32 alpha = min(0.99, o * exp(power)) is >= 1/255.  A pair whose
fp32 alpha lies within AMBIG_ULPS of 1/255 (at power != 0, where exp is not exact) may be decided either way by two
correct expf implementations; its Gaussian, and every Gaussian in front of it at that pixel (their T and colour
behind depend on the decision), are excluded.

Per pair, in float64: G, alpha, T (recovered from final_T by division, back to front, as the kernels do), the colour
blended behind (accum_rec), dL/dalpha with the background term (backward.cu's form) and the accumulator
contributions, in the layout of the GPU's per-Gaussian record:
    0 dL/dmean2D.x   1 dL/dmean2D.y   (with the 0.5 W, 0.5 H factor)
    2 dL/dconic a    3 dL/dconic b    4 dL/dconic c   (b as the reference stores it: -0.5 G dx dy dL/dG)
    5 dL/dopacity    6-8 dL/dcolour r g b (masked by the SH clamp bits when given)    9 dL/dvalue (feature channel)
Their signed sums per Gaussian are the reference value.

The bound E (units of U = 2^-24, the fp32 unit roundoff; first order) has two parts.  A worst-case bound (every
rounding of every term adding up with one sign) cannot be tight here: the geometric gradients of a Gaussian cancel
over its footprint, sum|term| / |sum| is 50-2000 for the Gaussians the per-tensor bar hides, so u sum|term| alone is
already near 1e-4 of them.  The roundings of different pixels are independent, so E adds them in quadrature:
  * E_pair, the rounding of each pair's term: C_PAIR U of the term's magnitude (the same expression on absolute
    values, dL/dalpha as T sum(|c| + |accum_rec|) |dL/dpixel| + the background term), and per splat behind it the
    division that recovers T, U (1 + 2 alpha / (1 - alpha)), summed back to front.  The oracle's sums are exact (it
    accumulates in double), so it must agree with the reference within E_pair alone (plus one rounding of the result).
  * E_sum, the summation order of a kernel that sums in fp32: a Gaussian's pairs are reduced over a block's pixels
    (D_BLOCK roundings deep, including the moment shift, whose magnitudes are |ax| + |cx| >= |dx| about a half-block
    centre) and then across its blocks by one fp32 atomic per block it touches.
E = SAFETY (E_pair + E_sum), SAFETY set from the measured ratios (below).
"""
import numpy as np

U = 2.0 ** -24
ALPHA_MIN = np.float32(1) / np.float32(255)
ALPHA_MAX = float(np.float32(0.99))
AMBIG_ULPS = 4
# C_PAIR: the roundings of one pair's chain (dx, power, the exp2 approximation, alpha, the products and fmas of the
# terms), 8; C_POWER: G's relative rounding per unit of |power| on absolute values (the power's three roundings and
# its scaling into exp2), 4.  D_BLOCK: the 16-pixel moment chains, the shift and the half-block shuffle of chunk_flush.
C_PAIR, C_POWER, D_BLOCK = 8.0, 4.0, 24.0
# SAFETY: with SAFETY = 1, the largest |oracle - ref| / E_pair over every Gaussian and component of the CPU scenes
# (test_blend64_cpu.py) is 0.57 (mid_tiles colours), and on an H100 the largest |gpu - ref| / E over every scene of
# test_gpu_grad_rows.py is 1.6 (lone_warp; 0.55 of E with SAFETY = 3).  E adds independent roundings in quadrature,
# so a correct kernel's error is a sum of many random-signed roundings: over ~10^5 Gaussians per scene the largest
# reaches ~4-5 standard deviations, which is what the quadrature sum approximates.  3 is about twice the largest
# measured ratio, and still leaves E below 1e-4 of the row for most of the rows the per-tensor bar hides.
SAFETY = 3.0
NAMES = ("mean2D_x", "mean2D_y", "conic_a", "conic_b", "conic_c", "opacity", "color_r", "color_g", "color_b", "value")
GROUPS = dict(means2D=(0, 1), conic=(2, 3, 4), opacity=(5,), colors=(6, 7, 8), values=(9,))


def _rev_cumsum(a, exclusive=False):
    c = np.flip(np.cumsum(np.flip(a, axis=-1), axis=-1), axis=-1)
    if exclusive:
        c = np.concatenate([c[..., 1:], np.zeros_like(c[..., :1])], axis=-1)
    return c


def _fma32(a, b, c):
    """fmaf(a, b, c) for fp32 arrays: the exact product in double, one double sum, rounded to fp32 (double rounding
    can differ from a single rounding only on exact ties of the double sum)."""
    return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(np.float32)


LY, LX = np.divmod(np.arange(256), 16)   # pixel offsets of a 16x16 tile, row-major (8x4 block = LY // 4 * 2 + LX // 8)


def tile_pairs(st, t):
    """The fp32 decisions of tile t: dict(ids [n] (the first n = max n_contrib list entries), px, py, inside [256],
    nc [256], p32 [256, n] (fp32 power), alpha32 [256, n] (fp32 alpha), V [256, n] (contributing pairs), amb [256, n]
    (ambiguous pairs)), or None for a tile without contributions."""
    H, W = st["final_T"].shape
    gx = (W + 15) // 16
    lo, hi = (int(x) for x in np.asarray(st["ranges"]).view(np.uint32).reshape(-1, 2)[t])
    if hi <= lo:
        return None
    ty, tx = divmod(int(t), gx)
    px, py = 16 * tx + LX, 16 * ty + LY
    inside = (px < W) & (py < H)
    pxc, pyc = np.minimum(px, W - 1), np.minimum(py, H - 1)
    nc = np.where(inside, np.asarray(st["n_contrib"]).view(np.uint32).astype(np.int64)[pyc, pxc], 0)
    n = int(nc.max())
    if n == 0:
        return None
    ids = np.asarray(st["point_list"]).view(np.uint32).astype(np.int64)[lo:lo + n]
    m = np.asarray(st["means2D"], np.float32)[ids]
    co = np.asarray(st["conic_opacity"], np.float32)[ids]
    # as the forward decided (ref_power: fma(fma(dx, dx*a, dy*(dy*c)), -0.5, -(dy*(dx*b))))
    dx32 = m[None, :, 0] - px[:, None].astype(np.float32)
    dy32 = m[None, :, 1] - py[:, None].astype(np.float32)
    q = _fma32(dx32, dx32 * co[:, 0], dy32 * (dy32 * co[:, 2]))
    p32 = _fma32(q, np.float32(-0.5), -(dy32 * (dx32 * co[:, 1])))
    cand = (np.arange(n)[None, :] < nc[:, None]) & ~(p32 > 0)
    a32 = np.minimum(np.float32(0.99), (co[:, 3] * np.exp(p32.astype(np.float64))).astype(np.float32))
    amb = cand & (np.abs(a32.astype(np.float64) - float(ALPHA_MIN)) <= AMBIG_ULPS * float(np.spacing(ALPHA_MIN))) \
        & (p32 != 0)
    return dict(ids=ids, px=px, py=py, pxc=pxc, pyc=pyc, inside=inside, nc=nc, p32=p32, alpha32=a32,
                V=cand & (a32 >= ALPHA_MIN), amb=amb, tx=tx, ty=ty)


def blend_backward64(st, bg, dL_dpix, colors, clamped=None, values=None, feat_bg=0.0, dL_dfeat=None, tiles=None):
    """st: the forward state (means2D [P,2], conic_opacity [P,4], point_list [R], ranges [T,2], n_contrib [H,W],
    final_T [H,W]), fp32/int arrays as _C.inspect_state or the oracle return them.  colors [P,3] (rgb or precomp),
    clamped [P,3] (SH clamp bits; masks the colour gradient) or None, values [P] / feat_bg / dL_dfeat [H,W] for the
    feature channel.  tiles: the tiles to walk (default all); a Gaussian's sums are complete only if every tile it is
    binned to is walked.

    Returns dict(ref [P,C], e_pair [P,C], e_sum [P,C], bound [P,C] = SAFETY (e_pair + e_sum), mag [P,C] (sum of the
    terms' magnitudes), touched [P] (has a contributing pair), excluded [P], n_ambiguous (pairs), n_blocks [P]).
    C = 10 with values, else 9."""
    H, W = st["final_T"].shape
    P = st["means2D"].shape[0]
    feat = values is not None
    NC = 10 if feat else 9
    means2D = np.asarray(st["means2D"], np.float32)
    co = np.asarray(st["conic_opacity"], np.float32)
    colors = np.asarray(colors, np.float32)
    ranges = np.asarray(st["ranges"]).view(np.uint32).reshape(-1, 2)
    finT = np.asarray(st["final_T"], np.float32).astype(np.float64)
    dpix_all = np.asarray(dL_dpix, np.float32).astype(np.float64).reshape(3, H, W)
    bg = np.asarray(bg, np.float32).astype(np.float64).reshape(3)
    cmask = np.ones((P, 3)) if clamped is None else (np.asarray(clamped).reshape(P, 3) == 0).astype(np.float64)
    ref, v_pair, v_sum, mag = (np.zeros((P, NC)) for _ in range(4))
    nblk = np.zeros(P, np.int64)
    touched = np.zeros(P, bool)
    excluded = np.zeros(P, bool)
    n_amb = 0
    tiles = range(ranges.shape[0]) if tiles is None else tiles
    lx, ly = LX, LY
    hcx = (lx // 8) * 8 + 3.5                                 # centres of the 8x2 halves of the 8x4 blocks
    hcy = (ly // 4) * 4 + ((ly % 4) // 2) * 2 + 0.5
    for t in tiles:
        tp = tile_pairs(st, t)
        if tp is None:
            continue
        ids, px, py, pxc, pyc, inside, V, amb = (tp[k] for k in ("ids", "px", "py", "pxc", "pyc", "inside", "V", "amb"))
        tx, ty, n = tp["tx"], tp["ty"], len(ids)
        m = means2D[ids]
        a32, b32, c32, o32 = co[ids, 0], co[ids, 1], co[ids, 2], co[ids, 3]
        if amb.any():
            n_amb += int(amb.sum())
            kmax = np.where(amb.any(1), n - 1 - np.argmax(amb[:, ::-1], axis=1), -1)
            front = (np.arange(n)[None, :] <= kmax[:, None]) & (V | amb)
            excluded[ids[front.any(0)]] = True
        # float64 pair values
        a, b, c, o = (x.astype(np.float64) for x in (a32, b32, c32, o32))
        dx = m[None, :, 0].astype(np.float64) - px[:, None]
        dy = m[None, :, 1].astype(np.float64) - py[:, None]
        pw = -0.5 * (a * dx * dx + c * dy * dy) - b * dx * dy
        G = np.where(V, np.exp(np.minimum(pw, 0.0)), 0.0)
        oG = o * G
        al = np.where(V, np.minimum(ALPHA_MAX, oG), 0.0)
        om = 1.0 - al
        R = np.flip(np.cumprod(np.flip(om, 1), 1), 1)                 # prod_{j >= k} (1 - alpha_j)
        Rn = np.concatenate([R[:, 1:], np.ones((R.shape[0], 1))], 1)  # prod_{j > k}
        fT = np.where(inside, finT[pyc, pxc], 1.0)[:, None]          # (pixels outside the image have no pairs)
        T = fT / R                                                    # transmittance in front of pair k
        Tb = fT / Rn                                                  # ... behind it: T (1 - alpha)
        dp = np.where(inside[None], dpix_all[:, pyc, pxc], 0.0)       # [3, npix]
        col = colors[ids].astype(np.float64)                          # [n, 3]
        chans = [(col[:, ch], dp[ch]) for ch in range(3)]
        bgdp = bg @ dp
        bgdp_abs = np.abs(bg) @ np.abs(dp)
        if feat:
            dpf = np.where(inside, np.asarray(dL_dfeat, np.float32).astype(np.float64)[pyc, pxc], 0.0)
            chans.append((np.asarray(values, np.float32).astype(np.float64).reshape(-1)[ids], dpf))
            fb = float(np.float32(feat_bg))
            bgdp = bgdp + fb * dpf
            bgdp_abs = bgdp_abs + abs(fb) * np.abs(dpf)
        dLda = -fT / om * bgdp[:, None]
        DA = fT / om * bgdp_abs[:, None]                              # dL/dalpha on absolute values
        for cj, dj in chans:
            w = np.where(V, al * T * cj[None, :], 0.0)
            accum = _rev_cumsum(w, exclusive=True) / Tb               # colour blended behind pair k
            dLda = dLda + T * (cj[None, :] - accum) * dj[:, None]
            DA = DA + T * (np.abs(cj[None, :]) + np.abs(accum)) * np.abs(dj)[:, None]
        dLda = np.where(V, dLda, 0.0)
        DA = np.where(V, DA, 0.0)
        # squared relative rounding of a pair's term (units of U): the pair's own roundings, and per splat behind it
        # the division that recovers T, (1 + 2 alpha / (1 - alpha)), summed back to front
        Pabs = 0.5 * (a * dx * dx + c * dy * dy) + np.abs(b * dx * dy)   # power on absolute values: G's rounding
        rel2 = (C_PAIR + C_POWER * Pabs) ** 2 + _rev_cumsum(np.where(V, 1.0 + 2.0 * al / om, 0.0)) ** 2
        dLdG = o * dLda
        gdx, gdy = G * dx, G * dy
        terms = [dLdG * (-gdx * a - gdy * b) * (0.5 * W), dLdG * (-gdy * c - gdx * b) * (0.5 * H),
                 -0.5 * gdx * dx * dLdG, -0.5 * gdx * dy * dLdG, -0.5 * gdy * dy * dLdG, G * dLda]
        adx, ady = np.abs(dx), np.abs(dy)
        wabs = [oG * (a * adx + np.abs(b) * ady) * (0.5 * W), oG * (c * ady + np.abs(b) * adx) * (0.5 * H),
                0.5 * oG * adx * adx, 0.5 * oG * adx * ady, 0.5 * oG * ady * ady, G]
        # the same weights in the moment form about the half-block centre: |dx| <= |ax| + |cx|
        X = np.abs(m[None, :, 0].astype(np.float64) - (16 * tx + hcx)[:, None]) + np.abs(lx % 8 - 3.5)[:, None]
        Y = np.abs(m[None, :, 1].astype(np.float64) - (16 * ty + hcy)[:, None]) + 0.5
        wmom = [oG * (a * X + np.abs(b) * Y) * (0.5 * W), oG * (c * Y + np.abs(b) * X) * (0.5 * H),
                0.5 * oG * X * X, 0.5 * oG * X * Y, 0.5 * oG * Y * Y, G]
        mags = [wk * DA for wk in wabs]
        moms = [wk * DA for wk in wmom]
        for ch, (cj, dj) in enumerate(chans):
            wc = np.where(V, al * T, 0.0) * dj[:, None]
            msk = cmask[ids, ch][None, :] if ch < 3 else 1.0
            terms.append(wc * msk)
            mags.append(np.abs(wc) * msk)
            moms.append(np.abs(wc) * msk)
        for k in range(NC):
            ref[ids, k] += terms[k].sum(0)
            mag[ids, k] += mags[k].sum(0)
            v_pair[ids, k] += (mags[k] ** 2 * rel2).sum(0)
            v_sum[ids, k] += (moms[k] ** 2).sum(0)
        touched[ids] |= V.any(0)
        nblk[ids] += V.reshape(4, 4, 2, 8, n).any(axis=(1, 3)).sum(axis=(0, 1))
    e_pair = U * (np.abs(ref) + np.sqrt(v_pair))    # + the final rounding of the sum to fp32
    e_sum = U * np.sqrt((D_BLOCK + nblk)[:, None] * v_sum)
    return dict(ref=ref, e_pair=e_pair, e_sum=e_sum, bound=SAFETY * (e_pair + e_sum), mag=mag, touched=touched,
                excluded=excluded, n_ambiguous=n_amb, n_blocks=nblk)


def oracle_accumulators(bw, P):
    """The CPU oracle's blend accumulators (raster_oracle.backward) as [P, 9] in the component order above."""
    c = bw["dL_dconic"].reshape(P, 4)
    return np.concatenate([bw["dL_dmeans2D"].reshape(P, 3)[:, :2], c[:, [0, 1, 3]], bw["dL_dopacity"].reshape(P, 1),
                           bw["dL_dcolors"].reshape(P, 3)], 1).astype(np.float64)


def gpu_accumulators(gacc, dL_dcolors, dL_dvalues=None):
    """The GPU's blend record gacc [P, 8] (dmean2D x y, conic a b c, opacity, -, -) and dL_dcolors [P, 3]
    (+ dL_dvalues [P]) as [P, 9] (or [P, 10])."""
    parts = [np.asarray(gacc, np.float64)[:, :6], np.asarray(dL_dcolors, np.float64).reshape(-1, 3)]
    if dL_dvalues is not None:
        parts.append(np.asarray(dL_dvalues, np.float64).reshape(-1, 1))
    return np.concatenate(parts, 1)


def row_norms(x, ncomp=None):
    """|row|_inf of each gradient group (GROUPS), broadcast back to its components: [P, C]."""
    C = x.shape[1] if ncomp is None else ncomp
    out = np.zeros((x.shape[0], C))
    for cols in GROUPS.values():
        cols = [c for c in cols if c < C]
        if cols:
            out[:, cols] = np.abs(x[:, cols]).max(1, keepdims=True)
    return out
