"""The view-parallel exchange (sugar_b200/parallel.py; csrc/sgr_peer.cu, csrc/sgr_exchange.cu and the MULTI pass of
csrc/sgr_backward.cu) Gaussian by Gaussian, on one GPU.

test_gpu_parallel.py holds the exchange's gradients to |a - b|_inf / |b|_inf <= 1e-4 per tensor, which only sees the
Gaussians near a tensor's largest entry: a zeroed row, a 16-byte unit left out of a slice or a view summed twice passes
there whenever the Gaussian involved is a small one.  Here ViewParallel.run_backward is driven directly with the test's
own buffers (not through the autograd op), so every intermediate can be read, and every row is checked:

1. The records before the reduce (the NCCL path's `records`, the peer path's own staging array) against the CPU
   oracle's per-Gaussian chain fed with this run's own blend accumulators and SH factor, with test_gpu_grad_rows'
   per-row bar (CHAIN_RTOL, and 5 x the row's sensitivity to 1e-6 noise on the accumulators).  The opacity entry is
   the accumulator, bit for bit; the rows of Gaussians culled in this view are zero.
2. The peer reduce: every rank's sum array S equals, bit for bit, the float32 sum STAGE[0] + STAGE[1] + ... +
   STAGE[N-1] taken left to right (sgr_peer.cu sums in rank order so that every owner of a slice gives the same bits).
3. The split: dL_dmeans3D | dL_dopacity | dL_dscales | dL_drotations == float32(S x scale) (NCCL path: records x
   scale), bit for bit, every row.
4. dL_dsh against float64  scale sum_v basis(normalize(mean - campos_v)) (x) factor_v,  element by element, within the
   rounding bound DSH_C (dsh_reference); coefficients at or above (deg + 1)^2, and the rows of Gaussians no view sees,
   are exactly zero.
5. The own view's blend accumulators (test_gpu_grad_rows.check_accumulators): this guards the scratch offset that 1
   and 4 read the accumulators and factors at.

Peer mode is emulated (emulate_peers): this GPU is rank `me` of N; the other N - 1 ranks are static stand-ins whose factor
blocks and records come from plain backwards of their own views and whose flag words are preset, and this process
reduces their record slices as well.  Everything a real N-rank run executes on one rank runs: the flag waits, the MULTI
pass pulling the other views' factor blocks through the pointer table, the reduce kernel for N ranks over N staging
arrays, the split.  The NCCL path runs as a forced single rank (no collective is issued), and the factor finalize
(sgr_view_grad_finalize) is driven directly with up to 13 views.
"""
import ctypes as C
import functools

import numpy as np
import pytest

import blend64 as b64
import helpers as h
import test_gpu_grad_rows as gr

pytestmark = pytest.mark.gpu

U = 2.0 ** -24           # unit roundoff of float32
P_SCENE, W, H = 6001, 160, 96     # P not a multiple of 64: every chunk range ends in a partial CTA
BG = (0.0, 0.0, 0.0)
MIN_CULLED_HERE = 36     # Gaussians culled in the own view and seen in another one: the MULTI pass's `!vis` rows

# |computed direction - exact direction|_2 <= DIR_ERR u: sh_dir rounds mean - campos (u |d_i| each), the squared length
# (<= 3u relative, half of it through the square root, + u) and the division (u): <= 4.5u per component, relative.
DIR_ERR = 5.0
# dL_dsh bound: |gpu - ref64| <= DSH_C u sum_v scale |factor_v| (|w_k(d_v)| + B_deg), B_deg = DIR_ERR x the largest
# |grad w_k| of the degree's basis functions on the unit sphere (basis_slope): what the direction's rounding moves w_k by,
# which also covers the cancellation inside the basis polynomials (w_6, w_11 ..: rounding ~ u |grad w_k|).  The |w_k|
# term covers fl(factor x scale), the product and the summation over the views (the fma chain rounds every partial sum).
# Largest |gpu - ref64| / (u sum_v ...) measured on an H100 (80 GB HBM3, 700 W power limit): 4.3, with 16 views of
# degree 0 (no B term: the fma chain over the 16 views' terms is all there is); single views of degree 0: 2.7.
DSH_C = 8.7


def view_offset(j):
    """Camera of rank j's view relative to view 0's: (yaw, shift).  View 2 is test_gpu_parallel's third view; its
    second, (0.15, (0.3, -0.1, 0.2)), is not used here: 62 of the 4742 Gaussians it renders (1.3%) take alpha
    decisions the float64 blend reference calls ambiguous, more than check_accumulators accepts."""
    if j == 1:
        return 0.1, (0.2, -0.15, 0.1)
    if j == 2:
        return -0.2, (-0.4, 0.2, 0.5)
    rng = np.random.Generator(np.random.PCG64(100 + j))
    return float(rng.uniform(-0.3, 0.3)), tuple(float(x) for x in rng.uniform(-0.5, 0.5, 3))


def view_scene(base, j):
    from sugar_b200 import scenes
    return base if j == 0 else scenes.with_camera_offset(base, *view_offset(j))


def with_M(sc, M):
    return sc._replace(shs=np.ascontiguousarray(sc.shs[:, :M]))


# ---------------------------------------------------------------------------------------------------------------------
# the references and checks (plain numpy: tests/test_exchange_rows_cpu.py runs them on synthetic arrays)
@functools.lru_cache(maxsize=None)
def basis_slope(deg):
    """max over unit directions d and k < (deg + 1)^2 of |grad w_k(d)|_2 (the basis polynomials in R^3, float64; 0 for
    degree 0), sampled on 4096 Fibonacci-sphere directions by central differences."""
    if deg == 0:
        return 0.0
    n = 4096
    i = np.arange(n) + 0.5
    z = 1 - 2 * i / n
    r, phi = np.sqrt(1 - z * z), np.pi * (1 + 5 ** 0.5) * i
    d = np.stack([r * np.cos(phi), r * np.sin(phi), z], 1)
    used, eps = (deg + 1) ** 2, 1e-6
    g2 = np.zeros((n, 16))
    for a in range(3):
        e = np.zeros(3)
        e[a] = eps
        g2 += ((h.sh_basis(d + e, deg) - h.sh_basis(d - e, deg)) / (2 * eps)) ** 2
    return float(np.sqrt(g2[:, :used]).max() * 1.01)


def dsh_reference(means, campos, factors, deg, scale):
    """float64  scale sum_v basis(normalize(mean - campos_v)) (x) factor_v  [P, 16, 3], and the bound weights
    sum_v scale |factor_v| (|w_k(d_v)| + DIR_ERR basis_slope(deg))  [P, 16, 3] (zero at and above (deg + 1)^2)."""
    m = np.asarray(means, np.float64).reshape(-1, 3)
    P, used = len(m), (deg + 1) ** 2
    scale = float(np.float32(scale))     # as the kernels receive it
    B = DIR_ERR * basis_slope(deg)
    ref, wt = np.zeros((P, 16, 3)), np.zeros((P, 16, 3))
    for cp, f in zip(campos, factors):
        d = m - np.asarray(cp, np.float64).reshape(1, 3)
        d /= np.linalg.norm(d, axis=1, keepdims=True)
        w = h.sh_basis(d, deg)
        fs = scale * np.asarray(f, np.float64).reshape(P, 3)
        ref += w[:, :, None] * fs[:, None, :]
        wt[:, :used] += (np.abs(w[:, :used]) + B)[:, :, None] * np.abs(fs)[:, None, :]
    return ref, wt


def check_dsh(label, got, ref, wt, deg):
    """dL_dsh [P, M, 3] element by element: |got - ref| <= DSH_C u wt; zero at and above (deg + 1)^2 and on the rows no
    view sees.  Returns the largest |got - ref| / (u wt), the c the bound would need."""
    g = np.asarray(got, np.float64)
    P, M = g.shape[:2]
    used = (deg + 1) ** 2
    assert not g[:, used:].any(), f"{label}: dL_dsh coefficients at or above (deg + 1)^2 = {used} are not zero"
    unseen = ~wt.reshape(P, -1).any(1)
    bad = np.flatnonzero(unseen & (g.reshape(P, -1) != 0).any(1))
    assert bad.size == 0, f"{label}: {bad.size} Gaussians that no view sees have dL_dsh rows, e.g. {bad[0]}"
    gm, rm, wm = g.reshape(P, -1), ref[:, :M].reshape(P, -1), wt[:, :M].reshape(P, -1)
    err = h.row_errors(gm, rm, DSH_C * U * wm)
    with np.errstate(divide="ignore", invalid="ignore"):
        c = np.where(wm > 0, np.abs(gm - rm) / (U * wm), 0.0)
    if err["ratio"] > 1.0:
        i, k = err["worst_row"], err["worst_col"]
        pytest.fail(f"{label}: dL_dsh of Gaussian {i} coefficient {k // 3} channel {k % 3}: gpu {gm[i, k]:.9g} "
                    f"ref64 {rm[i, k]:.9g}, |d| / bound {err['ratio']:.3g} (needs c = {c[i, k]:.3g}); "
                    f"{err['n_over']} Gaussians over")
    return float(c.max(initial=0.0))


def reduce_in_rank_order(stages):
    """float32 STAGE[0] + STAGE[1] + ... + STAGE[N-1], left to right (what every owner of a slice computes)."""
    acc = np.array(stages[0], np.float32, copy=True)
    for s in stages[1:]:
        acc = acc + np.asarray(s, np.float32)
    return acc


def check_sums(label, sums, stages):
    """Every rank's sum array S[0, 11P) == the rank-order float32 sum of the staging arrays, bit for bit."""
    want = np.ascontiguousarray(reduce_in_rank_order(stages)).view(np.uint32)
    for j, S in enumerate(sums):
        bad = np.flatnonzero(np.ascontiguousarray(S, np.float32).view(np.uint32) != want)
        if bad.size:
            e = int(bad[0])
            pytest.fail(f"{label}: S of rank {j} differs from the rank-order sum in {bad.size} floats, first at float "
                        f"{e} (16-byte unit {e // 4}, Gaussian {e // 11} entry {e % 11}): "
                        f"{np.float32(S[e])!r} != {want[e:e + 1].view(np.float32)[0]!r}")


SPLIT = dict(means3D=(0, 3), opacity=(3, 4), scales=(4, 7), rotations=(7, 11))   # the 44-byte record


def check_split(label, out, src, scale, rows=slice(None)):
    """out[name][rows] == float32(src[rows] x scale) bit for bit (src: [P, 11] records or sums)."""
    want = np.asarray(src, np.float32).reshape(-1, 11)[rows] * np.float32(scale)
    for k, (a, b) in SPLIT.items():
        g = np.ascontiguousarray(np.asarray(out[k], np.float32).reshape(-1, b - a)[rows]).view(np.uint32)
        bad = np.flatnonzero((g != np.ascontiguousarray(want[:, a:b]).view(np.uint32)).any(1))
        assert bad.size == 0, (f"{label}: dL_d{k} != float32(records x scale) in {bad.size} rows, e.g. row {bad[0]}: "
                               f"{g[bad[0]].view(np.float32)} != {want[bad[0], a:b]}")


def count_culled_here_seen_elsewhere(radii_me, other_factors):
    seen = np.zeros(len(radii_me), bool)
    for f in other_factors:
        seen |= (np.asarray(f).reshape(len(radii_me), 3) != 0).any(1)
    return int(((np.asarray(radii_me) == 0) & seen).sum())


# ---------------------------------------------------------------------------------------------------------------------
# the checks that need this run's forward (the oracle's chain, the blend reference)
def check_records(label, sc, deg, gacc, factor, rec, radii):
    """Check 1 (module docstring); returns compare_rows' report."""
    fw, _ = h.run_oracle(sc, np.asarray(BG, np.float32), None, use_sh=True, sh_degree=deg)
    assert np.array_equal(fw["radii"], radii), f"{label}: radii differ from the oracle's"
    vis = radii > 0
    assert not rec[~vis].any(), f"{label}: {int(rec[~vis].any(1).sum())} records of culled Gaussians are not zero"
    assert np.array_equal(rec[:, 3].view(np.uint32), np.ascontiguousarray(gacc[:, 5]).view(np.uint32)), \
        f"{label}: the records' opacity entry is not the blend accumulator"
    P = len(rec)
    dm2d, dconic = gr._accumulator_inputs(gacc, P)
    want = gr._oracle_chain(fw, dm2d, dconic, factor)
    pert = gr._oracle_chain(fw, *gr._noisy(dm2d, dconic), factor)
    got = {k: rec[:, a:b] for k, (a, b) in SPLIT.items() if k != "opacity"}
    return gr.compare_rows(label, {k: want[k] for k in got}, {k: pert[k] for k in got}, got, rows=vis)


def check_own_accumulators(label, f, gacc, factor, dL):
    st = f["st"]
    r = b64.blend_backward64(st, BG, dL, st["rgb"], clamped=st["clamped"])
    return gr.check_accumulators(label, st, b64.gpu_accumulators(gacc, factor), r)


# ---------------------------------------------------------------------------------------------------------------------
# driving the exchange with the test's own buffers
def plain_backward(sc, M, deg, dL):
    """A plain backward of view sc (no exchange): (factor block f32[3P+4] = dL_dcolors | campos | 0, records f32[P,11]
    in the 44-byte layout, the eight gradients)."""
    import torch
    from sugar_b200 import _C
    t = h.to_torch(sc)
    t["shs"] = t["shs"][:, :M].contiguous()
    E = torch.empty(0, device="cuda")
    bg = torch.tensor(BG, dtype=torch.float32, device="cuda")
    dLt = torch.from_numpy(dL).cuda()
    R, _color, radii, geom, binning, img = _C.rasterize_gaussians(
        bg, t["means3D"], E, t["opacities"], t["scales"], t["rotations"], 1.0, E, t["viewmatrix"], t["projmatrix"],
        sc.tanfovx, sc.tanfovy, H, W, t["shs"], deg, t["campos"], False, False)
    g = _C.rasterize_gaussians_backward(bg, t["means3D"], radii, E, t["scales"], t["rotations"], 1.0, E,
                                        t["viewmatrix"], t["projmatrix"], sc.tanfovx, sc.tanfovy, dLt, t["shs"], deg,
                                        t["campos"], geom, R, binning, img, False)
    block = torch.cat([g[1].reshape(-1), t["campos"].reshape(3), torch.zeros(1, device="cuda")]).contiguous()
    records = torch.cat([g[3], g[2], g[6], g[7]], dim=1).contiguous()
    return block, records, g


def _at_offset12(x):
    """x's values 12 bytes into a larger allocation: contiguous, not 16-byte aligned."""
    import torch
    buf = torch.zeros(x.numel() + 3, dtype=x.dtype, device=x.device)
    v = buf[3:].view(x.shape)
    v.copy_(x)
    return v


def own_view(sc, M, deg, offset12=False):
    """The forward of this rank's view (test_gpu_grad_rows._forward); offset12: the backward reads means3D from memory
    12 bytes off a 16-byte boundary, so no CTA of the per-Gaussian pass can bulk-load its inputs."""
    f = gr._forward(with_M(sc, M), BG, use_sh=True, sh_degree=deg)
    if offset12:
        a = list(f["args"])
        a[1] = _at_offset12(a[1])
        assert a[1].data_ptr() % 16 == 12
        f["args"] = tuple(a)
    return f


def launcher(f, bufs, dL):
    """`launch(plan, *, dL_dcolors, dL_dsh)` as _C.rasterize_gaussians_backward hands it to ViewParallel.run_backward:
    sgr_rasterize_backward_staged on f's forward buffers, gradients into `bufs`, accumulators into bufs' scratch."""
    import torch
    from sugar_b200 import _C, _lib
    (bgt, means3D, colors, _o, scales, rots, smod, cov, vm, pm, tfx, tfy, Hh, Ww, sh, deg, campos, _p, _d) = f["args"]
    view = _C._view_struct(bgt, smod, vm, pm, tfx, tfy, Hh, Ww, deg, campos, False, False)
    g = _C._gauss_struct(f["Pt"], f["M"], means3D, None, sh, colors, scales, rots, cov)
    dLt = torch.from_numpy(np.ascontiguousarray(dL, np.float32)).cuda()
    inputs = (C.byref(view), C.byref(g), f["radii"].data_ptr(), f["geom"].data_ptr(), f["binning"].data_ptr(),
              f["img"].data_ptr(), int(f["R"]), dLt.data_ptr())

    def launch(plan, *, dL_dcolors=bufs["colors"].data_ptr(), dL_dsh=None):
        _lib.check(_lib.lib.sgr_rasterize_backward_staged(
            *inputs, bufs["means2D"].data_ptr(), dL_dcolors, bufs["opacity"].data_ptr(), bufs["means3D"].data_ptr(),
            bufs["cov3D"].data_ptr(), dL_dsh, bufs["scales"].data_ptr(), bufs["rotations"].data_ptr(),
            bufs["scratch"].data_ptr(), torch.cuda.current_stream().cuda_stream, C.byref(plan)))
    launch.keep = (view, g, dLt)
    return launch


def _outputs(bufs):
    return {k: bufs[k].cpu().numpy() for k in ("means3D", "opacity", "scales", "rotations", "sh")}


def _poison(*tensors):
    for t in tensors:
        t.fill_(float("nan"))


class PeerEmulation:
    """This GPU as rank `me` of N in the peer-memory exchange (see the module docstring).  views[j] is rank j's view
    (views_sc: its scene with M coefficients, dL[j] its upstream gradient); blocks[j], records[j] and plain[j] come
    from a plain backward of view j; ranks j != me are stand-ins.  step() runs one backward of view `me` through
    ViewParallel.run_backward; close() frees the peer buffer."""

    def __init__(self, N, me, M, deg, chunks, taper, scale, P=P_SCENE, seed=41, offset12=False):
        import torch
        from sugar_b200 import _C, _lib, parallel, scenes
        assert 0 <= me < N
        self.N, self.me, self.M, self.deg, self.P, self.scale = N, me, M, deg, P, scale
        dev = torch.device("cuda", torch.cuda.current_device())
        base = scenes.make_scene(P, W, H, seed=seed, camera="posed")
        self.means = base.means3D
        self.views = [with_M(view_scene(base, j), M) for j in range(N)]
        self.dL = [scenes.upstream_grad(W, H, seed=5 + j) for j in range(N)]
        self.blocks, self.records, self.plain = [], [], []
        for j in range(N):
            b, r, g = plain_backward(self.views[j], M, deg, self.dL[j])
            self.blocks.append(b)
            self.records.append(r)
            self.plain.append(g)
        self.f = own_view(self.views[me], M, deg, offset12)
        self.bufs = _C._alloc_backward(P, M, dev, with_records=False)
        self.launch = launcher(self.f, self.bufs, self.dL[me])
        self.vp = vp = parallel.ViewParallel(chunks=chunks, scale=scale, force=True, peer=True, taper=taper)
        # rank `me` of a world of one with N staging arrays: R_ptr (where this rank's records go) is STAGE[me]
        st = parallel._PeerState(_lib.lib, _lib.check, P, me, 1, None, dev, nstage=N)
        self.st = st
        try:
            self.S_others = {j: torch.zeros(11 * P + 16, device=dev) for j in range(N) if j != me}
            i64 = lambda ptrs: torch.tensor(ptrs, dtype=torch.int64, device=dev)
            tab = lambda own, others: i64([own if j == me else others[j].data_ptr() for j in range(N)])
            st.world = N
            st.F_tab = [tab(st.base + st.off["F0"], self.blocks), tab(st.base + st.off["F1"], self.blocks)]
            st.S_tab = tab(st.S_ptr, self.S_others)
            st.stage_tab = i64([st.R_ptr] * N)        # every owner's array for this rank's records: this rank's own
            st.flag_tab = i64([st.base] * N)          # "every rank's flags" = this rank's
            for j in range(N):
                if j != me:
                    self.stage(j)[:11 * P].copy_(self.records[j].reshape(-1))
            self.flags = torch.as_tensor(type("Flags", (), {"__cuda_array_interface__": {
                "shape": (64, 64), "typestr": "<i4", "data": (st.base, False), "version": 2}})(), device=dev)
            self.others = [j for j in range(N) if j != me]
            self.flags[:63, self.others] = 1 << 30   # the stand-ins "have signalled" every slot (row 63: CTA counters)
            vp._emulated = tuple(self.others)
            self.check_tables()
            vp._peer_states[(P, dev)] = st
        except BaseException:
            st.world = 1
            st.close(_lib.lib)
            raise
        self.means3D = self.f["args"][1]
        self.campos = self.f["args"][16]

    def stage(self, j):
        from sugar_b200 import parallel
        import torch
        st = self.st
        return torch.as_tensor(parallel._DevMem(st.base + st.off["STAGE"] + j * st.stage_stride, 11 * self.P + 4),
                               device="cuda")

    def own_sums(self):
        from sugar_b200 import parallel
        import torch
        return torch.as_tensor(parallel._DevMem(self.st.S_ptr, 11 * self.P + 4), device="cuda")

    def check_tables(self):
        """On the host, before any kernel reads them: a wrong entry would show on the GPU as a flag wait that traps."""
        st, N, me, P = self.st, self.N, self.me, self.P
        rb, stage0 = st.stage_stride, st.base + st.off["STAGE"]
        tabs = dict(F0=st.F_tab[0], F1=st.F_tab[1], S=st.S_tab, stage=st.stage_tab, flags=st.flag_tab, rec=st.rec_tab)
        tabs = {k: v.cpu().tolist() for k, v in tabs.items()}
        for k, v in tabs.items():
            assert len(v) == N, (k, len(v), N)
        assert tabs["F0"][me] == st.base + st.off["F0"] and tabs["F1"][me] == st.base + st.off["F1"]
        assert tabs["S"][me] == st.S_ptr == st.base + st.off["S"]
        assert tabs["stage"] == [st.R_ptr] * N and st.R_ptr == stage0 + me * rb
        assert tabs["flags"] == [st.base] * N
        assert tabs["rec"] == [stage0 + j * rb for j in range(N)]
        for j in self.others:
            assert tabs["F0"][j] == tabs["F1"][j] == self.blocks[j].data_ptr()
            assert tabs["S"][j] == self.S_others[j].data_ptr()
            assert self.S_others[j].numel() >= 11 * P + 4
            assert np.array_equal(self.stage(j)[:11 * P].cpu().numpy(), self.records[j].reshape(-1).cpu().numpy())
        fl = self.flags.cpu().numpy()
        assert (fl[:63, self.others] == 1 << 30).all(), "stand-in flag presets"
        assert not fl[:, me].any() and not fl[63].any(), "the own flag column and the CTA counters start at zero"
        assert st.F_local[0].numel() == st.F_local[1].numel() == 3 * P + 4

    def step(self):
        """One backward of view `me` through ViewParallel.run_backward; every array the checks read, as numpy."""
        import torch
        st, P = self.st, self.P
        par = (st.seq + 1) & 1                      # the factor block this step's blend accumulates into
        S_all = [self.own_sums() if j == self.me else self.S_others[j] for j in range(self.N)]
        _poison(*(self.bufs[k] for k in ("means3D", "opacity", "scales", "rotations", "sh")),
                *(S[:11 * P] for S in S_all), self.stage(self.me)[:11 * P])
        self.vp.run_backward(self.launch, self.bufs, P, self.M, self.deg, self.means3D, self.campos,
                             has_cov_precomp=False)
        torch.cuda.synchronize()
        out = _outputs(self.bufs)
        out.update(gacc=gr.scratch_accumulators(self.bufs, P).cpu().numpy(),
                   factor=st.F_local[par][:3 * P].view(P, 3).cpu().numpy(),
                   stages=[self.stage(j)[:11 * P].cpu().numpy() for j in range(self.N)],
                   sums=[S[:11 * P].cpu().numpy() for S in S_all])
        out["records"] = out["stages"][self.me].reshape(P, 11)
        return out

    def close(self):
        import torch
        torch.cuda.synchronize()
        self.st.world = 1        # no process group: the close is local
        self.vp.close()


def emulate_peers(N, me, M, deg, chunks, taper, scale, **kw):
    return PeerEmulation(N, me, M, deg, chunks, taper, scale, **kw)


# ---------------------------------------------------------------------------------------------------------------------
# peer mode.  N, me, M, deg, chunks, taper, means3D 12 bytes off -- and the branch each case is there for
PEER_CASES = [
    (2, 0, 16, 3, 1, False, False),   # peer_reduce_kernel<2>, one chunk, rank 0 owns the first half
    (2, 1, 16, 3, 3, True, False),    # the own view skipped at index 1 of the factor table; rank 1 owns the second halves
    (3, 1, 9, 2, 16, True, False),    # M = 9 rows; tail chunks of 16 tapered ones have fewer blocks than ranks:
                                      #   this interior rank owns nothing there (q0 == q1, the handshake alone)
    (3, 2, 16, 3, 3, True, True),     # means3D 12 bytes off: every CTA stages word by word, the pulled factor blocks too
    (5, 2, 16, 2, 3, False, False),   # peer_reduce_kernel<8> with 5 ranks; degree 2 < 3: coefficients 9..15 zero
    (5, 4, 9, 1, 16, True, False),    # last rank, M = 9 with degree 1, empty tail chunks
    (8, 0, 16, 3, 16, True, False),   # 8 ranks: all 7 other views staged by the bulk copies (PB_VB = 7)
    (8, 7, 16, 3, 1, False, False),   # 8 ranks, last rank: the skip of the own view at the end of the table
    (9, 4, 16, 3, 3, True, False),    # peer_reduce_generic_kernel; the 8th other view loaded past PB_VB
    (9, 8, 9, 2, 1, False, False),    # the PB_VB overflow with M = 9 rows, last rank
    (16, 0, 16, 3, 16, False, False),  # 15 other views: 7 staged, 8 in the overflow loop (two batches)
    (16, 15, 16, 1, 3, True, False),   # 16 ranks, last rank, degree 1
    (16, 9, 9, 0, 16, True, False),    # 16 ranks, interior rank, M = 9 with degree 0, tail chunks owned by others
]


def _peer_id(c):
    N, me, M, deg, chunks, taper, off12 = c
    return f"N{N}-r{me}-M{M}-d{deg}-c{chunks}{'-taper' if taper else ''}{'-off12' if off12 else ''}"


@pytest.mark.parametrize("case", PEER_CASES, ids=[_peer_id(c) for c in PEER_CASES])
def test_peer_exchange_rows(case):
    N, me, M, deg, chunks, taper, off12 = case
    label = _peer_id(case)
    scale = 1.0 / N                      # the mean over the batch's views; not a power of two for most N
    em = emulate_peers(N, me, M, deg, chunks, taper, scale, offset12=off12)
    try:
        radii = em.f["radii"].cpu().numpy()
        others = [em.blocks[j][:3 * em.P].cpu().numpy() for j in em.others]
        n_elsewhere = count_culled_here_seen_elsewhere(radii, others)
        assert n_elsewhere >= MIN_CULLED_HERE, f"{label}: only {n_elsewhere} Gaussians culled here and seen elsewhere"
        rep = dict(culled_here_seen_elsewhere=n_elsewhere)
        for step in range(2):            # both factor-block parities
            o = em.step()
            lab = f"{label}/step{step}"
            if step == 0:
                rep["accumulators"] = check_own_accumulators(lab, em.f, o["gacc"], o["factor"], em.dL[me])
            rep[f"chain{step}"] = check_records(lab, em.views[me], deg, o["gacc"], o["factor"], o["records"], radii)
            check_sums(lab, o["sums"], o["stages"])
            check_split(lab, o, o["sums"][me], scale)
            factors = [o["factor"] if j == me else em.blocks[j][:3 * em.P].cpu().numpy() for j in range(N)]
            campos = [v.campos for v in em.views]
            ref, wt = dsh_reference(em.means, campos, factors, deg, scale)
            rep[f"dsh_c{step}"] = check_dsh(lab, o["sh"], ref, wt, deg)
        print(f"\n[exchange_rows] {label}: {rep}")
    finally:
        em.close()


# ---------------------------------------------------------------------------------------------------------------------
# the NCCL path as a forced single rank: records -> finalize (split + dL_dsh from the one view's factor)
NCCL_CASES = [   # M, deg, chunks, side_stream
    (16, 3, 1, False), (16, 3, 4, True), (16, 2, 7, False), (9, 2, 7, True), (9, 1, 4, False), (4, 1, 1, True),
    (4, 0, 7, False), (1, 0, 4, True), (1, 0, 1, False)]


@pytest.mark.parametrize("M,deg,chunks,side", NCCL_CASES)
def test_nccl_path_rows(M, deg, chunks, side):
    import torch
    from sugar_b200 import _C, parallel, scenes
    label = f"nccl-M{M}-d{deg}-c{chunks}{'-side' if side else ''}"
    scale = 0.3
    base = scenes.make_scene(P_SCENE, W, H, seed=41, camera="posed")
    sc = with_M(view_scene(base, 1), M)
    dL = scenes.upstream_grad(W, H, seed=6)
    f = own_view(sc, M, deg)
    bufs = _C._alloc_backward(P_SCENE, M, f["args"][1].device, with_records=True)
    vp = parallel.ViewParallel(chunks=chunks, scale=scale, force=True, side_stream=side, peer=False)
    assert not vp.uses_peer_memory(M, False)
    _poison(*(bufs[k] for k in ("means3D", "opacity", "scales", "rotations", "sh", "records")))
    vp.run_backward(launcher(f, bufs, dL), bufs, P_SCENE, M, deg, f["args"][1], f["args"][16], has_cov_precomp=False)
    torch.cuda.synchronize()
    o = _outputs(bufs)
    gacc = gr.scratch_accumulators(bufs, P_SCENE).cpu().numpy()
    factor, rec = bufs["colors"].cpu().numpy(), bufs["records"].cpu().numpy()
    radii = f["radii"].cpu().numpy()
    rep = dict(accumulators=check_own_accumulators(label, f, gacc, factor, dL))
    rep["chain"] = check_records(label, sc, deg, gacc, factor, rec, radii)
    check_split(label, o, rec, scale)
    ref, wt = dsh_reference(base.means3D, [sc.campos], [factor], deg, scale)
    rep["dsh_c"] = check_dsh(label, o["sh"], ref, wt, deg)
    print(f"\n[exchange_rows] {label}: {rep}")


# ---------------------------------------------------------------------------------------------------------------------
# sgr_view_grad_finalize with many views: the m16 kernel's view batches of SF_VB = 4 (its reload branch from the 5th
# view on), the generic kernel (M = 9, and M = 16 with a dL_dsh 12 bytes off alignment), full and partial ranges
def synthetic_factors(P, nviews, seed):
    """Per-view factors spread over four decades, a third of each view's rows zero (not visible there), and every
    twentieth Gaussian seen by no view."""
    rng = np.random.Generator(np.random.PCG64(seed))
    f = rng.normal(size=(nviews, P, 3)) * 10.0 ** rng.uniform(-4, 0, (nviews, P, 1))
    f[rng.uniform(size=(nviews, P)) < 1 / 3] = 0
    f[:, ::20] = 0
    return f.astype(np.float32)


def synthetic_records(P, seed):
    rng = np.random.Generator(np.random.PCG64(seed))
    return (rng.normal(size=(P, 11)) * 10.0 ** rng.uniform(-6, 0, (P, 1))).astype(np.float32)


FINALIZE_KINDS = {"m16": (16, 3, False), "generic_m9": (9, 2, False), "m16_offset12": (16, 3, True)}


@pytest.mark.parametrize("kind", list(FINALIZE_KINDS))
@pytest.mark.parametrize("nviews", [1, 4, 5, 8, 9, 13])
def test_finalize_many_views(nviews, kind):
    import torch
    from sugar_b200 import _lib, scenes
    M, deg, off12 = FINALIZE_KINDS[kind]
    P, scale = P_SCENE, 0.3
    base = scenes.make_scene(P, W, H, seed=41, camera="posed")
    campos = [view_scene(base, j).campos for j in range(nviews)]
    factors = synthetic_factors(P, nviews, seed=nviews)
    rec = synthetic_records(P, seed=100 + nviews)
    stride = 3 * P + 4                          # the exchange's factor block: [P, 3] factors, camera position, pad
    blocks = np.zeros((nviews, stride), np.float32)
    blocks[:, :3 * P] = factors.reshape(nviews, -1)
    blocks[:, 3 * P:3 * P + 3] = np.asarray(campos, np.float32)
    dev = torch.device("cuda", torch.cuda.current_device())
    blocks_t, rec_t = torch.from_numpy(blocks).to(dev), torch.from_numpy(rec).to(dev)
    means_t = torch.from_numpy(base.means3D).to(dev)
    ref, wt = dsh_reference(base.means3D, campos, factors, deg, scale)
    nan_bits = np.float32(np.nan).view(np.uint32)
    for p0, p1 in ((0, P), (1003, 4517)):
        label = f"finalize-{kind}-v{nviews}[{p0},{p1})"
        flat = torch.full((P * M * 3 + 3,), float("nan"), device=dev)
        dsh = (flat[3:] if off12 else flat[:-3]).view(P, M, 3)
        assert (dsh.data_ptr() % 16 == 12) == off12
        out = {k: torch.full((P, w), float("nan"), device=dev) for k, w in (("means3D", 3), ("opacity", 1),
                                                                             ("scales", 3), ("rotations", 4))}
        _lib.check(_lib.lib.sgr_view_grad_finalize(
            P, p0, p1, M, deg, nviews, means_t.data_ptr(), blocks_t.data_ptr() + 12 * P, blocks_t.data_ptr(), stride,
            stride, dsh.data_ptr(), rec_t.data_ptr(), scale, out["means3D"].data_ptr(), out["opacity"].data_ptr(),
            out["scales"].data_ptr(), out["rotations"].data_ptr(), torch.cuda.current_stream().cuda_stream))
        torch.cuda.synchronize()
        got = dsh.cpu().numpy()
        o = {k: v.cpu().numpy() for k, v in out.items()}
        outside = np.ones(P, bool)
        outside[p0:p1] = False
        for k, v in [("sh", got)] + list(o.items()):
            assert (v[outside].view(np.uint32) == nan_bits).all(), f"{label}: {k} rows outside [p0, p1) were written"
        check_split(label, o, rec, scale, rows=slice(p0, p1))
        c = check_dsh(label, got[p0:p1], ref[p0:p1], wt[p0:p1], deg)
        print(f"\n[exchange_rows] {label}: dsh_c {c:.3g}")
