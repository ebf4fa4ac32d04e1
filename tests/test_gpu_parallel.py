"""View-parallel exchange (sugar_b200/parallel.py) on ONE GPU: `ViewParallel(force=True)` drives the same
record / chunk / factor / finalize path as a multi-rank run, with the collectives left out, so its gradients
must equal the plain backward's.  The multi-rank numbers are checked by bench.py itself at N > 1 (`exchange_check`
in its JSON line) and by scripts/check_view_parallel.py under torchrun."""
import numpy as np
import pytest

import helpers as h

pytestmark = pytest.mark.gpu


def _err(a, b):
    return h.rel_err(a.detach().float().cpu().numpy(), b.detach().float().cpu().numpy())


def _render_loss(mod, t, sc, dL, deg, ps, bg=(0.1, 0.2, 0.3), colors=None):
    import torch
    means2D = torch.zeros_like(ps["means3D"], requires_grad=True)
    st = mod.GaussianRasterizationSettings(
        image_height=sc.height, image_width=sc.width, tanfovx=sc.tanfovx, tanfovy=sc.tanfovy,
        bg=torch.tensor(bg, device="cuda"), scale_modifier=1.0, viewmatrix=t["viewmatrix"], projmatrix=t["projmatrix"],
        sh_degree=deg, campos=t["campos"], prefiltered=False, debug=False)
    kw = dict(colors_precomp=colors) if colors is not None else dict(shs=ps["shs"])
    color, radii = mod.GaussianRasterizer(st)(means3D=ps["means3D"], means2D=means2D, opacities=ps["opacities"],
                                              scales=ps["scales"], rotations=ps["rotations"], **kw)
    return (color * dL).sum(), means2D


@pytest.mark.parametrize("deg,chunks,factors,side", [(3, 4, True, False), (1, 3, True, False), (0, 1, True, False),
                                                     (3, 4, False, False), (2, 7, True, False), (3, 4, True, True),
                                                     (2, 3, False, True)])
@pytest.mark.parametrize("peer", [True, False])
def test_forced_exchange_matches_plain_backward(deg, chunks, factors, side, peer):
    check_forced_exchange(16, deg, chunks, factors, side, peer)


# M = 1 / 4 / 9 stored SH coefficients: the generic finalize kernel (M = 16 has its own), and in peer mode the
# per-Gaussian pass with rows that are not 48 floats; deg < sqrt(M) - 1 leaves trailing coefficients that must be zero
@pytest.mark.parametrize("M,deg,chunks,factors,side", [
    (9, 2, 3, True, False), (9, 2, 4, True, True), (9, 1, 2, False, True), (4, 1, 4, True, False), (4, 1, 3, True, True),
    (4, 0, 2, False, False), (1, 0, 1, True, True), (1, 0, 3, True, False)])
@pytest.mark.parametrize("peer", [True, False])
def test_forced_exchange_with_fewer_stored_sh_coefficients(M, deg, chunks, factors, side, peer):
    check_forced_exchange(M, deg, chunks, factors, side, peer)


def check_forced_exchange(M, deg, chunks, factors, side, peer):
    """ViewParallel(force=True) with [P, M, 3] SH coefficients: scale x the plain backward's gradients."""
    import torch
    from sugar_b200 import diff_gaussian_rasterization as mod
    from sugar_b200 import parallel, scenes
    P, W, H = 6001, 160, 96          # not a multiple of the CTA size: partial last block, ragged chunks
    sc = scenes.make_scene(P, W, H, seed=31 + deg, camera="posed")
    dL = torch.from_numpy(scenes.upstream_grad(W, H, seed=5)).cuda()
    t = h.to_torch(sc)
    t["shs"] = t["shs"][:, :M].contiguous()
    leaf = lambda x: x.clone().requires_grad_(True)
    names = ("means3D", "opacities", "shs", "scales", "rotations")
    ps_a = {k: leaf(t[k]) for k in names}
    loss, m2a = _render_loss(mod, t, sc, dL, deg, ps_a)
    loss.backward()
    # peer=True: the peer-memory exchange (csrc/sgr_peer.cu) with this GPU as its only rank -- flags, two-shot
    # record reduce, pointer-table finalize, both side streams
    vp = parallel.ViewParallel(sh_factors=factors, chunks=chunks, scale=0.5, force=True, side_stream=side, peer=peer)
    for _ in range(3 if peer else 1):      # step parity alternates the factor blocks
        ps_b = {k: leaf(t[k]) for k in names}
        with vp.context():
            loss, m2b = _render_loss(mod, t, sc, dL, deg, ps_b)
            loss.backward()
    assert vp.stats["backwards"] == (3 if peer else 1)
    assert any(v is not None for v in vp._peer_states.values()) == (peer and factors)
    vp.close()
    for k in names:
        assert _err(ps_b[k].grad, 0.5 * ps_a[k].grad) <= 1e-4, k   # fp32 atomics: run-to-run order differs
    assert _err(m2b.grad, m2a.grad) <= 1e-4                        # per-view statistic: neither summed nor scaled
    used = (deg + 1) ** 2
    assert ps_b["shs"].grad.shape == (P, M, 3)
    if used < M:
        assert float(ps_b["shs"].grad[:, used:].abs().max()) == 0.0
        assert float(ps_a["shs"].grad[:, used:].abs().max()) == 0.0


def test_exchange_with_precomputed_colours_and_activations_in_front():
    """The trainers' path: raw parameters -> exp / sigmoid / normalize (+ python colours) -> rasterizer.  The
    exchange acts on the op's output gradients, so non-leaf inputs need nothing special."""
    import torch
    from sugar_b200 import diff_gaussian_rasterization as mod
    from sugar_b200 import parallel, scenes
    P, W, H = 5000, 160, 96
    sc = scenes.make_scene(P, W, H, seed=3, camera="posed")
    dL = torch.from_numpy(scenes.upstream_grad(W, H, seed=9)).cuda()
    t = h.to_torch(sc)

    def raw():
        r = dict(means3D=t["means3D"].clone(), log_scales=t["scales"].log(), quats=t["rotations"] * 1.7,
                 logit=torch.logit(t["opacities"].clamp(1e-4, 1 - 1e-4)), colors=t["colors_precomp"].clone())
        return {k: v.requires_grad_(True) for k, v in r.items()}

    def run(r):
        ps = dict(means3D=r["means3D"], opacities=torch.sigmoid(r["logit"]), scales=torch.exp(r["log_scales"]),
                  rotations=torch.nn.functional.normalize(r["quats"], dim=-1))
        loss, _ = _render_loss(mod, t, sc, dL, 0, ps, colors=r["colors"] * 1.0)
        loss.backward()

    a = raw()
    run(a)
    b = raw()
    vp = parallel.ViewParallel(chunks=4, force=True)
    with vp.context():
        run(b)
    for k in a:
        assert _err(b[k].grad, a[k].grad) <= 1e-4, k


def test_two_backwards_per_step_accumulate():
    """Two views rendered by one rank in one step (gradient accumulation): each backward runs its own exchange."""
    import torch
    from sugar_b200 import diff_gaussian_rasterization as mod
    from sugar_b200 import parallel, scenes
    P, W, H, deg = 5000, 160, 96, 3
    sc1 = scenes.make_scene(P, W, H, seed=77, camera="posed")
    sc2 = scenes.with_camera_offset(sc1, 0.15, (0.3, -0.1, 0.2))
    dL = torch.from_numpy(scenes.upstream_grad(W, H, seed=9)).cuda()
    names = ("means3D", "opacities", "shs", "scales", "rotations")
    t1, t2 = h.to_torch(sc1), h.to_torch(sc2)

    def both(ctxmgr):
        ps = {k: t1[k].clone().requires_grad_(True) for k in names}
        with ctxmgr:
            for t, sc in ((t1, sc1), (t2, sc2)):
                loss, _ = _render_loss(mod, t, sc, dL, deg, ps)
                loss.backward()
        return ps
    import contextlib
    a = both(contextlib.nullcontext())
    vp = parallel.ViewParallel(chunks=2, force=True)
    b = both(vp.context())
    assert vp.stats["backwards"] == 2
    for k in names:
        assert _err(b[k].grad, a[k].grad) <= 1e-4, k


def test_sh_factors_of_three_views_rebuild_the_summed_dsh():
    check_sh_factors_rebuild(16, 3)


def test_sh_factors_rebuild_the_summed_dsh_with_nine_stored_coefficients():
    """M = 9 stored coefficients, degree 1: the generic kernel, and coefficients 4..8 must come back zero."""
    check_sh_factors_rebuild(9, 1)


def check_sh_factors_rebuild(M, deg):
    """sh_grad_from_factors (sgr_view_grad_finalize) on the gathered factors of several views == the sum of the views'
    dL_dsh; the factor of a view is the dL_dcolors the backward returns with SH colours (clamp-masked dL/dRGB).  Also against
    sum_v basis(normalize(mean - campos_v)) (x) factor_v evaluated in float64.  On one view's factor alone it gives
    that view's dL_dsh exactly: the backward and the factor kernels evaluate the same basis at the same direction."""
    import torch
    from sugar_b200 import _C, parallel, scenes
    P, W, H = 6000, 160, 96
    base = scenes.make_scene(P, W, H, seed=34, camera="posed")
    views = [base, scenes.with_camera_offset(base, 0.15, (0.3, -0.1, 0.2)),
             scenes.with_camera_offset(base, -0.2, (-0.4, 0.2, 0.5))]
    want, factors, campos, dsh = None, [], [], []
    E = torch.Tensor([])
    for v, sc in enumerate(views):
        t = h.to_torch(sc)
        t["shs"] = t["shs"][:, :M].contiguous()
        dL = torch.from_numpy(scenes.upstream_grad(W, H, seed=5 + v)).cuda()
        bg = torch.zeros(3, device="cuda")
        R, color, radii, geom, binning, img = _C.rasterize_gaussians(
            bg, t["means3D"], E, t["opacities"], t["scales"], t["rotations"], 1.0, E, t["viewmatrix"], t["projmatrix"],
            sc.tanfovx, sc.tanfovy, H, W, t["shs"], deg, t["campos"], False, False)
        g = _C.rasterize_gaussians_backward(bg, t["means3D"], radii, E, t["scales"], t["rotations"], 1.0, E,
                                            t["viewmatrix"], t["projmatrix"], sc.tanfovx, sc.tanfovy, dL, t["shs"], deg,
                                            t["campos"], geom, R, binning, img, False)
        factors.append(g[1].clone())
        campos.append(t["campos"].clone())
        dsh.append(g[5].clone())
        want = g[5].double() if want is None else want + g[5].double()
    means = torch.from_numpy(base.means3D).cuda()
    got = parallel.sh_grad_from_factors(means, torch.stack(campos).contiguous(), torch.stack(factors).contiguous(), M, deg)
    assert got.shape == (P, M, 3)
    assert _err(got, want) <= 1e-4
    exact = 0.0
    for f, cp in zip(factors, campos):
        d = base.means3D.astype(np.float64) - cp.cpu().numpy().astype(np.float64).reshape(1, 3)
        d /= np.linalg.norm(d, axis=1, keepdims=True)
        exact = exact + h.sh_basis(d, deg)[:, :M, None] * f.cpu().numpy().astype(np.float64)[:, None, :]
    assert h.rel_err(got.cpu().numpy(), exact) <= 1e-5
    for f, cp, dsh_v in zip(factors, campos, dsh):
        one = parallel.sh_grad_from_factors(means, cp[None].contiguous(), f[None].contiguous(), M, deg)
        assert torch.equal(one, dsh_v)                 # ==, so +0 and -0 match
    used = (deg + 1) ** 2
    if used < M:
        assert float(got[:, used:].abs().max()) == 0.0 and float(want[:, used:].abs().max()) == 0.0


def test_peer_exchange_with_three_emulated_ranks():
    check_peer_exchange_with_three_emulated_ranks(16, 3)


def test_peer_exchange_with_three_emulated_ranks_and_nine_stored_coefficients():
    check_peer_exchange_with_three_emulated_ranks(9, 2)


def check_peer_exchange_with_three_emulated_ranks(M, deg):
    """The peer-memory exchange (csrc/sgr_peer.cu) as rank 0 of THREE, on one GPU: ranks 1 and 2 are static stand-ins --
    their factor blocks and record arrays are filled from plain backwards of their views, their flag words are preset,
    and this process reduces their record slices as well (test_gpu_exchange_rows.emulate_peers).  Everything the real
    multi-rank run executes runs here: the flag waits, the per-Gaussian pass summing three views' SH gradients through the
    pointer table, the two-shot reduce over three record arrays, the split.  The result must be scale x (sum of the three
    views' plain gradients)."""
    import torch
    from sugar_b200 import diff_gaussian_rasterization as mod
    import test_gpu_exchange_rows as ex
    P, scale = 6001, 0.25
    names = ("means3D", "opacities", "shs", "scales", "rotations")
    em = ex.emulate_peers(3, 0, M, deg, chunks=3, taper=True, scale=scale, P=P, seed=41)
    try:
        plain = [{"means3D": g[3].double(), "opacities": g[2].double(), "shs": g[5].double(), "scales": g[6].double(),
                  "rotations": g[7].double()} for g in em.plain]
        want = {k: scale * sum(p[k] for p in plain) for k in names}
        records = em.records
        t0, sc0 = h.to_torch(em.views[0]), em.views[0]
        dL0 = torch.from_numpy(em.dL[0]).cuda()
        for step in range(2):       # both factor-block parities
            ps = {k: t0[k].clone().requires_grad_(True) for k in names}
            with em.vp.context():
                loss, _ = _render_loss(mod, t0, sc0, dL0, deg, ps, bg=(0.0, 0.0, 0.0))
                loss.backward()
            for k in names:
                assert _err(ps[k].grad, want[k].float()) <= 1e-4, (step, k)
            for S in em.S_others.values():        # every rank's sum array received every slice
                assert _err(S[:11 * P], (records[0].double() + records[1].double() + records[2].double()).float().reshape(-1)) <= 1e-4
    finally:
        em.close()
