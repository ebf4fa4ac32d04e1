"""Float64 restatement of the per-Gaussian backward chain: the reference's computeCov2DCUDA (with the guard-band clamp
and its gradient gates), the projection term of preprocessCUDA and computeCov3D's backward.

TEST INFRASTRUCTURE ONLY.  `oracle/raster_oracle.c` restates the reference's fp32 arithmetic; this module restates
the same formulas in float64 and says, for every Gaussian and output group, how far a correct fp32 kernel may land
from them.  Like tests/blend64.py it holds each Gaussian to a bar of its own.

Rules.
* Inputs are fp32 and bit-identical between ours, the oracle and the reference: the means, scales, rotations, the
  forward's cov3D (or cov3D_precomp), the camera, and the blend accumulators dL/dmeans2D and dL/dconic (a, b, c).
* Decisions are taken from the fp32 values, not re-decided in float64: visibility (radius > 0), the clamp side and
  the gates (edge_scenes.gates: txtz and its comparison with limx = fl32(1.3 tanfov), as the kernels compute them) and
  denom2inv == 0 (denom_overflows).  On a clamped axis t.x = +-limx t.z, limx the fp32 constant.
* The formulas are the reference's, including its two departures from the derivative of its own forward, which a
  kernel must reproduce:
    - a clamped axis has dL/dt.x = 0 (the gate), and dL/dt.z takes the clamped t.x as if it were constant in t.z, so
      its J02 term is 2 h_x limx / t.z^2 where the clamped forward's derivative is h_x limx / t.z^2;
    - dL/dscale is dL/d(s), s = scale_modifier * scale, without the factor scale_modifier.
  denom - a c is -b^2 in exact arithmetic and is taken as such.
* SH is not restated: on scenes with SH colours only cov3D, scales and rotations are held here (dL/dmeans3D carries
  the SH colour's view-direction term, which the oracle checks).
* Bar.  Per row and output group (means3D, cov3D, scales, rotations): max(RTOL |row|_inf, SENS x the row's change
  when the accumulators and cov3D carry 1e-6 relative noise), test_gpu_grad_rows' rule.  The largest
  |oracle - project64| / bar over every row of every edge scene (tests/test_projection_edges_cpu.py) is 0.13, and
  the largest |gpu - project64| / bar on an H100 80GB HBM3 at its 700 W limit (tests/test_gpu_projection_edges.py,
  both id formats) is 0.18, both dL/drotations of scale_mod_1.7_posed_sh3; on the guard-band, near-plane and
  off-screen scenes no group exceeds 0.05.  The mutations those tests apply miss the oracle by more than 10x.
"""
import numpy as np

import edge_scenes as es

RTOL, SENS, NOISE = 1e-4, 5.0, 1e-6
GROUPS = ("means3D", "cov3D", "scales", "rotations")


def _cov2d(sc, cov3D, gx, gy):
    """computeCov2DCUDA's forward pieces in float64, t.x (t.y) clamped to +-limx t.z where gx (gy) is False:
    dict(tx, ty, tz, hx, hy, T0, T1 [P,3] (the rows of W J), p = V T0, q = V T1, a, b, c (+0.3 included))."""
    v = es.fp32_view(sc)
    vm = np.asarray(sc.viewmatrix, np.float32).reshape(-1).astype(np.float64)
    m = sc.means3D.astype(np.float64)
    t = [m @ vm[[r, 4 + r, 8 + r]] + vm[12 + r] for r in range(3)]
    tz = t[2]
    limx, limy = float(v["limx"]), float(v["limy"])
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):   # culled rows (tz <= 0.2) are masked later
        tx = np.where(gx, t[0], np.sign(v["txtz"]) * limx * tz)
        ty = np.where(gy, t[1], np.sign(v["tytz"]) * limy * tz)
        hx = es.W / (2.0 * float(np.float32(sc.tanfovx)))
        hy = es.H / (2.0 * float(np.float32(sc.tanfovy)))
        J00, J02, J11, J12 = hx / tz, -hx * tx / tz ** 2, hy / tz, -hy * ty / tz ** 2
        T0 = np.stack([vm[4 * r] * J00 + vm[2 + 4 * r] * J02 for r in range(3)], 1)
        T1 = np.stack([vm[1 + 4 * r] * J11 + vm[2 + 4 * r] * J12 for r in range(3)], 1)
        c3 = np.asarray(cov3D, np.float64)
        V = c3[:, [0, 1, 2, 1, 3, 4, 2, 4, 5]].reshape(-1, 3, 3)
        p = np.einsum("pkj,pj->pk", V, T0)
        q = np.einsum("pkj,pj->pk", V, T1)
        return dict(tx=tx, ty=ty, tz=tz, hx=hx, hy=hy, T0=T0, T1=T1, p=p, q=q, a=(T0 * p).sum(1) + 0.3,
                    b=(T0 * q).sum(1), c=(T1 * q).sum(1) + 0.3)


def denom_overflows(sc, cov3D, rows):
    """denom2inv == 0 in fp32: denom^2 rounds to infinity.  Decided on the float64 denom = a c - b^2; a row within 4x
    of the threshold would be decided by the rounding of the fp32 chain, and the edge scenes keep none there."""
    k = _cov2d(sc, cov3D, *es.gates(sc))
    with np.errstate(invalid="ignore", over="ignore"):
        d2 = (k["a"] * k["c"] - k["b"] * k["b"]) ** 2
    near = rows & (d2 > es.F32_MAX / 4) & (d2 < 4 * es.F32_MAX)
    assert not near.any(), f"rows {np.flatnonzero(near)} have denom^2 within 4x of FLT_MAX"
    return rows & (d2 >= 4 * es.F32_MAX)


def chain64(sc, cov3D, radii, dm2d, dconic, scale_modifier=1.0, scales=True, gate_clamp=True, mod_in_dscale=False,
            honour_overflow=True, flip_gates=None):
    """dict(means3D [P,3], cov3D [P,6], scales [P,3], rotations [P,4]) in float64, zero for culled rows.
    dm2d [P,>=2], dconic [P,3] (a, b, c).  The keyword flags switch on the mutations the sensitivity tests use:
    gate_clamp=False (gates 1, t unclamped), mod_in_dscale=True (dL/dscale times scale_modifier),
    honour_overflow=False (the denom2inv == 0 branch ignored) and flip_gates=(fx, fy) (bool [P]: the gate of
    those rows decided the other way; the clamp unchanged)."""
    P = sc.means3D.shape[0]
    vis = np.asarray(radii) > 0
    gx, gy = es.gates(sc)
    if not gate_clamp:
        gx, gy = np.ones(P, bool), np.ones(P, bool)
    mx, my = gx, gy                                                # the gradient gates
    if flip_gates is not None:
        mx, my = gx ^ flip_gates[0], gy ^ flip_gates[1]
    over = denom_overflows(sc, cov3D, vis) if honour_overflow else np.zeros(P, bool)
    vm = np.asarray(sc.viewmatrix, np.float32).reshape(-1).astype(np.float64)
    pm = np.asarray(sc.projmatrix, np.float32).reshape(-1).astype(np.float64)
    m = sc.means3D.astype(np.float64)
    k = _cov2d(sc, cov3D, gx, gy)
    tx, ty, tz, hx, hy, T0, T1, p, q, a, b, c = (k[n] for n in ("tx", "ty", "tz", "hx", "hy", "T0", "T1", "p", "q",
                                                               "a", "b", "c"))
    dc = np.asarray(dconic, np.float64)
    dcx, dcy, dcz = dc[:, 0], dc[:, 1], dc[:, 2]
    denom = a * c - b * b
    d2inv = np.where(over | ~vis, 0.0, 1.0 / (denom * denom + 1e-7))
    nb2 = -b * b                                                   # denom - a c
    dL_da = d2inv * (-c * c * dcx + 2 * b * c * dcy + nb2 * dcz)
    dL_dc = d2inv * (-a * a * dcz + 2 * a * b * dcy + nb2 * dcx)
    dL_db = d2inv * 2 * (b * c * dcx - (denom + 2 * b * b) * dcy + a * b * dcz)
    dcov = np.stack([T0[:, 0] ** 2 * dL_da + T0[:, 0] * T1[:, 0] * dL_db + T1[:, 0] ** 2 * dL_dc,
                     2 * T0[:, 0] * T0[:, 1] * dL_da + (T0[:, 0] * T1[:, 1] + T0[:, 1] * T1[:, 0]) * dL_db
                     + 2 * T1[:, 0] * T1[:, 1] * dL_dc,
                     2 * T0[:, 0] * T0[:, 2] * dL_da + (T0[:, 0] * T1[:, 2] + T0[:, 2] * T1[:, 0]) * dL_db
                     + 2 * T1[:, 0] * T1[:, 2] * dL_dc,
                     T0[:, 1] ** 2 * dL_da + T0[:, 1] * T1[:, 1] * dL_db + T1[:, 1] ** 2 * dL_dc,
                     2 * T0[:, 2] * T0[:, 1] * dL_da + (T0[:, 1] * T1[:, 2] + T0[:, 2] * T1[:, 1]) * dL_db
                     + 2 * T1[:, 1] * T1[:, 2] * dL_dc,
                     T0[:, 2] ** 2 * dL_da + T0[:, 2] * T1[:, 2] * dL_db + T1[:, 2] ** 2 * dL_dc], 1)
    dT0 = 2 * p * dL_da[:, None] + q * dL_db[:, None]
    dT1 = 2 * q * dL_dc[:, None] + p * dL_db[:, None]
    dJ00 = dT0 @ vm[[0, 4, 8]]
    dJ02 = dT0 @ vm[[2, 6, 10]]
    dJ11 = dT1 @ vm[[1, 5, 9]]
    dJ12 = dT1 @ vm[[2, 6, 10]]
    with np.errstate(divide="ignore", invalid="ignore"):
        itz = 1.0 / tz
        dtx = np.where(mx, 1.0, 0.0) * -hx * itz ** 2 * dJ02
        dty = np.where(my, 1.0, 0.0) * -hy * itz ** 2 * dJ12
        dtz = (-hx * itz ** 2 * dJ00 - hy * itz ** 2 * dJ11 + 2 * hx * tx * itz ** 3 * dJ02
               + 2 * hy * ty * itz ** 3 * dJ12)
    dmean = np.stack([vm[0] * dtx + vm[1] * dty + vm[2] * dtz, vm[4] * dtx + vm[5] * dty + vm[6] * dtz,
                      vm[8] * dtx + vm[9] * dty + vm[10] * dtz], 1)
    # projection term (preprocessCUDA)
    hw = m @ pm[[3, 7, 11]] + pm[15]
    m_w = 1.0 / (hw + 1e-7)
    mul1 = (m @ pm[[0, 4, 8]] + pm[12]) * m_w * m_w
    mul2 = (m @ pm[[1, 5, 9]] + pm[13]) * m_w * m_w
    g = np.asarray(dm2d, np.float64)
    gxm, gym = g[:, 0], g[:, 1]
    for k in range(3):
        dmean[:, k] += ((pm[4 * k] * m_w - pm[4 * k + 3] * mul1) * gxm
                        + (pm[4 * k + 1] * m_w - pm[4 * k + 3] * mul2) * gym)
    out = dict(means3D=dmean, cov3D=dcov)
    if scales:
        out.update(_cov3d_backward(sc.scales, sc.rotations, scale_modifier, dcov, mod_in_dscale))
    return {k: np.where(vis[:, None], x, 0.0) for k, x in out.items()}


def _cov3d_backward(scales, rots, mod, dcov, mod_in_dscale):
    """computeCov3D's backward (backward.cu:278-341) in float64: dL/dscale (as dL/ds, s = mod scale) and dL/drot."""
    q = np.asarray(rots, np.float64)
    r, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    # R[col][row] as glm stores it
    R = np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y)], 1),
                  np.stack([2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x)], 1),
                  np.stack([2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], 1)], 1)
    s = float(np.float32(mod)) * np.asarray(scales, np.float64)
    d = dcov
    dS = np.stack([np.stack([d[:, 0], 0.5 * d[:, 1], 0.5 * d[:, 2]], 1),
                   np.stack([0.5 * d[:, 1], d[:, 3], 0.5 * d[:, 4]], 1),
                   np.stack([0.5 * d[:, 2], 0.5 * d[:, 4], d[:, 5]], 1)], 1)
    # dMt[w][c] = 2 s[w] sum_j R[j][w] dS[c][j]
    dMt = 2 * s[:, :, None] * np.einsum("pjw,pcj->pwc", R, dS)
    dscale = np.einsum("pjk,pkj->pk", R, dMt)
    if mod_in_dscale:
        dscale = dscale * float(np.float32(mod))
    dMt = dMt * s[:, :, None]
    M = dMt
    dq = np.stack([
        2 * z * (M[:, 0, 1] - M[:, 1, 0]) + 2 * y * (M[:, 2, 0] - M[:, 0, 2]) + 2 * x * (M[:, 1, 2] - M[:, 2, 1]),
        2 * y * (M[:, 1, 0] + M[:, 0, 1]) + 2 * z * (M[:, 2, 0] + M[:, 0, 2]) + 2 * r * (M[:, 1, 2] - M[:, 2, 1])
        - 4 * x * (M[:, 2, 2] + M[:, 1, 1]),
        2 * x * (M[:, 1, 0] + M[:, 0, 1]) + 2 * r * (M[:, 2, 0] - M[:, 0, 2]) + 2 * z * (M[:, 1, 2] + M[:, 2, 1])
        - 4 * y * (M[:, 2, 2] + M[:, 0, 0]),
        2 * r * (M[:, 0, 1] - M[:, 1, 0]) + 2 * x * (M[:, 2, 0] + M[:, 0, 2]) + 2 * y * (M[:, 1, 2] + M[:, 2, 1])
        - 4 * z * (M[:, 1, 1] + M[:, 0, 0])], 1)
    return dict(scales=dscale, rotations=dq)


def _noisy(*arrays, seed=0):
    rng = np.random.default_rng(seed)
    return [np.asarray(a, np.float64) * (1 + NOISE * rng.standard_normal(np.shape(a))) for a in arrays]


def reference(sc, cov3D, radii, dm2d, dconic, scale_modifier=1.0, scales=True, **mutation):
    """(ref, bar): the float64 chain and each row's bar per group ([P, C] arrays, the bar broadcast over a group)."""
    ref = chain64(sc, cov3D, radii, dm2d, dconic, scale_modifier, scales, **mutation)
    nm, nc, ncov = _noisy(dm2d, dconic, cov3D)
    pert = chain64(sc, ncov, radii, nm, nc, scale_modifier, scales, **mutation)
    bar = {}
    for k in ref:
        sens = np.abs(pert[k] - ref[k]).max(1)
        bar[k] = np.maximum(RTOL * np.abs(ref[k]).max(1), SENS * sens)[:, None] * np.ones_like(ref[k])
    return ref, bar


def accumulators_of(bw, P):
    """(dm2d [P,2], dconic [P,3] (a, b, c)) of raster_oracle.backward's result."""
    return bw["dL_dmeans2D"].reshape(P, 3)[:, :2], bw["dL_dconic"].reshape(P, 4)[:, [0, 1, 3]]
