"""Surface-shaped inputs for the field, better-normal and density-estimation kernels, and the per-row rule they are
held to against float64.  TEST INFRASTRUCTURE ONLY (like tests/blend64.py).

fo.make_case draws isotropic blobs, on which nothing is hard.  SuGaR's coarse training makes flat Gaussians whose
smallest axis is the surface normal, identity quaternions at initialisation and samples hugging the surface; there the
1/s clamp, the Mahalanobis^2 clamp, the opacity_min_clamp branch, sign(<n_k, n_own>) = 0, the clamps of min_scaling and
wsum and the first-minimum tie rule actually run.  `surface_case` draws such a cloud, `with_edges` appends named
groups of Gaussians and samples that sit on each of those boundaries, and each group is checked on its own.

The rule.  Every value and gradient row is compared with the oracle (oracle/field_oracle.py, densest_oracle.py) in
float64, allowing a small floor plus what the reference's own float32 chain is off on the same inputs:
    p = max(|o32 - o64|, |o32r - o64|) + 2 |ours - ours'|
o32 is the oracle in float32, o32r the same with each sample's K neighbour columns reversed (a second summation
order), ours' a second GPU run (the order of the atomics).
    values     |ours - v64| <= floor_v (|v64| + scale) + 3 p          per sample or entry
    gradients  |ours - g64| <= 1e-4 rowmax|g64| + 4 p + 2 G + floor_T max|g64|   per row (h.row_errors), the max
               taken over the row's group (the surface cloud, or one edge group) so an edge's large rows do not hide
               the rest; G = grad_term_error, the per-term rounding that two summation orders cannot show
Normal-loss samples with a neighbour where 0 < |<n_k, n_own>| <= 1e-6 (the sign is a coin toss in float32) or a
Gaussian whose two smallest scales are 1 ulp apart are excluded; exact zeros and exact ties are not.
"""
import numpy as np
import torch

import helpers as h
from oracle import densest_oracle as deo
from oracle import field_oracle as fo

LEAVES = ("x", "points", "scaling", "quaternions", "strengths")
FIELD_OUTPUTS = ("density", "beta", "sdf", "closest_gaussian_opacities")

# Value floors (relative to |v64| + scale) and gradient floors floor_T (relative to the group's largest |g64|).  The
# smallest floors under which the float32 oracle with its neighbour columns in a random order passes every case of
# test_field_rows_cpu.py (the measured value in the comment) are raised to at least 1e-6: the permutation changes only
# the order of the sums, while the kernels also round each term differently (FMA contraction, expf, the product order
# of L^-T (x - mu)).  check() reports, per group and tensor, the share of rows whose allowance the floor dominates.
VALUE_FLOOR = dict(density=1e-6,                       # 7.6e-8
                   closest_gaussian_opacities=1e-6,    # 0: p holds each term's own rounding
                   beta=1e-6,                          # 1.8e-7
                   sdf=1e-6,                           # 1.7e-7
                   sdf_grad=4e-6,                      # 1.6e-6
                   densest=5e-6,                       # 2.6e-6
                   normal=1e-6)                        # see value_scale
# Gradient floors: with 2 G in the allowance, the smallest floor the float32 oracle in four orders and the kernels'
# float32 stand-in need over G is at most 4.4e-9 (k16_df1's dL/dstrengths; 0 to 1e-41 elsewhere,
# test_field_grad_rows_cpu), so every gradient takes the 1e-6 default.
GRAD_FLOOR = dict(field={}, densest={}, normal={})
# Gradients that are zero in exact arithmetic, so that every entry is the rounding of cancelling terms: the normal
# loss's dL/dq in groups where each sample's weighted neighbour normals sum to its own (v = 0) or no weight is left
# (|n_own|^2 = 1 for every q).  Their values are checked.
NOISE_ONLY = {("normal", g, "quaternions") for g in ("inv_s_clamp", "zero_weights", "mahalanobis_clamp", "far_samples",
                                                     "sdf_grad_clip", "dense_center")}
SIGN_EPS = 1e-6
EXCLUDED_MAX = 0.005


# ---------------------------------------------------------------------------------------------------------- inputs
def _quat_from_matrix(R):
    """Unit quaternions (real part first, r >= 0) of rotation matrices [P, 3, 3], float64."""
    R = np.asarray(R, np.float64)
    t = np.trace(R, axis1=1, axis2=2)
    q = np.empty((len(R), 4))
    m = np.stack([t, R[:, 0, 0], R[:, 1, 1], R[:, 2, 2]], 1).argmax(1)
    for i in range(len(R)):
        a = R[i]
        if m[i] == 0:
            s = 2.0 * np.sqrt(1.0 + t[i])
            q[i] = [0.25 * s, (a[2, 1] - a[1, 2]) / s, (a[0, 2] - a[2, 0]) / s, (a[1, 0] - a[0, 1]) / s]
        elif m[i] == 1:
            s = 2.0 * np.sqrt(1.0 + a[0, 0] - a[1, 1] - a[2, 2])
            q[i] = [(a[2, 1] - a[1, 2]) / s, 0.25 * s, (a[0, 1] + a[1, 0]) / s, (a[0, 2] + a[2, 0]) / s]
        elif m[i] == 2:
            s = 2.0 * np.sqrt(1.0 + a[1, 1] - a[0, 0] - a[2, 2])
            q[i] = [(a[0, 2] - a[2, 0]) / s, (a[0, 1] + a[1, 0]) / s, 0.25 * s, (a[1, 2] + a[2, 1]) / s]
        else:
            s = 2.0 * np.sqrt(1.0 + a[2, 2] - a[0, 0] - a[1, 1])
            q[i] = [(a[1, 0] - a[0, 1]) / s, (a[0, 2] + a[2, 0]) / s, (a[1, 2] + a[2, 1]) / s, 0.25 * s]
    return q * np.where(q[:, :1] < 0, -1.0, 1.0)


def _rot(q):
    return fo.quaternion_to_matrix(torch.from_numpy(np.asarray(q, np.float64))).numpy()


def surface_case(P=4000, N=16000, K=16, seed=0, thin=1e-3, identity_frac=0.3, q_norm=True, density_factor=1.0 / 16,
                 thin_abs=None):
    """Flat Gaussians on a unit sphere and on a tilted plane below it, each rotated so that its smallest axis is the
    surface normal (the thin column is drawn at random); `thin` is the smallest scale over the in-plane ones, or
    `thin_abs` the smallest scale itself.  `identity_frac` of the Gaussians have identity quaternions (their normal is
    the coordinate axis of the thin column); with `q_norm`, a tenth have |q| = 0.5 and a tenth |q| = 3 (two_s != 2).
    Strengths are sigmoids mostly near 1.  Samples are drawn like sample_points_in_gaussians (multinomial over
    volumes, x = mu + R(q) (1.5 s N(0,1))); neighbours are the sample's Gaussian's exact K nearest (fo.knn_idx)."""
    rng = np.random.default_rng(seed)
    Ps = P // 2
    v = rng.normal(size=(Ps, 3))
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    npl = np.array([0.3, -0.2, 1.0]) / np.linalg.norm([0.3, -0.2, 1.0])
    ua = np.cross(npl, [1.0, 0.0, 0.0])
    ua /= np.linalg.norm(ua)
    uv = rng.uniform(-1, 1, (P - Ps, 2))
    pl = np.array([0.0, 0.0, -1.2]) + uv[:, :1] * ua + uv[:, 1:] * np.cross(npl, ua)
    points = np.r_[v, pl]
    normal = np.r_[v, np.tile(npl, (P - Ps, 1))]
    spacing = np.r_[np.full(Ps, np.sqrt(4 * np.pi / Ps)), np.full(P - Ps, np.sqrt(4.0 / (P - Ps)))]
    inplane = 0.6 * spacing[:, None] * np.exp(rng.normal(0.0, 0.3, (P, 2)))
    small = thin_abs if thin_abs is not None else thin * np.sqrt(inplane[:, 0] * inplane[:, 1])
    col = rng.integers(0, 3, P)
    scaling = np.empty((P, 3))
    R = np.empty((P, 3, 3))
    for i in range(P):
        n = normal[i]
        a = np.cross(n, [1.0, 0.0, 0.0] if abs(n[0]) < 0.9 else [0.0, 1.0, 0.0])
        a /= np.linalg.norm(a)
        b = np.cross(n, a)
        th = rng.uniform(0, 2 * np.pi)
        t1, t2 = np.cos(th) * a + np.sin(th) * b, -np.sin(th) * a + np.cos(th) * b
        others = [c for c in range(3) if c != col[i]]
        R[i][:, col[i]], R[i][:, others[0]] = n, t1
        R[i][:, others[1]] = np.cross(R[i][:, (others[1] + 1) % 3], R[i][:, (others[1] + 2) % 3])
        scaling[i, col[i]] = small if np.isscalar(small) else small[i]
        scaling[i, others] = inplane[i]
    q = _quat_from_matrix(R)
    q *= np.where(rng.random(P) < 0.5, -1.0, 1.0)[:, None]
    q[rng.random(P) < identity_frac] = [1.0, 0.0, 0.0, 0.0]
    if q_norm:
        u = rng.random(P)
        q[u < 0.1] *= 0.5
        q[u > 0.9] *= 3.0
    strengths = 1.0 / (1.0 + np.exp(-rng.normal(3.0, 1.5, P)))
    points, scaling, q = (np.ascontiguousarray(a, np.float32) for a in (points, scaling, q))
    vol = scaling.astype(np.float64).prod(1)
    gi = rng.choice(P, N, p=vol / vol.sum())
    x = points[gi] + np.einsum("nij,nj->ni", _rot(q[gi]), 1.5 * scaling[gi] * rng.normal(size=(N, 3)))
    nbr = fo.knn_idx(torch.from_numpy(points), K).numpy()[gi]
    return dict(x=np.ascontiguousarray(x, np.float32), nbr_idx=np.ascontiguousarray(nbr), gaussian_idx=gi.astype(np.int64),
                points=points, scaling=scaling, quaternions=q, strengths=strengths.astype(np.float32),
                density_factor=density_factor, density_threshold=1.0)


# Surface cases: the smallest scale over the in-plane ones at K = 16 and the coarse_sdf trainer's density factor, one
# absolute smallest scale below 1e-6, and K = 8, 5 (a partial lane group), 33 (two pairs per lane) at both factors.
SURFACE = {"thin1e-1": dict(thin=1e-1), "thin1e-2": dict(thin=1e-2), "thin1e-3": dict(thin=1e-3),
           "thin1e-4": dict(thin=1e-4), "abs5e-7": dict(thin_abs=5e-7),
           "k16_df1": dict(thin=1e-3, density_factor=1.0),
           "k8": dict(K=8, thin=1e-3, density_factor=1.0 / 8), "k8_df1": dict(K=8, thin=1e-2, density_factor=1.0),
           "k5": dict(K=5, thin=1e-3, N=12001, density_factor=1.0 / 5), "k5_df1": dict(K=5, thin=1e-3, N=12001, density_factor=1.0),
           "k33": dict(K=33, thin=1e-3, N=8000, density_factor=1.0 / 33), "k33_df1": dict(K=33, thin=1e-2, N=8000, density_factor=1.0)}


def surface(name, edges=True):
    cfg = dict(dict(P=3000, N=12000, K=16, seed=sum(map(ord, name))), **SURFACE[name])
    case = surface_case(**cfg)
    return with_edges(case) if edges else dict(case, groups={"surface": _all(case)})


def _all(case):
    return (np.arange(len(case["x"])), np.arange(len(case["points"])))


# --------------------------------------------------------------------------------------------------------- edges
F32 = np.float32
UP = lambda v: np.nextafter(F32(v), F32(np.inf))
DOWN = lambda v: np.nextafter(F32(v), F32(0))
ID = (1.0, 0.0, 0.0, 0.0)
TILT = [(0.9, 0.3, -0.2, 0.1), (0.7, -0.4, 0.5, 0.2), (0.8, 0.1, 0.4, -0.3), (0.6, 0.5, 0.3, 0.5)]


class _Edges:
    """Appends groups of Gaussians and samples; a group's neighbour rows name only its own Gaussians (cycled to K)."""

    def __init__(self, case):
        self.c = {k: list(case[k]) for k in ("points", "scaling", "quaternions", "strengths")}
        self.x, self.own, self.nbr = [], [], []
        self.K = case["nbr_idx"].shape[1]
        self.P0, self.N0 = len(case["points"]), len(case["x"])
        self.groups = {"surface": _all(case)}
        self.origin = 0

    def group(self, name, gaussians, samples):
        """gaussians: (offset, scaling, q, strength); samples: (offset, own, row) with `own` and `row` indices into
        this group's Gaussians.  Each group sits at its own exactly representable origin far from the rest."""
        self.origin += 1
        o = np.array([100.0 + 10.0 * self.origin, -50.0, 0.0])
        g0, n0 = len(self.c["points"]), self.N0 + len(self.x)
        for off, s, q, st in gaussians:
            self.c["points"].append(F32(o + np.asarray(off, np.float64)))
            self.c["scaling"].append(np.asarray(s, F32))
            self.c["quaternions"].append(np.asarray(q, F32))
            self.c["strengths"].append(F32(st))
        for off, own, row in samples:
            self.x.append(np.asarray(o + np.asarray(off, np.float64), F32))
            self.own.append(g0 + own)
            self.nbr.append([g0 + row[k % len(row)] for k in range(self.K)])
        self.groups[name] = (np.arange(n0, self.N0 + len(self.x)), np.arange(g0, len(self.c["points"])))
        return g0


def with_edges(case):
    """`case` with the named edge groups appended (case['groups']: name -> (sample rows, Gaussian rows))."""
    e = _Edges(case)
    thin = lambda v, c=2: [0.05 if j != c else v for j in range(3)]
    # 1/scaling.clamp(min=1e-8): the clamped entry, the bound itself (torch's clamp passes the gradient at equality)
    # and one ulp above.  mu.z = 0 and x.z = 3e-9 make the shift exact, so w = 3e-9 / s stays O(1).
    e.group("inv_s_clamp", [((0.25 * i, 0, 0), thin(v), ID, 0.9) for i, v in enumerate((DOWN(1e-8), F32(1e-8), UP(1e-8)))],
            [((0.25 * i + dx, -0.015, 3e-9), i, [i, 0, 1, 2]) for i in range(3) for dx in (0.01, -0.02)])
    # min_scaling.clamp(min=1e-6) of the normal loss, tilted normals
    e.group("min_scaling_clamp", [((0.02 * i, 0.01 * i, 0), thin(v, i), TILT[i], 0.95)
                                  for i, v in enumerate((DOWN(1e-6), F32(1e-6), UP(1e-6)))],
            [((0.02 * i + dx, 0.01 * i - dx, 5e-7), i, [i, (i + 1) % 3, (i + 2) % 3]) for i in range(3)
             for dx in (0.004, -0.007)])
    # equal smallest scales: beta's ds column and the normal are the first minimum's
    tied = [(0.01, 0.01, 0.05), (0.05, 0.01, 0.01), (0.01, 0.05, 0.01), (0.01, 0.01, 0.01)]
    rng = np.random.default_rng(7)
    e.group("tied_scales", [((0.02 * i, 0, 0.01 * i), s, TILT[i], 0.9) for i, s in enumerate(tied)],
            [(np.array([0.02 * i, 0, 0.01 * i]) + 0.015 * rng.normal(size=3), i, [i, (i + 1) % 4, (i + 2) % 4, (i + 3) % 4])
             for i in range(4) for _ in range(3)])
    # identity quaternions with different thin columns: the normals are z, x, y and <n_k, n_own> is exactly 0
    e.group("orthogonal_normals", [((0, 0, 0), thin(0.005, 2), ID, 0.9), ((0.03, 0, 0), thin(0.005, 0), ID, 0.9),
                                   ((0, 0.03, 0), thin(0.005, 1), ID, 0.9), ((0.02, 0.02, 0), thin(0.004, 2), TILT[2], 0.8)],
            [((0.01, 0.012, 0.002), 0, [0, 1, 2, 3]), ((0.02, 0.003, -0.001), 0, [0, 1, 2, 3]),
             ((0.025, 0.004, 0.003), 1, [1, 0, 2, 3]), ((0.002, 0.025, 0.003), 2, [2, 0, 1, 3])])
    # a sample exactly on its Gaussian's plane: e = 0
    e.group("on_plane", [((0, 0, 0), thin(0.001), ID, 0.9), ((0.03, 0, 0.002), thin(0.002), TILT[0], 0.9)],
            [((0.01, 0.02, 0), 0, [0, 1]), ((-0.02, 0.005, 0), 0, [0, 1])])
    # every neighbour weight 0 (all on the sample's plane): wsum is clamped to 1e-6, the loss is |n_own|^2
    e.group("zero_weights", [((0.03 * i, 0.01 * i, 0), (0.05, 0.03, 0.001), ID, 0.9) for i in range(3)],
            [((0.01, 0.005, 0), 0, [0, 1, 2]), ((0.04, 0.0, 0), 1, [1, 0, 2])])
    # Mahalanobis^2 across its 1e8 clamp: s = 1e-6 and the sample ~1e-2 off the plane (a round neighbour keeps rho > 0)
    e.group("mahalanobis_clamp", [((0, 0, 0), thin(F32(1e-6)), ID, 0.9), ((0, 0, 0.01), (0.05, 0.04, 0.06), ID, 0.9)],
            [((0.003, 0.001, 1e-2 * (1 + d)), 0, [0, 1]) for d in (-1e-3, -1e-6, 0.0, 1e-6, 1e-3)])
    # samples far from every neighbour: rho underflows below opacity_min_clamp, or to 0
    e.group("far_samples", [((0, 0, 0), (0.02, 0.025, 0.015), TILT[3], 0.9), ((0, 0.01, 0), (0.02, 0.02, 0.02), ID, 0.9)],
            [((0.02 * np.sqrt(d2), -0.005, 0), 0, [0, 1]) for d2 in (60.0, 70.0, 75.0, 80.0, 1e6)])
    # sdf_grad on both sides of +-10: a thin tilted Gaussian, its other neighbour slots a far round one (beta ~ 0.1)
    qt = np.asarray(TILT[1], np.float64)
    n = _rot(qt[None])[0][:, 0]
    e.group("sdf_grad_clip", [((0, 0, 0), (0.001, 0.05, 0.05), TILT[1], 0.95), ((5, 0, 0), (0.1, 0.12, 0.08), ID, 0.9)],
            [(sgn * t * 0.001 * n + (0.003, -0.002, 0.001), 0, [0, 1]) for t in np.geomspace(0.01, 3, 10)
             for sgn in (1, -1)])
    # three coincident Gaussians: rho >= 1 at density factor 1 (the sdf's gradient is non-finite there in the
    # reference's float32 chain, and no trainer reaches it: forward values only)
    e.group("dense_center", [((0.001 * i, 0, 0), (0.05, 0.04, 0.03), ID, 0.95) for i in range(3)],
            [((0.004 * s, 0.003, -0.002), 0, [0, 1, 2]) for s in (-1, 0, 1)])
    out = dict(case)
    for k, v in e.c.items():
        out[k] = np.ascontiguousarray(np.array(v), np.float32)
    out["x"] = np.ascontiguousarray(np.r_[case["x"], np.array(e.x, np.float32).reshape(-1, 3)], np.float32)
    out["gaussian_idx"] = np.r_[case["gaussian_idx"], np.array(e.own, np.int64)]
    out["nbr_idx"] = np.ascontiguousarray(np.r_[case["nbr_idx"], np.array(e.nbr, np.int64).reshape(-1, e.K)])
    out["groups"] = e.groups
    return out


# ------------------------------------------------------------------------------------------------------- oracles
def weights(N, K, seed=1):
    rng = np.random.default_rng(seed)
    return {"density": rng.normal(size=N), "sdf": rng.normal(size=N), "beta": rng.normal(size=N),
            "closest_gaussian_opacities": rng.normal(size=(N, K)), "normal": rng.normal(size=N),
            "densest": rng.normal(size=N)}


def field_weights(case):
    """The field's output weights.  At density factor 1 the sdf is left out of the loss: rho >= 1 makes its gradient
    non-finite in the reference (its values are still checked)."""
    N, K = case["nbr_idx"].shape
    w = weights(N, K)
    keys = FIELD_OUTPUTS if case["density_factor"] < 1 else ("density", "beta", "closest_gaussian_opacities")
    return {k: w[k] for k in keys}


def _leaves(case, dtype, perturb=None):
    arr = {k: case[k] for k in LEAVES}
    if perturb:
        arr = perturb(dict(arr))
    return {k: torch.from_numpy(np.ascontiguousarray(arr[k])).to(dtype).clone().requires_grad_(True) for k in LEAVES}


def _order(case, order):
    """The column permutation of each sample's neighbours: None, 'reversed' or a seed."""
    N, K = case["nbr_idx"].shape
    if order is None:
        return np.arange(K)
    if order == "reversed":
        return np.arange(K)[::-1].copy()
    return np.random.default_rng(order).permutation(K)


def field_oracle(case, w, dtype, order=None, perturb=None):
    """Values (density, beta, sdf, closest_gaussian_opacities, sdf_grad) and the gradients of sum_k w_k . out_k,
    float64 numpy, with the neighbour columns in `order` (outputs reported in the original column order)."""
    perm = _order(case, order)
    inv = np.argsort(perm)
    leaf = _leaves(case, dtype, perturb)
    nbr = torch.from_numpy(case["nbr_idx"][:, perm])
    out = fo.field_values_torch(leaf["x"], nbr, leaf["points"], leaf["scaling"], leaf["quaternions"],
                                leaf["strengths"], case["density_factor"], 1.0, return_sdf_grad=True)
    loss = 0
    for k, v in w.items():
        wk = v[:, perm] if k == "closest_gaussian_opacities" else v
        loss = loss + (out[k] * torch.from_numpy(np.ascontiguousarray(wk)).to(dtype)).sum()
    loss.backward()
    vals = {k: out[k].detach().double().numpy() for k in FIELD_OUTPUTS + ("sdf_grad",)}
    vals["closest_gaussian_opacities"] = vals["closest_gaussian_opacities"][:, inv]
    return vals, {k: v.grad.double().numpy() for k, v in leaf.items()}


def normal_oracle(case, opac, w, dtype, order=None, perturb=None):
    perm = _order(case, order)
    leaf = _leaves(case, dtype, perturb)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a))
    loss = fo.better_normal_loss_torch(leaf["x"].detach(), t(case["gaussian_idx"]), t(case["nbr_idx"][:, perm]),
                                       leaf["points"].detach(), leaf["scaling"].detach(), leaf["quaternions"],
                                       t(opac[:, perm]).to(dtype))
    (loss * t(w).to(dtype)).sum().backward()
    return {"normal": loss.detach().double().numpy()}, {"quaternions": leaf["quaternions"].grad.double().numpy()}


def densest_oracle(case, w, dtype, order=None, perturb=None):
    perm = _order(case, order)
    inv = np.argsort(perm)
    leaf = _leaves(case, dtype, perturb)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a))
    loss, opac = deo.density_estimation_loss_torch(leaf["x"], t(case["gaussian_idx"]), t(case["nbr_idx"][:, perm]),
                                                   leaf["points"], leaf["scaling"], leaf["quaternions"],
                                                   leaf["strengths"], case["density_factor"], True)
    (loss * t(w).to(dtype)).sum().backward()
    vals = {"densest": loss.detach().double().numpy(),
            "closest_gaussian_opacities": opac.double().numpy()[:, inv]}
    return vals, {k: v.grad.double().numpy() for k, v in leaf.items()}


def probes(run, *args):
    """run(*args, dtype, order) in float64, float32 and float32 with the neighbour columns reversed."""
    return run(*args, torch.float64), run(*args, torch.float32), run(*args, torch.float32, "reversed")


# ---------------------------------------------------------------------------------------------------------- rule
def normal_exclusions(case):
    """bool [N]: samples with a neighbour whose |<n_k, n_own>| is in (0, SIGN_EPS], or whose own or neighbour
    Gaussians have two smallest scales 1 ulp apart."""
    s = case["scaling"]
    t = lambda k: torch.from_numpy(case[k]).double()
    n = fo.smallest_axis(t("scaling"), t("quaternions")).numpy()
    dot = np.abs(np.einsum("nkc,nc->nk", n[case["nbr_idx"]], n[case["gaussian_idx"]]))
    ss = np.sort(s, 1)
    near_tie = (ss[:, 1] != ss[:, 0]) & (np.nextafter(ss[:, 0], F32(np.inf)) >= ss[:, 1])
    return (((dot > 0) & (dot <= SIGN_EPS)).any(1) | near_tie[case["nbr_idx"]].any(1) |
            near_tie[case["gaussian_idx"]])


def _p(o32, o32r, o64, ours2=None, ours=None):
    p = np.maximum(np.abs(o32 - o64), np.abs(o32r - o64))
    if ours2 is not None:
        p = p + 2.0 * np.abs(np.asarray(ours, np.float64) - np.asarray(ours2, np.float64))
    return p


def value_scale(k, case, v64):
    """The `scale` of a value's floor: density_factor for densities and opacities, beta for the sdf, rho for the
    density-estimation loss |rho - target|, and |v| + 1e-6 for the normal loss |v|^2 (its error is 2 |v| |dv| + |dv|^2,
    with |dv| a few float32 ulps of the unit normals)."""
    if k in ("density", "closest_gaussian_opacities"):
        return case["density_factor"]
    if k == "sdf":
        return np.abs(v64["beta"]) if "beta" in v64 else field_oracle_beta(case)
    if k == "densest":
        return np.abs(v64["closest_gaussian_opacities"].sum(1))
    if k == "normal":
        return np.sqrt(np.abs(v64["normal"])) + 1e-6
    return 0.0


def value_bound(k, v64, v32, v32r, scale, ours=None, ours2=None, model=None):
    """floor_v (|v64| + scale) + 3 p, plus 2 E for the values term_error bounds (E is passed as `model`)."""
    floor = VALUE_FLOOR[k] * (np.abs(v64) + scale)
    b = floor + 3.0 * _p(v32, v32r, v64, ours2, ours)
    return (b if model is None else b + 2.0 * model), floor


def grad_bound(kind, leaf, g64, g32, g32r, rows, ours=None, ours2=None, model=None):
    """The allowance of each entry of g [R, C] for the rows of one group, its floor part and its 2 G part (G the
    per-term rounding bound grad_term_error, passed as `model`)."""
    g64 = g64.reshape(len(g64), -1)
    sh = lambda a: None if a is None else np.asarray(a).reshape(g64.shape)
    gmax = np.abs(g64[rows]).max() if len(rows) else 0.0
    floor = np.broadcast_to(GRAD_FLOOR.get(kind, {}).get(leaf, 1e-6) * gmax, g64.shape)
    b = (1e-4 * np.abs(g64).max(1, keepdims=True) + 4.0 * _p(sh(g32), sh(g32r), g64, sh(ours2), sh(ours)) + floor)
    gm = np.zeros(g64.shape) if model is None else 2.0 * sh(model)
    return b + gm, floor, gm


def check(kind, case, got, ref, got2=None, excluded=None, value_keys=None, model=None, gmodel=None):
    """Hold `got` = (values, grads) to the rule against ref = probes(...), gradients with gmodel = grad_term_error(...)
    when given.  Returns a report {(group, tensor): dict(ratio, worst, n_over, rows, floor_dominated)}; a gradient's
    entry also has g_dominated (the share of rows whose allowance 2 G dominates) and `by`, what dominates the worst
    row's allowance ('floor', 'G' or 'p', the 1e-4 and float32-order part)."""
    (v64, g64), (v32, g32), (v32r, g32r) = ref
    vals, grads = got
    vals2, grads2 = got2 if got2 is not None else (None, None)
    rep = {}
    keep = np.ones(len(case["x"]), bool) if excluded is None else ~excluded
    for k in (value_keys or vals):
        b, fl = value_bound(k, v64[k], v32[k], v32r[k], value_scale(k, case, v64), vals[k],
                            None if vals2 is None else vals2[k], None if model is None else model.get(k))
        for gname, (srows, _) in case["groups"].items():
            rows = srows[keep[srows]]
            r = h.row_errors(vals[k][rows], v64[k][rows], b[rows])
            rep[(gname, k)] = dict(ratio=r["ratio"], worst=int(rows[r["worst_row"]]) if len(rows) else -1,
                                   n_over=r["n_over"], rows=len(rows),
                                   floor_dominated=float((fl[rows] * 2 >= b[rows]).mean()) if len(rows) else 0.0)
    for k in grads:
        for gname, (srows, grows) in case["groups"].items():
            if (kind, gname, k) in NOISE_ONLY:
                continue
            rows = srows[keep[srows]] if k == "x" else grows
            b, fl, gm = grad_bound(kind, k, g64[k], g32[k], g32r[k], rows, grads[k],
                                   None if grads2 is None else grads2[k], None if gmodel is None else gmodel[k])
            want = g64[k].reshape(len(g64[k]), -1)
            r = h.row_errors(np.asarray(grads[k]).reshape(want.shape)[rows], want[rows], b[rows])
            by = "-"
            if len(rows):
                i, c = rows[r["worst_row"]], r["worst_col"]
                by = max((fl[i, c], "floor"), (gm[i, c], "G"), (b[i, c] - fl[i, c] - gm[i, c], "p"))[1]
            rep[(gname, "d" + k)] = dict(ratio=r["ratio"], worst=int(rows[r["worst_row"]]) if len(rows) else -1,
                                         n_over=r["n_over"], rows=len(rows), by=by,
                                         floor_dominated=float((fl[rows] * 2 >= b[rows]).mean()) if len(rows) else 0.0,
                                         g_dominated=float((gm[rows] * 2 >= b[rows]).mean()) if len(rows) else 0.0)
    return rep


def field_oracle_beta(case):
    s = case["scaling"].astype(np.float64).min(1)
    return s[case["nbr_idx"]].mean(1)


def failures(rep):
    """{(group, tensor): (worst ratio, worst row, rows over, what dominates the worst row's allowance)}"""
    return {k: (round(v["ratio"], 3), v["worst"], v["n_over"], v.get("by", "-")) for k, v in rep.items() if v["n_over"]}


def worst(rep):
    """The largest error over allowance per tensor, over all groups."""
    out = {}
    for (g, k), v in rep.items():
        if v["ratio"] >= out.get(k, (0.0, None))[0]:
            out[k] = (round(v["ratio"], 3), g)
    return out


# ------------------------------------------------------------------------------------------- per-term error model
U = 2.0 ** -24     # float32 unit roundoff
C_TERM = 16.0      # roundings of one term (sh = x - mu, the entries of R(q), the 3-term dot, 1/s, the squares, expf), x2


def term_error(case):
    """First-order bounds on the rounding of a float32 evaluation of the forward values, float64 [N, K] / [N].

    Two neighbour orders of the float32 oracle only sample the rounding of the sums; every per-term rounding is the
    same in both, so at an entry where the oracle happens to land near float64 they say nothing about a kernel that
    rounds the same term differently.  On flat Gaussians that per-term rounding dominates: u_j = sum_i R_ij sh_i
    cancels (|u_j| ~ s_j while |sh| ~ the in-plane scale), and the Mahalanobis term w_j = u_j / s_j carries an
    absolute error of a few U (sum_i |R_ij||sh_i| + |sh|_1) / s_j, which the exponent turns into a relative error of
    o of sum_j |w_j| times that.  This bound holds for any order of the same operations (test_field_rows_cpu checks
    that it holds for the float32 oracle in every order it runs).
        opacity   E_o = o (C U sum_j |w_j| / s_j (sum_i |R_ij||sh_i| + |sh|_1) + C U (d2 + 1))
        density   E_rho = sum_k E_o + K U sum_k o
        sdf       beta / (rho sqrt(-2 ln rho)) E_rho, 0 where rho is clamped
        densest   E_rho + t (|e| / beta^2 dE + e^2 / beta^2 K U + C U), dE = C U (sum_i |d_i||n_i| + |d|_1)"""
    t = lambda k: torch.from_numpy(np.ascontiguousarray(case[k])).double()
    nb = torch.from_numpy(case["nbr_idx"])
    R = fo.quaternion_to_matrix(t("quaternions"))
    inv = 1.0 / t("scaling").clamp(min=float(F32(1e-8)))
    sh = t("x")[:, None] - t("points")[nb]                                   # [N, K, 3]
    Rk = R[nb]                                                               # [N, K, 3, 3]
    u = torch.einsum("nkij,nki->nkj", Rk, sh)
    a = torch.einsum("nkij,nki->nkj", Rk.abs(), sh.abs()) + sh.abs().sum(-1, keepdim=True)
    w = u * inv[nb]
    d2raw = (w * w).sum(-1)
    d2 = d2raw.clamp(0.0, 1e8)
    o = case["density_factor"] * t("strengths")[nb] * torch.exp(-0.5 * d2)
    E_o = o * (C_TERM * U * (w.abs() * inv[nb] * a).sum(-1) + C_TERM * U * (d2 + 1.0))
    K = nb.shape[1]
    rho = o.sum(1)
    E_rho = E_o.sum(1) + K * U * o.sum(1)
    beta = t("scaling").min(1)[0][nb].mean(1)
    omc = float(F32(1e-16))
    cl = torch.where(rho >= 1.0, rho / (rho + 1e-12), rho).clamp(min=omc)
    root = torch.sqrt(-2.0 * torch.log(cl))
    E_sdf = torch.where((rho > omc) & (rho < 1.0), beta / (cl * root) * E_rho, torch.zeros_like(rho))
    gi = torch.from_numpy(case["gaussian_idx"])
    n = fo.smallest_axis(t("scaling"), t("quaternions"))[gi]
    d = t("x") - t("points")[gi]
    e = (d * n).sum(-1)
    dE = C_TERM * U * ((d.abs() * n.abs()).sum(-1) + d.abs().sum(-1))
    tgt = torch.exp(-0.5 * e * e / (beta * beta))
    E_t = tgt * (e.abs() / beta ** 2 * dE + e * e / beta ** 2 * K * U + C_TERM * U)
    f = lambda v: v.numpy()
    return {"closest_gaussian_opacities": f(E_o), "density": f(E_rho), "sdf": f(E_sdf), "beta": f(K * U * beta),
            "densest": f(E_rho + E_t)}


# ----------------------------------------------------------------------------------- per-term error model: gradients
# The backward kernels (field_pair_backward, densest_backward_kernel's lane-0 terms, normal_loss_backward_kernel and
# smallest_axis_backward) restated once, op for op, over an arithmetic `F`:
#   _Err   float64 values, each carrying a first-order bound on the absolute error of computing it in float32: every
#          result is rounded once (U |v|; expf 2 ulp) and carries its operands' errors through its partials, a group
#          sum of n terms adds (n - 1) U sum |c|, a per-Gaussian sum K U sum |c|.  grad_term_error is C_GRAD times that.
#   _F32   float32 torch, in the kernels' lane order (lane l takes slots l, l + G, ...; then the xor butterfly): a CPU
#          stand-in for the kernels (kernel_stand_in).
# Two neighbour orders of the float32 oracle only change the order of its sums.  On flat Gaussians the gradients'
# per-term rounding dominates (u = R^T (x - mu) cancels to ~s while |x - mu| is the in-plane scale, and dL/ds ~ 1/s^3
# amplifies it), and a kernel that rounds those terms differently misses a p-only allowance by orders of magnitude.
class _E:
    """A float64 value and a first-order bound on the absolute error of its float32 evaluation."""
    __slots__ = ("v", "e")

    def __init__(self, v, e=None):
        self.v = v
        self.e = torch.zeros_like(v) if e is None else e

    def __getitem__(self, i):
        return _E(self.v[i], self.e[i])

    def __add__(a, b):
        b = _lift(b)
        return _rnd(a.v + b.v, a.e + b.e)

    def __sub__(a, b):
        b = _lift(b)
        return _rnd(a.v - b.v, a.e + b.e)

    def __mul__(a, b):
        b = _lift(b)
        return _rnd(a.v * b.v, a.e * b.v.abs() + b.e * a.v.abs())

    def __truediv__(a, b):
        b = _lift(b)
        v = a.v / b.v
        return _rnd(v, (a.e + v.abs() * b.e) / b.v.abs())

    __radd__ = lambda a, b: _lift(b) + a
    __rsub__ = lambda a, b: _lift(b) - a
    __rmul__ = lambda a, b: _lift(b) * a
    __rtruediv__ = lambda a, b: _lift(b) / a
    __neg__ = lambda a: _E(-a.v, a.e)


def _lift(a):
    return a if isinstance(a, _E) else _E(torch.as_tensor(a, dtype=torch.float64))


def _rnd(v, e):
    return _E(v, e + U * v.abs())


def _group_width(K):
    G = 1
    while G < K and G < 32:
        G *= 2
    return G


class _Err:
    @staticmethod
    def exact(a):
        return _E(torch.from_numpy(np.asarray(a, np.float64)))

    val = staticmethod(lambda a: a.v)

    @staticmethod
    def exp(a):
        v = torch.exp(a.v)
        return _E(v, v * (a.e + 4 * U))

    @staticmethod
    def log(a):
        v = torch.log(a.v)
        return _E(v, a.e / a.v + 2 * U * v.abs())

    @staticmethod
    def sqrt(a):
        v = torch.sqrt(a.v)
        return _E(v, a.e / (2 * v) + U * v)

    @staticmethod
    def abs(a):
        return _E(a.v.abs(), a.e)

    @staticmethod
    def where(c, a, b):
        a, b = _lift(a), _lift(b)
        return _E(torch.where(c, a.v, b.v), torch.where(c, a.e, b.e))

    @staticmethod
    def group(a):
        n = a.v.shape[1]
        return _E(a.v.sum(1), a.e.sum(1) + (n - 1) * U * a.v.abs().sum(1))

    @staticmethod
    def scatter(P, idx, a, K):
        z = lambda t: torch.zeros(P, dtype=torch.float64).index_add_(0, idx, t.reshape(-1))
        return _E(z(a.v), z(a.e) + K * U * z(a.v.abs()))


class _F32:
    @staticmethod
    def exact(a):
        return torch.from_numpy(np.ascontiguousarray(a, np.float32))

    val = staticmethod(lambda a: a)
    exp, log, sqrt, abs = torch.exp, torch.log, torch.sqrt, torch.abs

    @staticmethod
    def where(c, a, b):
        f = lambda t: t if torch.is_tensor(t) else torch.tensor(t, dtype=torch.float32)
        return torch.where(c, f(a), f(b))

    @staticmethod
    def lanes(a):
        """The G lanes' partial sums of a [N, K] (lane l: slots l, l + G, ... in order)."""
        K = a.shape[1]
        G = _group_width(K)
        out = []
        for l in range(G):
            s = torch.zeros(a.shape[0], dtype=torch.float32)
            for k in range(l, K, G):
                s = s + a[:, k]
            out.append(s)
        return out

    @staticmethod
    def group(a):
        s = _F32.lanes(a)
        o = len(s) // 2
        while o:
            s = [s[l] + s[l ^ o] for l in range(len(s))]
            o //= 2
        return s[0]

    @staticmethod
    def scatter(P, idx, a, K):
        return torch.zeros(P, dtype=torch.float32).index_add_(0, idx, a.reshape(-1))


def _quat_rot(q):
    """quat_to_rot: R (rows of columns) and two_s of q = (r, i, j, k)."""
    r, i, j, k = q
    ts = 2.0 / (r * r + i * i + j * j + k * k)
    m = [[1 - ts * (j * j + k * k), ts * (i * j - k * r), ts * (i * k + j * r)],
         [ts * (i * j + k * r), 1 - ts * (i * i + k * k), ts * (j * k - i * r)],
         [ts * (i * k - j * r), ts * (j * k + i * r), 1 - ts * (i * i + j * j)]]
    return m, ts


def _rot_backward(A, q, ts):
    qr, qi, qj, qk = q
    dts = (A[0][0] * -(qj * qj + qk * qk) + A[0][1] * (qi * qj - qk * qr) + A[0][2] * (qi * qk + qj * qr) +
           A[1][0] * (qi * qj + qk * qr) + A[1][1] * -(qi * qi + qk * qk) + A[1][2] * (qj * qk - qi * qr) +
           A[2][0] * (qi * qk - qj * qr) + A[2][1] * (qj * qk + qi * qr) + A[2][2] * -(qi * qi + qj * qj))
    c = -ts * ts * dts
    dqr = ts * (-qk * A[0][1] + qj * A[0][2] + qk * A[1][0] - qi * A[1][2] - qj * A[2][0] + qi * A[2][1]) + c * qr
    dqi = ts * (qj * (A[0][1] + A[1][0]) + qk * (A[0][2] + A[2][0]) + qr * (A[2][1] - A[1][2]) -
                2.0 * qi * (A[1][1] + A[2][2])) + c * qi
    dqj = ts * (qi * (A[0][1] + A[1][0]) + qr * (A[0][2] - A[2][0]) + qk * (A[1][2] + A[2][1]) -
                2.0 * qj * (A[0][0] + A[2][2])) + c * qj
    dqk = ts * (qr * (A[1][0] - A[0][1]) + qi * (A[0][2] + A[2][0]) + qj * (A[1][2] + A[2][1]) -
                2.0 * qk * (A[0][0] + A[1][1])) + c * qk
    return [dqr, dqi, dqj, dqk]


def _axis_backward(F, col, q, ts, dn):
    """smallest_axis_backward: dL/dR is dn in column `col`."""
    A = [[F.where(col == j, dn[i], 0.0) for j in range(3)] for i in range(3)]
    return _rot_backward(A, q, ts)


def _column(F, m, col):
    return [F.where(col == 0, m[i][0], F.where(col == 1, m[i][1], m[i][2])) for i in range(3)]


def _pair_backward(F, x, mu, strength, q, invs, s_ok, col, df, Gk, gbK):
    """field_pair_backward over all (sample, slot) pairs: dL/dx (= -dL/dmu), dL/dsigma, dL/dq, dL/ds."""
    m, ts = _quat_rot(q)
    sh = [x[i] - mu[i] for i in range(3)]
    u = [m[0][j] * sh[0] + m[1][j] * sh[1] + m[2][j] * sh[2] for j in range(3)]
    w = [u[j] * invs[j] for j in range(3)]
    d2raw = w[0] * w[0] + w[1] * w[1] + w[2] * w[2]
    big = F.val(d2raw) > 1e8
    e = df * F.exp(-0.5 * F.where(big, 1e8, d2raw))
    o = strength * e
    dsig = Gk * e
    dd2 = F.where(big, 0.0, Gk * o * -0.5)
    du, ds = [], []
    for j in range(3):
        dw = dd2 * 2.0 * w[j]
        du.append(dw * invs[j])
        dsj = F.where(s_ok[j], -(dw * u[j]) * invs[j] * invs[j], 0.0)
        ds.append(F.where(col == j, dsj + gbK, dsj))
    dsh = [m[i][0] * du[0] + m[i][1] * du[1] + m[i][2] * du[2] for i in range(3)]
    A = [[sh[i] * du[j] for j in range(3)] for i in range(3)]
    return dsh, dsig, _rot_backward(A, q, ts), ds


def _first_min(s):
    return torch.from_numpy(np.argmin(np.asarray(s), 1))


def _kernel_backward(case, kind, w, F, opac=None):
    """The kernels' gradients of sum_n w_n . out_n under F: {leaf: [rows, C]} (and, for the float32 stand-in, the
    per-pair and per-lane pieces the planted defects of the CPU tests take out)."""
    N, K = case["nbr_idx"].shape
    P = len(case["points"])
    nb, gi = torch.from_numpy(case["nbr_idx"]), torch.from_numpy(case["gaussian_idx"])
    sraw = case["scaling"]
    xs, pts, qs = F.exact(case["x"]), F.exact(case["points"]), F.exact(case["quaternions"])
    x = [xs[:, i:i + 1] for i in range(3)]
    mu = [pts[:, i][nb] for i in range(3)]
    q = [qs[:, c][nb] for c in range(4)]
    col_g = _first_min(sraw)
    extra = {}
    if kind == "normal":
        # normal_pack_kernel: n, 1 / max(s_col, 1e-6)^2
        mg, _ = _quat_rot([qs[:, c] for c in range(4)])
        ng = _column(F, mg, col_g)
        cmin = F.exact(np.maximum(sraw[np.arange(P), col_g.numpy()], F32(1e-6)))
        cg = 1.0 / (cmin * cmin)
        n_k = [ng[i][nb] for i in range(3)]
        n0 = [ng[i][gi][:, None] for i in range(3)]
        dot = n_k[0] * n0[0] + n_k[1] * n0[1] + n_k[2] * n0[2]
        sg = torch.sign(F.val(dot))
        op = F.exact(opac)
        wk = op * F.abs(((x[0] - mu[0]) * n_k[0] + (x[1] - mu[1]) * n_k[1] + (x[2] - mu[2]) * n_k[2]) * sg) * cg[nb]
        wsum = F.group(wk)
        sv = [F.group(wk * sg * n_k[i]) for i in range(3)]
        inv = 1.0 / F.where(F.val(wsum) < 1e-6, 1e-6, wsum)
        v = [n0[i][:, 0] - sv[i] * inv for i in range(3)]
        g2 = 2.0 * F.exact(w)
        c = -g2[:, None] * (wk * inv[:, None]) * sg
        idx = torch.cat([gi, nb.reshape(-1)])
        dn = [F.scatter(P, idx, _cat(F, [g2 * v[i], c * v[i][:, None]]), K) for i in range(3)]
        qg = [qs[:, c] for c in range(4)]
        dq = _axis_backward(F, col_g, qg, _quat_rot(qg)[1], dn)
        return {"quaternions": _stack(F, dq)}, {"normal": v[0] * v[0] + v[1] * v[1] + v[2] * v[2]}
    # pass 1: rho and beta of the sample in the forward's lane order
    st = F.exact(case["strengths"])[nb]
    invs_g = 1.0 / F.exact(np.maximum(sraw, F32(1e-8)))
    invs = [invs_g[:, j][nb] for j in range(3)]
    m, _ = _quat_rot(q)
    sh = [x[i] - mu[i] for i in range(3)]
    wv = [(m[0][j] * sh[0] + m[1][j] * sh[1] + m[2][j] * sh[2]) * invs[j] for j in range(3)]
    d2 = wv[0] * wv[0] + wv[1] * wv[1] + wv[2] * wv[2]
    dens = F.group(case["density_factor"] * st * F.exp(-0.5 * F.where(F.val(d2) > 1e8, 1e8, d2)))
    b = F.group(F.exact(sraw.min(1))[nb]) / float(K)
    zero = F.exact(np.zeros(N))
    if kind == "field":
        gd = F.exact(w["density"]) if "density" in w else zero
        gb = F.exact(w["beta"]) if "beta" in w else zero
        if "sdf" in w:                        # sdf_from_density, sdf_offset = 0 at density_threshold 1
            gs = F.exact(w["sdf"])
            ge1 = F.val(dens) >= 1.0
            d = F.where(ge1, dens / (dens + 1e-12), dens)
            dd = F.where(ge1, 1.0 / (dens + 1e-12), 1.0)
            low = F.val(d) < float(F32(1e-16))
            cl = F.where(low, float(F32(1e-16)), d)
            dd = F.where(low, 0.0, dd)
            root = F.sqrt(-2.0 * F.log(cl))
            gb = gb + gs * root
            gd = F.where(F.val(dd) != 0, gd + gs * (-b / (cl * root)) * dd, gd)
        Gk = gd[:, None]
        if "closest_gaussian_opacities" in w:
            Gk = Gk + F.exact(w["closest_gaussian_opacities"])
    else:                                     # densest: |rho - t| at lane 0
        og = [qs[:, c][gi] for c in range(4)]
        mo, tso = _quat_rot(og)
        n = _column(F, mo, col_g[gi])
        dvec = [xs[:, i] - pts[:, i][gi] for i in range(3)]
        e = dvec[0] * n[0] + dvec[1] * n[1] + dvec[2] * n[2]
        t = F.exp(-0.5 * (e * e) / (b * b))
        s = torch.sign(F.val(dens - t)) * F.exact(w)
        ib2 = 1.0 / (b * b)
        gd, gb, ge = s, -s * t * (e * e) * ib2 / b, s * t * e * ib2
        Gk = gd[:, None]
    col = col_g[nb]
    s_ok = [torch.from_numpy(sraw[:, j] >= F32(1e-8))[nb] for j in range(3)]
    dsh, dsig, dq, ds = _pair_backward(F, x, mu, st, q, invs, s_ok, col, case["density_factor"], Gk,
                                       (gb / float(K))[:, None])
    dx = [F.group(dsh[i]) for i in range(3)]
    per_pair = {"points": [-v for v in dsh], "strengths": [dsig], "quaternions": dq, "scaling": ds}
    own = {}
    if kind == "densest":
        dx = [dx[i] + ge * n[i] for i in range(3)]
        own = {"points": [-ge * n[i] for i in range(3)],
               "quaternions": _axis_backward(F, col_g[gi], og, tso, [ge * dvec[i] for i in range(3)])}
    if F is _F32:
        extra = {"pair": per_pair, "lanes": [_F32.lanes(v) for v in dsh], "gbK": gb / float(K)}
    out = {"x": _stack(F, dx)}
    for k, cs in per_pair.items():
        rows = []
        for c, v in enumerate(cs):
            if k in own:
                rows.append(F.scatter(P, torch.cat([nb.reshape(-1), gi]), _cat(F, [v, own[k][c]]), K))
            else:
                rows.append(F.scatter(P, nb.reshape(-1), v, K))
        out[k] = _stack(F, rows)
    return out, extra


def _cat(F, parts):
    flat = lambda a: a.reshape(-1)
    if F is _Err:
        return _E(torch.cat([flat(p.v) for p in parts]), torch.cat([flat(p.e) for p in parts]))
    return torch.cat([flat(p) for p in parts])


def _stack(F, cols):
    if F is _Err:
        return _E(torch.stack([c.v for c in cols], 1), torch.stack([c.e for c in cols], 1))
    return torch.stack(cols, 1)


# The bound's own factor.  The float32 oracle evaluates the same gradients in another algebraic order
# (L^-1 = R diag(1/s) first, dL/dR summed over a Gaussian's pairs before one quaternion backward, dL/ds through
# d(1/s)), so its per-op roundings are not the stand-in's.  At C_GRAD = 1 the worst error over floor + G in test_field_grad_rows_cpu is 0.38
# for the stand-in and 0.38 for the oracle in four orders (k5's dL/dx; <= 0.22 for the normal's dL/dq), so no
# extra factor is needed.
C_GRAD = 1.0


def grad_term_error(case, kind, w, opac=None):
    """First-order bound G on the per-term float32 rounding of every gradient entry ('field', 'densest', 'normal'):
    {leaf: float64 array shaped like the gradient}.  w: field_weights(case) for 'field', the per-sample weights for
    'densest' and 'normal'; opac: the float32 neighbour opacities the normal loss is given."""
    rows, _ = _kernel_backward(case, kind, w, _Err, opac)
    return {k: C_GRAD * v.e.numpy().reshape(_shape(case, k)) for k, v in rows.items()}


def kernel_stand_in(case, kind, w, opac=None):
    """The kernels' float32 gradients on the CPU (grads, pieces): {leaf: float64 array}, and the per-pair and per-lane
    float32 pieces of the field and densest backwards."""
    rows, extra = _kernel_backward(case, kind, w, _F32, opac)
    return {k: v.double().numpy().reshape(_shape(case, k)) for k, v in rows.items()}, extra


def _shape(case, k):
    return {"x": case["x"].shape, "points": case["points"].shape, "scaling": case["scaling"].shape,
            "quaternions": case["quaternions"].shape, "strengths": case["strengths"].shape}[k]


def sdf_grad_error(case):
    """First-order bound on the float32 rounding of sdf_grad = beta / (rho sqrt(-2 ln rho)) (-d rho / dx), [N, 3]:
    the coefficient times the field backward's bound on d rho / dx (grad_term_error with a loss on the density alone),
    plus |d rho / dx| times the coefficient's own error (E_rho through (rho r)' = r - 1/r, r = sqrt(-2 ln rho), and
    beta's K U); without the E_rho part where rho is clamped below, and 0 at rho >= 1 (no trainer reaches it)."""
    N, K = case["nbr_idx"].shape
    ones = {"density": np.ones(N)}
    rows, _ = _kernel_backward(case, "field", ones, _Err)
    gx, Gx = rows["x"].v.numpy(), C_GRAD * rows["x"].e.numpy()
    t = lambda k: torch.from_numpy(np.ascontiguousarray(case[k])).double()
    v = fo.field_values_torch(t("x"), torch.from_numpy(case["nbr_idx"]), t("points"), t("scaling"), t("quaternions"),
                              t("strengths"), case["density_factor"])
    rho, beta = v["density"].numpy(), v["beta"].numpy()
    omc = float(F32(1e-16))
    live = (rho > omc) & (rho < 1.0)
    cl = np.where(live, rho, np.where(rho >= 1.0, 0.5, omc))
    r = np.sqrt(-2.0 * np.log(cl))
    coef = np.where(rho < 1.0, beta / np.maximum(cl * r, omc), 0.0)
    dcoef = coef * (np.where(live, np.abs(r - 1.0 / r) / (cl * r) * term_error(case)["density"], 0.0) + (K + 8) * U)
    return coef[:, None] * Gx + dcoef[:, None] * np.abs(gx)


def normal_value_error(case, opac):
    """First-order bound on the float32 rounding of the better-normal loss |v|^2 per sample, [N] (the same op-by-op
    propagation as grad_term_error through the normals, weights, their sums and v = n_own - sum_k w_k m_k)."""
    _, extra = _kernel_backward(case, "normal", np.zeros(len(case["x"])), _Err, opac)
    return C_GRAD * extra["normal"].e.numpy()
