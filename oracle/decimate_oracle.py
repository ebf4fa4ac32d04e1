"""Quadric edge-collapse decimation and open3d's mesh clean-up passes, in numpy (float64).

The reference ends both coarse-mesh extraction branches (sugar_extractors/coarse_mesh.py:433-463, :716-744) with

    decimated = mesh.simplify_quadric_decimation(decimation_target)        # open3d 0.17
    decimated.remove_degenerate_triangles(); decimated.remove_duplicated_triangles()
    decimated.remove_duplicated_vertices();  decimated.remove_non_manifold_edges()

with open3d's defaults maximum_error = inf and boundary_weight = 1.  This module restates those calls from open3d's
published algorithm (TriangleMesh::SimplifyQuadricDecimation and the four Remove* passes).  open3d is not installed
where this package is built or tested, so nothing here has been checked against open3d itself.  The rules below are
the rules this package implements; the CUDA op (csrc/sgr_decimate.cu) equals `decimate_rounds` array for array.

Arithmetic (float64, every product and sum rounded on its own, in the order written; the kernels use _rn intrinsics):
  * Plane of a face p0 p1 p2: n = (p1 - p0) x (p2 - p0), with (u x w)_x = u_y w_z - u_z w_y and cyclic; |n| =
    sqrt((n_x^2 + n_y^2) + n_z^2); unit normal = n / |n| per component; d = -((n_x p0_x + n_y p0_y) + n_z p0_z).
    If |n| = 0 the plane is zero (normal 0, d = 0).
  * Quadric of a plane (n, d) with weight w: A_ij = w (n_i n_j), b_i = (w d) n_i, c = (w d) d; stored as
    (A00, A01, A02, A11, A12, A22, b0, b1, b2, c).  Quadrics add component by component.
  * Face quadric: the face's plane, weight = its area 0.5 |n|.  Each vertex sums the quadrics of its faces in face
    order, starting from zero.
  * Boundary quadric (boundary_weight = 1): for each face slot k, edge (v0, v1) = (f[k], f[k+1 mod 3]), that belongs to
    exactly one face: the plane through v0 with unit normal m / |m|, m = (p1 - p0) x (the face's unit normal), zero if
    |m| = 0, weight 1; added to v0 and v1.  Once, at the start, after all face quadrics: each vertex walks its faces in
    face order and their slots 0, 1, 2, and adds the boundary quadric of every boundary slot it is an end of.
  * Edge cost of (a, b), a < b: Q = Q_a + Q_b.  With the cofactors C00 = A11 A22 - A12 A12, C01 = A02 A12 - A01 A22,
    C02 = A01 A12 - A02 A11, C11 = A00 A22 - A02 A02, C12 = A01 A02 - A00 A12, C22 = A00 A11 - A01 A01 and
    det = (A00 C00 + A01 C01) + A02 C02, A counts as invertible when |det| > 1e-4 (open3d's Quadric::IsInvertible: an
    absolute threshold, so whether the solve is used depends on the mesh's scale).  Then v = -t / det per component,
    t_i = (C_i0 b0 + C_i1 b1) + C_i2 b2 (the adjugate; open3d solves with an LDLT factorisation instead, which can
    differ in the last bits).  Otherwise v is the midpoint m = (p_a + p_b) * 0.5, replaced by p_a if cost(p_a) <
    cost(m), then by p_b if cost(p_b) < the cost so far: ties prefer the midpoint, then p_a, then p_b.
    cost(x) = (x.Ax + 2 b.x) + c with (Ax)_i = (A_i0 x0 + A_i1 x1) + A_i2 x2, x.Ax and b.x summed ((0 + 1) + 2).
    The cost gets + 0.0 (so -0 sorts with +0).  A NaN cost is never collapsed.
  * Key of an edge: (cost, a, b), compared lexicographically.  open3d leaves equal costs to its heap; the lower (a, b)
    first is this package's rule.
  * Flip test of collapsing (a, b) into v: for every live face of b that does not contain a, the unit normals before
    and after moving b to v (n / |n| per component) have dot product (x + y) + z < 0 -> the collapse is skipped.
    Only b's faces are tested, as in open3d.  A zero normal gives NaN, which does not count as a flip.
  * Collapse: delete the live faces that contain both a and b, rewrite b to a in the other faces of b, p_a = v,
    Q_a = Q_a + Q_b, colour_a = 0.5 (colour_a + colour_b) and the same for normals (kept in float64 until the end),
    b is dead.
  * After the loop: the live faces in index order; the vertices that a live face references, in index order.

decimate_greedy is the sequential loop: a min-heap of edge keys; while the face count is above the target, pop the
least key and skip it if it is stale (its edge was pushed again since), if a or b is dead, if no live face contains
the edge, or if it fails the flip test; otherwise collapse and push again every edge that a shares with a live face.
A skipped (flipped) edge returns only when it is pushed again that way.  Where it departs from open3d on purpose:
  * open3d keeps a popped edge whose faces were all deleted by earlier collapses in its heap and may collapse it;
    here, as in the rounds, an edge counts only while a live face contains it.
  * open3d keeps vertices that no face references any more; here they are dropped (the output holds only referenced
    vertices), and vertex colours and normals are averaged in float64 rather than in the mesh's storage type.

decimate_rounds is the parallel form the kernels compute.  Each round: every edge of a live face that is not blocked
and has a non-NaN cost is a candidate; vmin[v] = least key of v's candidate edges, fmin[f] = least vmin of f's
vertices, rmin[v] = least fmin of v's live faces; (a, b) is selected when its key equals rmin[a] and rmin[b].  No
face then holds vertices of two selected edges, so their collapses touch disjoint stars and applying them together
equals applying them one by one in key order.  The selected edges are flip-tested in the state at the round's start;
a failing edge is blocked (a flag on each face slot that holds the edge) until a or b survives a later collapse, which
is the greedy loop's "pushed again" rule.  The passing edges are accepted in key order while the face count is still
above the target; the removed-face count of the collapse that took it to the target or below is reported.  Accepted
collapses are applied, and the live faces compacted in order.  The loop stops at the target or when nothing can be
selected.  With max_collapses_per_round = 1 only the least key is considered per round, and the result equals
decimate_greedy exactly.

Clean-up passes, the reference's order (clean_mesh):
  * remove_degenerate_triangles: drop faces with two equal vertex ids.
  * remove_duplicated_triangles: faces equal up to rotation (not reflection) are duplicates; the first is kept.
  * remove_duplicated_vertices: vertices with exactly equal float64 coordinates (-0 equals +0) are merged into the
    first; its colour and normal are kept, faces are remapped and the kept vertices keep their order.
  * remove_non_manifold_edges: repeat until no edge has more than two faces: visit the edges with more than two faces
    in ascending (a, b) order (open3d visits them in hash-map order), and on each delete the smallest-area faces (area
    0.5 |n| as above; equal areas: the lower face index first) not yet deleted in this sweep until two remain; then
    drop the deleted faces.
  None of the passes drops vertices that no face references, as in open3d.
"""
import heapq
import math

import numpy as np

INV_DET = 1e-4


# ---------------------------------------------------------------------------------------------------------------------
# arithmetic shared by the scalar (Python float) and vector (numpy) paths
# ---------------------------------------------------------------------------------------------------------------------
def _is_vec(*xs):
    return any(isinstance(x, np.ndarray) for x in xs)


def _sqrt(x):
    return np.sqrt(x) if isinstance(x, np.ndarray) else math.sqrt(x)


def _div(x, y):
    if _is_vec(x, y):
        return x / y
    try:
        return x / y
    except ZeroDivisionError:
        if x != x or x == 0.0:
            return math.nan
        return math.copysign(math.inf, x) * math.copysign(1.0, y)


def _where(cond, x, y):
    if _is_vec(cond, x, y):
        return np.where(cond, x, y)
    return x if cond else y


def _cross(u, w):
    return (u[1] * w[2] - u[2] * w[1], u[2] * w[0] - u[0] * w[2], u[0] * w[1] - u[1] * w[0])


def _sub(p, q):
    return (p[0] - q[0], p[1] - q[1], p[2] - q[2])


def _norm(n):
    return _sqrt((n[0] * n[0] + n[1] * n[1]) + n[2] * n[2])


def _unit(n):
    ln = _norm(n)
    return (_div(n[0], ln), _div(n[1], ln), _div(n[2], ln)), ln


def _plane_through(nrm, p0):
    """Unit normal and offset of the plane through p0 with normal direction `nrm`; zero when |nrm| = 0."""
    u, ln = _unit(nrm)
    d = -((u[0] * p0[0] + u[1] * p0[1]) + u[2] * p0[2])
    z = ln == 0.0
    return (_where(z, 0.0, u[0]), _where(z, 0.0, u[1]), _where(z, 0.0, u[2])), _where(z, 0.0, d), ln


def _quadric(n, d, w):
    wd = w * d
    return (w * (n[0] * n[0]), w * (n[0] * n[1]), w * (n[0] * n[2]), w * (n[1] * n[1]), w * (n[1] * n[2]),
            w * (n[2] * n[2]), wd * n[0], wd * n[1], wd * n[2], wd * d)


def face_plane(p0, p1, p2):
    """-> (unit normal, d, |n|) of the face; zero plane when |n| = 0."""
    return _plane_through(_cross(_sub(p1, p0), _sub(p2, p0)), p0)


def _eval(q, x):
    A00, A01, A02, A11, A12, A22, b0, b1, b2, c = q
    ax = (A00 * x[0] + A01 * x[1]) + A02 * x[2]
    ay = (A01 * x[0] + A11 * x[1]) + A12 * x[2]
    az = (A02 * x[0] + A12 * x[1]) + A22 * x[2]
    vav = (x[0] * ax + x[1] * ay) + x[2] * az
    bv = (b0 * x[0] + b1 * x[1]) + b2 * x[2]
    return (vav + 2.0 * bv) + c


def edge_solution(Qa, Qb, pa, pb):
    """-> (cost, (vx, vy, vz)) of collapsing edge (a, b), a < b (module docstring)."""
    q = tuple(Qa[i] + Qb[i] for i in range(10))
    A00, A01, A02, A11, A12, A22, b0, b1, b2, c = q
    C00 = A11 * A22 - A12 * A12
    C01 = A02 * A12 - A01 * A22
    C02 = A01 * A12 - A02 * A11
    C11 = A00 * A22 - A02 * A02
    C12 = A01 * A02 - A00 * A12
    C22 = A00 * A11 - A01 * A01
    det = (A00 * C00 + A01 * C01) + A02 * C02
    inv = abs(det) > INV_DET
    vec = _is_vec(det, pa[0], pb[0])
    if vec or inv:
        t0 = (C00 * b0 + C01 * b1) + C02 * b2
        t1 = (C01 * b0 + C11 * b1) + C12 * b2
        t2 = (C02 * b0 + C12 * b1) + C22 * b2
        vi = (_div(-t0, det), _div(-t1, det), _div(-t2, det))
        ci = _eval(q, vi)
        if not vec:
            return ci + 0.0, vi
    m = ((pa[0] + pb[0]) * 0.5, (pa[1] + pb[1]) * 0.5, (pa[2] + pb[2]) * 0.5)
    cost, v = _eval(q, m), m
    ca, cb = _eval(q, pa), _eval(q, pb)
    t = ca < cost
    cost, v = _where(t, ca, cost), tuple(_where(t, pa[i], v[i]) for i in range(3))
    t = cb < cost
    cost, v = _where(t, cb, cost), tuple(_where(t, pb[i], v[i]) for i in range(3))
    if vec:
        cost = np.where(inv, ci, cost)
        v = tuple(np.where(inv, vi[i], v[i]) for i in range(3))
    return cost + 0.0, v


def flips(q0, q1, q2, slot, v):
    """True where moving corner `slot` of face (q0, q1, q2) to v turns its unit normal by more than 90 degrees."""
    before, _ = _unit(_cross(_sub(q1, q0), _sub(q2, q0)))
    r = [q0, q1, q2]
    if _is_vec(slot):
        r = [tuple(_where(slot == s, v[i], r[s][i]) for i in range(3)) for s in range(3)]
    else:
        r[slot] = v
    after, _ = _unit(_cross(_sub(r[1], r[0]), _sub(r[2], r[0])))
    return (before[0] * after[0] + before[1] * after[1]) + before[2] * after[2] < 0.0


def _rows(a):
    return tuple(a[:, i] for i in range(a.shape[1]))


# ---------------------------------------------------------------------------------------------------------------------
# set-up shared by both loops
# ---------------------------------------------------------------------------------------------------------------------
def _check(verts, faces):
    P = np.asarray(verts, np.float64).reshape(-1, 3).copy()
    F = np.asarray(faces, np.int64).reshape(-1, 3).copy()
    if F.size and (F.min() < 0 or F.max() >= len(P)):
        raise ValueError("face ids must lie in [0, V)")
    if ((F[:, 0] == F[:, 1]) | (F[:, 1] == F[:, 2]) | (F[:, 0] == F[:, 2])).any():
        raise ValueError("faces must not repeat a vertex")
    return P, F


def _incidence(F, V):
    """Vertex -> faces in face order as (order of corners sorted by (vertex, face), degree, rank of each corner)."""
    fid = np.repeat(np.arange(len(F)), 3)
    vid = F.reshape(-1)
    order = np.lexsort((fid, vid))
    deg = np.bincount(vid, minlength=V)
    start = np.concatenate([[0], np.cumsum(deg)[:-1]])
    rank = np.empty(len(vid), np.int64)
    rank[order] = np.arange(len(vid)) - start[vid[order]]
    return vid, fid, rank, deg


def initial_quadrics(P, F):
    """Per-vertex quadrics [V, 10]: face quadrics in face order, then boundary quadrics (module docstring)."""
    V = len(P)
    Q = np.zeros((V, 10))
    if not len(F):
        return Q
    with np.errstate(all="ignore"):
        p = [P[F[:, k]] for k in range(3)]
        n, d, ln = face_plane(_rows(p[0]), _rows(p[1]), _rows(p[2]))
        fq = np.stack(_quadric(n, d, 0.5 * ln), 1)
        e = np.sort(np.stack([F, np.roll(F, -1, 1)], 2).reshape(-1, 2), 1)
        _, inv, cnt = np.unique(e, axis=0, return_inverse=True, return_counts=True)
        boundary = (cnt[inv.reshape(-1)] == 1).reshape(-1, 3)
        bq = np.zeros((len(F), 3, 10))
        for k in range(3):
            v0, v1 = p[k], p[(k + 1) % 3]
            m = _cross(_rows(v1 - v0), n)
            bn, bd, _ = _plane_through(m, _rows(v0))
            bq[:, k] = np.stack(_quadric(bn, bd, 1.0), 1)
    vid, fid, rank, deg = _incidence(F, V)
    for r in range(int(deg.max())):
        s = rank == r
        Q[vid[s]] += fq[fid[s]]
    for r in range(int(deg.max())):
        s = rank == r
        v, f = vid[s], fid[s]
        for k in range(3):
            t = boundary[f, k] & ((F[f, k] == v) | (F[f, (k + 1) % 3] == v))
            Q[v[t]] += bq[f[t], k]
    return Q


def _finish(P, F, colors, normals, rounds, last_removed):
    ref = np.zeros(len(P), bool)
    ref[F.reshape(-1)] = True
    remap = np.cumsum(ref) - 1
    return {"verts": P[ref], "faces": remap[F].reshape(-1, 3).astype(np.int64),
            "colors": None if colors is None else colors[ref], "normals": None if normals is None else normals[ref],
            "rounds": rounds, "last_removed": last_removed}


def _attr(x, V):
    return None if x is None else np.asarray(x, np.float64).reshape(V, 3).copy()


# ---------------------------------------------------------------------------------------------------------------------
# the sequential loop
# ---------------------------------------------------------------------------------------------------------------------
def decimate_greedy(verts, faces, target, colors=None, normals=None):
    """The sequential heap loop (module docstring) -> dict verts f64 [V',3], faces i64 [F',3], colors, normals,
    rounds (0), last_removed (faces removed by the collapse that reached the target, else 0)."""
    P0, F0 = _check(verts, faces)
    V = len(P0)
    Qa = initial_quadrics(P0, F0)
    col, nrm = _attr(colors, V), _attr(normals, V)
    P = [tuple(r) for r in P0.tolist()]
    Q = [tuple(r) for r in Qa.tolist()]
    F = F0.tolist()
    vf = [[] for _ in range(V)]
    for i, f in enumerate(F):
        for v in f:
            vf[v].append(i)
    alive = [True] * V
    fdead = [False] * len(F)
    current = {}
    heap = []

    def push(x, y):
        a, b = (x, y) if x < y else (y, x)
        cost, v = edge_solution(Q[a], Q[b], P[a], P[b])
        current[(a, b)] = (cost, v)
        if cost == cost:
            heapq.heappush(heap, (cost, a, b))

    for f in F:
        for k in range(3):
            e = (min(f[k], f[(k + 1) % 3]), max(f[k], f[(k + 1) % 3]))
            if e not in current:
                push(*e)
    n_f = len(F)
    last_removed = 0
    while n_f > int(target) and heap:
        cost, a, b = heapq.heappop(heap)
        if not (alive[a] and alive[b]) or current[(a, b)][0] != cost:
            continue
        live_b = [t for t in vf[b] if not fdead[t]]
        both = [t for t in live_b if a in F[t]]
        if not both:
            continue
        v = current[(a, b)][1]
        if any(flips(P[F[t][0]], P[F[t][1]], P[F[t][2]], F[t].index(b), v) for t in live_b if a not in F[t]):
            continue
        for t in live_b:
            if a in F[t]:
                fdead[t] = True
            else:
                F[t][F[t].index(b)] = a
                vf[a].append(t)
        n_f -= len(both)
        last_removed = len(both)
        P[a] = v
        Q[a] = tuple(Q[a][i] + Q[b][i] for i in range(10))
        for x in (col, nrm):
            if x is not None:
                x[a] = (x[a] + x[b]) * 0.5
        alive[b] = False
        vf[a] = [t for t in vf[a] if not fdead[t]]
        nbrs = {x for t in vf[a] for x in F[t] if x != a}
        for x in sorted(nbrs):
            push(a, x)
    if n_f > int(target):
        last_removed = 0
    keep = [t for t in range(len(F)) if not fdead[t]]
    Fo = np.array([F[t] for t in keep], np.int64).reshape(-1, 3)
    return _finish(np.array(P, np.float64).reshape(-1, 3), Fo, col, nrm, 0, last_removed)


# ---------------------------------------------------------------------------------------------------------------------
# the rounds
# ---------------------------------------------------------------------------------------------------------------------
def decimate_rounds(verts, faces, target, colors=None, normals=None, max_collapses_per_round=None):
    """The round algorithm of csrc/sgr_decimate.cu in numpy (module docstring) -> the dict of decimate_greedy, with
    `rounds` = the number of rounds that selected an edge.  max_collapses_per_round (tests only) considers only the
    first so many selected edges in key order."""
    P, F = _check(verts, faces)
    V = len(P)
    Q = initial_quadrics(P, F)
    col, nrm = _attr(colors, V), _attr(normals, V)
    blk = np.zeros(F.shape, bool)
    target = int(target)
    rounds = last_removed = 0
    never = np.iinfo(np.int64).max
    while len(F) > target:
        ea = np.minimum(F, np.roll(F, -1, 1)).reshape(-1)
        eb = np.maximum(F, np.roll(F, -1, 1)).reshape(-1)
        with np.errstate(all="ignore"):
            cost, vbar = edge_solution(_rows(Q[ea]), _rows(Q[eb]), _rows(P[ea]), _rows(P[eb]))
        cand = ~blk.reshape(-1) & ~np.isnan(cost)
        rank = np.full(len(ea), never)
        ci = np.nonzero(cand)[0]
        if len(ci):
            o = ci[np.lexsort((eb[ci], ea[ci], cost[ci]))]
            new = np.ones(len(o), bool)
            new[1:] = (ea[o[1:]] != ea[o[:-1]]) | (eb[o[1:]] != eb[o[:-1]])
            rank[o] = np.cumsum(new) - 1
        vmin = np.full(V, never)
        np.minimum.at(vmin, ea, rank)
        np.minimum.at(vmin, eb, rank)
        fmin = vmin[F].min(1)
        rmin = np.full(V, never)
        np.minimum.at(rmin, F.reshape(-1), np.repeat(fmin, 3))
        sel_slot = cand & (rank == rmin[ea]) & (rank == rmin[eb])
        s = np.nonzero(sel_slot)[0]
        s = s[np.unique(rank[s], return_index=True)[1]]          # one slot per selected edge, in key order
        if not len(s):
            break
        rounds += 1
        if max_collapses_per_round:
            s = s[:max_collapses_per_round]
        sa, sb = ea[s], eb[s]
        sv = tuple(vbar[i][s] for i in range(3))
        n = len(s)
        # the faces of b, per corner: flip test and removed-face count
        of_b = np.full(V, -1)
        of_b[sb] = np.arange(n)
        of_a = np.full(V, -1)
        of_a[sa] = np.arange(n)
        fc, kc = np.nonzero(of_b[F] >= 0)
        e = of_b[F[fc, kc]]
        has_a = (F[fc] == sa[e][:, None]).any(1)
        removed = np.bincount(e[has_a], minlength=n)
        t = ~has_a
        with np.errstate(all="ignore"):
            fl = flips(*(_rows(P[F[fc[t], k]]) for k in range(3)), kc[t], tuple(x[e[t]] for x in sv))
        flipped = np.zeros(n, bool)
        flipped[e[t][fl]] = True
        # a failing edge is blocked on every slot that holds it
        se = (ea * (V + 1) + eb).reshape(F.shape)
        bad = np.isin(se, sa[flipped] * (V + 1) + sb[flipped])
        blk |= bad
        # budget: accept the passing edges in key order while the face count is above the target
        ok = np.nonzero(~flipped)[0]
        before = len(F) - (np.cumsum(removed[ok]) - removed[ok])
        acc = ok[before > target]
        if len(acc) and len(F) - removed[acc].sum() <= target:
            last_removed = int(removed[acc[-1]])
        if not len(acc):
            continue
        aa, ab = sa[acc], sb[acc]
        dead_b = np.zeros(V, bool)
        dead_b[ab] = True
        surv = np.full(V, -1)
        surv[ab] = aa
        # delete faces holding both ends, rewrite b -> a, unblock every slot touching a or b
        hb = dead_b[F]
        partner = np.where(hb, surv[F], -1).max(1)
        delete = hb.any(1) & (F == partner[:, None]).any(1)
        touch = np.zeros(V, bool)
        touch[aa] = True
        touch[ab] = True
        tf = touch[F]
        blk &= ~(tf | np.roll(tf, -1, 1))
        F = np.where(hb, surv[F], F)
        P[aa] = np.stack([x[acc] for x in sv], 1)
        Q[aa] = Q[aa] + Q[ab]
        for x in (col, nrm):
            if x is not None:
                x[aa] = (x[aa] + x[ab]) * 0.5
        F, blk = F[~delete], blk[~delete]
    if len(F) > target:
        last_removed = 0
    return _finish(P, F, col, nrm, rounds, last_removed)


# ---------------------------------------------------------------------------------------------------------------------
# clean-up passes
# ---------------------------------------------------------------------------------------------------------------------
def remove_degenerate_triangles(faces):
    F = np.asarray(faces, np.int64).reshape(-1, 3)
    return F[(F[:, 0] != F[:, 1]) & (F[:, 1] != F[:, 2]) & (F[:, 0] != F[:, 2])]


def remove_duplicated_triangles(faces):
    F = np.asarray(faces, np.int64).reshape(-1, 3)
    seen, keep = set(), []
    for f in F.tolist():
        k = f.index(min(f))
        key = tuple(f[k:] + f[:k])
        keep.append(key not in seen)
        seen.add(key)
    return F[np.array(keep, bool)] if len(F) else F


def remove_duplicated_vertices(verts, faces, colors=None, normals=None):
    P = np.asarray(verts, np.float64).reshape(-1, 3)
    F = np.asarray(faces, np.int64).reshape(-1, 3)
    first, keep, remap = {}, [], np.empty(len(P), np.int64)
    for i, r in enumerate(P.tolist()):
        key = tuple(r)
        if key not in first:
            first[key] = len(keep)
            keep.append(i)
        remap[i] = first[key]
    keep = np.array(keep, np.int64)
    pick = lambda x: None if x is None else np.asarray(x)[keep]
    return P[keep], remap[F].reshape(-1, 3), pick(colors), pick(normals)


def triangle_areas(verts, faces):
    P = np.asarray(verts, np.float64)
    F = np.asarray(faces, np.int64).reshape(-1, 3)
    p = [_rows(P[F[:, k]]) for k in range(3)]
    return 0.5 * _norm(_cross(_sub(p[1], p[0]), _sub(p[2], p[0])))


def remove_non_manifold_edges(verts, faces):
    F = np.asarray(faces, np.int64).reshape(-1, 3)
    while True:
        area = triangle_areas(verts, F)
        e = np.sort(np.stack([F, np.roll(F, -1, 1)], 2).reshape(-1, 2), 1)
        edges, inv, cnt = np.unique(e, axis=0, return_inverse=True, return_counts=True)
        inv = inv.reshape(-1)
        bad = np.nonzero(cnt > 2)[0]
        if not len(bad):
            return F
        dead = np.zeros(len(F), bool)
        fid = np.repeat(np.arange(len(F)), 3)
        for g in bad:                                   # ascending (a, b): np.unique sorts the edges
            fs = [int(t) for t in fid[inv == g] if not dead[t]]
            fs.sort(key=lambda t: (area[t], t))
            for t in fs[:max(len(fs) - 2, 0)]:
                dead[t] = True
        F = F[~dead]


def clean_mesh(verts, faces, colors=None, normals=None):
    """The four passes in the reference's order -> (verts, faces, colors, normals)."""
    F = remove_duplicated_triangles(remove_degenerate_triangles(faces))
    P, F, c, n = remove_duplicated_vertices(verts, F, colors, normals)
    return P, remove_non_manifold_edges(P, F), c, n
