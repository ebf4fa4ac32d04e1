// sgr_decimate.cu -- quadric edge-collapse decimation of a triangle mesh (sm_90a).
//
// Replaces open3d's TriangleMesh::simplify_quadric_decimation as the reference calls it at the end of both coarse-mesh
// extraction branches (sugar_extractors/coarse_mesh.py:433-463, :716-744).  The rules (planes, quadrics, boundary
// quadrics, edge cost, key order, flip test, collapse) are written down in oracle/decimate_oracle.py, whose
// decimate_rounds this file equals array for array: every product and sum below is a _rn intrinsic in the oracle's
// order, so nvcc's contraction cannot change a bit.  Positions, quadrics, colours and normals are float64 here.
//
// open3d's sequential heap becomes rounds of independent collapses.  Per round:
//   1. CSR list of each vertex's live faces in face order: count (integer atomics), scan (sgr_knn.cu's), scatter, and a
//      per-vertex insertion sort of the (short) list.
//   2. One thread per face slot (edge f[k] -> f[k+1]) evaluates the edge's key (cost, a, b); NaN or a blocked slot is
//      "never".  Then three gathers through the CSR list, no atomics: vmin[v] over v's edges, fmin[f] over f's vertices,
//      rmin[v] over v's faces.
//   3. (a, b) is selected when its key equals rmin[a] and rmin[b]: no face holds vertices of two selected edges, so the
//      collapses touch disjoint stars and need no synchronisation.  One thread per a runs the flip test over b's faces
//      and counts the faces that hold both; a failing edge sets the blocked bit of its slots (cleared when a or b
//      survives a later collapse).
//   4. One host read: the number selected and the faces the passing collapses would remove.  If that reaches the
//      target, the passing edges are compacted and one CTA bisects the key at which the running count first reaches
//      the target (the greedy loop's stop rule; a is unique among selected edges, so (cost, a) orders them).
//   5. One thread per accepted collapse rewrites b's faces, deletes the shared ones, moves a, adds the quadrics and
//      averages colour and normal; then the live faces are compacted in order (a scan), so the work shrinks each round.
// After the loop the vertices that a face references are compacted in order and written as float32.
#include <math.h>

#include "sgr_knn.cuh"

namespace sgr {

namespace {

constexpr unsigned long long DEC_NEVER = ~0ull;

struct DKey {
    unsigned long long c;  // order-preserving bits of the cost; DEC_NEVER: not a candidate
    uint32_t a, b;
};

struct PassRec {
    unsigned long long c;
    uint32_t a, r;  // r: faces the collapse removes
};

__device__ __forceinline__ bool key_lt(const DKey &x, const DKey &y)
{
    return x.c < y.c || (x.c == y.c && (x.a < y.a || (x.a == y.a && x.b < y.b)));
}
__device__ __forceinline__ bool key_eq(const DKey &x, const DKey &y) { return x.c == y.c && x.a == y.a && x.b == y.b; }
__device__ __forceinline__ DKey key_never() { return DKey{DEC_NEVER, 0xffffffffu, 0xffffffffu}; }

__device__ __forceinline__ unsigned long long cost_bits(double c)
{
    if (c != c) return DEC_NEVER;
    const unsigned long long u = (unsigned long long)__double_as_longlong(c);
    return (u >> 63) ? ~u : (u | 0x8000000000000000ull);
}

struct D3 {
    double x, y, z;
};

__device__ __forceinline__ D3 ld3(const double *p, uint32_t i) { return D3{p[3 * (size_t)i], p[3 * (size_t)i + 1], p[3 * (size_t)i + 2]}; }
__device__ __forceinline__ D3 sub3(D3 p, D3 q) { return D3{__dsub_rn(p.x, q.x), __dsub_rn(p.y, q.y), __dsub_rn(p.z, q.z)}; }
__device__ __forceinline__ D3 cross3(D3 u, D3 w)
{
    return D3{__dsub_rn(__dmul_rn(u.y, w.z), __dmul_rn(u.z, w.y)), __dsub_rn(__dmul_rn(u.z, w.x), __dmul_rn(u.x, w.z)),
              __dsub_rn(__dmul_rn(u.x, w.y), __dmul_rn(u.y, w.x))};
}
__device__ __forceinline__ double dot3(D3 u, D3 w)
{
    return __dadd_rn(__dadd_rn(__dmul_rn(u.x, w.x), __dmul_rn(u.y, w.y)), __dmul_rn(u.z, w.z));
}
__device__ __forceinline__ D3 unit3(D3 n, double &ln)
{
    ln = __dsqrt_rn(dot3(n, n));
    return D3{__ddiv_rn(n.x, ln), __ddiv_rn(n.y, ln), __ddiv_rn(n.z, ln)};
}
// the plane through p0 with normal direction m: unit normal u and offset d, zero when |m| = 0
__device__ __forceinline__ double plane_through(D3 m, D3 p0, D3 &u)
{
    double ln;
    u = unit3(m, ln);
    const double d = -dot3(u, p0);
    if (ln == 0.0) {
        u = D3{0.0, 0.0, 0.0};
        return 0.0;
    }
    return d;
}
__device__ __forceinline__ void add_quadric(double *q, D3 n, double d, double w)
{
    const double wd = __dmul_rn(w, d);
    q[0] = __dadd_rn(q[0], __dmul_rn(w, __dmul_rn(n.x, n.x)));
    q[1] = __dadd_rn(q[1], __dmul_rn(w, __dmul_rn(n.x, n.y)));
    q[2] = __dadd_rn(q[2], __dmul_rn(w, __dmul_rn(n.x, n.z)));
    q[3] = __dadd_rn(q[3], __dmul_rn(w, __dmul_rn(n.y, n.y)));
    q[4] = __dadd_rn(q[4], __dmul_rn(w, __dmul_rn(n.y, n.z)));
    q[5] = __dadd_rn(q[5], __dmul_rn(w, __dmul_rn(n.z, n.z)));
    q[6] = __dadd_rn(q[6], __dmul_rn(wd, n.x));
    q[7] = __dadd_rn(q[7], __dmul_rn(wd, n.y));
    q[8] = __dadd_rn(q[8], __dmul_rn(wd, n.z));
    q[9] = __dadd_rn(q[9], __dmul_rn(wd, d));
}

__device__ __forceinline__ double qeval(const double *q, D3 x)
{
    const double ax = __dadd_rn(__dadd_rn(__dmul_rn(q[0], x.x), __dmul_rn(q[1], x.y)), __dmul_rn(q[2], x.z));
    const double ay = __dadd_rn(__dadd_rn(__dmul_rn(q[1], x.x), __dmul_rn(q[3], x.y)), __dmul_rn(q[4], x.z));
    const double az = __dadd_rn(__dadd_rn(__dmul_rn(q[2], x.x), __dmul_rn(q[4], x.y)), __dmul_rn(q[5], x.z));
    const double vav = __dadd_rn(__dadd_rn(__dmul_rn(x.x, ax), __dmul_rn(x.y, ay)), __dmul_rn(x.z, az));
    const double bv = __dadd_rn(__dadd_rn(__dmul_rn(q[6], x.x), __dmul_rn(q[7], x.y)), __dmul_rn(q[8], x.z));
    return __dadd_rn(__dadd_rn(vav, __dmul_rn(2.0, bv)), q[9]);
}

// cost (+ 0.0) and target position of collapsing (a, b), a < b
__device__ double edge_solve(const double *__restrict__ Q, const double *__restrict__ pos, uint32_t a, uint32_t b, D3 &v)
{
    double q[10];
#pragma unroll
    for (int i = 0; i < 10; i++) q[i] = __dadd_rn(Q[10 * (size_t)a + i], Q[10 * (size_t)b + i]);
    const double C00 = __dsub_rn(__dmul_rn(q[3], q[5]), __dmul_rn(q[4], q[4]));
    const double C01 = __dsub_rn(__dmul_rn(q[2], q[4]), __dmul_rn(q[1], q[5]));
    const double C02 = __dsub_rn(__dmul_rn(q[1], q[4]), __dmul_rn(q[2], q[3]));
    const double C11 = __dsub_rn(__dmul_rn(q[0], q[5]), __dmul_rn(q[2], q[2]));
    const double C12 = __dsub_rn(__dmul_rn(q[1], q[2]), __dmul_rn(q[0], q[4]));
    const double C22 = __dsub_rn(__dmul_rn(q[0], q[3]), __dmul_rn(q[1], q[1]));
    const double det = __dadd_rn(__dadd_rn(__dmul_rn(q[0], C00), __dmul_rn(q[1], C01)), __dmul_rn(q[2], C02));
    double cost;
    if (fabs(det) > 1e-4) {
        const double t0 = __dadd_rn(__dadd_rn(__dmul_rn(C00, q[6]), __dmul_rn(C01, q[7])), __dmul_rn(C02, q[8]));
        const double t1 = __dadd_rn(__dadd_rn(__dmul_rn(C01, q[6]), __dmul_rn(C11, q[7])), __dmul_rn(C12, q[8]));
        const double t2 = __dadd_rn(__dadd_rn(__dmul_rn(C02, q[6]), __dmul_rn(C12, q[7])), __dmul_rn(C22, q[8]));
        v = D3{__ddiv_rn(-t0, det), __ddiv_rn(-t1, det), __ddiv_rn(-t2, det)};
        cost = qeval(q, v);
    } else {
        const D3 pa = ld3(pos, a), pb = ld3(pos, b);
        v = D3{__dmul_rn(__dadd_rn(pa.x, pb.x), 0.5), __dmul_rn(__dadd_rn(pa.y, pb.y), 0.5),
               __dmul_rn(__dadd_rn(pa.z, pb.z), 0.5)};
        cost = qeval(q, v);
        const double ca = qeval(q, pa), cb = qeval(q, pb);
        if (ca < cost) {
            cost = ca;
            v = pa;
        }
        if (cb < cost) {
            cost = cb;
            v = pb;
        }
    }
    return __dadd_rn(cost, 0.0);
}

__device__ __forceinline__ bool flips(D3 q0, D3 q1, D3 q2, int slot, D3 v)
{
    double l;
    const D3 before = unit3(cross3(sub3(q1, q0), sub3(q2, q0)), l);
    if (slot == 0) q0 = v;
    else if (slot == 1) q1 = v;
    else q2 = v;
    const D3 after = unit3(cross3(sub3(q1, q0), sub3(q2, q0)), l);
    return dot3(before, after) < 0.0;
}

__device__ __forceinline__ bool has(const int *f, uint32_t v) { return f[0] == (int)v || f[1] == (int)v || f[2] == (int)v; }

// ---------------------------------------------------------------------------------------------------------------------
// kernels
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) dec_init_kernel(int V, int F, const float *__restrict__ verts,
                                                       const int64_t *__restrict__ faces, const float *__restrict__ colors,
                                                       const float *__restrict__ normals, double *__restrict__ pos,
                                                       double *__restrict__ col, double *__restrict__ nrm,
                                                       int *__restrict__ fc, uint8_t *__restrict__ blk,
                                                       unsigned long long *__restrict__ bad)
{
    const int n = max(V, F);
    for (int i = blockIdx.x * 256 + threadIdx.x; i < n; i += gridDim.x * 256) {
        if (i < V) {
            for (int k = 0; k < 3; k++) {
                pos[3 * (size_t)i + k] = (double)verts[3 * (size_t)i + k];
                if (col) col[3 * (size_t)i + k] = (double)colors[3 * (size_t)i + k];
                if (nrm) nrm[3 * (size_t)i + k] = (double)normals[3 * (size_t)i + k];
            }
        }
        if (i < F) {
            const int64_t a = faces[3 * (size_t)i], b = faces[3 * (size_t)i + 1], c = faces[3 * (size_t)i + 2];
            const bool ok = a >= 0 && b >= 0 && c >= 0 && a < V && b < V && c < V && a != b && b != c && a != c;
            if (!ok) atomicOr(bad, 1ull);
            fc[3 * (size_t)i] = ok ? (int)a : 0;
            fc[3 * (size_t)i + 1] = ok ? (int)b : 0;
            fc[3 * (size_t)i + 2] = ok ? (int)c : 0;
            blk[i] = 0;
        }
    }
}

__global__ void __launch_bounds__(256) dec_count_kernel(int n3, const int *__restrict__ fc, uint32_t *__restrict__ cnt)
{
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i < n3) atomicAdd(&cnt[fc[i]], 1u);
}

__global__ void __launch_bounds__(256) dec_scatter_kernel(int n3, const int *__restrict__ fc, uint32_t *__restrict__ cursor,
                                                          uint32_t *__restrict__ csr)
{
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i < n3) csr[atomicAdd(&cursor[fc[i]], 1u)] = (uint32_t)(i / 3);
}

// the scatter's order depends on the atomics: sort each list into face order
__global__ void __launch_bounds__(256) dec_sort_kernel(int V, const uint32_t *__restrict__ vstart, uint32_t *__restrict__ csr)
{
    const int v = blockIdx.x * 256 + threadIdx.x;
    if (v >= V) return;
    const uint32_t s = vstart[v], e = vstart[v + 1];
    for (uint32_t i = s + 1; i < e; i++) {
        const uint32_t x = csr[i];
        uint32_t j = i;
        while (j > s && csr[j - 1] > x) {
            csr[j] = csr[j - 1];
            j--;
        }
        csr[j] = x;
    }
}

// face quadrics in face order, then the boundary quadrics of the vertex's boundary slots in (face, slot) order
__global__ void __launch_bounds__(128) dec_quadric_kernel(int V, const int *__restrict__ fc, const uint32_t *__restrict__ vstart,
                                                          const uint32_t *__restrict__ csr, const double *__restrict__ pos,
                                                          double *__restrict__ Q)
{
    const int v = blockIdx.x * 128 + threadIdx.x;
    if (v >= V) return;
    const uint32_t s = vstart[v], e = vstart[v + 1];
    double q[10];
#pragma unroll
    for (int i = 0; i < 10; i++) q[i] = 0.0;
    for (uint32_t j = s; j < e; j++) {
        const int *f = fc + 3 * (size_t)csr[j];
        const D3 p0 = ld3(pos, f[0]), p1 = ld3(pos, f[1]), p2 = ld3(pos, f[2]);
        double ln;
        unit3(cross3(sub3(p1, p0), sub3(p2, p0)), ln);
        D3 n;
        const double d = plane_through(cross3(sub3(p1, p0), sub3(p2, p0)), p0, n);
        add_quadric(q, n, d, __dmul_rn(0.5, ln));
    }
    for (uint32_t j = s; j < e; j++) {
        const int *f = fc + 3 * (size_t)csr[j];
        const D3 p0 = ld3(pos, f[0]), p1 = ld3(pos, f[1]), p2 = ld3(pos, f[2]);
        D3 n;
        plane_through(cross3(sub3(p1, p0), sub3(p2, p0)), p0, n);
        for (int k = 0; k < 3; k++) {
            const int v0 = f[k], v1 = f[(k + 1) % 3];
            if (v0 != v && v1 != v) continue;
            const int other = v0 == v ? v1 : v0;
            int count = 0;
            for (uint32_t t = s; t < e; t++) count += has(fc + 3 * (size_t)csr[t], (uint32_t)other);
            if (count != 1) continue;
            const D3 a = ld3(pos, v0);
            D3 m;
            const double d = plane_through(cross3(sub3(ld3(pos, v1), a), n), a, m);
            add_quadric(q, m, d, 1.0);
        }
    }
#pragma unroll
    for (int i = 0; i < 10; i++) Q[10 * (size_t)v + i] = q[i];
}

__global__ void __launch_bounds__(256) dec_cost_kernel(int n3, const int *__restrict__ fc, const uint8_t *__restrict__ blk,
                                                       const double *__restrict__ pos, const double *__restrict__ Q,
                                                       unsigned long long *__restrict__ slotc)
{
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= n3) return;
    const int f = i / 3, k = i - 3 * f;
    if (blk[f] >> k & 1) {
        slotc[i] = DEC_NEVER;
        return;
    }
    const uint32_t x = (uint32_t)fc[i], y = (uint32_t)fc[3 * f + (k + 1) % 3];
    D3 v;
    slotc[i] = cost_bits(edge_solve(Q, pos, min(x, y), max(x, y), v));
}

__global__ void __launch_bounds__(256) dec_vmin_kernel(int V, const int *__restrict__ fc, const uint32_t *__restrict__ vstart,
                                                       const uint32_t *__restrict__ csr,
                                                       const unsigned long long *__restrict__ slotc, DKey *__restrict__ vmin)
{
    const int v = blockIdx.x * 256 + threadIdx.x;
    if (v >= V) return;
    DKey best = key_never();
    for (uint32_t j = vstart[v]; j < vstart[v + 1]; j++) {
        const uint32_t f = csr[j];
        const int *t = fc + 3 * (size_t)f;
        const int c = t[0] == v ? 0 : (t[1] == v ? 1 : 2);
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const int s = h ? (c + 2) % 3 : c;  // the two slots with an end at v
            const unsigned long long cb = slotc[3 * (size_t)f + s];
            if (cb == DEC_NEVER) continue;
            const uint32_t x = (uint32_t)t[s], y = (uint32_t)t[(s + 1) % 3];
            const DKey k{cb, min(x, y), max(x, y)};
            if (key_lt(k, best)) best = k;
        }
    }
    vmin[v] = best;
}

__global__ void __launch_bounds__(256) dec_fmin_kernel(int F, const int *__restrict__ fc, const DKey *__restrict__ vmin,
                                                       DKey *__restrict__ fmin)
{
    const int f = blockIdx.x * 256 + threadIdx.x;
    if (f >= F) return;
    DKey best = vmin[fc[3 * (size_t)f]];
    for (int k = 1; k < 3; k++) {
        const DKey x = vmin[fc[3 * (size_t)f + k]];
        if (key_lt(x, best)) best = x;
    }
    fmin[f] = best;
}

__global__ void __launch_bounds__(256) dec_rmin_kernel(int V, const uint32_t *__restrict__ vstart, const uint32_t *__restrict__ csr,
                                                       const DKey *__restrict__ fmin, DKey *__restrict__ rmin)
{
    const int v = blockIdx.x * 256 + threadIdx.x;
    if (v >= V) return;
    DKey best = key_never();
    for (uint32_t j = vstart[v]; j < vstart[v + 1]; j++) {
        const DKey x = fmin[csr[j]];
        if (key_lt(x, best)) best = x;
    }
    rmin[v] = best;
}

struct SelArgs {
    int V;
    int *fc;
    uint8_t *blk;
    const uint32_t *vstart, *csr;
    const double *pos, *Q;
    const DKey *vmin, *rmin;
    uint8_t *state;  // 0 not selected, 1 selected and passes the flip test, 2 selected and flips
    uint32_t *removed, *partner;
    double *vbar;
    unsigned long long *ctr;  // [0] selected, [1] passing, [2] faces the passing collapses remove
};

__global__ void __launch_bounds__(256) dec_select_kernel(const SelArgs g)
{
    const int a = blockIdx.x * 256 + threadIdx.x;
    uint32_t sel = 0, pass = 0, rem = 0;
    if (a < g.V) {
        const DKey k = g.vmin[a];
        uint8_t st = 0;
        if (k.c != DEC_NEVER && k.a == (uint32_t)a && key_eq(g.rmin[a], k) && key_eq(g.rmin[k.b], k)) {
            const uint32_t b = k.b;
            D3 v;
            edge_solve(g.Q, g.pos, a, b, v);
            bool flip = false;
            for (uint32_t j = g.vstart[b]; j < g.vstart[b + 1]; j++) {
                const int *t = g.fc + 3 * (size_t)g.csr[j];
                if (has(t, a)) {
                    rem++;
                    continue;
                }
                if (!flip) {
                    const int slot = t[0] == (int)b ? 0 : (t[1] == (int)b ? 1 : 2);
                    flip = flips(ld3(g.pos, t[0]), ld3(g.pos, t[1]), ld3(g.pos, t[2]), slot, v);
                }
            }
            sel = 1;
            if (flip) {
                st = 2;
                rem = 0;
                for (uint32_t j = g.vstart[a]; j < g.vstart[a + 1]; j++) {
                    const uint32_t f = g.csr[j];
                    const int *t = g.fc + 3 * (size_t)f;
                    for (int s = 0; s < 3; s++) {
                        const uint32_t x = (uint32_t)t[s], y = (uint32_t)t[(s + 1) % 3];
                        if ((x == (uint32_t)a && y == b) || (x == b && y == (uint32_t)a)) g.blk[f] |= (uint8_t)(1 << s);
                    }
                }
            } else {
                st = 1;
                pass = 1;
                g.removed[a] = rem;
                g.partner[a] = b;
                g.vbar[3 * (size_t)a] = v.x;
                g.vbar[3 * (size_t)a + 1] = v.y;
                g.vbar[3 * (size_t)a + 2] = v.z;
            }
        }
        g.state[a] = st;
    }
    sel = __reduce_add_sync(0xffffffffu, sel);
    pass = __reduce_add_sync(0xffffffffu, pass);
    rem = __reduce_add_sync(0xffffffffu, rem);
    if ((threadIdx.x & 31) == 0 && sel) {
        atomicAdd(g.ctr, (unsigned long long)sel);
        atomicAdd(g.ctr + 1, (unsigned long long)pass);
        atomicAdd(g.ctr + 2, (unsigned long long)rem);
    }
}

__global__ void __launch_bounds__(256) dec_pass_flags_kernel(int V, const uint8_t *__restrict__ state, uint32_t *__restrict__ flags)
{
    const int v = blockIdx.x * 256 + threadIdx.x;
    if (v < V) flags[v] = state[v] == 1;
}

__global__ void __launch_bounds__(256) dec_pass_list_kernel(int V, const uint8_t *__restrict__ state, const uint32_t *__restrict__ off,
                                                            const DKey *__restrict__ vmin, const uint32_t *__restrict__ removed,
                                                            PassRec *__restrict__ list)
{
    const int v = blockIdx.x * 256 + threadIdx.x;
    if (v < V && state[v] == 1) list[off[v]] = PassRec{vmin[v].c, (uint32_t)v, removed[v]};
}

__device__ unsigned long long block_sum_u64(unsigned long long x, unsigned long long *s_w)
{
    for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = x;
    __syncthreads();
    unsigned long long t = 0;
    for (int w = 0; w < 32; w++) t += s_w[w];
    return t;
}

// Budget of the last round: the least key (c*, a*) over the passing edges at which the removed faces of the edges up
// to it reach `need`.  ctr[4], ctr[5] <- (c*, a*), ctr[6] <- faces removed up to it, ctr[7] <- faces its collapse removes.
__global__ void __launch_bounds__(1024) dec_cutoff_kernel(uint32_t n, const PassRec *__restrict__ list,
                                                          unsigned long long need, unsigned long long *__restrict__ ctr)
{
    __shared__ unsigned long long s_w[32];
    unsigned long long lo = 0, hi = DEC_NEVER - 1;
    while (lo < hi) {
        const unsigned long long mid = lo + (hi - lo) / 2;
        unsigned long long s = 0;
        for (uint32_t i = threadIdx.x; i < n; i += 1024) s += list[i].c <= mid ? list[i].r : 0u;
        if (block_sum_u64(s, s_w) >= need) hi = mid;
        else lo = mid + 1;
    }
    const unsigned long long cs = lo;
    unsigned long long base = 0;
    for (uint32_t i = threadIdx.x; i < n; i += 1024) base += list[i].c < cs ? list[i].r : 0u;
    base = block_sum_u64(base, s_w);
    uint32_t alo = 0, ahi = 0xffffffffu;
    unsigned long long acc = 0;
    while (alo < ahi) {
        const uint32_t mid = alo + (ahi - alo) / 2;
        unsigned long long s = 0;
        for (uint32_t i = threadIdx.x; i < n; i += 1024) s += (list[i].c == cs && list[i].a <= mid) ? list[i].r : 0u;
        s = base + block_sum_u64(s, s_w);
        if (s >= need) ahi = mid;
        else alo = mid + 1;
    }
    for (uint32_t i = threadIdx.x; i < n; i += 1024) {
        if (list[i].c == cs && list[i].a == alo) ctr[7] = list[i].r;
        acc += (list[i].c < cs || (list[i].c == cs && list[i].a <= alo)) ? list[i].r : 0u;
    }
    acc = block_sum_u64(acc, s_w);
    if (threadIdx.x == 0) {
        ctr[4] = cs;
        ctr[5] = alo;
        ctr[6] = acc;
    }
}

struct ApplyArgs {
    int V;
    int *fc;
    uint8_t *blk;
    const uint32_t *vstart, *csr;
    const uint8_t *state;
    const DKey *vmin;
    const uint32_t *partner;
    const double *vbar;
    const unsigned long long *thr;  // (cost bits, a) of the last accepted edge; all ones: every passing edge
    double *pos, *Q, *col, *nrm;
};

__device__ __forceinline__ void unblock(uint8_t *blk, const int *t, uint32_t f, int a)
{
    uint8_t m = blk[f];
    for (int s = 0; s < 3; s++)
        if (t[s] == a || t[(s + 1) % 3] == a) m &= (uint8_t)~(1 << s);
    blk[f] = m;
}

__global__ void __launch_bounds__(256) dec_apply_kernel(const ApplyArgs g)
{
    const int a = blockIdx.x * 256 + threadIdx.x;
    if (a >= g.V || g.state[a] != 1) return;
    const unsigned long long c = g.vmin[a].c;
    if (!(c < g.thr[0] || (c == g.thr[0] && (unsigned long long)a <= g.thr[1]))) return;
    const uint32_t b = g.partner[a];
    for (uint32_t j = g.vstart[b]; j < g.vstart[b + 1]; j++) {
        const uint32_t f = g.csr[j];
        int *t = g.fc + 3 * (size_t)f;
        if (has(t, a)) {
            t[0] = -1;  // deleted; compacted away below
            continue;
        }
        for (int s = 0; s < 3; s++)
            if (t[s] == (int)b) t[s] = a;
        unblock(g.blk, t, f, a);
    }
    for (uint32_t j = g.vstart[a]; j < g.vstart[a + 1]; j++) {
        const uint32_t f = g.csr[j];
        const int *t = g.fc + 3 * (size_t)f;
        if (t[0] >= 0) unblock(g.blk, t, f, a);
    }
    for (int k = 0; k < 3; k++) g.pos[3 * (size_t)a + k] = g.vbar[3 * (size_t)a + k];
    for (int i = 0; i < 10; i++) g.Q[10 * (size_t)a + i] = __dadd_rn(g.Q[10 * (size_t)a + i], g.Q[10 * (size_t)b + i]);
    for (int k = 0; k < 3; k++) {
        if (g.col) g.col[3 * (size_t)a + k] = __dmul_rn(__dadd_rn(g.col[3 * (size_t)a + k], g.col[3 * (size_t)b + k]), 0.5);
        if (g.nrm) g.nrm[3 * (size_t)a + k] = __dmul_rn(__dadd_rn(g.nrm[3 * (size_t)a + k], g.nrm[3 * (size_t)b + k]), 0.5);
    }
}

__global__ void __launch_bounds__(256) dec_face_flags_kernel(int F, const int *__restrict__ fc, uint32_t *__restrict__ flags)
{
    const int f = blockIdx.x * 256 + threadIdx.x;
    if (f < F) flags[f] = fc[3 * (size_t)f] >= 0;
}

__global__ void __launch_bounds__(256) dec_face_scatter_kernel(int F, const int *__restrict__ fc, const uint8_t *__restrict__ blk,
                                                               const uint32_t *__restrict__ off, int *__restrict__ fc_out,
                                                               uint8_t *__restrict__ blk_out)
{
    const int f = blockIdx.x * 256 + threadIdx.x;
    if (f >= F || fc[3 * (size_t)f] < 0) return;
    const uint32_t o = off[f];
    for (int k = 0; k < 3; k++) fc_out[3 * (size_t)o + k] = fc[3 * (size_t)f + k];
    blk_out[o] = blk[f];
}

__global__ void __launch_bounds__(256) dec_mark_kernel(int n3, const int *__restrict__ fc, uint32_t *__restrict__ used)
{
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i < n3) used[fc[i]] = 1u;
}

__global__ void __launch_bounds__(256) dec_out_verts_kernel(int V, const uint32_t *__restrict__ off, const double *__restrict__ pos,
                                                            const double *__restrict__ col, const double *__restrict__ nrm,
                                                            float *__restrict__ verts, float *__restrict__ colors,
                                                            float *__restrict__ normals)
{
    const int v = blockIdx.x * 256 + threadIdx.x;
    if (v >= V || off[v + 1] == off[v]) return;
    const size_t o = off[v];
    for (int k = 0; k < 3; k++) {
        verts[3 * o + k] = (float)pos[3 * (size_t)v + k];
        if (colors) colors[3 * o + k] = (float)col[3 * (size_t)v + k];
        if (normals) normals[3 * o + k] = (float)nrm[3 * (size_t)v + k];
    }
}

__global__ void __launch_bounds__(256) dec_out_faces_kernel(int n3, const int *__restrict__ fc, const uint32_t *__restrict__ off,
                                                            int64_t *__restrict__ faces)
{
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i < n3) faces[i] = (int64_t)off[fc[i]];
}

// ---------------------------------------------------------------------------------------------------------------------
// scratch
// ---------------------------------------------------------------------------------------------------------------------
struct DecScratch {
    unsigned long long *ctr;
    double *pos, *Q, *col, *nrm, *vbar;
    int *fc[2];
    uint8_t *blk[2], *state;
    uint32_t *vcnt, *vstart, *csr, *fflag, *bsums, *removed, *partner;
    unsigned long long *slotc;
    DKey *vmin, *rmin, *fmin;
    PassRec *list;
};

DecScratch dec_scratch(Layout &l, size_t V, size_t F)
{
    const size_t n = (V > F ? V : F) + 1;
    DecScratch t;
    t.ctr = l.take<unsigned long long>(8);
    t.pos = l.take<double>(3 * V);
    t.Q = l.take<double>(10 * V);
    t.col = l.take<double>(3 * V);
    t.nrm = l.take<double>(3 * V);
    t.vbar = l.take<double>(3 * V);
    t.fc[0] = l.take<int>(3 * F);
    t.fc[1] = l.take<int>(3 * F);
    t.blk[0] = l.take<uint8_t>(F);
    t.blk[1] = l.take<uint8_t>(F);
    t.state = l.take<uint8_t>(V);
    t.vcnt = l.take<uint32_t>(V + 1);
    t.vstart = l.take<uint32_t>(V + 1);
    t.csr = l.take<uint32_t>(3 * F);
    t.fflag = l.take<uint32_t>(n);
    t.bsums = l.take<uint32_t>(scan_block_sums(n));
    t.removed = l.take<uint32_t>(V);
    t.partner = l.take<uint32_t>(V);
    t.slotc = l.take<unsigned long long>(3 * F);
    t.vmin = l.take<DKey>(V);
    t.rmin = l.take<DKey>(V);
    t.fmin = l.take<DKey>(F);
    t.list = l.take<PassRec>(V);
    return t;
}

static bool dec_sizes_ok(int32_t V, int32_t F)
{
    return V >= 0 && F >= 0 && V <= (1 << 30) && F <= (1 << 29) && !(F > 0 && V == 0);
}

static unsigned grid(size_t n, int block) { return (unsigned)((n + block - 1) / block); }

// vertex -> live faces in face order (vstart has V + 1 entries)
static int build_csr(int V, int F, const DecScratch &s, const int *fc, cudaStream_t st)
{
    SGR_CUDA(cudaMemsetAsync(s.vcnt, 0, ((size_t)V + 1) * 4, st));
    if (F) SGR_LAUNCH(K_MISC, st, dec_count_kernel<<<grid(3 * (size_t)F, 256), 256, 0, st>>>(3 * F, fc, s.vcnt));
    exclusive_scan_u32(K_MISC, V + 1, s.vcnt, s.vstart, s.bsums, s.vcnt, st);
    if (F) SGR_LAUNCH(K_MISC, st, dec_scatter_kernel<<<grid(3 * (size_t)F, 256), 256, 0, st>>>(3 * F, fc, s.vcnt, s.csr));
    SGR_LAUNCH(K_MISC, st, dec_sort_kernel<<<grid(V, 256), 256, 0, st>>>(V, s.vstart, s.csr));
    return SGR_OK;
}

static int read_back(void *dst, const void *src, size_t bytes, cudaStream_t st)
{
    SGR_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, st));
    SGR_CUDA(cudaStreamSynchronize(st));
    return SGR_OK;
}

}  // namespace

}  // namespace sgr

using namespace sgr;

extern "C" {

size_t sgr_decimate_scratch_bytes(int32_t V, int32_t F)
{
    return dec_sizes_ok(V, F) ? layout_bytes([&](Layout &l) { dec_scratch(l, V, F); }) : 0;
}

int sgr_decimate(int32_t V, int32_t F, int64_t target, const float *verts, const int64_t *faces, const float *colors,
                 const float *normals, float *verts_out, int64_t *faces_out, float *colors_out, float *normals_out,
                 int64_t *result, void *scratch, void *stream)
{
    if (!dec_sizes_ok(V, F) || target < 0) {
        set_error("sgr_decimate: need 0 <= V <= 2^30, 0 <= F <= 2^29 (F > 0 only with V > 0) and target >= 0 "
                  "(V=%d F=%d target=%lld)", V, F, (long long)target);
        return SGR_EINVAL;
    }
    if (!result || ((V > 0 || F > 0) && !scratch) || (V > 0 && (!verts || !verts_out)) ||
        (F > 0 && (!faces || !faces_out)) || (!colors != !colors_out) || (!normals != !normals_out)) {
        set_error("sgr_decimate: null pointer (colours and normals go in and out together)");
        return SGR_EINVAL;
    }
    result[0] = result[1] = result[2] = result[3] = 0;
    if (V == 0) return SGR_OK;
    cudaStream_t st = (cudaStream_t)stream;
    Layout l(scratch);
    const DecScratch s = dec_scratch(l, V, F);
    double *col = colors ? s.col : nullptr, *nrm = normals ? s.nrm : nullptr;
    unsigned long long ctr[8];
    SGR_CUDA(cudaMemsetAsync(s.ctr, 0, 64, st));
    SGR_LAUNCH(K_MISC, st, dec_init_kernel<<<device_sm_count() * 4, 256, 0, st>>>(V, F, verts, faces, colors, normals, s.pos,
                                                                                  col, nrm, s.fc[0], s.blk[0], s.ctr + 3));
    int rc = read_back(ctr, s.ctr, 64, st);
    if (rc) return rc;
    if (ctr[3]) {
        set_error("sgr_decimate: a face id outside [0, %d) or a face that repeats a vertex", V);
        return SGR_EINVAL;
    }
    int cur = 0, Fc = F;
    int64_t rounds = 0, last = 0;
    if ((rc = build_csr(V, Fc, s, s.fc[cur], st))) return rc;
    SGR_LAUNCH(K_MISC, st, dec_quadric_kernel<<<grid(V, 128), 128, 0, st>>>(V, s.fc[cur], s.vstart, s.csr, s.pos, s.Q));
    bool fresh = true;  // the CSR lists match the current faces
    while ((int64_t)Fc > target) {
        if (!fresh && (rc = build_csr(V, Fc, s, s.fc[cur], st))) return rc;
        fresh = false;
        SGR_CUDA(cudaMemsetAsync(s.ctr, 0, 24, st));
        SGR_LAUNCH(K_MISC, st, dec_cost_kernel<<<grid(3 * (size_t)Fc, 256), 256, 0, st>>>(3 * Fc, s.fc[cur], s.blk[cur], s.pos,
                                                                                         s.Q, s.slotc));
        SGR_LAUNCH(K_MISC, st, dec_vmin_kernel<<<grid(V, 256), 256, 0, st>>>(V, s.fc[cur], s.vstart, s.csr, s.slotc, s.vmin));
        SGR_LAUNCH(K_MISC, st, dec_fmin_kernel<<<grid(Fc, 256), 256, 0, st>>>(Fc, s.fc[cur], s.vmin, s.fmin));
        SGR_LAUNCH(K_MISC, st, dec_rmin_kernel<<<grid(V, 256), 256, 0, st>>>(V, s.vstart, s.csr, s.fmin, s.rmin));
        const SelArgs sa{V, s.fc[cur], s.blk[cur], s.vstart, s.csr, s.pos, s.Q, s.vmin, s.rmin, s.state, s.removed,
                         s.partner, s.vbar, s.ctr};
        SGR_LAUNCH(K_MISC, st, dec_select_kernel<<<grid(V, 256), 256, 0, st>>>(sa));
        if ((rc = read_back(ctr, s.ctr, 24, st))) return rc;
        if (ctr[0] == 0) break;
        rounds++;
        const unsigned long long need = (unsigned long long)((int64_t)Fc - target);
        const bool cutoff = ctr[2] >= need;
        if (cutoff) {
            SGR_LAUNCH(K_MISC, st, dec_pass_flags_kernel<<<grid(V, 256), 256, 0, st>>>(V, s.state, s.fflag));
            exclusive_scan_u32(K_MISC, V, s.fflag, s.fflag, s.bsums, s.fflag, st);
            SGR_LAUNCH(K_MISC, st, dec_pass_list_kernel<<<grid(V, 256), 256, 0, st>>>(V, s.state, s.fflag, s.vmin, s.removed,
                                                                                     s.list));
            SGR_LAUNCH(K_MISC, st, dec_cutoff_kernel<<<1, 1024, 0, st>>>((uint32_t)ctr[1], s.list, need, s.ctr));
        } else {
            SGR_CUDA(cudaMemsetAsync(s.ctr + 4, 0xff, 16, st));
        }
        const ApplyArgs aa{V, s.fc[cur], s.blk[cur], s.vstart, s.csr, s.state, s.vmin, s.partner, s.vbar, s.ctr + 4,
                           s.pos, s.Q, col, nrm};
        SGR_LAUNCH(K_MISC, st, dec_apply_kernel<<<grid(V, 256), 256, 0, st>>>(aa));
        SGR_LAUNCH(K_MISC, st, dec_face_flags_kernel<<<grid(Fc, 256), 256, 0, st>>>(Fc, s.fc[cur], s.fflag));
        exclusive_scan_u32(K_MISC, Fc, s.fflag, s.fflag, s.bsums, s.fflag, st);
        SGR_LAUNCH(K_MISC, st, dec_face_scatter_kernel<<<grid(Fc, 256), 256, 0, st>>>(Fc, s.fc[cur], s.blk[cur], s.fflag,
                                                                                      s.fc[cur ^ 1], s.blk[cur ^ 1]));
        cur ^= 1;
        if (cutoff) {
            if ((rc = read_back(ctr, s.ctr, 64, st))) return rc;
            Fc -= (int)ctr[6];
            last = (int64_t)ctr[7];
        } else {
            Fc -= (int)ctr[2];
        }
    }
    // the vertices that a face references, in order
    SGR_CUDA(cudaMemsetAsync(s.vcnt, 0, ((size_t)V + 1) * 4, st));
    if (Fc) SGR_LAUNCH(K_MISC, st, dec_mark_kernel<<<grid(3 * (size_t)Fc, 256), 256, 0, st>>>(3 * Fc, s.fc[cur], s.vcnt));
    exclusive_scan_u32(K_MISC, V + 1, s.vcnt, s.vstart, s.bsums, s.vcnt, st);
    SGR_LAUNCH(K_MISC, st, dec_out_verts_kernel<<<grid(V, 256), 256, 0, st>>>(V, s.vstart, s.pos, col, nrm, verts_out,
                                                                             colors_out, normals_out));
    if (Fc) SGR_LAUNCH(K_MISC, st, dec_out_faces_kernel<<<grid(3 * (size_t)Fc, 256), 256, 0, st>>>(3 * Fc, s.fc[cur], s.vstart,
                                                                                                 faces_out));
    uint32_t nv;
    if ((rc = read_back(&nv, s.vstart + V, 4, st))) return rc;
    result[0] = nv;
    result[1] = Fc;
    result[2] = rounds;
    result[3] = last;
    SGR_CUDA(cudaGetLastError());
    return SGR_OK;
}

}  // extern "C"
