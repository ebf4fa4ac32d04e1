// sgr_meshloss.cu -- the refinement stage's mesh normal-consistency regulariser, forward and backward.
//
// Replaces pytorch3d 0.7.4's mesh_normal_consistency as sugar_trainers/refine.py:775-783 calls it on the surface
// mesh of the bound Gaussians: every call rebuilds the mesh's edge table, lists the pairs of faces that share an
// edge in a Python loop over all 3F (face, edge) entries, and runs ~15 gather / cross / cosine kernels plus their
// autograd.  The faces never change during refinement, so the pair table is built once (sugar_b200/meshloss.py:
// mesh_topology, torch sort / unique on the device) and what is left per step is:
//
// Forward, one thread per pair (v0, v1, a, b): gather the four vertices, n_a = (v1 - v0) x (a - v0), n_b the same
//   with b, the term 1 - cos(n_a, -n_b); one double per CTA, summed in a fixed order by a second kernel (no float
//   atomics: the result is identical from run to run).
// Backward, one thread per pair writes the term's gradient for its four vertices (48 B), then one thread per vertex
//   sums its entries over the vertex -> (pair, slot) CSR list in ascending order (deterministic, no atomics).
//
// Numerics.  The per-pair arithmetic is in double.  On the smooth meshes refinement produces, adjacent normals are
// ~0.01 rad apart and 1 - cos leaves a term near 5e-5; with both normals longer than eps the term is evaluated as
// |n_a/|n_a| + n_b/|n_b||^2 / 2 (= 1 - cos for unit vectors), which keeps its digits.  Where a normal is shorter than
// torch.cosine_similarity's eps the identity does not hold; there the term is torch's 1 - (x1 / max(|x1|, eps)) .
// (x2 / max(|x2|, eps)) and its gradient is the one autograd gives for that expression (the clamp is applied without
// gradient, the norm keeps its own: x / |x|, zero at x = 0), so a zero normal gives a term of 1.
#include <math.h>

#include "sgr_internal.cuh"
#include "sgr_reduce.cuh"

// The per-pair arithmetic is plain C++: tests/test_meshloss_cpu.py compiles this file with
// -DSGR_MESHLOSS_HOST_TEST and runs the same function on the host against the oracle's float64 autograd.
#define SGR_HD __host__ __device__ __forceinline__

namespace sgr {

struct NcVec {
    double x, y, z;
};
SGR_HD NcVec operator+(NcVec a, NcVec b) { return {a.x + b.x, a.y + b.y, a.z + b.z}; }
SGR_HD NcVec operator-(NcVec a, NcVec b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
SGR_HD NcVec operator-(NcVec a) { return {-a.x, -a.y, -a.z}; }
SGR_HD NcVec operator*(double s, NcVec a) { return {s * a.x, s * a.y, s * a.z}; }
SGR_HD double nc_dot(NcVec a, NcVec b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
SGR_HD NcVec nc_cross(NcVec a, NcVec b) { return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }
SGR_HD NcVec nc_vert(const float *__restrict__ verts, int i)
{
    const float *p = verts + 3 * (size_t)i;
    return {(double)p[0], (double)p[1], (double)p[2]};
}

constexpr double NC_EPS = 1e-8;  // torch.cosine_similarity's default

// adjoint of y = x / max(|x|, eps) as autograd differentiates torch's expression: g / c - x <g, x> / (c^2 |x|)
SGR_HD NcVec nc_clamped_normalize_adj(NcVec x, double len, double c, NcVec g)
{
    NcVec r = (1.0 / c) * g;
    if (len > 0.0) r = r - (nc_dot(g, x) / (c * c * len)) * x;
    return r;
}

// The term of one pair; with gv != nullptr also the gradient of g * term for (v0, v1, a, b) in gv[0..3].
SGR_HD double nc_pair(const float *__restrict__ verts, int v0, int v1, int a, int b, double g, NcVec *gv)
{
    const NcVec p0 = nc_vert(verts, v0), p1 = nc_vert(verts, v1);
    const NcVec e = p1 - p0, wa = nc_vert(verts, a) - p0, wb = nc_vert(verts, b) - p0;
    const NcVec na = nc_cross(e, wa), nb = nc_cross(e, wb);
    const double la = sqrt(nc_dot(na, na)), lb = sqrt(nc_dot(nb, nb));
    double term;
    NcVec ga, gb;
    if (la >= NC_EPS && lb >= NC_EPS) {
        const NcVec ua = (1.0 / la) * na, ub = (-1.0 / lb) * nb;  // the two unit vectors compared
        const NcVec d = ua - ub;
        term = 0.5 * nc_dot(d, d);
        if (!gv) return term;
        // d term / d ua projected on the tangent plane = d - term ua (and -d - term ub for ub = -nb / |nb|)
        ga = (g / la) * (d - term * ua);
        gb = (g / lb) * (d + term * ub);
    } else {
        const double ca = fmax(la, NC_EPS), cb = fmax(lb, NC_EPS);
        const NcVec x2 = -nb, y1 = (1.0 / ca) * na, y2 = (1.0 / cb) * x2;
        term = 1.0 - nc_dot(y1, y2);
        if (!gv) return term;
        ga = nc_clamped_normalize_adj(na, la, ca, (-g) * y2);
        gb = -nc_clamped_normalize_adj(x2, lb, cb, (-g) * y1);
    }
    // n = e x w:  d/de = w x g_n,  d/dw = g_n x e
    const NcVec ge = nc_cross(wa, ga) + nc_cross(wb, gb);
    const NcVec gwa = nc_cross(ga, e), gwb = nc_cross(gb, e);
    gv[0] = -(ge + gwa + gwb);
    gv[1] = ge;
    gv[2] = gwa;
    gv[3] = gwb;
    return term;
}

constexpr int NC_THREADS = 256;

__global__ void __launch_bounds__(NC_THREADS) mesh_nc_forward_kernel(int Q, const float *__restrict__ verts,
                                                                     const int4 *__restrict__ pairs,
                                                                     double *__restrict__ partials)
{
    __shared__ double red[NC_THREADS / 32];
    const int q = blockIdx.x * NC_THREADS + threadIdx.x;
    double t = 0.0;
    if (q < Q) {
        const int4 r = __ldg(pairs + q);
        t = nc_pair(verts, r.x, r.y, r.z, r.w, 0.0, nullptr);
    }
    const double s = cta_sum_by_warps<NC_THREADS>(t, red);
    if (threadIdx.x == 0) partials[blockIdx.x] = s;
}

__global__ void __launch_bounds__(NC_THREADS) mesh_nc_pair_grad_kernel(int Q, const float *__restrict__ verts,
                                                                       const int4 *__restrict__ pairs,
                                                                       const float *__restrict__ g_loss, double inv_q,
                                                                       float4 *__restrict__ pair_grads)
{
    const int q = blockIdx.x * NC_THREADS + threadIdx.x;
    if (q >= Q) return;
    const int4 r = __ldg(pairs + q);
    NcVec gv[4];
    nc_pair(verts, r.x, r.y, r.z, r.w, (double)__ldg(g_loss) * inv_q, gv);
    float4 *o = pair_grads + 3 * (size_t)q;  // [Q, 4 slots, 3] floats
    o[0] = make_float4((float)gv[0].x, (float)gv[0].y, (float)gv[0].z, (float)gv[1].x);
    o[1] = make_float4((float)gv[1].y, (float)gv[1].z, (float)gv[2].x, (float)gv[2].y);
    o[2] = make_float4((float)gv[2].z, (float)gv[3].x, (float)gv[3].y, (float)gv[3].z);
}

__global__ void __launch_bounds__(NC_THREADS) mesh_nc_vertex_sum_kernel(int V, const int *__restrict__ vert_ptr,
                                                                        const int *__restrict__ vert_inc,
                                                                        const float *__restrict__ pair_grads,
                                                                        float *__restrict__ g_verts)
{
    const int v = blockIdx.x * NC_THREADS + threadIdx.x;
    if (v >= V) return;
    double x = 0.0, y = 0.0, z = 0.0;
    const int k1 = __ldg(vert_ptr + v + 1);
    for (int k = __ldg(vert_ptr + v); k < k1; k++) {
        const float *p = pair_grads + 3 * (size_t)__ldg(vert_inc + k);
        x += p[0];
        y += p[1];
        z += p[2];
    }
    g_verts[3 * (size_t)v] = (float)x;
    g_verts[3 * (size_t)v + 1] = (float)y;
    g_verts[3 * (size_t)v + 2] = (float)z;
}

static int nc_blocks(int n) { return (n + NC_THREADS - 1) / NC_THREADS; }

// the forward's per-block partial sums; the backward's per-pair gradients (four vertices x 3 floats)
static double *nc_partials(Layout &l, int Q) { return l.take<double>(nc_blocks(Q)); }
static float4 *nc_pair_grads(Layout &l, int Q) { return l.take<float4>(3 * (size_t)Q); }

static bool nc_sizes_ok(int32_t Q, int32_t V, const char *who)
{
    if (Q < 0 || V < 0 || Q > INT32_MAX / 4) {
        set_error("%s: bad sizes Q=%d V=%d (0 <= Q <= (2^31 - 1) / 4, V >= 0)", who, Q, V);
        return false;
    }
    return true;
}

}  // namespace sgr

using namespace sgr;

#ifdef SGR_MESHLOSS_HOST_TEST
// test-only build (never part of libsugar_b200.so): the per-pair function looped on the host, terms in double
extern "C" void mesh_nc_host(int Q, const float *verts, const int *pairs, double g, double *terms, double *pair_grads)
{
    for (int q = 0; q < Q; q++) {
        NcVec gv[4];
        const int *r = pairs + 4 * (size_t)q;
        terms[q] = nc_pair(verts, r[0], r[1], r[2], r[3], g, gv);
        for (int s = 0; s < 4; s++) {
            pair_grads[12 * (size_t)q + 3 * s] = gv[s].x;
            pair_grads[12 * (size_t)q + 3 * s + 1] = gv[s].y;
            pair_grads[12 * (size_t)q + 3 * s + 2] = gv[s].z;
        }
    }
}
#else
extern "C" {

// Q == 0 needs no scratch
size_t sgr_mesh_nc_forward_scratch_bytes(int32_t Q)
{
    return Q > 0 && Q <= INT32_MAX / 4 ? layout_bytes([&](Layout &l) { nc_partials(l, Q); }) : 0;
}

size_t sgr_mesh_nc_backward_scratch_bytes(int32_t Q)
{
    return Q > 0 && Q <= INT32_MAX / 4 ? layout_bytes([&](Layout &l) { nc_pair_grads(l, Q); }) : 0;
}

int sgr_mesh_nc_forward(int32_t Q, int32_t V, const float *verts, const int32_t *pairs, float *loss, void *scratch,
                        void *stream)
{
    if (!nc_sizes_ok(Q, V, "sgr_mesh_nc_forward")) return SGR_EINVAL;
    if (!loss || (Q > 0 && (!verts || !pairs || !scratch))) {
        set_error("sgr_mesh_nc_forward: null pointer");
        return SGR_EINVAL;
    }
    cudaStream_t st = (cudaStream_t)stream;
    if (Q == 0) {  // no face shares an edge with another: the mean over no pairs is 0
        SGR_CUDA(cudaMemsetAsync(loss, 0, sizeof(float), st));
        return SGR_OK;
    }
    Layout l(scratch);
    double *partials = nc_partials(l, Q);
    const int nb = nc_blocks(Q);
    SGR_LAUNCH(K_MESH_NC_FWD, st,
               mesh_nc_forward_kernel<<<nb, NC_THREADS, 0, st>>>(Q, verts, (const int4 *)pairs, partials));
    SGR_LAUNCH(K_MESH_NC_FWD, st, sum_partials_kernel<1024><<<1, 1024, 0, st>>>(nb, 1.0 / (double)Q, partials, loss));
    SGR_CUDA(cudaGetLastError());
    return SGR_OK;
}

int sgr_mesh_nc_backward(int32_t Q, int32_t V, const float *verts, const int32_t *pairs, const int32_t *vert_ptr,
                         const int32_t *vert_inc, const float *g_loss, float *g_verts, void *scratch, void *stream)
{
    if (!nc_sizes_ok(Q, V, "sgr_mesh_nc_backward")) return SGR_EINVAL;
    if ((V > 0 && !g_verts) ||
        (Q > 0 && (!verts || !pairs || !vert_ptr || !vert_inc || !g_loss || !scratch))) {
        set_error("sgr_mesh_nc_backward: null pointer");
        return SGR_EINVAL;
    }
    cudaStream_t st = (cudaStream_t)stream;
    if (Q == 0) {
        if (V > 0) SGR_CUDA(cudaMemsetAsync(g_verts, 0, sizeof(float) * 3 * (size_t)V, st));
        return SGR_OK;
    }
    Layout l(scratch);
    float4 *pair_grads = nc_pair_grads(l, Q);
    SGR_LAUNCH(K_MESH_NC_BWD, st,
               mesh_nc_pair_grad_kernel<<<nc_blocks(Q), NC_THREADS, 0, st>>>(Q, verts, (const int4 *)pairs, g_loss,
                                                                             1.0 / (double)Q, pair_grads));
    if (V > 0)
        SGR_LAUNCH(K_MESH_NC_BWD, st,
                   mesh_nc_vertex_sum_kernel<<<nc_blocks(V), NC_THREADS, 0, st>>>(V, vert_ptr, vert_inc,
                                                                                  (const float *)pair_grads, g_verts));
    SGR_CUDA(cudaGetLastError());
    return SGR_OK;
}

}  // extern "C"
#endif  // SGR_MESHLOSS_HOST_TEST
