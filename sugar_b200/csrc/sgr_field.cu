// sgr_field.cu -- SuGaR surface-regularisation field as fused kernels.
//
// Replaces the PyTorch op chain of SuGaR.get_field_values / compute_density
// (sugar_scene/sugar_model.py:1247-1316, 1345-1368) with its inputs
//   get_covariance(return_sqrt, inverse_scales)   sugar_model.py:730-750   (L^-1 = R(q) diag(1/s))
//   get_beta, beta_mode 'average'                 sugar_model.py:1172-1195
//   pytorch3d.transforms.quaternion_to_matrix     (pytorch3d 0.7.4, real-first, two_s = 2/|q|^2)
// The reference materialises N x K x 3 x 3 inverse-scaled rotations (576 MB at N=1M, K=16) plus
// several N x K x 3 temporaries and their autograd copies; here one lane owns one
// (sample, neighbour) pair, gathers a 48-byte packed Gaussian record, and the K partial
// opacities are summed with shuffles.  Backward recomputes the pair and scatters with
// 16-byte vector reductions into a packed per-Gaussian gradient record.
// The coarse_density trainer's density estimation loss (densest_*_kernel) runs the same per-pair passes and adds the
// sample's own Gaussian's terms.
#include "sgr_field.cuh"

namespace sgr {

__global__ void __launch_bounds__(256) field_pack_kernel(int P, const float *__restrict__ points,
                                                         const float *__restrict__ scaling,
                                                         const float *__restrict__ quats,
                                                         const float *__restrict__ strengths, float4 *__restrict__ rec)
{
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= P) return;
    const float s0 = scaling[3 * i], s1 = scaling[3 * i + 1], s2 = scaling[3 * i + 2];
    rec[(size_t)i * 3] = make_float4(points[3 * i], points[3 * i + 1], points[3 * i + 2], strengths[i]);
    rec[(size_t)i * 3 + 1] = make_float4(quats[4 * i], quats[4 * i + 1], quats[4 * i + 2], quats[4 * i + 3]);
    // 1 / scaling.clamp(min=1e-8)   (sugar_model.py:732-733)
    rec[(size_t)i * 3 + 2] =
        make_float4(1.0f / fmaxf(s0, 1e-8f), 1.0f / fmaxf(s1, 1e-8f), 1.0f / fmaxf(s2, 1e-8f), fminf(s0, fminf(s1, s2)));
}

template <int G>
__device__ __forceinline__ float group_sum(float v)
{
#pragma unroll
    for (int o = G / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

struct FieldArgs {
    int N, K, P, group;
    float density_factor, sdf_offset, opacity_min_clamp;
    const float *x;
    const int64_t *idx;
    const float4 *rec;
};

// straight-through clamp of sugar_model.py:1280-1281 followed by the SDF of :1303-1306
__device__ __forceinline__ void sdf_from_density(float density, float beta, float opacity_min_clamp, float sdf_offset,
                                                 float &sdf, float &root, float &cl, float &dcl_ddens)
{
    float d = density;
    dcl_ddens = 1.0f;
    if (density >= 1.0f) {
        d = density / (density + 1e-12f);
        dcl_ddens = 1.0f / (density + 1e-12f);
    }
    cl = fmaxf(d, opacity_min_clamp);
    if (d < opacity_min_clamp) dcl_ddens = 0.0f;
    root = sqrtf(-2.0f * logf(cl));
    sdf = beta * (root - sdf_offset);
}

template <int G>
__global__ void __launch_bounds__(256) field_forward_kernel(const FieldArgs a, float *__restrict__ density,
                                                            float *__restrict__ nbr_opacity, float *__restrict__ beta,
                                                            float *__restrict__ sdf)
{
    constexpr int SPB = 256 / G;  // samples per block
    const int g = threadIdx.x / G, l = threadIdx.x % G;
    const int n = blockIdx.x * SPB + g;
    const bool live = n < a.N;
    const int nrow = a.group > 1 ? n / a.group : n;  // neighbour row shared by `group` consecutive samples
    float dens = 0.f, bsum = 0.f;
    if (live) {
        const float x0 = a.x[3 * n], x1 = a.x[3 * n + 1], x2 = a.x[3 * n + 2];
        for (int k = l; k < a.K; k += G) {
            const int64_t id = a.idx[(size_t)nrow * a.K + k];
            const float4 r0 = __ldg(a.rec + id * 3), r1 = __ldg(a.rec + id * 3 + 1), r2 = __ldg(a.rec + id * 3 + 2);
            const float o = field_term(x0, x1, x2, r0, r1, r2, a.density_factor);
            if (nbr_opacity) nbr_opacity[(size_t)n * a.K + k] = o;
            dens += o;
            bsum += r2.w;
        }
    }
    dens = group_sum<G>(dens);
    bsum = group_sum<G>(bsum);
    if (live && l == 0) {
        const float b = bsum / (float)a.K;
        if (density) density[n] = dens;
        if (beta) beta[n] = b;
        if (sdf) {
            float s, root, cl, dd;
            sdf_from_density(dens, b, a.opacity_min_clamp, a.sdf_offset, s, root, cl, dd);
            sdf[n] = s;
        }
    }
}

__device__ __forceinline__ void red_v4(float *addr, float a, float b, float c, float d)
{
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}

// dL/dq from A = dL/dR, R = I + ts * E(q) with ts = two_s = 2 / |q|^2 (pytorch3d's quaternion_to_matrix)
__device__ __forceinline__ float4 rot_backward(const float (&A)[3][3], float4 q, float ts)
{
    const float qr = q.x, qi = q.y, qj = q.z, qk = q.w;
    const float dts = A[0][0] * -(qj * qj + qk * qk) + A[0][1] * (qi * qj - qk * qr) + A[0][2] * (qi * qk + qj * qr) +
                      A[1][0] * (qi * qj + qk * qr) + A[1][1] * -(qi * qi + qk * qk) + A[1][2] * (qj * qk - qi * qr) +
                      A[2][0] * (qi * qk - qj * qr) + A[2][1] * (qj * qk + qi * qr) + A[2][2] * -(qi * qi + qj * qj);
    const float c = -ts * ts * dts;  // d ts / d q_c = -ts^2 q_c
    const float dqr = ts * (-qk * A[0][1] + qj * A[0][2] + qk * A[1][0] - qi * A[1][2] - qj * A[2][0] + qi * A[2][1]) + c * qr;
    const float dqi = ts * (qj * (A[0][1] + A[1][0]) + qk * (A[0][2] + A[2][0]) + qr * (A[2][1] - A[1][2]) -
                            2.f * qi * (A[1][1] + A[2][2])) + c * qi;
    const float dqj = ts * (qi * (A[0][1] + A[1][0]) + qr * (A[0][2] - A[2][0]) + qk * (A[1][2] + A[2][1]) -
                            2.f * qj * (A[0][0] + A[2][2])) + c * qj;
    const float dqk = ts * (qr * (A[1][0] - A[0][1]) + qi * (A[0][2] + A[2][0]) + qj * (A[1][2] + A[2][1]) -
                            2.f * qk * (A[0][0] + A[1][1])) + c * qk;
    return make_float4(dqr, dqi, dqj, dqk);
}

// Pass 2 of a field backward for one (sample x, neighbour id) pair.  Gk = dL/d(the pair's opacity) in total, gb = dL/d
// beta of the sample.  Adds dL/dx to gx and scatters dL/d(mu, sigma, q, s) into the Gaussian's 12-float gradient record:
// dmu.xyz dsig | dq.rijk | ds.xyz -
__device__ __forceinline__ void field_pair_backward(float x0, float x1, float x2, int64_t id, const float4 *__restrict__ rec,
                                                    const float *__restrict__ scaling, float density_factor, float Gk,
                                                    float gb, int K, float *__restrict__ grec, float &gx0, float &gx1,
                                                    float &gx2)
{
    const float4 r0 = __ldg(rec + id * 3), r1 = __ldg(rec + id * 3 + 1), r2 = __ldg(rec + id * 3 + 2);
    const Rot R = quat_to_rot(r1);
    const float sh[3] = {x0 - r0.x, x1 - r0.y, x2 - r0.z};
    float u[3], w[3];
#pragma unroll
    for (int j = 0; j < 3; j++) u[j] = R.m[0][j] * sh[0] + R.m[1][j] * sh[1] + R.m[2][j] * sh[2];
    w[0] = u[0] * r2.x;
    w[1] = u[1] * r2.y;
    w[2] = u[2] * r2.z;
    const float d2raw = w[0] * w[0] + w[1] * w[1] + w[2] * w[2];
    const float d2 = fminf(fmaxf(d2raw, 0.f), 1e8f);
    const float e = density_factor * expf(-0.5f * d2);
    const float o = r0.w * e;
    const float dsig = Gk * e;
    const float dd2 = (d2raw > 1e8f || d2raw < 0.f) ? 0.f : Gk * o * -0.5f;
    const float invs[3] = {r2.x, r2.y, r2.z};
    float du[3], ds[3];
    const float *sc = scaling + id * 3;
    int amin = 0;
    float smin = sc[0];
#pragma unroll
    for (int j = 0; j < 3; j++) {
        const float dw = dd2 * 2.0f * w[j];
        du[j] = dw * invs[j];
        const float sj = sc[j];
        ds[j] = (sj >= 1e-8f) ? -(dw * u[j]) * invs[j] * invs[j] : 0.f;
        if (j > 0 && sj < smin) {
            smin = sj;
            amin = j;
        }
    }
    ds[amin] += gb / (float)K;
    float dsh[3];
#pragma unroll
    for (int i = 0; i < 3; i++) dsh[i] = R.m[i][0] * du[0] + R.m[i][1] * du[1] + R.m[i][2] * du[2];
    gx0 += dsh[0];
    gx1 += dsh[1];
    gx2 += dsh[2];
    // dL/dR[i][j] = sh[i] * du[j]
    float A[3][3];
#pragma unroll
    for (int i = 0; i < 3; i++)
#pragma unroll
        for (int j = 0; j < 3; j++) A[i][j] = sh[i] * du[j];
    const float4 dq = rot_backward(A, r1, R.ts);
    float *gr = grec + id * 12;
    red_v4(gr, -dsh[0], -dsh[1], -dsh[2], dsig);
    red_v4(gr + 4, dq.x, dq.y, dq.z, dq.w);
    red_v4(gr + 8, ds[0], ds[1], ds[2], 0.f);
}

template <int G>
__global__ void __launch_bounds__(256) field_backward_kernel(const FieldArgs a, const float *__restrict__ scaling,
                                                             const float *__restrict__ g_density,
                                                             const float *__restrict__ g_nbr, const float *__restrict__ g_beta,
                                                             const float *__restrict__ g_sdf, float *__restrict__ g_x,
                                                             float *__restrict__ grec)
{
    constexpr int SPB = 256 / G;
    const int g = threadIdx.x / G, l = threadIdx.x % G;
    const int n = blockIdx.x * SPB + g;
    const bool live = n < a.N;
    const int nrow = a.group > 1 ? n / a.group : n;
    float x0 = 0, x1 = 0, x2 = 0;
    if (live) x0 = a.x[3 * n], x1 = a.x[3 * n + 1], x2 = a.x[3 * n + 2];
    // pass 1: recompute density and beta for the sample (needed for d sdf / d density)
    float dens = 0.f, bsum = 0.f;
    if (live)
        for (int k = l; k < a.K; k += G) {
            const int64_t id = a.idx[(size_t)nrow * a.K + k];
            const float4 r0 = __ldg(a.rec + id * 3), r1 = __ldg(a.rec + id * 3 + 1), r2 = __ldg(a.rec + id * 3 + 2);
            const Rot R = quat_to_rot(r1);
            const float sh0 = x0 - r0.x, sh1 = x1 - r0.y, sh2 = x2 - r0.z;
            const float w0 = (R.m[0][0] * sh0 + R.m[1][0] * sh1 + R.m[2][0] * sh2) * r2.x;
            const float w1 = (R.m[0][1] * sh0 + R.m[1][1] * sh1 + R.m[2][1] * sh2) * r2.y;
            const float w2 = (R.m[0][2] * sh0 + R.m[1][2] * sh1 + R.m[2][2] * sh2) * r2.z;
            const float d2 = fminf(fmaxf(w0 * w0 + w1 * w1 + w2 * w2, 0.f), 1e8f);
            dens += a.density_factor * r0.w * expf(-0.5f * d2);
            bsum += r2.w;
        }
    dens = group_sum<G>(dens);
    bsum = group_sum<G>(bsum);
    float gd = 0.f, gb = 0.f;  // dL/d density (total), dL/d beta (total)
    if (live) {
        const float b = bsum / (float)a.K;
        gd = g_density ? g_density[n] : 0.f;
        gb = g_beta ? g_beta[n] : 0.f;
        if (g_sdf) {
            float s, root, cl, dd;
            sdf_from_density(dens, b, a.opacity_min_clamp, a.sdf_offset, s, root, cl, dd);
            const float gs = g_sdf[n];
            gb += gs * (root - a.sdf_offset);
            if (dd != 0.f) gd += gs * (-b / (cl * root)) * dd;
        }
    }
    // pass 2: per-pair gradients
    float gx0 = 0.f, gx1 = 0.f, gx2 = 0.f;
    if (live)
        for (int k = l; k < a.K; k += G) {
            const int64_t id = a.idx[(size_t)nrow * a.K + k];
            const float Gk = gd + (g_nbr ? g_nbr[(size_t)n * a.K + k] : 0.f);
            field_pair_backward(x0, x1, x2, id, a.rec, scaling, a.density_factor, Gk, gb, a.K, grec, gx0, gx1, gx2);
        }
    gx0 = group_sum<G>(gx0);
    gx1 = group_sum<G>(gx1);
    gx2 = group_sum<G>(gx2);
    if (live && l == 0 && g_x) {
        g_x[3 * n] = gx0;
        g_x[3 * n + 1] = gx1;
        g_x[3 * n + 2] = gx2;
    }
}

// Density estimation loss of the coarse_density trainer in projection mode (coarse_density.py:654-656, 684-691):
//   e = <x - mu_g, n_g>,  n_g = column argmin_j scaling[g][j] of R(q_g) (the first minimum, like torch.min),
//   target = exp(-0.5 e^2 / beta^2),  loss = |rho - target|
// with rho and beta the field's density (before the straight-through clamp) and beta at x.  The K terms are the field
// forward's, in its lane order and butterfly, so rho and the neighbour opacities carry the field's bits.

// <x - mu_g, n_g> for the sample's own Gaussian g; the column index comes from the float scaling row, so the 1e-8
// clamp of the packed 1/s cannot change the pick
struct OwnAxis {
    float e, n[3], d[3];  // d = x - mu_g
    int col;
    float4 q;
    float ts;  // two_s of q
};

__device__ __forceinline__ OwnAxis own_axis(float x0, float x1, float x2, int64_t g, const float4 *__restrict__ rec,
                                            const float *__restrict__ scaling)
{
    OwnAxis o;
    const float4 r0 = __ldg(rec + g * 3);
    o.q = __ldg(rec + g * 3 + 1);
    const float *sc = scaling + g * 3;
    const float s0 = sc[0], s1 = sc[1], s2 = sc[2];
    o.col = 0;
    float smin = s0;
    if (s1 < smin) smin = s1, o.col = 1;
    if (s2 < smin) o.col = 2;
    const Rot R = quat_to_rot(o.q);
    o.ts = R.ts;
#pragma unroll
    for (int i = 0; i < 3; i++) o.n[i] = o.col == 0 ? R.m[i][0] : (o.col == 1 ? R.m[i][1] : R.m[i][2]);
    o.d[0] = x0 - r0.x;
    o.d[1] = x1 - r0.y;
    o.d[2] = x2 - r0.z;
    o.e = o.d[0] * o.n[0] + o.d[1] * o.n[1] + o.d[2] * o.n[2];
    return o;
}

// exp(-0.5 * e.pow(2) / beta.pow(2)) in the reference's evaluation order
__device__ __forceinline__ float density_target(float e, float beta) { return expf(-0.5f * (e * e) / (beta * beta)); }

template <int G>
__global__ void __launch_bounds__(256) densest_forward_kernel(const FieldArgs a, const int64_t *__restrict__ own,
                                                              const float *__restrict__ scaling, float *__restrict__ loss,
                                                              float *__restrict__ nbr_opacity)
{
    constexpr int SPB = 256 / G;
    const int g = threadIdx.x / G, l = threadIdx.x % G;
    const int n = blockIdx.x * SPB + g;
    const bool live = n < a.N;
    float x0 = 0.f, x1 = 0.f, x2 = 0.f, dens = 0.f, bsum = 0.f;
    if (live) {
        x0 = a.x[3 * n], x1 = a.x[3 * n + 1], x2 = a.x[3 * n + 2];
        for (int k = l; k < a.K; k += G) {
            const int64_t id = a.idx[(size_t)n * a.K + k];
            const float4 r0 = __ldg(a.rec + id * 3), r1 = __ldg(a.rec + id * 3 + 1), r2 = __ldg(a.rec + id * 3 + 2);
            const float o = field_term(x0, x1, x2, r0, r1, r2, a.density_factor);
            if (nbr_opacity) nbr_opacity[(size_t)n * a.K + k] = o;
            dens += o;
            bsum += r2.w;
        }
    }
    dens = group_sum<G>(dens);
    bsum = group_sum<G>(bsum);
    if (live && l == 0) {
        const float b = bsum / (float)a.K;
        const OwnAxis ax = own_axis(x0, x1, x2, own[n], a.rec, scaling);
        loss[n] = fabsf(dens - density_target(ax.e, b));
    }
}

template <int G>
__global__ void __launch_bounds__(256) densest_backward_kernel(const FieldArgs a, const int64_t *__restrict__ own,
                                                               const float *__restrict__ scaling,
                                                               const float *__restrict__ g_loss, float *__restrict__ g_x,
                                                               float *__restrict__ grec)
{
    constexpr int SPB = 256 / G;
    const int g = threadIdx.x / G, l = threadIdx.x % G;
    const int n = blockIdx.x * SPB + g;
    const bool live = n < a.N;
    float x0 = 0.f, x1 = 0.f, x2 = 0.f;
    if (live) x0 = a.x[3 * n], x1 = a.x[3 * n + 1], x2 = a.x[3 * n + 2];
    // pass 1: rho and beta of the sample, as the forward
    float dens = 0.f, bsum = 0.f;
    if (live)
        for (int k = l; k < a.K; k += G) {
            const int64_t id = a.idx[(size_t)n * a.K + k];
            const float4 r0 = __ldg(a.rec + id * 3), r1 = __ldg(a.rec + id * 3 + 1), r2 = __ldg(a.rec + id * 3 + 2);
            dens += field_term(x0, x1, x2, r0, r1, r2, a.density_factor);
            bsum += r2.w;
        }
    dens = group_sum<G>(dens);
    bsum = group_sum<G>(bsum);
    // lane 0 of the group: dL/drho, dL/dbeta and dL/de of |rho - t|, t = exp(-e^2 / (2 beta^2))
    float gd = 0.f, gb = 0.f, ge = 0.f;
    if (live && l == 0) {
        const float b = bsum / (float)a.K;
        const OwnAxis ax = own_axis(x0, x1, x2, own[n], a.rec, scaling);
        const float t = density_target(ax.e, b);
        const float r = dens - t;
        const float s = (r > 0.f ? 1.f : (r < 0.f ? -1.f : 0.f)) * g_loss[n];  // torch's abs: 0 at rho == t
        const float ib2 = 1.0f / (b * b);
        gd = s;
        gb = -s * t * (ax.e * ax.e) * ib2 / b;
        ge = s * t * ax.e * ib2;
    }
    const int lead = (threadIdx.x & 31) & ~(G - 1);
    gd = __shfl_sync(0xffffffffu, gd, lead);
    gb = __shfl_sync(0xffffffffu, gb, lead);
    ge = __shfl_sync(0xffffffffu, ge, lead);
    // pass 2: the field backward's per-pair scatter with dL/d opacity = dL/drho
    float gx0 = 0.f, gx1 = 0.f, gx2 = 0.f;
    if (live)
        for (int k = l; k < a.K; k += G) {
            const int64_t id = a.idx[(size_t)n * a.K + k];
            field_pair_backward(x0, x1, x2, id, a.rec, scaling, a.density_factor, gd, gb, a.K, grec, gx0, gx1, gx2);
        }
    gx0 = group_sum<G>(gx0);
    gx1 = group_sum<G>(gx1);
    gx2 = group_sum<G>(gx2);
    if (!live || l != 0) return;
    // the own Gaussian's terms of e = <x - mu_g, n_g>: x, mu_g, and q_g through column `col` of R(q_g).  The axis is
    // gathered again rather than kept live through pass 2 (fewer registers for every lane)
    const int64_t og = own[n];
    const OwnAxis ax = own_axis(x0, x1, x2, og, a.rec, scaling);
    if (g_x) {
        g_x[3 * n] = gx0 + ge * ax.n[0];
        g_x[3 * n + 1] = gx1 + ge * ax.n[1];
        g_x[3 * n + 2] = gx2 + ge * ax.n[2];
    }
    if (ge == 0.f) return;
    float A[3][3];
#pragma unroll
    for (int i = 0; i < 3; i++) {
        const float dn = ge * ax.d[i];
        A[i][0] = ax.col == 0 ? dn : 0.f;
        A[i][1] = ax.col == 1 ? dn : 0.f;
        A[i][2] = ax.col == 2 ? dn : 0.f;
    }
    const float4 dq = rot_backward(A, ax.q, ax.ts);
    float *gr = grec + og * 12;
    red_v4(gr, -ge * ax.n[0], -ge * ax.n[1], -ge * ax.n[2], 0.f);
    red_v4(gr + 4, dq.x, dq.y, dq.z, dq.w);
}

__global__ void __launch_bounds__(256) field_unpack_kernel(int P, const float4 *__restrict__ grec, float *g_points,
                                                           float *g_scaling, float *g_quats, float *g_strengths)
{
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= P) return;
    const float4 a = grec[(size_t)i * 3], b = grec[(size_t)i * 3 + 1], c = grec[(size_t)i * 3 + 2];
    if (g_points) g_points[3 * i] = a.x, g_points[3 * i + 1] = a.y, g_points[3 * i + 2] = a.z;
    if (g_strengths) g_strengths[i] = a.w;
    if (g_quats) ((float4 *)g_quats)[i] = b;
    if (g_scaling) g_scaling[3 * i] = c.x, g_scaling[3 * i + 1] = c.y, g_scaling[3 * i + 2] = c.z;
}

void field_pack(int kind, int P, const float *points, const float *scaling, const float *quats, const float *strengths,
                float4 *rec, cudaStream_t st)
{
    SGR_LAUNCH(kind, st, field_pack_kernel<<<(P + 255) / 256, 256, 0, st>>>(P, points, scaling, quats, strengths, rec));
}

// the packed records, then the backward's per-Gaussian gradient records
struct FieldScratch {
    float4 *rec;
    float *grec;
};

static FieldScratch field_scratch(Layout &l, size_t P) { return {l.take<float4>(3 * P), l.take<float>(12 * P)}; }

}  // namespace sgr

using namespace sgr;

extern "C" {

size_t sgr_field_scratch_bytes(int32_t P) { return P > 0 ? layout_bytes([&](Layout &l) { field_scratch(l, P); }) : 0; }

static int field_check(const SgrFieldParams *p, const void *x, const void *idx, const void *a, const void *b,
                       const void *c, const void *d, const void *scratch)
{
    if (!p || p->N < 0 || p->K <= 0 || p->P <= 0) {
        set_error("bad field sizes");
        return SGR_EINVAL;
    }
    if (p->N > 0 && (!x || !idx || !a || !b || !c || !d || !scratch)) {
        set_error("null pointer passed to sgr_field_*");
        return SGR_EINVAL;
    }
    return SGR_OK;
}

static FieldArgs make_args(const SgrFieldParams *p, const float *x, const int64_t *idx, const float4 *rec)
{
    FieldArgs a;
    a.N = p->N;
    a.K = p->K;
    a.P = p->P;
    a.group = p->samples_per_idx_row > 1 ? p->samples_per_idx_row : 1;
    a.density_factor = p->density_factor;
    // np.sqrt(-2. * np.log(min(density_threshold, 1.)))   (sugar_model.py:1305), evaluated in double like numpy
    const double thr = p->density_threshold < 1.0f ? (double)p->density_threshold : 1.0;
    a.sdf_offset = (float)sqrt(-2.0 * log(thr));
    a.opacity_min_clamp = p->opacity_min_clamp;
    a.x = x;
    a.idx = idx;
    a.rec = rec;
    return a;
}

int sgr_field_forward(const SgrFieldParams *p, const float *x, const int64_t *nbr_idx, const float *points,
                      const float *scaling, const float *quaternions, const float *strengths, float *density,
                      float *nbr_opacity, float *beta, float *sdf, void *scratch, void *stream)
{
    int rc = field_check(p, x, nbr_idx, points, scaling, quaternions, strengths, scratch);
    if (rc) return rc;
    if (p->N == 0) return SGR_OK;
    cudaStream_t st = (cudaStream_t)stream;
    Layout l(scratch);
    float4 *rec = field_scratch(l, p->P).rec;
    field_pack(K_FIELD_PACK, p->P, points, scaling, quaternions, strengths, rec, st);
    const FieldArgs a = make_args(p, x, nbr_idx, rec);
    const int G = group_width(p->K);
    const int blocks = (p->N + 256 / G - 1) / (256 / G);
    sgr::prof_begin(K_FIELD_FWD, st);
    switch (G) {
        case 1: field_forward_kernel<1><<<blocks, 256, 0, st>>>(a, density, nbr_opacity, beta, sdf); break;
        case 2: field_forward_kernel<2><<<blocks, 256, 0, st>>>(a, density, nbr_opacity, beta, sdf); break;
        case 4: field_forward_kernel<4><<<blocks, 256, 0, st>>>(a, density, nbr_opacity, beta, sdf); break;
        case 8: field_forward_kernel<8><<<blocks, 256, 0, st>>>(a, density, nbr_opacity, beta, sdf); break;
        case 16: field_forward_kernel<16><<<blocks, 256, 0, st>>>(a, density, nbr_opacity, beta, sdf); break;
        default: field_forward_kernel<32><<<blocks, 256, 0, st>>>(a, density, nbr_opacity, beta, sdf); break;
    }
    sgr::prof_end(st);
    SGR_CUDA(cudaGetLastError());
    return SGR_OK;
}

int sgr_field_backward(const SgrFieldParams *p, const float *x, const int64_t *nbr_idx, const float *points,
                       const float *scaling, const float *quaternions, const float *strengths,
                       const float *g_density, const float *g_nbr_opacity, const float *g_beta, const float *g_sdf,
                       float *g_x, float *g_points, float *g_scaling, float *g_quaternions, float *g_strengths,
                       void *scratch, void *stream)
{
    int rc = field_check(p, x, nbr_idx, points, scaling, quaternions, strengths, scratch);
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    Layout l(scratch);
    const auto [rec, grec] = field_scratch(l, p->P);
    SGR_CUDA(cudaMemsetAsync(grec, 0, (size_t)p->P * 48, st));
    if (p->N > 0) {
        field_pack(K_FIELD_PACK, p->P, points, scaling, quaternions, strengths, rec, st);
        const FieldArgs a = make_args(p, x, nbr_idx, rec);
        const int G = group_width(p->K);
        const int blocks = (p->N + 256 / G - 1) / (256 / G);
#define SGR_FB(GW)                                                                                                   \
    field_backward_kernel<GW><<<blocks, 256, 0, st>>>(a, scaling, g_density, g_nbr_opacity, g_beta, g_sdf, g_x, grec)
        sgr::prof_begin(K_FIELD_BWD, st);
        switch (G) {
            case 1: SGR_FB(1); break;
            case 2: SGR_FB(2); break;
            case 4: SGR_FB(4); break;
            case 8: SGR_FB(8); break;
            case 16: SGR_FB(16); break;
            default: SGR_FB(32); break;
        }
        sgr::prof_end(st);
#undef SGR_FB
    }
    SGR_LAUNCH(K_FIELD_UNPACK, st,
               field_unpack_kernel<<<(p->P + 255) / 256, 256, 0, st>>>(p->P, (const float4 *)grec, g_points, g_scaling,
                                                                       g_quaternions, g_strengths));
    SGR_CUDA(cudaGetLastError());
    return SGR_OK;
}

// the density estimation loss takes the field's sizes and one index row per sample
static int densest_check(const SgrFieldParams *p, const void *own, const void *out)
{
    if (p && p->samples_per_idx_row > 1) {
        set_error("bad field sizes: sgr_density_estimation_* takes one index row per sample");
        return SGR_EINVAL;
    }
    if (p && p->N > 0 && (!own || !out)) {
        set_error("null pointer passed to sgr_density_estimation_*");
        return SGR_EINVAL;
    }
    return SGR_OK;
}

int sgr_density_estimation_forward(const SgrFieldParams *p, const float *x, const int64_t *own_idx,
                                   const int64_t *nbr_idx, const float *points, const float *scaling,
                                   const float *quaternions, const float *strengths, float *loss, float *nbr_opacity,
                                   void *scratch, void *stream)
{
    int rc = field_check(p, x, nbr_idx, points, scaling, quaternions, strengths, scratch);
    if (!rc) rc = densest_check(p, own_idx, loss);
    if (rc) return rc;
    if (p->N == 0) return SGR_OK;
    cudaStream_t st = (cudaStream_t)stream;
    Layout l(scratch);
    float4 *rec = field_scratch(l, p->P).rec;
    field_pack(K_FIELD_PACK, p->P, points, scaling, quaternions, strengths, rec, st);
    const FieldArgs a = make_args(p, x, nbr_idx, rec);
    const int G = group_width(p->K);
    const int blocks = (p->N + 256 / G - 1) / (256 / G);
#define SGR_DF(GW) densest_forward_kernel<GW><<<blocks, 256, 0, st>>>(a, own_idx, scaling, loss, nbr_opacity)
    sgr::prof_begin(K_DENSEST_FWD, st);
    switch (G) {
        case 1: SGR_DF(1); break;
        case 2: SGR_DF(2); break;
        case 4: SGR_DF(4); break;
        case 8: SGR_DF(8); break;
        case 16: SGR_DF(16); break;
        default: SGR_DF(32); break;
    }
    sgr::prof_end(st);
#undef SGR_DF
    SGR_CUDA(cudaGetLastError());
    return SGR_OK;
}

int sgr_density_estimation_backward(const SgrFieldParams *p, const float *x, const int64_t *own_idx,
                                    const int64_t *nbr_idx, const float *points, const float *scaling,
                                    const float *quaternions, const float *strengths, const float *g_loss, float *g_x,
                                    float *g_points, float *g_scaling, float *g_quaternions, float *g_strengths,
                                    void *scratch, void *stream)
{
    int rc = field_check(p, x, nbr_idx, points, scaling, quaternions, strengths, scratch);
    if (!rc) rc = densest_check(p, own_idx, g_loss);
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    Layout l(scratch);
    const auto [rec, grec] = field_scratch(l, p->P);
    SGR_CUDA(cudaMemsetAsync(grec, 0, (size_t)p->P * 48, st));
    if (p->N > 0) {
        field_pack(K_FIELD_PACK, p->P, points, scaling, quaternions, strengths, rec, st);
        const FieldArgs a = make_args(p, x, nbr_idx, rec);
        const int G = group_width(p->K);
        const int blocks = (p->N + 256 / G - 1) / (256 / G);
#define SGR_DB(GW) densest_backward_kernel<GW><<<blocks, 256, 0, st>>>(a, own_idx, scaling, g_loss, g_x, grec)
        sgr::prof_begin(K_DENSEST_BWD, st);
        switch (G) {
            case 1: SGR_DB(1); break;
            case 2: SGR_DB(2); break;
            case 4: SGR_DB(4); break;
            case 8: SGR_DB(8); break;
            case 16: SGR_DB(16); break;
            default: SGR_DB(32); break;
        }
        sgr::prof_end(st);
#undef SGR_DB
    }
    SGR_LAUNCH(K_FIELD_UNPACK, st,
               field_unpack_kernel<<<(p->P + 255) / 256, 256, 0, st>>>(p->P, (const float4 *)grec, g_points, g_scaling,
                                                                       g_quaternions, g_strengths));
    SGR_CUDA(cudaGetLastError());
    return SGR_OK;
}

}  // extern "C"
