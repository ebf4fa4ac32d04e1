// sgr_normal.cu -- SuGaR's "better normal" regularisation as fused kernels.
//
// Replaces the PyTorch op chain inlined in the trainers (sugar_trainers/coarse_sdf.py:688-716, same
// block in coarse_density.py / refine.py) together with SuGaR.get_normals(estimate_from_points=False)
// -> get_smallest_axis (sugar_scene/sugar_model.py:930-968):
//     n_g      = column argmin_j scaling[g][j] of R(quaternions[g])
//     m_k      = sign(<n_k, n_own>) n_k                                (sign detached)
//     w_k      = o_k |<x - mu_k, m_k>| / max(min_j scaling[k][j], 1e-6)^2,  w_k /= max(sum_k w_k, 1e-6)
//     loss     = | n_own - sum_k w_k m_k |^2                           (weights detached)
// with the trainers' only setting sdf_better_normal_gradient_through_normal_only = True
// (coarse_sdf.py:144): gradients reach the quaternions through the normals only.
// The reference gathers N x K x 3 normals, points and several N x K temporaries through autograd;
// here every Gaussian's normal is packed once (32 B record), one lane owns one (sample, neighbour)
// pair, and the backward scatters dL/dn with 16-byte vector reductions before one per-Gaussian
// pass maps dL/dn to dL/dquaternion (pytorch3d quaternion_to_matrix, two_s = 2/|q|^2).  The normal, its quaternion
// backward, the lane groups and their sums are the field kernels' (sgr_field.cuh).
#include "sgr_field.cuh"

namespace sgr {

// per-Gaussian record, 8 floats: n.xyz, 1/max(s_min,1e-6)^2 | mu.xyz, -
__global__ void __launch_bounds__(256) normal_pack_kernel(int P, const float *__restrict__ points,
                                                          const float *__restrict__ scaling,
                                                          const float *__restrict__ quats, float4 *__restrict__ rec)
{
    const int g = blockIdx.x * 256 + threadIdx.x;
    if (g >= P) return;
    const float s[3] = {scaling[3 * g], scaling[3 * g + 1], scaling[3 * g + 2]};
    const SmallestAxis ax = smallest_axis(s, ((const float4 *)quats)[g]);
    const float c = fmaxf(ax.col == 0 ? s[0] : (ax.col == 1 ? s[1] : s[2]), 1e-6f);
    rec[(size_t)g * 2] = make_float4(ax.n[0], ax.n[1], ax.n[2], 1.0f / (c * c));
    rec[(size_t)g * 2 + 1] = make_float4(points[3 * g], points[3 * g + 1], points[3 * g + 2], 0.f);
}

struct NormalArgs {
    int N, K;
    const float *x;
    const int64_t *own, *idx;
    const float4 *rec;
    const float *opac;
};

// residual v = n_own - sum_k w_k m_k of one sample, reduced over its G lanes; returns 1/max(sum w,1e-6)
template <int G>
__device__ __forceinline__ float sample_residual(const NormalArgs &a, bool live, int n, int l, float4 n0, float &vx,
                                                 float &vy, float &vz)
{
    // every lane of the warp reaches the shuffles below through this one call site; dead groups
    // (n >= N) just contribute nothing
    float x0 = 0.f, x1 = 0.f, x2 = 0.f;
    if (live) x0 = a.x[3 * n], x1 = a.x[3 * n + 1], x2 = a.x[3 * n + 2];
    float sx = 0.f, sy = 0.f, sz = 0.f, wsum = 0.f;
    const int Kn = live ? a.K : 0;
    for (int k = l; k < Kn; k += G) {
        const int64_t id = a.idx[(size_t)n * a.K + k];
        const float4 r0 = __ldg(a.rec + id * 2), r1 = __ldg(a.rec + id * 2 + 1);
        const float dot = r0.x * n0.x + r0.y * n0.y + r0.z * n0.z;
        const float sg = dot > 0.f ? 1.f : (dot < 0.f ? -1.f : 0.f);
        const float w = a.opac[(size_t)n * a.K + k] *
                        fabsf(((x0 - r1.x) * r0.x + (x1 - r1.y) * r0.y + (x2 - r1.z) * r0.z) * sg) * r0.w;
        wsum += w;
        sx += w * sg * r0.x;
        sy += w * sg * r0.y;
        sz += w * sg * r0.z;
    }
    wsum = group_sum<G>(wsum);
    sx = group_sum<G>(sx);
    sy = group_sum<G>(sy);
    sz = group_sum<G>(sz);
    const float inv = 1.0f / fmaxf(wsum, 1e-6f);
    vx = n0.x - sx * inv;
    vy = n0.y - sy * inv;
    vz = n0.z - sz * inv;
    return inv;
}

template <int G>
__global__ void __launch_bounds__(256) normal_loss_forward_kernel(const NormalArgs a, float *__restrict__ loss)
{
    constexpr int SPB = 256 / G;
    const int n = blockIdx.x * SPB + threadIdx.x / G, l = threadIdx.x % G;
    const bool live = n < a.N;  // uniform within a group
    float vx, vy, vz;
    float4 n0 = make_float4(0, 0, 0, 0);
    if (live) n0 = __ldg(a.rec + a.own[n] * 2);
    sample_residual<G>(a, live, n, l, n0, vx, vy, vz);
    if (live && l == 0) loss[n] = vx * vx + vy * vy + vz * vz;
}

template <int G>
__global__ void __launch_bounds__(256) normal_loss_backward_kernel(const NormalArgs a, const float *__restrict__ g_loss,
                                                                   float *__restrict__ dnrm /* float4[P] */)
{
    constexpr int SPB = 256 / G;
    const int n = blockIdx.x * SPB + threadIdx.x / G, l = threadIdx.x % G;
    const bool live = n < a.N;
    float vx, vy, vz;
    const int64_t own = live ? a.own[n] : 0;
    float4 n0 = make_float4(0, 0, 0, 0);
    if (live) n0 = __ldg(a.rec + own * 2);
    const float inv = sample_residual<G>(a, live, n, l, n0, vx, vy, vz);
    if (!live) return;
    const float g2 = 2.0f * g_loss[n];
    if (g2 == 0.f) return;
    if (l == 0) red_add_v4(dnrm + own * 4, g2 * vx, g2 * vy, g2 * vz, 0.f);
    const float x0 = a.x[3 * n], x1 = a.x[3 * n + 1], x2 = a.x[3 * n + 2];
    for (int k = l; k < a.K; k += G) {
        const int64_t id = a.idx[(size_t)n * a.K + k];
        const float4 r0 = __ldg(a.rec + id * 2), r1 = __ldg(a.rec + id * 2 + 1);
        const float dot = r0.x * n0.x + r0.y * n0.y + r0.z * n0.z;
        const float sg = dot > 0.f ? 1.f : (dot < 0.f ? -1.f : 0.f);
        const float w = a.opac[(size_t)n * a.K + k] *
                        fabsf(((x0 - r1.x) * r0.x + (x1 - r1.y) * r0.y + (x2 - r1.z) * r0.z) * sg) * r0.w * inv;
        const float c = -g2 * w * sg;
        if (c != 0.f) red_add_v4(dnrm + id * 4, c * vx, c * vy, c * vz, 0.f);
    }
}

// dL/dq from dL/dn
__global__ void __launch_bounds__(256) normal_unpack_kernel(int P, const float *__restrict__ scaling,
                                                            const float *__restrict__ quats,
                                                            const float4 *__restrict__ dnrm, float4 *__restrict__ g_quats)
{
    const int g = blockIdx.x * 256 + threadIdx.x;
    if (g >= P) return;
    const float4 d = dnrm[g];
    if (d.x == 0.f && d.y == 0.f && d.z == 0.f) {
        g_quats[g] = make_float4(0, 0, 0, 0);
        return;
    }
    const float4 q = ((const float4 *)quats)[g];
    const float dn[3] = {d.x, d.y, d.z};
    g_quats[g] = smallest_axis_backward(smallest_axis(scaling + 3 * g, q), q, dn);
}

// the packed records, then the backward's per-Gaussian normal gradients
struct NormalScratch {
    float4 *rec;
    float *dnrm;
};

static NormalScratch normal_scratch(Layout &l, size_t P) { return {l.take<float4>(2 * P), l.take<float>(4 * P)}; }

}  // namespace sgr

using namespace sgr;

extern "C" {

size_t sgr_normal_scratch_bytes(int32_t P) { return P > 0 ? layout_bytes([&](Layout &l) { normal_scratch(l, P); }) : 0; }

static int normal_check(int N, int K, int P, const void *x, const void *own, const void *idx, const void *a,
                        const void *b, const void *c, const void *d, const void *e, const void *scratch)
{
    if (N < 0 || K <= 0 || P <= 0) {
        set_error("bad sizes passed to sgr_normal_loss_*");
        return SGR_EINVAL;
    }
    if (!a || !b || !c || !scratch || (N > 0 && (!x || !own || !idx || !d || !e))) {
        set_error("null pointer passed to sgr_normal_loss_*");
        return SGR_EINVAL;
    }
    return SGR_OK;
}

int sgr_normal_loss_forward(int32_t N, int32_t K, int32_t P, const float *x, const int64_t *own_idx,
                            const int64_t *nbr_idx, const float *points, const float *scaling,
                            const float *quaternions, const float *nbr_opacity, float *loss, void *scratch, void *stream)
{
    int rc = normal_check(N, K, P, x, own_idx, nbr_idx, points, scaling, quaternions, nbr_opacity, loss, scratch);
    if (rc) return rc;
    if (N == 0) return SGR_OK;
    cudaStream_t st = (cudaStream_t)stream;
    Layout l(scratch);
    float4 *rec = normal_scratch(l, P).rec;
    SGR_LAUNCH(K_FIELD_PACK, st, normal_pack_kernel<<<(P + 255) / 256, 256, 0, st>>>(P, points, scaling, quaternions, rec));
    NormalArgs a{N, K, x, own_idx, nbr_idx, rec, nbr_opacity};
    SGR_LAUNCH(K_FIELD_FWD, st, with_group_width(K, [&](auto G) {
                   normal_loss_forward_kernel<G><<<(N + 256 / G - 1) / (256 / G), 256, 0, st>>>(a, loss);
               }));
    SGR_CUDA(cudaGetLastError());
    return SGR_OK;
}

int sgr_normal_loss_backward(int32_t N, int32_t K, int32_t P, const float *x, const int64_t *own_idx,
                             const int64_t *nbr_idx, const float *points, const float *scaling,
                             const float *quaternions, const float *nbr_opacity, const float *g_loss,
                             float *g_quaternions, void *scratch, void *stream)
{
    int rc = normal_check(N, K, P, x, own_idx, nbr_idx, points, scaling, quaternions, nbr_opacity, g_loss, scratch);
    if (rc) return rc;
    if (!g_quaternions) {
        set_error("null pointer passed to sgr_normal_loss_backward");
        return SGR_EINVAL;
    }
    cudaStream_t st = (cudaStream_t)stream;
    Layout l(scratch);
    const NormalScratch s = normal_scratch(l, P);
    SGR_CUDA(cudaMemsetAsync(s.dnrm, 0, (size_t)P * 16, st));
    if (N > 0) {
        SGR_LAUNCH(K_FIELD_PACK, st, normal_pack_kernel<<<(P + 255) / 256, 256, 0, st>>>(P, points, scaling, quaternions, s.rec));
        NormalArgs a{N, K, x, own_idx, nbr_idx, s.rec, nbr_opacity};
        SGR_LAUNCH(K_FIELD_BWD, st, with_group_width(K, [&](auto G) {
                       normal_loss_backward_kernel<G><<<(N + 256 / G - 1) / (256 / G), 256, 0, st>>>(a, g_loss, s.dnrm);
                   }));
    }
    SGR_LAUNCH(K_FIELD_UNPACK, st,
               normal_unpack_kernel<<<(P + 255) / 256, 256, 0, st>>>(P, scaling, quaternions, (const float4 *)s.dnrm,
                                                                     (float4 *)g_quaternions));
    SGR_CUDA(cudaGetLastError());
    return SGR_OK;
}

}  // extern "C"
