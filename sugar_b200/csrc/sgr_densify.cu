// sgr_densify.cu -- densification and pruning of the coarse model's Gaussians (SuGaRDensifier,
// sugar_scene/sugar_densifier.py), restated in oracle/densify_oracle.py.
//
// densify_stats_kernel     one thread per Gaussian: for rows with visibility set, max_radii = max(max_radii,
//                          float(radii)), accum += |grad_means2D[:2]|, denom += 1.  The norm is torch's vector_norm
//                          over two floats on the device: each square rounded, then one add, then sqrtf.
// densify_classify_kernel  one thread per original row: the four per-row flags of densify_and_prune from the float32
//                          gates (the caller rounds the thresholds to float32, as torch does with Python scalars).
//                          The clone and split copies share the parent's density, clones its scale, and both children
//                          exp(log(exp(s) * inv_split)), so every row's fate follows from its parent alone.  The
//                          screen-size clause compares max_radii2D after the appends, which are all zeros.
// densify_map_kernel       one thread per original row: scatters each output row's parent and tag into src_row from
//                          the inclusive scans of the flags (the output order of the reference).
// densify_emit_kernel      one launch over every column, flattened [P' x width] per column so the stores are coalesced
//                          whatever the row width (sh_rest rows are 180 B).  Rows tagged clone or child copy the
//                          parameter and zero the moments; a child's position and log-scale come from its parent and
//                          normal k*S + rank_in_split; a SGR_DENSIFY_POINTS_VANILLA column takes R from vanilla
//                          3DGS's build_rotation instead of pytorch3d's quaternion_to_matrix.
#include <math.h>

#include "sgr_internal.cuh"

namespace sgr {

constexpr int DNS_THREADS = 256;
constexpr int DNS_UNROLL = 4;   // elements per thread of the emit: independent loads in flight

// src_row: parent index in the low 30 bits, tag in the top two
constexpr unsigned TAG_SHIFT = 30, TAG_ORIG = 0u, TAG_CLONE = 1u, TAG_CHILD0 = 2u, TAG_CHILD1 = 3u;

struct DensifyColumns {
    SgrDensifyColumn col[SGR_DENSIFY_MAX_COLUMNS];
    unsigned first_block[SGR_DENSIFY_MAX_COLUMNS + 1];   // block prefix over the columns
    int n;
};

__device__ __forceinline__ float nan_max(float a, float b) { return (isnan(a) || a > b) ? a : b; }  // torch max

__device__ __forceinline__ float sigmoid_f(float x) { return __fdiv_rn(1.0f, __fadd_rn(1.0f, expf(-x))); }

__global__ void __launch_bounds__(DNS_THREADS) densify_stats_kernel(int P, const float *__restrict__ g, int stride,
                                                                    const int *__restrict__ radii,
                                                                    const unsigned char *__restrict__ vis,
                                                                    float *__restrict__ accum, float *__restrict__ denom,
                                                                    float *__restrict__ max_radii)
{
    const int i = blockIdx.x * DNS_THREADS + threadIdx.x;
    if (i >= P || !vis[i]) return;
    const float r = (float)radii[i], m = max_radii[i];
    max_radii[i] = isnan(m) ? m : nan_max(r, m);
    const float gx = g[(size_t)i * stride], gy = g[(size_t)i * stride + 1];
    accum[i] = __fadd_rn(accum[i], sqrtf(__fadd_rn(__fmul_rn(gx, gx), __fmul_rn(gy, gy))));
    denom[i] = __fadd_rn(denom[i], 1.0f);
}

__global__ void __launch_bounds__(DNS_THREADS) densify_classify_kernel(int P, const float *__restrict__ accum,
                                                                       const float *__restrict__ denom,
                                                                       const float *__restrict__ scales,
                                                                       const float *__restrict__ densities,
                                                                       SgrDensifyGates t, unsigned char *__restrict__ flags)
{
    const int i = blockIdx.x * DNS_THREADS + threadIdx.x;
    if (i >= P) return;
    float g = __fdiv_rn(accum[i], denom[i]);
    if (isnan(g)) g = 0.0f;
    float s[3], m = 0.0f, cm = 0.0f;
#pragma unroll
    for (int d = 0; d < 3; d++) {
        s[d] = expf(scales[3 * (size_t)i + d]);
        const float cs = expf(logf(__fmul_rn(s[d], t.inv_split)));   // exp of the child's stored log-scale
        m = d == 0 ? s[d] : nan_max(m, s[d]);
        cm = d == 0 ? cs : nan_max(cm, cs);
    }
    // clone: torch.norm over the size-1 gradient dimension, sqrt of the rounded square
    const bool clone = sqrtf(__fmul_rn(g, g)) >= t.max_grad && m <= t.clone_scale;
    const bool split = g >= t.max_grad && m > t.clone_scale;
    const bool low = sigmoid_f(densities[i]) < t.min_opacity;
    const bool screen = t.use_screen && 0.0f > t.screen_size;   // max_radii2D is zeros after the appends
    const bool prune = low || (t.use_screen && (screen || m > t.big_scale));
    const bool prune_child = low || (t.use_screen && (screen || cm > t.big_scale));
    flags[i] = !split && !prune;
    flags[(size_t)P + i] = clone && !prune;
    flags[2 * (size_t)P + i] = split;
    flags[3 * (size_t)P + i] = split && !prune_child;
}

__global__ void __launch_bounds__(DNS_THREADS) densify_map_kernel(int P, const int *__restrict__ scan, int n_keep,
                                                                  int n_clone, int n_child, int *__restrict__ src_row)
{
    const int i = blockIdx.x * DNS_THREADS + threadIdx.x;
    if (i >= P) return;
    int at[4], f[4];
#pragma unroll
    for (int k = 0; k < 4; k++) {
        const int *sc = scan + (size_t)k * P;
        at[k] = sc[i];
        f[k] = at[k] - (i ? sc[i - 1] : 0);
    }
    if (f[0]) src_row[at[0] - 1] = i | (int)(TAG_ORIG << TAG_SHIFT);
    if (f[1]) src_row[n_keep + at[1] - 1] = i | (int)(TAG_CLONE << TAG_SHIFT);
    if (f[3]) {
        src_row[n_keep + n_clone + at[3] - 1] = i | (int)(TAG_CHILD0 << TAG_SHIFT);
        src_row[n_keep + n_clone + n_child + at[3] - 1] = i | (int)(TAG_CHILD1 << TAG_SHIFT);
    }
}

// R . (normal * exp(scale)) + point for row R of the child's rotation (the bmm's dot product as an fma chain)
__device__ __forceinline__ float child_offset(int p, int d, int copy, int S, const int *__restrict__ split_scan,
                                              const float *__restrict__ points, const float *__restrict__ scales,
                                              const float *__restrict__ normals, const float R[3])
{
    const size_t z = 3 * ((size_t)copy * S + (split_scan[p] - 1));
    float x = 0.0f;
#pragma unroll
    for (int c = 0; c < 3; c++) x = fmaf(R[c], __fmul_rn(normals[z + c], expf(scales[3 * (size_t)p + c])), x);
    return __fadd_rn(x, points[3 * (size_t)p + d]);
}

// row d of vanilla 3DGS's build_rotation(q) (utils/general_utils.py:78-99), each torch op rounded on its own:
// norm = sqrt(((r*r + x*x) + y*y) + z*z), no epsilon; q / norm a true division; then the entries as written
__device__ void vanilla_rotation_row(float4 q, int d, float R[3])
{
    const float n = sqrtf(__fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(q.x, q.x), __fmul_rn(q.y, q.y)), __fmul_rn(q.z, q.z)),
                                    __fmul_rn(q.w, q.w)));
    const float r = __fdiv_rn(q.x, n), x = __fdiv_rn(q.y, n), y = __fdiv_rn(q.z, n), z = __fdiv_rn(q.w, n);
    if (d == 0) {
        R[0] = __fsub_rn(1.0f, __fmul_rn(2.0f, __fadd_rn(__fmul_rn(y, y), __fmul_rn(z, z))));
        R[1] = __fmul_rn(2.0f, __fsub_rn(__fmul_rn(x, y), __fmul_rn(r, z)));
        R[2] = __fmul_rn(2.0f, __fadd_rn(__fmul_rn(x, z), __fmul_rn(r, y)));
    } else if (d == 1) {
        R[0] = __fmul_rn(2.0f, __fadd_rn(__fmul_rn(x, y), __fmul_rn(r, z)));
        R[1] = __fsub_rn(1.0f, __fmul_rn(2.0f, __fadd_rn(__fmul_rn(x, x), __fmul_rn(z, z))));
        R[2] = __fmul_rn(2.0f, __fsub_rn(__fmul_rn(y, z), __fmul_rn(r, x)));
    } else {
        R[0] = __fmul_rn(2.0f, __fsub_rn(__fmul_rn(x, z), __fmul_rn(r, y)));
        R[1] = __fmul_rn(2.0f, __fadd_rn(__fmul_rn(y, z), __fmul_rn(r, x)));
        R[2] = __fsub_rn(1.0f, __fmul_rn(2.0f, __fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y))));
    }
}

// position (d) of child copy k of parent p: R(q^) (normal * scale) + point, R as pytorch3d's quaternion_to_matrix, or
// as vanilla 3DGS's build_rotation when `vanilla`
__device__ float child_position(int p, int d, int copy, int S, const int *__restrict__ split_scan,
                                const float *__restrict__ points, const float *__restrict__ scales,
                                const float *__restrict__ quats, const float *__restrict__ normals, bool vanilla)
{
    const float4 q = reinterpret_cast<const float4 *>(quats)[p];
    float R[3];
    if (vanilla) {
        vanilla_rotation_row(q, d, R);
        return child_offset(p, d, copy, S, split_scan, points, scales, normals, R);
    }
    // F.normalize: q / max(|q|, 1e-12), |q| summed pairwise as torch's reduction does
    const float n = fmaxf(sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(q.x, q.x), __fmul_rn(q.y, q.y)),
                                          __fadd_rn(__fmul_rn(q.z, q.z), __fmul_rn(q.w, q.w)))), 1e-12f);
    const float r = __fdiv_rn(q.x, n), qi = __fdiv_rn(q.y, n), qj = __fdiv_rn(q.z, n), qk = __fdiv_rn(q.w, n);
    const float two_s = __fdiv_rn(2.0f, __fadd_rn(__fadd_rn(__fmul_rn(r, r), __fmul_rn(qi, qi)),
                                                  __fadd_rn(__fmul_rn(qj, qj), __fmul_rn(qk, qk))));
    if (d == 0) {
        R[0] = __fsub_rn(1.0f, __fmul_rn(two_s, __fadd_rn(__fmul_rn(qj, qj), __fmul_rn(qk, qk))));
        R[1] = __fmul_rn(two_s, __fsub_rn(__fmul_rn(qi, qj), __fmul_rn(qk, r)));
        R[2] = __fmul_rn(two_s, __fadd_rn(__fmul_rn(qi, qk), __fmul_rn(qj, r)));
    } else if (d == 1) {
        R[0] = __fmul_rn(two_s, __fadd_rn(__fmul_rn(qi, qj), __fmul_rn(qk, r)));
        R[1] = __fsub_rn(1.0f, __fmul_rn(two_s, __fadd_rn(__fmul_rn(qi, qi), __fmul_rn(qk, qk))));
        R[2] = __fmul_rn(two_s, __fsub_rn(__fmul_rn(qj, qk), __fmul_rn(qi, r)));
    } else {
        R[0] = __fmul_rn(two_s, __fsub_rn(__fmul_rn(qi, qk), __fmul_rn(qj, r)));
        R[1] = __fmul_rn(two_s, __fadd_rn(__fmul_rn(qj, qk), __fmul_rn(qi, r)));
        R[2] = __fsub_rn(1.0f, __fmul_rn(two_s, __fadd_rn(__fmul_rn(qi, qi), __fmul_rn(qj, qj))));
    }
    return child_offset(p, d, copy, S, split_scan, points, scales, normals, R);
}

__global__ void __launch_bounds__(DNS_THREADS) densify_emit_kernel(DensifyColumns cols, int P_out, int S,
                                                                   const int *__restrict__ src_row,
                                                                   const int *__restrict__ split_scan,
                                                                   const float *__restrict__ points,
                                                                   const float *__restrict__ scales,
                                                                   const float *__restrict__ quats,
                                                                   const float *__restrict__ normals, float inv_split)
{
    int c = 0;
    while (c + 1 < cols.n && blockIdx.x >= cols.first_block[c + 1]) c++;
    const SgrDensifyColumn col = cols.col[c];
    const unsigned w = (unsigned)col.width, total = (unsigned)P_out * w;
    const unsigned base = (blockIdx.x - cols.first_block[c]) * (DNS_THREADS * DNS_UNROLL) + threadIdx.x;
    float v[DNS_UNROLL];
#pragma unroll
    for (int u = 0; u < DNS_UNROLL; u++) {
        const unsigned e = base + u * DNS_THREADS;
        v[u] = 0.0f;
        if (e >= total) continue;
        const unsigned row = e / w, d = e - row * w;
        const unsigned code = (unsigned)src_row[row], p = code & ((1u << TAG_SHIFT) - 1), tag = code >> TAG_SHIFT;
        if (tag != TAG_ORIG && col.kind == SGR_DENSIFY_ZERO_NEW) continue;
        if (tag >= TAG_CHILD0 && (col.kind == SGR_DENSIFY_POINTS || col.kind == SGR_DENSIFY_POINTS_VANILLA))
            v[u] = child_position((int)p, (int)d, (int)(tag - TAG_CHILD0), S, split_scan, points, scales, quats,
                                  normals, col.kind == SGR_DENSIFY_POINTS_VANILLA);
        else if (tag >= TAG_CHILD0 && col.kind == SGR_DENSIFY_SCALES)
            v[u] = logf(__fmul_rn(expf(col.src[(size_t)p * 3 + d]), inv_split));
        else
            v[u] = col.src[(size_t)p * w + d];
    }
#pragma unroll
    for (int u = 0; u < DNS_UNROLL; u++) {
        const unsigned e = base + u * DNS_THREADS;
        if (e < total) col.dst[e] = v[u];
    }
}

static int dns_blocks(long long n, int per) { return (int)((n + per - 1) / per); }

}  // namespace sgr

using namespace sgr;

extern "C" {

int sgr_densify_stats(int32_t P, const float *grad_means2D, int32_t grad_stride, const int32_t *radii,
                      const uint8_t *visibility, float *accum, float *denom, float *max_radii, void *stream)
{
    if (P < 0 || grad_stride < 2 || (long long)P * grad_stride > INT32_MAX) {
        set_error("sgr_densify_stats: bad sizes P=%d grad_stride=%d (stride >= 2, P*stride <= 2^31 - 1)", P,
                  grad_stride);
        return SGR_EINVAL;
    }
    if (P == 0) return SGR_OK;
    if (!grad_means2D || !radii || !visibility || !accum || !denom || !max_radii) {
        set_error("sgr_densify_stats: null pointer");
        return SGR_EINVAL;
    }
    cudaStream_t st = (cudaStream_t)stream;
    SGR_LAUNCH(K_MISC, st,
               densify_stats_kernel<<<dns_blocks(P, DNS_THREADS), DNS_THREADS, 0, st>>>(
                   P, grad_means2D, grad_stride, radii, visibility, accum, denom, max_radii));
    SGR_CUDA(cudaGetLastError());
    return SGR_OK;
}

int sgr_densify_classify(int32_t P, const float *accum, const float *denom, const float *scales,
                         const float *densities, const SgrDensifyGates *gates, uint8_t *flags, void *stream)
{
    if (P < 0 || P >= (1 << 30) || !gates) {
        set_error("sgr_densify_classify: bad sizes P=%d (P < 2^30) or null gates", P);
        return SGR_EINVAL;
    }
    if (P == 0) return SGR_OK;
    if (!accum || !denom || !scales || !densities || !flags) {
        set_error("sgr_densify_classify: null pointer");
        return SGR_EINVAL;
    }
    cudaStream_t st = (cudaStream_t)stream;
    SGR_LAUNCH(K_MISC, st,
               densify_classify_kernel<<<dns_blocks(P, DNS_THREADS), DNS_THREADS, 0, st>>>(
                   P, accum, denom, scales, densities, *gates, flags));
    SGR_CUDA(cudaGetLastError());
    return SGR_OK;
}

int sgr_densify_emit(int32_t P, int32_t n_keep, int32_t n_clone, int32_t S, int32_t n_child, const int32_t *scan,
                     int32_t n_cols, const SgrDensifyColumn *cols, const float *points, const float *scales,
                     const float *quaternions, const float *normals, float inv_split, int32_t *src_row, void *stream)
{
    const long long P_out = (long long)n_keep + n_clone + 2LL * n_child;
    if (P < 0 || P >= (1 << 30) || n_keep < 0 || n_clone < 0 || S < 0 || n_child < 0 || S > P || n_child > S ||
        n_keep > P - S || n_clone > P - S) {
        set_error("sgr_densify_emit: counts disagree with P=%d: n_keep=%d n_clone=%d S=%d n_child=%d (kept and "
                  "cloned rows are not split, n_child <= S <= P < 2^30)", P, n_keep, n_clone, S, n_child);
        return SGR_EINVAL;
    }
    if (n_cols < 0 || n_cols > SGR_DENSIFY_MAX_COLUMNS || (n_cols > 0 && !cols)) {
        set_error("sgr_densify_emit: n_cols=%d (0..%d, cols on the host)", n_cols, SGR_DENSIFY_MAX_COLUMNS);
        return SGR_EINVAL;
    }
    DensifyColumns tab;
    tab.n = n_cols;
    tab.first_block[0] = 0;
    long long blocks = 0;
    for (int c = 0; c < n_cols; c++) {
        const SgrDensifyColumn &k = cols[c];
        if (k.width <= 0 || k.kind < SGR_DENSIFY_COPY || k.kind > SGR_DENSIFY_POINTS_VANILLA ||
            (k.kind >= SGR_DENSIFY_POINTS && k.width != 3) || P_out * k.width > INT32_MAX) {
            set_error("sgr_densify_emit: column %d: width=%d kind=%d (width > 0, 3 for points and scales, "
                      "P' * width <= 2^31 - 1 with P'=%lld)", c, k.width, k.kind, P_out);
            return SGR_EINVAL;
        }
        if (P_out > 0 && (!k.dst || !k.src)) {
            set_error("sgr_densify_emit: column %d: null pointer", c);
            return SGR_EINVAL;
        }
        tab.col[c] = k;
        blocks += dns_blocks(P_out * k.width, DNS_THREADS * DNS_UNROLL);
        tab.first_block[c + 1] = (unsigned)blocks;
    }
    if (P_out == 0 || n_cols == 0) return SGR_OK;
    if (!scan || !src_row || (n_child > 0 && (!points || !scales || !quaternions || !normals))) {
        set_error("sgr_densify_emit: null pointer");
        return SGR_EINVAL;
    }
    if ((size_t)quaternions & 15) {
        set_error("sgr_densify_emit: quaternions must be 16-byte aligned");
        return SGR_EINVAL;
    }
    cudaStream_t st = (cudaStream_t)stream;
    SGR_LAUNCH(K_MISC, st,
               densify_map_kernel<<<dns_blocks(P, DNS_THREADS), DNS_THREADS, 0, st>>>(P, scan, n_keep, n_clone,
                                                                                       n_child, src_row));
    SGR_LAUNCH(K_MISC, st,
               densify_emit_kernel<<<(unsigned)blocks, DNS_THREADS, 0, st>>>(
                   tab, (int)P_out, S, src_row, scan + 2 * (size_t)P, points, scales, quaternions, normals,
                   inv_split));
    SGR_CUDA(cudaGetLastError());
    return SGR_OK;
}

}  // extern "C"
