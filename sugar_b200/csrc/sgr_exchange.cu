// sgr_exchange.cu -- the view-parallel step's epilogue after its gradient exchange (NCCL path; the peer exchange's record
// split) and the chunk geometry of the per-Gaussian backward pass; no counterpart in the reference (1 view / 1 GPU,
// sugar_trainers/coarse_sdf.py:98,507).  The epilogue runs one thread per Gaussian of a chunk:
//  * dL_dsh from the views' factors: dL_dsh[i] = sum_v basis(normalize(mean_i - campos_v)) (x) dRGB_v[i]
//    (the SH part of backward.cu:20-139 is an outer product per view).  The 3*M accumulators stay in
//    registers over the views and the rows leave through shared memory as coalesced stores.
//  * the all-reduced 44-byte records (means3D 3 | opacity 1 | scales 3 | rotations 4) are split into
//    the four gradient arrays autograd expects.
// Either half is optional.
#include "sgr_internal.cuh"
#include "sgr_sh.cuh"

namespace sgr {

// Where view v's factor block [P,3] starts: a slice of one gathered buffer (base + v * stride), or -- peer mode -- an
// entry of a device-resident pointer table whose entries may point into OTHER GPUs' memory (CUDA IPC mappings over
// NVLink): the all-gather is then fused into this kernel's loads and no gathered copy exists.
__device__ __forceinline__ const float *view_block(const float *base, size_t stride, const float *const *tab, int v)
{
    return tab ? tab[v] : base + (size_t)v * stride;
}

constexpr int SF_T = 256;  // 64 Gaussians per CTA, four threads each
constexpr int SF_VB = 4;  // views whose factors a thread fetches before it uses any

// Four threads per Gaussian: thread q owns SH coefficients 4q .. 4q+3, i.e. 48 contiguous bytes of the row
// (three 16-byte stores; the four threads of a Gaussian cover its 192-byte row, a warp 1.5 KB without gaps), and
// evaluates only those four basis functions per view -- 12 accumulators instead of 48 per thread, no shared-memory
// transpose, 4x the threads in flight.  Rows with M != 16 use the generic path below (one thread per Gaussian).
// `view_stride` is the distance in floats between two views' factor blocks (>= 3P: the exchange appends each view's
// camera position to its block); campos[v] may live there too.
__global__ void __launch_bounds__(SF_T) view_grad_finalize_m16_kernel(int p0, int p1, int deg, int nviews,
                                                                       const float *__restrict__ means,
                                                                       const float *__restrict__ campos, int campos_stride,
                                                                       const float *__restrict__ dRGB, size_t view_stride,
                                                                       const float *const *__restrict__ view_tab,
                                                                       size_t campos_off, float *__restrict__ dsh,
                                                                       const float *__restrict__ rec11, float scale,
                                                                       float *__restrict__ dmeans3D,
                                                                       float *__restrict__ dopacity,
                                                                       float *__restrict__ dscales, float *__restrict__ drots)
{
    const int t = blockIdx.x * SF_T + threadIdx.x;
    const int i = p0 + (t >> 2), q = t & 3;
    if (i >= p1) return;
    // Every load of the thread is issued before its first store or use: the kernel is a latency chain per thread
    // (records -> stores, mean + factors -> rows), and what hides DRAM latency here is bytes in flight per thread.
    float rv[4] = {0.f, 0.f, 0.f, 0.f};
    if (rec11 && q < 3) {
        // the 11 reduced floats of a Gaussian, split over its four threads: means3D | opacity + scales | rotations
        const float *r = rec11 + (size_t)i * 11 + (q == 0 ? 0 : q == 1 ? 3 : 7);
        rv[0] = __ldcs(r);
        rv[1] = __ldcs(r + 1);
        rv[2] = __ldcs(r + 2);
        if (q) rv[3] = __ldcs(r + 3);
    }
    float mx = 0.f, my = 0.f, mz = 0.f;
    float gv[SF_VB][3];
    if (dsh) {
        mx = __ldg(means + 3 * (size_t)i);
        my = __ldg(means + 3 * (size_t)i + 1);
        mz = __ldg(means + 3 * (size_t)i + 2);
#pragma unroll
        for (int u = 0; u < SF_VB; u++) {
            const bool on = u < nviews;
            const float *g = view_block(dRGB, view_stride, view_tab, on ? u : 0) + (size_t)i * 3;
            gv[u][0] = on ? __ldcs(g) : 0.f;
            gv[u][1] = on ? __ldcs(g + 1) : 0.f;
            gv[u][2] = on ? __ldcs(g + 2) : 0.f;
        }
    }
    if (rec11) {
        if (q == 0) {
            __stcs(dmeans3D + 3 * (size_t)i, rv[0] * scale);
            __stcs(dmeans3D + 3 * (size_t)i + 1, rv[1] * scale);
            __stcs(dmeans3D + 3 * (size_t)i + 2, rv[2] * scale);
        } else if (q == 1) {
            __stcs(dopacity + i, rv[0] * scale);
            __stcs(dscales + 3 * (size_t)i, rv[1] * scale);
            __stcs(dscales + 3 * (size_t)i + 1, rv[2] * scale);
            __stcs(dscales + 3 * (size_t)i + 2, rv[3] * scale);
        } else if (q == 2) {
            __stcs((float4 *)(drots + 4 * (size_t)i), make_float4(rv[0] * scale, rv[1] * scale, rv[2] * scale, rv[3] * scale));
        }
    }
    if (!dsh) return;
    const int used = (deg + 1) * (deg + 1);
    float acc[4][3];
#pragma unroll
    for (int k = 0; k < 4; k++) acc[k][0] = acc[k][1] = acc[k][2] = 0.f;
    // The views' factors are independent 12-byte reads 3P floats apart: a thread fetches SF_VB views' worth at a time
    // (the first batch above, with everything else), so 8 views cost 2 dependent DRAM round trips, not 8.
    for (int v0 = 0; v0 < nviews; v0 += SF_VB) {
        if (v0) {
#pragma unroll
            for (int u = 0; u < SF_VB; u++) {
                const bool on = v0 + u < nviews;
                const float *g = view_block(dRGB, view_stride, view_tab, on ? v0 + u : v0) + (size_t)i * 3;
                gv[u][0] = on ? __ldcs(g) : 0.f;
                gv[u][1] = on ? __ldcs(g + 1) : 0.f;
                gv[u][2] = on ? __ldcs(g + 2) : 0.f;
            }
        }
#pragma unroll
        for (int u = 0; u < SF_VB; u++) {
            const float gr = gv[u][0] * scale, gg = gv[u][1] * scale, gb = gv[u][2] * scale;
            if (gr == 0.f && gg == 0.f && gb == 0.f) continue;  // not visible in this view (or past the last view)
            const float *cp = view_tab ? view_tab[v0 + u] + campos_off : campos + (size_t)(v0 + u) * campos_stride;
            const f3 d = sh_dir(mx, my, mz, __ldg(cp), __ldg(cp + 1), __ldg(cp + 2));
            float w[4] = {0.f, 0.f, 0.f, 0.f};  // basis functions 4q .. 4q + 3, zero at and above (deg + 1)^2
            auto quad = [&](auto q4) {
                constexpr int K0 = 4 * decltype(q4)::value;
                sh_for<K0, K0 + 4>([&](auto k) {
                    constexpr int K = decltype(k)::value;
                    if (K < used) w[K - K0] = sh_basis<K>(d);
                });
            };
            if (q == 0) quad(std::integral_constant<int, 0>{});
            else if (q == 1) quad(std::integral_constant<int, 1>{});
            else if (q == 2) quad(std::integral_constant<int, 2>{});
            else quad(std::integral_constant<int, 3>{});
#pragma unroll
            for (int k = 0; k < 4; k++) {
                acc[k][0] = fmaf(w[k], gr, acc[k][0]);
                acc[k][1] = fmaf(w[k], gg, acc[k][1]);
                acc[k][2] = fmaf(w[k], gb, acc[k][2]);
            }
        }
    }
    // written once, 576 MB per backward at 3M Gaussians: streaming stores keep them from displacing the L2's contents
    float4 *dst = (float4 *)(dsh + (size_t)i * 48 + q * 12);
    __stcs(dst, make_float4(acc[0][0], acc[0][1], acc[0][2], acc[1][0]));
    __stcs(dst + 1, make_float4(acc[1][1], acc[1][2], acc[2][0], acc[2][1]));
    __stcs(dst + 2, make_float4(acc[2][2], acc[3][0], acc[3][1], acc[3][2]));
}

constexpr int SFG_T = 128;

__global__ void __launch_bounds__(SFG_T) view_grad_finalize_kernel(int p0, int p1, int P, int M, int deg, int nviews,
                                                                   const float *__restrict__ means,
                                                                   const float *__restrict__ campos, int campos_stride,
                                                                   const float *__restrict__ dRGB, size_t view_stride,
                                                                   const float *const *__restrict__ view_tab,
                                                                   size_t campos_off, float *__restrict__ dsh,
                                                                   const float *__restrict__ rec11, float scale,
                                                                   float *__restrict__ dmeans3D, float *__restrict__ dopacity,
                                                                   float *__restrict__ dscales, float *__restrict__ drots)
{
    extern __shared__ __align__(16) float s_rows[];  // SFG_T rows x stride floats (SH half only)
    const int tid = threadIdx.x, base = p0 + blockIdx.x * SFG_T, i = base + tid;
    const int n = min(SFG_T, p1 - base);
    if (rec11 && tid < n) {
        const float *r = rec11 + (size_t)i * 11;
        float v[11];
#pragma unroll
        for (int k = 0; k < 11; k++) v[k] = r[k] * scale;
        dmeans3D[3 * (size_t)i] = v[0];
        dmeans3D[3 * (size_t)i + 1] = v[1];
        dmeans3D[3 * (size_t)i + 2] = v[2];
        dopacity[i] = v[3];
        dscales[3 * (size_t)i] = v[4];
        dscales[3 * (size_t)i + 1] = v[5];
        dscales[3 * (size_t)i + 2] = v[6];
        drots[4 * (size_t)i] = v[7];
        drots[4 * (size_t)i + 1] = v[8];
        drots[4 * (size_t)i + 2] = v[9];
        drots[4 * (size_t)i + 3] = v[10];
    }
    if (!dsh) return;
    const int row_f = M * 3;
    int vec;
    const int stride = sh_row_stride(M, false, &vec);
    float acc[48];
#pragma unroll
    for (int k = 0; k < 48; k++) acc[k] = 0.f;
    if (tid < n) {
        const float mx = means[3 * (size_t)i], my = means[3 * (size_t)i + 1], mz = means[3 * (size_t)i + 2];
        for (int v = 0; v < nviews; v++) {
            const float *g = view_block(dRGB, view_stride, view_tab, v) + (size_t)i * 3;
            const float gr = g[0] * scale, gg = g[1] * scale, gb = g[2] * scale;
            if (gr == 0.f && gg == 0.f && gb == 0.f) continue;  // not visible in this view
            const float *cp = view_tab ? view_tab[v] + campos_off : campos + (size_t)v * campos_stride;
            sh_accumulate(deg, acc, sh_dir(mx, my, mz, cp[0], cp[1], cp[2]), {gr, gg, gb});
        }
        float *row = s_rows + tid * stride;
#pragma unroll
        for (int k = 0; k < 48; k++)
            if (k < row_f) row[k] = acc[k];
        for (int k = 48; k < row_f; k++) row[k] = 0.f;
    }
    __syncthreads();
    float *dst = dsh + (size_t)base * row_f;
    sh_rows_walk<SFG_T, 1>(n, row_f, stride, [&](int g, int s) { dst[g] = s_rows[s]; });
}

// CTA range [b0, b1) of chunk c of the per-Gaussian pass.  taper == 0: equal chunks.  taper != 0: every chunk half the size
// of the one before it (weights 2^(n-1-c)), so that what a caller does with a finished chunk while the next one is
// computed (the peer exchange: reduce + split) is matched by that next chunk's shorter run, and little is left after the
// last, smallest chunk.
void chunk_blocks(int blocks, int nchunks, int c, int taper, int *b0, int *b1)
{
    if (!taper || nchunks > 30) {
        *b0 = (int)((int64_t)blocks * c / nchunks);
        *b1 = (int)((int64_t)blocks * (c + 1) / nchunks);
        return;
    }
    const int64_t full = ((int64_t)1 << nchunks) - 1;
    auto edge = [&](int k) { return (int)((int64_t)blocks * ((((int64_t)1 << nchunks) - ((int64_t)1 << (nchunks - k)))) / full); };
    *b0 = edge(c);
    *b1 = c + 1 == nchunks ? blocks : edge(c + 1);
}

int finalize_impl(int32_t P, int32_t p0, int32_t p1, int32_t M, int32_t sh_degree, int32_t num_views,
                  const float *means3D, const float *campos, const float *dRGB, int64_t view_stride, int32_t campos_stride,
                  float *dL_dsh, const float *reduced_records, float scale,
                  float *dL_dmeans3D, float *dL_dopacity, float *dL_dscales, float *dL_drotations, void *stream,
                  const char *who)
{
    const bool sh = dL_dsh != nullptr, rec = reduced_records != nullptr;
    const bool src_ok = campos && dRGB && view_stride >= (int64_t)3 * P && campos_stride >= 3;
    if (P < 0 || p0 < 0 || p1 < p0 || p1 > P || (!sh && !rec) ||
        (sh && (M <= 0 || sh_degree < 0 || sh_degree > 3 || (sh_degree + 1) * (sh_degree + 1) > M || num_views <= 0 ||
                !means3D || !src_ok)) ||
        (rec && (!dL_dmeans3D || !dL_dopacity || !dL_dscales || !dL_drotations))) {
        set_error(who);
        return SGR_EINVAL;
    }
    if (p1 == p0) return SGR_OK;
    cudaStream_t st = (cudaStream_t)stream;
    // the kernels' view-table mode (campos_off: where a table entry keeps its camera position) has no caller
    const size_t campos_off = (size_t)3 * P;
    const bool al16 = (((uintptr_t)dL_dsh | (uintptr_t)dL_drotations) & 15u) == 0;
    if ((!sh || M == 16) && al16) {
        const int threads = (p1 - p0) * 4;
        SGR_LAUNCH(K_FINALIZE, st,
                   view_grad_finalize_m16_kernel<<<(threads + SF_T - 1) / SF_T, SF_T, 0, st>>>(
                       p0, p1, sh_degree, num_views, means3D, campos, campos_stride, dRGB, (size_t)view_stride, nullptr,
                       campos_off, dL_dsh, reduced_records, scale, dL_dmeans3D, dL_dopacity, dL_dscales, dL_drotations));
    } else {
        int vec;
        const size_t dyn = sh ? (size_t)SFG_T * sh_row_stride(M, false, &vec) * sizeof(float) : 0;
        SGR_LAUNCH(K_FINALIZE, st,
                   view_grad_finalize_kernel<<<(p1 - p0 + SFG_T - 1) / SFG_T, SFG_T, dyn, st>>>(
                       p0, p1, P, M, sh_degree, num_views, means3D, campos, campos_stride, dRGB, (size_t)view_stride,
                       nullptr, campos_off, dL_dsh, reduced_records, scale, dL_dmeans3D, dL_dopacity, dL_dscales,
                       dL_drotations));
    }
    SGR_CUDA(cudaGetLastError());
    return SGR_OK;
}

}  // namespace sgr

extern "C" int sgr_backward_chunk_range(int32_t P, int32_t num_chunks, int32_t chunk, int32_t taper, int32_t *p0,
                                        int32_t *p1)
{
    using namespace sgr;
    if (P < 0 || num_chunks < 1 || chunk < 0 || chunk >= num_chunks || !p0 || !p1) {
        set_error("bad arguments to sgr_backward_chunk_range");
        return SGR_EINVAL;
    }
    const int blocks = (P + PB_T - 1) / PB_T, nchunks = backward_chunks(P, num_chunks);
    if (chunk >= nchunks) {
        *p0 = *p1 = P;
        return SGR_OK;
    }
    int b0, b1;
    chunk_blocks(blocks, nchunks, chunk, taper, &b0, &b1);
    *p0 = b0 * PB_T;
    *p1 = b1 * PB_T;
    if (*p1 > P) *p1 = P;
    if (*p0 > P) *p0 = P;
    return SGR_OK;
}

extern "C" int sgr_view_grad_finalize(int32_t P, int32_t p0, int32_t p1, int32_t M, int32_t sh_degree, int32_t num_views,
                                      const float *means3D, const float *campos, const float *dRGB, int64_t view_stride,
                                      int32_t campos_stride, float *dL_dsh, const float *reduced_records, float scale,
                                      float *dL_dmeans3D, float *dL_dopacity, float *dL_dscales, float *dL_drotations,
                                      void *stream)
{
    return sgr::finalize_impl(P, p0, p1, M, sh_degree, num_views, means3D, campos, dRGB, view_stride, campos_stride, dL_dsh, reduced_records, scale, dL_dmeans3D, dL_dopacity, dL_dscales, dL_drotations, stream,
                              "bad arguments to sgr_view_grad_finalize");
}
