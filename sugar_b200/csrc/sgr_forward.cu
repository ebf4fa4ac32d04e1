// sgr_forward.cu -- forward path of the H100 rasterizer.
//
// Replaces (reference: gaussian_splatting/submodules/diff-gaussian-rasterization/cuda_rasterizer/)
//   preprocessCUDA            forward.cu:155-256      -> preprocess_kernel   (+ per-tile counting)
//   InclusiveSum + D2H sync   rasterizer_impl.cu:277-281 -> tile_scan_kernel (over TILES, not Gaussians)
//   duplicateWithKeys         rasterizer_impl.cu:70-111  -> scatter_kernel   (atomic cursor per tile)
//   cub SortPairs (6 passes)  rasterizer_impl.cu:303-308 -> tile_sort_{bucket,merge}_kernel (per tile, in smem),
//                                                          tile_sort_global_kernel (tiles above SORT_CAP)
//   identifyTileRanges        rasterizer_impl.cu:116-138 -> (ranges fall out of the tile scan)
//   renderCUDA                forward.cu:261-374      -> blend_forward_kernel
//
// Binning design: the 64-bit key (tile<<32 | depth) is sorted MSD-first.  The tile digit is a
// counting sort (per-tile counts by L2 atomics in preprocess, exclusive scan over tiles, atomic
// cursor scatter), the remaining (depth, gaussian-id) order is sorted by one CTA per tile in its
// shared memory (bucket or merge sort by size class; tiles of more than SORT_CAP instances take an
// 8-bit LSD radix sort through global memory).  Instances move through HBM once (8 B write,
// 8 B read, 4 B write) instead of ~150 B for six global radix passes, and the sorted order is
// exactly the reference's: by tile, then depth bits, then Gaussian index (the reference's
// stable sort keeps emission order = index order among equal keys).
#include <stdarg.h>
#include <stdio.h>

#include <mutex>
#include <vector>

#include "sgr_internal.cuh"
#include "sgr_sh.cuh"

namespace sgr {

// ------------------------------------------------------------------------------------------------
// preprocess
// ------------------------------------------------------------------------------------------------
constexpr int PRE_T = 128;

struct PreArgs {
    int P;
    const float *means, *scales, *rots, *opac, *shs, *colors, *cov_pre;
    // raw-parameter mode (SgrGaussians.activations != 0): opac = logits, scales = logs, rots un-normalised, the SH
    // coefficients in the model's own two arrays: shs = the DC term [P,1,3], sh_rest = the others [P,M-1,3]
    const float *sh_rest;
    ViewConsts v;
    int bulk_ok;      // all staged arrays 16B-aligned
    int sh_stride;    // padded smem row stride in floats (0 = no SH)
    int sh_vec;       // 1: rows copied as 16-byte cp.async, 0: 4-byte
    GeomState geom;
    int32_t *radii;
    uint32_t *tile_count;
};

// Cooperative, coalesced copy of n floats into shared memory (fallback when bulk copy is not legal).
__device__ __forceinline__ void stage_plain(float *dst, const float *__restrict__ src, int n)
{
    for (int i = threadIdx.x; i < n; i += PRE_T) dst[i] = __ldg(src + i);
}

// RAW: SuGaR's activations (sugar_model.py:400-479: sigmoid of the densities, exp of the scales, normalize of
// the quaternions) are applied to the staged values here and the SH coefficients come from the model's own
// (dc, rest) arrays, so a training step needs no elementwise prologue kernels in front of the op.  The rest block
// of a CTA is one contiguous run -> a single bulk copy into rows of M-1 coefficients (stride 3(M-1) floats: odd
// for M = 16, conflict-free).
template <bool RAW>
__global__ void __launch_bounds__(PRE_T) preprocess_kernel(const PreArgs a)
{
    extern __shared__ __align__(16) float s_sh[];  // PRE_T rows x sh_stride floats (only with SH)
    __shared__ __align__(16) float s_means[PRE_T * 3];
    __shared__ __align__(16) float4 s_rots[PRE_T];
    __shared__ __align__(16) float s_opac[PRE_T];
    __shared__ __align__(16) float s_col[PRE_T * 3];
    // scales (3 floats) and cov3D_precomp (6) of the CTA's Gaussians; once every thread is past the geometry phase the
    // same 36 bytes per Gaussian hold its SH Jacobian row on the way out (a separate array would cost the kernel one
    // of its six CTAs per SM)
    __shared__ __align__(16) float s_geo[PRE_T * 9];
    float *const s_scales = s_geo, *const s_cov = s_geo + PRE_T * 3, *const s_jac = s_geo;
    __shared__ __align__(8) uint64_t s_bar;

    const int tid = threadIdx.x;
    const int base = blockIdx.x * PRE_T;
    const int n = min(PRE_T, a.P - base);
    const int idx = base + tid;
    const bool full = (n == PRE_T);

    // ---- stage inputs: one elected thread drives the TMA engine with 1-D bulk copies -----------
    if (a.bulk_ok && full) {
        if (tid == 0) {
            mbar_init(&s_bar, 1);
            mbar_fence_init();
            uint32_t bytes = PRE_T * 12 + PRE_T * 4;
            if (a.scales) bytes += PRE_T * 12 + PRE_T * 16;
            if (a.cov_pre) bytes += PRE_T * 24;
            if (a.colors) bytes += PRE_T * 12;
            if (RAW && a.shs) bytes += PRE_T * 12 + PRE_T * (uint32_t)(a.v.M - 1) * 12;
            mbar_expect_tx(&s_bar, bytes);
            if (RAW && a.shs) {
                bulk_g2s(s_col, a.shs + (size_t)base * 3, PRE_T * 12, &s_bar);  // DC terms (colours are absent with SH)
                if (a.v.M > 1)
                    bulk_g2s(s_sh, a.sh_rest + (size_t)base * (a.v.M - 1) * 3, PRE_T * (uint32_t)(a.v.M - 1) * 12, &s_bar);
            }
            bulk_g2s(s_means, a.means + (size_t)base * 3, PRE_T * 12, &s_bar);
            bulk_g2s(s_opac, a.opac + base, PRE_T * 4, &s_bar);
            if (a.scales) {
                bulk_g2s(s_scales, a.scales + (size_t)base * 3, PRE_T * 12, &s_bar);
                bulk_g2s(s_rots, a.rots + (size_t)base * 4, PRE_T * 16, &s_bar);
            }
            if (a.cov_pre) bulk_g2s(s_cov, a.cov_pre + (size_t)base * 6, PRE_T * 24, &s_bar);
            if (a.colors) bulk_g2s(s_col, a.colors + (size_t)base * 3, PRE_T * 12, &s_bar);
        }
    } else {
        stage_plain(s_means, a.means + (size_t)base * 3, n * 3);
        stage_plain(s_opac, a.opac + base, n);
        if (a.scales) {
            stage_plain(s_scales, a.scales + (size_t)base * 3, n * 3);
            stage_plain((float *)s_rots, a.rots + (size_t)base * 4, n * 4);
        }
        if (a.cov_pre) stage_plain(s_cov, a.cov_pre + (size_t)base * 6, n * 6);
        if (a.colors) stage_plain(s_col, a.colors + (size_t)base * 3, n * 3);
        if (RAW && a.shs) {
            stage_plain(s_col, a.shs + (size_t)base * 3, n * 3);
            stage_plain(s_sh, a.sh_rest + (size_t)base * (a.v.M - 1) * 3, n * (a.v.M - 1) * 3);
        }
    }
    // ---- SH rows: coalesced cp.async into bank-conflict-free padded rows -----------------------
    if (!RAW && a.shs) {
        const int row_f = a.v.M * 3;
        const float *src = a.shs + (size_t)base * row_f;
        if (a.sh_vec) sh_rows_walk<PRE_T, 4>(n, row_f, a.sh_stride, [&](int g, int s) { cp_async16(s_sh + s, src + g); });
        else sh_rows_walk<PRE_T, 1>(n, row_f, a.sh_stride, [&](int g, int s) { cp_async4(s_sh + s, src + g); });
        cp_async_commit();
    }
    __syncthreads();  // barrier init visible / plain staging complete
    if (a.bulk_ok && full) mbar_wait(&s_bar, 0);

    // ---- per-Gaussian projection, cull, covariance, radius, tile rect (bit-exact chain) --------
    int x0 = 0, y0 = 0, x1 = 0, y1 = 0, radius = 0;
    bool visible = false;
    float depth = 0.f, px = 0.f, py = 0.f, con_a = 0.f, con_b = 0.f, con_c = 0.f, opacity = 0.f;
    float mx = 0.f, my = 0.f, mz = 0.f;
    if (tid < n) {
        mx = s_means[tid * 3], my = s_means[tid * 3 + 1], mz = s_means[tid * 3 + 2];
        const float *vm = a.v.viewmatrix, *pm = a.v.projmatrix;
        depth = xf_row(vm, 2, mx, my, mz);
        if (depth <= 0.2f) {
            if (a.v.prefiltered) {  // auxiliary.h:156-160
                printf("Point is filtered although prefiltered is set. This shouldn't happen!");
                __trap();
            }
        } else {
            const float hx = xf_row(pm, 0, mx, my, mz), hy = xf_row(pm, 1, mx, my, mz), hw = xf_row(pm, 3, mx, my, mz);
            const float p_w = __frcp_rn(__fadd_rn(hw, 0.0000001f));
            const float projx = __fmul_rn(hx, p_w), projy = __fmul_rn(hy, p_w);
            float c3[6];
            if (a.cov_pre) {
#pragma unroll
                for (int k = 0; k < 6; k++) c3[k] = s_cov[tid * 6 + k];
            } else {
                float s0 = s_scales[tid * 3], s1 = s_scales[tid * 3 + 1], s2 = s_scales[tid * 3 + 2];
                float4 q = s_rots[tid];
                if (RAW) {  // scale_activation = exp, quaternions = F.normalize(_quaternions) (sugar_model.py:417,479)
                    s0 = expf(s0), s1 = expf(s1), s2 = expf(s2);
                    const float inv = __fdiv_rn(1.0f, fmaxf(sqrtf(q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w), 1e-12f));
                    q = make_float4(q.x * inv, q.y * inv, q.z * inv, q.w * inv);
                }
                cov3d_from_scale_rot(s0, s1, s2, a.v.scale_modifier, q, c3);
            }
            const float tx0 = xf_row(vm, 0, mx, my, mz), ty0 = xf_row(vm, 1, mx, my, mz);
            const Cov2D cv = cov2d_project(tx0, ty0, depth, a.v.focal_x, a.v.focal_y, a.v.tanfovx, a.v.tanfovy, c3, vm);
            const float det = __fmaf_rn(cv.a, cv.c, -__fmul_rn(cv.b, cv.b));
            if (det != 0.0f) {
                const float det_inv = __frcp_rn(det);
                con_a = __fmul_rn(cv.c, det_inv);
                con_b = __fmul_rn(cv.b, -det_inv);
                con_c = __fmul_rn(cv.a, det_inv);
                const float mid = __fmul_rn(__fadd_rn(cv.a, cv.c), 0.5f);
                const float s = __fsqrt_rn(fmaxf(0.1f, __fmaf_rn(mid, mid, -det)));
                const float lmax = fmaxf(__fadd_rn(mid, s), __fsub_rn(mid, s));
                radius = (int)ceilf(__fmul_rn(3.0f, __fsqrt_rn(lmax)));
                px = ndc2pix(projx, a.v.W);
                py = ndc2pix(projy, a.v.H);
                tile_rect(px, py, radius, a.v.gx, a.v.gy, x0, y0, x1, y1);
                visible = (x1 - x0) * (y1 - y0) != 0;
                opacity = s_opac[tid];
                if (RAW) opacity = __fdiv_rn(1.0f, 1.0f + expf(-opacity));  // strengths = sigmoid(all_densities) (:403)
            }
        }
    }
    if (a.shs) {
        if (!RAW) cp_async_wait<0>();
        __syncthreads();  // SH rows landed; no thread reads s_scales / s_cov any more, s_jac may overwrite them
    }
    if (tid < n) {
        float jac[9];  // (dRGBdx, dRGBdy, dRGBdz) as RGB triples; zero for culled Gaussians and degree 0
#pragma unroll
        for (int k = 0; k < 9; k++) jac[k] = 0.f;
        if (visible) {
            float r, g, b;
            uint32_t clamp_bits = 0;
            if (a.colors) {
                r = s_col[tid * 3], g = s_col[tid * 3 + 1], b = s_col[tid * 3 + 2];
            } else {
                const float *cp = a.v.campos;
                const f3 d = sh_dir(mx, my, mz, cp[0], cp[1], cp[2]);
                const float *dc, *rest;
                if (RAW) {
                    dc = s_col + tid * 3;
                    rest = s_sh + tid * (a.v.M - 1) * 3;
                } else {
                    dc = s_sh + tid * a.sh_stride;
                    rest = dc + 3;
                }
                auto channel = [&](int c) {
                    return sh_channel(a.v.D, d, [&](int k) { return k == 0 ? dc[c] : rest[(k - 1) * 3 + c]; });
                };
                r = channel(0), g = channel(1), b = channel(2);
                if (a.v.D > 0) {
#pragma unroll
                    for (int c = 0; c < 3; c++) sh_channel_jacobian(a.v.D, rest + c, d.x, d.y, d.z, jac[c], jac[3 + c], jac[6 + c]);
                }
                // clamped <=> result + 0.5 < 0 (forward.cu:63-70)
                clamp_bits = (r < -0.5f ? 1u : 0u) | (g < -0.5f ? 2u : 0u) | (b < -0.5f ? 4u : 0u);
                r = (clamp_bits & 1u) ? 0.0f : __fadd_rn(r, 0.5f);
                g = (clamp_bits & 2u) ? 0.0f : __fadd_rn(g, 0.5f);
                b = (clamp_bits & 4u) ? 0.0f : __fadd_rn(b, 0.5f);
            }
            // Conservative cull threshold: alpha = min(.99, o*exp(power)) < 1/255 is certain when
            // power < tau = ln(1/(255 o)) - 1e-4 (margin >> ulp error of expf/logf; DESIGN.md).
            // "Always skipped" is exactly the blend's own rejection of the largest alpha, o < 1/255: at
            // o == 1/255 (where o * 255 rounds to 1) a pixel with power == 0 has alpha == 1/255 and is drawn,
            // and tau = -1e-4 keeps it.
            float tau;
            if (opacity < 1.0f / 255.0f) tau = __int_as_float(0x7f800000);  // never reaches 1/255: always skipped
            else if (opacity == opacity) tau = -logf(opacity * 255.0f) - 1e-4f;
            else tau = -__int_as_float(0x7f800000);                          // NaN opacity: take the exact path
            float4 *rec = a.geom.rec + (size_t)idx * 3;
            rec[0] = make_float4(px, py, con_a, con_b);
            rec[1] = make_float4(con_c, tau, opacity, r);
            // the SH clamp bits and the Gaussian's own index ride in the record's spare words: the backward
            // blend masks dL/dRGB with the bits and addresses its accumulators with the index
            rec[2] = make_float4(g, b, __uint_as_float(clamp_bits), __uint_as_float((uint32_t)idx));
            a.geom.depth[idx] = depth;
            a.geom.rect[idx] = make_ushort4((unsigned short)x0, (unsigned short)y0, (unsigned short)x1, (unsigned short)y1);
            a.radii[idx] = radius;
        } else {
            a.geom.rect[idx] = make_ushort4(0, 0, 0, 0);
            a.radii[idx] = 0;
        }
        if (a.shs) {
#pragma unroll
            for (int k = 0; k < 9; k++) s_jac[tid * 9 + k] = jac[k];  // stride 9: conflict-free
        }
    }
    // the CTA's Jacobian rows are one contiguous block of sh_jac: coalesced 16-byte stores, evict-first (only the
    // backward reads them, long after this pass; a single bulk store per CTA measured the same)
    if (a.shs) {
        __syncthreads();
        float *dst = a.geom.sh_jac + (size_t)base * 9;
        if (full) {
            for (int k = tid; k < PRE_T * 9 / 4; k += PRE_T) __stcs((float4 *)dst + k, ((const float4 *)s_jac)[k]);
        } else {
            for (int k = tid; k < n * 9; k += PRE_T) __stcs(dst + k, s_jac[k]);
        }
    }

    // ---- per-tile instance counts.  Small rects (the common case) are walked by their own thread;
    // rects of more than SMALL tiles are walked by the whole warp so one huge splat cannot stall it.
    constexpr int SMALL = 6;
    const unsigned lane = tid & 31;
    const int rw = x1 - x0, rcnt = visible ? rw * (y1 - y0) : 0;
    if (rcnt > 0 && rcnt <= SMALL) {
        for (int ty = y0; ty < y1; ty++)
            for (int tx = x0; tx < x1; tx++) atomicAdd(a.tile_count + ty * a.v.gx + tx, 1u);
    }
    unsigned todo = __ballot_sync(0xffffffffu, rcnt > SMALL);
    while (todo) {
        const int src = __ffs(todo) - 1;
        todo &= todo - 1;
        const int rx0 = __shfl_sync(0xffffffffu, x0, src), ry0 = __shfl_sync(0xffffffffu, y0, src);
        const int w = __shfl_sync(0xffffffffu, rw, src), cnt = __shfl_sync(0xffffffffu, rcnt, src);
        for (int k = lane; k < cnt; k += 32) {
            const int ty = k / w, tx = k - ty * w;
            atomicAdd(a.tile_count + (ry0 + ty) * a.v.gx + rx0 + tx, 1u);
        }
    }
}

// ------------------------------------------------------------------------------------------------
// exclusive scan over tile counts -> tile_start[0..T], cursor copy, R
// ------------------------------------------------------------------------------------------------
// Also orders the tiles by decreasing instance count (counting sort on count / 8, 1024 classes): the
// blend kernels take their tile from this list, so the hardware's in-order block dispatch starts the
// heaviest tiles first and the tail of the grid consists of the lightest ones (longest-processing-time
// -first; the order within a class is arbitrary and has no effect on any result).  The weights are the full
// counts, dead instances included: the live counts are only known after scatter, and the order is a schedule
// that no result depends on.
__global__ void __launch_bounds__(1024) tile_scan_kernel(const uint32_t *__restrict__ count, uint32_t *__restrict__ start,
                                                         uint32_t *__restrict__ cursor, uint32_t *__restrict__ order,
                                                         uint32_t *__restrict__ counters, int T, uint32_t *host_mirror)
{
    __shared__ uint32_t s_warp[32];
    __shared__ uint32_t s_carry;
    __shared__ uint32_t s_class[1024];
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    if (tid == 0) s_carry = 0;
    __syncthreads();
    for (int base = 0; base < T; base += 1024 * 4) {
        const int i0 = base + tid * 4;
        uint32_t v[4], sum = 0;
#pragma unroll
        for (int k = 0; k < 4; k++) {
            v[k] = (i0 + k < T) ? count[i0 + k] : 0u;
            sum += v[k];
        }
        uint32_t inc = sum;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o);
            if (lane >= o) inc += t;
        }
        if (lane == 31) s_warp[wid] = inc;
        __syncthreads();
        if (wid == 0) {
            uint32_t w = s_warp[lane], winc = w;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t t = __shfl_up_sync(0xffffffffu, winc, o);
                if (lane >= o) winc += t;
            }
            s_warp[lane] = winc - w;  // exclusive
        }
        __syncthreads();
        uint32_t excl = s_carry + s_warp[wid] + inc - sum;
#pragma unroll
        for (int k = 0; k < 4; k++) {
            if (i0 + k < T) {
                start[i0 + k] = excl;
                cursor[i0 + k] = excl;
            }
            excl += v[k];
        }
        __syncthreads();
        if (tid == 1023) s_carry = excl;
        __syncthreads();
    }
    if (tid == 0) {
        start[T] = s_carry;
        counters[0] = s_carry;
        if (host_mirror) *host_mirror = s_carry;
    }
    // ---- tile order: class 0 = heaviest ----
    s_class[tid] = 0;
    __syncthreads();
    for (int i = tid; i < T; i += 1024) atomicAdd(&s_class[1023u - min(count[i] >> 3, 1023u)], 1u);
    __syncthreads();
    {
        const uint32_t c = s_class[tid];
        uint32_t inc = c;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o);
            if (lane >= o) inc += t;
        }
        if (lane == 31) s_warp[wid] = inc;
        __syncthreads();
        if (wid == 0) {
            uint32_t w = s_warp[lane], winc = w;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t t = __shfl_up_sync(0xffffffffu, winc, o);
                if (lane >= o) winc += t;
            }
            s_warp[lane] = winc - w;
        }
        __syncthreads();
        s_class[tid] = s_warp[wid] + inc - c;  // exclusive start of this class
    }
    __syncthreads();
    for (int i = tid; i < T; i += 1024) order[atomicAdd(&s_class[1023u - min(count[i] >> 3, 1023u)], 1u)] = (uint32_t)i;
}

// ------------------------------------------------------------------------------------------------
// scatter: one (depth | id [| footprint mask]) word per LIVE (Gaussian, tile) instance into its tile's
// segment.  The kernel is bound by the round trip of its returning atomics (one slot claim per instance), so
// the arithmetic it does while they are in flight is free: this is where the exact footprint mask of every
// instance (sgr_internal.cuh, block_mask) is computed -- once, for both blend kernels.
// An instance whose mask is 0 cannot reach any pixel of its tile (the masks are conservative), so it claims
// no slot: the live words of tile t fill [tile_start[t], cursor[t]) and the rest of the segment, which
// preprocess sized by the full count, stays unused.  The sorts and both blend kernels walk the live range only.
// The plain-id format (packed = 0) carries no mask in the word but computes it all the same, to drop the dead.
// KEEP_DEAD: every instance claims its slot (cursor[t] ends at tile_start[t + 1]): the reference's full list,
// rebuilt by sgr_inspect_state.
// ------------------------------------------------------------------------------------------------
template <bool KEEP_DEAD>
__global__ void __launch_bounds__(256) scatter_kernel(int P, int gx, const ushort4 *__restrict__ rect,
                                                      const float *__restrict__ depth, const float4 *__restrict__ rec,
                                                      uint32_t *__restrict__ cursor,
                                                      const uint32_t *__restrict__ counters, uint64_t capacity,
                                                      int packed, uint64_t *__restrict__ inst)
{
    if ((uint64_t)counters[0] > capacity) return;  // overflow: host re-runs with a bigger buffer
    const int idx = blockIdx.x * 256 + threadIdx.x;
    const unsigned lane = threadIdx.x & 31;
    ushort4 rc = make_ushort4(0, 0, 0, 0);
    uint32_t dbits = 0;
    EllipseBands eb;
    eb.all = true;
    eb.dead = false;
    if (idx < P) {
        rc = rect[idx];
        if (rc.z > rc.x && rc.w > rc.y) {
            dbits = __float_as_uint(depth[idx]);
            const float4 r0 = __ldg(rec + (size_t)idx * 3), r1 = __ldg(rec + (size_t)idx * 3 + 1);
            eb = ellipse_bands(r0.x, r0.y, r0.z, r0.w, r1.x, r1.y);
        }
    }
    // Rects of up to SMALL tiles are walked by their own thread: masks first (pure arithmetic), then all
    // the slot claims back to back (the returning atomics are in flight together), then the stores.
    // Larger rects are walked cooperatively by the whole warp, one tile per lane.
    constexpr int SMALL = 6;
    static_assert(SMALL <= 8, "masks of a small rect are packed into one 64-bit register");
    const int rw = (int)rc.z - (int)rc.x, rcnt = (rc.z > rc.x && rc.w > rc.y) ? rw * ((int)rc.w - (int)rc.y) : 0;
    const uint32_t low_id = packed ? ((uint32_t)idx << 8) : (uint32_t)idx;
    const uint32_t word_mask = packed ? 0xffu : 0u;  // the mask rides in the word only in the packed format
    if (rcnt > 0 && rcnt <= SMALL) {
        uint64_t masks = 0;
        if (!eb.dead) {
            // the columns a band reaches do not depend on the tile column: once per tile row, then every
            // tile of the row only compares its two 8-column halves with them
            int k = 0;
            for (int ty = rc.y; ty < rc.w; ty++) {
                int lo[4], hi[4];
#pragma unroll
                for (int band = 0; band < 4; band++) {
                    lo[band] = 1;
                    hi[band] = 0;  // empty
                    if (eb.all) {
                        lo[band] = -(1 << 30);
                        hi[band] = 1 << 30;
                    } else {
                        const int ra = max(ty * SGR_TILE + 4 * band, eb.r_lo), rb = min(ty * SGR_TILE + 4 * band + 3, eb.r_hi);
                        if (ra <= rb) band_columns(eb, ra, rb, lo[band], hi[band]);
                    }
                }
                for (int tx = rc.x; tx < rc.z; tx++, k++) {
                    const int x0 = tx * SGR_TILE;
                    uint32_t m = 0;
#pragma unroll
                    for (int band = 0; band < 4; band++) {
                        const bool any = hi[band] >= lo[band];
                        const uint32_t left = (any && lo[band] <= x0 + 7 && hi[band] >= x0) ? 1u : 0u;
                        const uint32_t right = (any && lo[band] <= x0 + 15 && hi[band] >= x0 + 8) ? 2u : 0u;
                        m |= (left | right) << (2 * band);
                    }
                    masks |= (uint64_t)m << (8 * k);
                }
            }
        }
        uint32_t slot[SMALL];
        int tx = 0, trow = (int)rc.y * gx + (int)rc.x;
#pragma unroll
        for (int k = 0; k < SMALL; k++) {
            if (k < rcnt) {
                if (KEEP_DEAD || ((masks >> (8 * k)) & 0xffu)) slot[k] = atomicAdd(cursor + trow + tx, 1u);
                if (++tx == rw) {
                    tx = 0;
                    trow += gx;
                }
            }
        }
#pragma unroll
        for (int k = 0; k < SMALL; k++) {
            const uint32_t m = (uint32_t)(masks >> (8 * k)) & 0xffu;
            if (k < rcnt && (KEEP_DEAD || m)) inst[slot[k]] = ((uint64_t)dbits << 32) | low_id | (m & word_mask);
        }
    }
    unsigned todo = __ballot_sync(0xffffffffu, rcnt > SMALL);
    while (todo) {
        const int src = __ffs(todo) - 1;
        todo &= todo - 1;
        const int rx0 = __shfl_sync(0xffffffffu, (int)rc.x, src), ry0 = __shfl_sync(0xffffffffu, (int)rc.y, src);
        const int w = __shfl_sync(0xffffffffu, rw, src), cnt = __shfl_sync(0xffffffffu, rcnt, src);
        const uint32_t db = __shfl_sync(0xffffffffu, dbits, src);
        const uint32_t lid = __shfl_sync(0xffffffffu, low_id, src);
        EllipseBands es;
        es.gx = __shfl_sync(0xffffffffu, eb.gx, src);
        es.gy = __shfl_sync(0xffffffffu, eb.gy, src);
        es.k_a = __shfl_sync(0xffffffffu, eb.k_a, src);
        es.det_a2 = __shfl_sync(0xffffffffu, eb.det_a2, src);
        es.b_a = __shfl_sync(0xffffffffu, eb.b_a, src);
        es.v_r = __shfl_sync(0xffffffffu, eb.v_r, src);
        es.r_lo = __shfl_sync(0xffffffffu, eb.r_lo, src);
        es.r_hi = __shfl_sync(0xffffffffu, eb.r_hi, src);
        es.all = __shfl_sync(0xffffffffu, (int)eb.all, src) != 0;
        es.dead = __shfl_sync(0xffffffffu, (int)eb.dead, src) != 0;
        for (int k = lane; k < cnt; k += 32) {
            const int ty = k / w, tx = k - ty * w;
            const uint32_t m = block_mask(es, (rx0 + tx) * SGR_TILE, (ry0 + ty) * SGR_TILE);
            if (!KEEP_DEAD && m == 0u) continue;
            const uint32_t slot = atomicAdd(cursor + (ry0 + ty) * gx + rx0 + tx, 1u);
            inst[slot] = ((uint64_t)db << 32) | lid | (m & word_mask);
        }
    }
}

// ------------------------------------------------------------------------------------------------
// per-tile sort of the tiles with more than SORT_CAP instances: LSD radix on the (depth|id) words,
// 8-bit digits, warp-private histograms, match_any ranking (stable), constant bytes skipped; the
// words ping-pong between inst_a and inst_b in L2/HBM.
// ------------------------------------------------------------------------------------------------
constexpr int SORT_CAP = 8192;  // largest shared-memory (merge sort) class; above it: global radix
constexpr int GSORT_T = 1024;

__global__ void __launch_bounds__(GSORT_T) tile_sort_global_kernel(const uint32_t *__restrict__ tile_start,
                                                                   const uint32_t *__restrict__ tile_end,
                                                                   const uint32_t *__restrict__ counters,
                                                                   uint64_t capacity, uint64_t *__restrict__ inst_a,
                                                                   uint64_t *__restrict__ inst_b,
                                                                   uint32_t *__restrict__ plist, int num_tiles)
{
    constexpr int NW = GSORT_T / 32;
    __shared__ uint32_t s_hist[NW][256];
    __shared__ uint32_t s_diff[2];
    __shared__ uint32_t s_wsum[32];

    if ((uint64_t)counters[0] > capacity) return;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const uint32_t lo = tile_start[tile];
    const int n = (int)(tile_end[tile] - lo);
    if (n <= SORT_CAP) continue;

    uint64_t *src = inst_a + lo, *dst = inst_b + lo;

    // find which key bytes vary inside this tile
    if (tid < 2) s_diff[tid] = 0;
    __syncthreads();
    {
        const uint64_t k0 = inst_a[lo];
        uint32_t dlo = 0, dhi = 0;
        for (int i = tid; i < n; i += GSORT_T) {
            const uint64_t x = inst_a[lo + i] ^ k0;
            dlo |= (uint32_t)x;
            dhi |= (uint32_t)(x >> 32);
        }
        dlo = __reduce_or_sync(0xffffffffu, dlo);
        dhi = __reduce_or_sync(0xffffffffu, dhi);
        if (lane == 0) {
            if (dlo) atomicOr(&s_diff[0], dlo);
            if (dhi) atomicOr(&s_diff[1], dhi);
        }
    }
    __syncthreads();
    const uint64_t diff = ((uint64_t)s_diff[1] << 32) | s_diff[0];

    // contiguous chunk per warp (multiple of 32 so that lanes map to consecutive elements)
    const int chunk = ((n + NW - 1) / NW + 31) & ~31;
    const int w_lo = min(n, wid * chunk), w_hi = min(n, w_lo + chunk);

    for (int shift = 0; shift < 64; shift += 8) {
        if (((diff >> shift) & 0xffull) == 0) continue;
        for (int i = tid; i < NW * 256; i += GSORT_T) (&s_hist[0][0])[i] = 0;
        __syncthreads();
        // pass 1: warp-private digit histogram
        for (int i = w_lo + lane; i - lane < w_hi; i += 32) {
            const bool ok = i < w_hi;
            const unsigned act = __ballot_sync(0xffffffffu, ok);
            if (ok) {
                const uint32_t d = (uint32_t)(src[i] >> shift) & 0xffu;
                const unsigned peers = __match_any_sync(act, d);
                if ((int)(__ffs(peers) - 1) == lane) s_hist[wid][d] += __popc(peers);
            }
            __syncwarp();
        }
        __syncthreads();
        // digit-major exclusive scan over (digit, warp)
        {
            uint32_t tot = 0;
            if (tid < 256) {
#pragma unroll 4
                for (int w = 0; w < NW; w++) tot += s_hist[w][tid];
            }
            uint32_t inc = tot;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o);
                if (lane >= o) inc += t;
            }
            if (tid < 256 && lane == 31) s_wsum[wid] = inc;
            __syncthreads();
            if (tid < 256) {
                uint32_t basev = inc - tot;
                for (int w = 0; w < wid; w++) basev += s_wsum[w];
                for (int w = 0; w < NW; w++) {
                    const uint32_t c = s_hist[w][tid];
                    s_hist[w][tid] = basev;
                    basev += c;
                }
            }
            __syncthreads();
        }
        // pass 2: stable scatter
        for (int i = w_lo + lane; i - lane < w_hi; i += 32) {
            const bool ok = i < w_hi;
            const unsigned act = __ballot_sync(0xffffffffu, ok);
            if (ok) {
                const uint64_t k = src[i];
                const uint32_t d = (uint32_t)(k >> shift) & 0xffu;
                const unsigned peers = __match_any_sync(act, d);
                const uint32_t pos = s_hist[wid][d] + __popc(peers & ((1u << lane) - 1u));
                dst[pos] = k;
                __syncwarp(act);
                if ((int)(__ffs(peers) - 1) == lane) s_hist[wid][d] += __popc(peers);
            }
            __syncwarp();
        }
        __syncthreads();
        uint64_t *t = src;
        src = dst;
        dst = t;
    }
    for (int i = tid; i < n; i += GSORT_T) plist[lo + i] = (uint32_t)src[i];
    __syncthreads();
    }
}

// ------------------------------------------------------------------------------------------------
// per-tile sort, shared-memory path: merge sort on the 64-bit (depth|id) words of one tile.
// Every thread sorts VT=8 words in registers with a 19-comparator network, then log2(n/8) rounds
// of pairwise run merging in shared memory; in each round a thread finds its output window with a
// merge-path binary search and merges 8 outputs serially.  The words are distinct (the id is part
// of the key) so the result is the unique total order = the reference's stable sort by depth.
// Size classes (LOWER, CAP]: each class is its own launch over all tiles with early exit, so the
// shared-memory footprint (and occupancy) matches the tile population.  Every sort kernel sorts the
// words of [tile_start[t], tile_end[t]) -- the live instances scatter wrote -- and picks its class by that count.
// ------------------------------------------------------------------------------------------------
constexpr int SORT_VT = 8;  // words per thread in the per-tile merge sort

__device__ __forceinline__ void cswap(uint64_t &a, uint64_t &b)
{
    const uint64_t lo = a < b ? a : b, hi = a < b ? b : a;
    a = lo;
    b = hi;
}

// In-place merge sort of s_keys[0..n) by the NT threads of the CTA (all must call).  s_keys must
// have room for ceil(n/VT)*VT words; n <= NT*VT.
template <int NT>
__device__ __forceinline__ void block_merge_sort(uint64_t *s_keys, const int n)
{
    constexpr int VT = SORT_VT;
    const int tid = threadIdx.x;
    const int nact = (n + VT - 1) / VT;  // threads that own a window
    const int L = nact * VT;             // padded length (pad words = all ones sort last)
    uint64_t r[VT];
    if (tid < nact) {
#pragma unroll
        for (int k = 0; k < VT; k++) {
            const int i = tid * VT + k;
            r[k] = i < n ? s_keys[i] : ~0ull;
        }
        // Batcher odd-even merge sort network on the VT registers (19 comparators)
        static_assert(VT == 8, "sorting network written out for 8 words per thread");
        cswap(r[0], r[1]); cswap(r[2], r[3]); cswap(r[4], r[5]); cswap(r[6], r[7]); cswap(r[0], r[2]);
        cswap(r[1], r[3]); cswap(r[4], r[6]); cswap(r[5], r[7]); cswap(r[1], r[2]); cswap(r[5], r[6]);
        cswap(r[0], r[4]); cswap(r[1], r[5]); cswap(r[2], r[6]); cswap(r[3], r[7]); cswap(r[2], r[4]);
        cswap(r[3], r[5]); cswap(r[1], r[2]); cswap(r[3], r[4]); cswap(r[5], r[6]);
    }
    __syncthreads();  // every thread has read its window before anyone overwrites it
    if (tid < nact) {
#pragma unroll
        for (int k = 0; k < VT; k++) s_keys[tid * VT + k] = r[k];
    }
    for (int run = VT; run < L; run <<= 1) {
        __syncthreads();
        if (tid < nact) {
            const int out0 = tid * VT;
            const int a0 = out0 & ~(2 * run - 1);
            const int la = min(run, L - a0);
            const int b0 = a0 + run;
            const int lb = max(0, min(run, L - b0));
            const int diag = out0 - a0;
            int slo = max(0, diag - lb), shi = min(diag, la);
            while (slo < shi) {
                const int mid = (slo + shi) >> 1;
                if (s_keys[a0 + mid] <= s_keys[b0 + diag - 1 - mid]) slo = mid + 1;
                else shi = mid;
            }
            int i = slo, j = diag - slo;
            uint64_t ka = i < la ? s_keys[a0 + i] : ~0ull;
            uint64_t kb = j < lb ? s_keys[b0 + j] : ~0ull;
#pragma unroll
            for (int k = 0; k < VT; k++) {
                const bool takeA = (j >= lb) || (i < la && ka <= kb);
                r[k] = takeA ? ka : kb;
                if (takeA) {
                    i++;
                    ka = i < la ? s_keys[a0 + i] : ~0ull;
                } else {
                    j++;
                    kb = j < lb ? s_keys[b0 + j] : ~0ull;
                }
            }
        }
        __syncthreads();
        if (tid < nact) {
#pragma unroll
            for (int k = 0; k < VT; k++) s_keys[tid * VT + k] = r[k];
        }
    }
    __syncthreads();
}

template <int CAP, int LOWER>
__global__ void __launch_bounds__(CAP / SORT_VT) tile_sort_merge_kernel(const uint32_t *__restrict__ tile_start,
                                                                        const uint32_t *__restrict__ tile_end,
                                                                        const uint32_t *__restrict__ counters,
                                                                        uint64_t capacity,
                                                                        const uint64_t *__restrict__ inst,
                                                                        uint32_t *__restrict__ plist, int num_tiles)
{
    extern __shared__ __align__(16) uint64_t s_keys[];  // CAP words
    if ((uint64_t)counters[0] > capacity) return;
    const int tid = threadIdx.x;
    // grid-stride over tiles: rare size classes are launched with a small grid and skip cheaply
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const uint32_t lo = tile_start[tile];
        const int n = (int)(tile_end[tile] - lo);
        if (n <= LOWER || n > CAP) continue;
        for (int i = tid; i < n; i += CAP / SORT_VT) s_keys[i] = inst[lo + i];
        __syncthreads();
        block_merge_sort<CAP / SORT_VT>(s_keys, n);
        for (int i = tid; i < n; i += CAP / SORT_VT) plist[lo + i] = (uint32_t)s_keys[i];
        __syncthreads();  // s_keys is reused by the next tile of this CTA
    }
}

// ------------------------------------------------------------------------------------------------
// per-tile sort, fast path for the common size class (512 < n <= 2048): one MSD bucket pass on the
// depth bits + insertion sort inside the (tiny) buckets.
//   bucket(word) = (depth_bits - min_bits) >> sh   with sh chosen so that the tile's depth range
// maps onto at most NB = 1024 buckets: monotone in the key, so concatenating the sorted buckets
// is the sorted tile.  Counting (shared int atomics), one exclusive scan, an atomic-cursor
// scatter, then every thread insertion-sorts NB/256 buckets on the full 64-bit words (total
// order incl. the Gaussian id, so the result is identical to the merge sort's).  Depth
// distributions that put more than BUCKET_MAX words in one bucket (e.g. many equal depths) take
// the merge sort instead -- same kernel, same buffers.
// ------------------------------------------------------------------------------------------------
constexpr int BK_CAP = 2048, BK_T = 256, BK_NB = 1024, BK_LOG2NB = 10, BUCKET_MAX = 24;

__global__ void __launch_bounds__(BK_T) tile_sort_bucket_kernel(const uint32_t *__restrict__ tile_start,
                                                                 const uint32_t *__restrict__ tile_end,
                                                                 const uint32_t *__restrict__ counters, uint64_t capacity,
                                                                 const uint64_t *__restrict__ inst,
                                                                 uint32_t *__restrict__ plist, int num_tiles, int lower)
{
    __shared__ __align__(16) uint64_t s_a[BK_CAP];
    __shared__ __align__(16) uint64_t s_b[BK_CAP];
    __shared__ uint32_t s_cnt[BK_NB];
    __shared__ uint32_t s_off[BK_NB];
    __shared__ uint32_t s_red[4];  // min bits, max bits, max bucket count, scan carry helper
    __shared__ uint32_t s_wsum[BK_T / 32];
    if ((uint64_t)counters[0] > capacity) return;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const uint32_t lo = tile_start[tile];
        const int n = (int)(tile_end[tile] - lo);
        if (n <= lower || n > BK_CAP) continue;
        if (tid == 0) {
            s_red[0] = 0xffffffffu;
            s_red[1] = 0u;
            s_red[2] = 0u;
        }
        for (int i = tid; i < BK_NB; i += BK_T) s_cnt[i] = 0;
        __syncthreads();
        uint32_t mn = 0xffffffffu, mx = 0u;
        for (int i = tid; i < n; i += BK_T) {
            const uint64_t k = inst[lo + i];
            s_a[i] = k;
            const uint32_t d = (uint32_t)(k >> 32);
            mn = min(mn, d);
            mx = max(mx, d);
        }
        mn = __reduce_min_sync(0xffffffffu, mn);
        mx = __reduce_max_sync(0xffffffffu, mx);
        if (lane == 0) {
            atomicMin(&s_red[0], mn);
            atomicMax(&s_red[1], mx);
        }
        __syncthreads();
        const uint32_t dmin = s_red[0], range = s_red[1] - dmin;
        const int sh = max(0, 32 - __clz(range) - BK_LOG2NB);  // (range >> sh) < NB
        for (int i = tid; i < n; i += BK_T) atomicAdd(&s_cnt[((uint32_t)(s_a[i] >> 32) - dmin) >> sh], 1u);
        __syncthreads();
        // exclusive scan of the NB counts (4 consecutive buckets per thread) + max count
        {
            uint32_t c[4], sum = 0, cm = 0;
#pragma unroll
            for (int k = 0; k < 4; k++) {
                c[k] = s_cnt[tid * 4 + k];
                sum += c[k];
                cm = max(cm, c[k]);
            }
            cm = __reduce_max_sync(0xffffffffu, cm);
            uint32_t inc = sum;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o);
                if (lane >= o) inc += t;
            }
            if (lane == 31) s_wsum[wid] = inc;
            if (lane == 0) atomicMax(&s_red[2], cm);
            __syncthreads();
            uint32_t basev = inc - sum;
            for (int w = 0; w < wid; w++) basev += s_wsum[w];
#pragma unroll
            for (int k = 0; k < 4; k++) {
                s_off[tid * 4 + k] = basev;
                s_cnt[tid * 4 + k] = 0;  // reused as the scatter cursor
                basev += c[k];
            }
        }
        __syncthreads();
        if (s_red[2] > (uint32_t)BUCKET_MAX) {
            block_merge_sort<BK_T>(s_a, n);  // skewed depths: generic path (ends with a barrier)
            for (int i = tid; i < n; i += BK_T) plist[lo + i] = (uint32_t)s_a[i];
        } else {
            for (int i = tid; i < n; i += BK_T) {
                const uint64_t k = s_a[i];
                const uint32_t b = ((uint32_t)(k >> 32) - dmin) >> sh;
                s_b[s_off[b] + atomicAdd(&s_cnt[b], 1u)] = k;
            }
            __syncthreads();
            for (int b = tid; b < BK_NB; b += BK_T) {
                const int c = (int)s_cnt[b];
                uint64_t *q = s_b + s_off[b];
                for (int i = 1; i < c; i++) {
                    const uint64_t key = q[i];
                    int j = i - 1;
                    while (j >= 0 && q[j] > key) {
                        q[j + 1] = q[j];
                        j--;
                    }
                    q[j + 1] = key;
                }
            }
            __syncthreads();
            for (int i = tid; i < n; i += BK_T) plist[lo + i] = (uint32_t)s_b[i];
        }
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------------------
// forward blend: one CTA per 16x16 tile, one thread per pixel, one warp per 8x4 pixel block
// (block w = band * 2 + half, sgr_internal.cuh).  The records of a batch of the tile's live list
// [tile_start, tile_end) are gathered once into shared memory -- the dead instances (empty footprint mask, a
// third of them) never entered the list -- and each warp walks only the splats whose mask has its block's
// bit (clz over a bit-reversed per-block membership word).  power / alpha / T / C follow the reference's rounding
// exactly (forward.cu:261-374), so final_T and the image are bit-identical to the reference; the masks and the
// `power < tau` test only skip pairs the exact alpha test would reject.  n_contrib is the last contributor's
// position + 1 in the LIVE list (the backward bounds its walk by it; sgr_inspect_state maps it back to the
// reference's count over the full list).  Tiles are taken heaviest first (tile_order).
// ------------------------------------------------------------------------------------------------
constexpr int BLEND_T = 256;

// -DSGR_BLEND_STATS: count what the blend loops do (scripts/blend_stats.py); never in the shipped build
#ifdef SGR_BLEND_STATS
__device__ unsigned long long g_fwd_stats[8];
#define FWD_STAT(k, v) atomicAdd(&g_fwd_stats[k], (unsigned long long)(v))
#endif

// (1 << n) - 1 for n = 0..31 in one instruction (BMSK); nvcc makes a shift of a materialised -1 and a LOP3 of it
__device__ __forceinline__ uint32_t low_mask(uint32_t n)
{
    uint32_t r;
    asm("bmsk.clamp.b32 %0, 0, %1;" : "=r"(r) : "r"(n));
    return r;
}

// No minimum CTA count in the launch bounds: with a minimum of 1 nvcc gives the packed format 38 registers (6 CTAs per
// SM) instead of 32 (8 CTAs), and the unpacked one 53 instead of 48.  The extra CTAs outweigh the one instruction per
// visit the 32-register code spends (DESIGN.md §3).
// FEAT: also blend one per-Gaussian scalar (values[P]) over its own background (*feat_bg) into out_feature[H,W],
// with the colour channels' exact operations; the FEAT = false instantiations ignore the last three arguments.
template <bool packed, bool FEAT>
__global__ void __launch_bounds__(BLEND_T) blend_forward_kernel(const uint32_t *__restrict__ tile_order,
                                                                const uint32_t *__restrict__ tile_start,
                                                                const uint32_t *__restrict__ tile_end,
                                                                const uint32_t *__restrict__ plist,
                                                                const float4 *__restrict__ rec,
                                                                const uint32_t *__restrict__ counters, uint64_t capacity,
                                                                int W, int H, int gx, const float *__restrict__ bg,
                                                                float *__restrict__ final_T,
                                                                uint32_t *__restrict__ n_contrib,
                                                                float *__restrict__ out_color,
                                                                const float *__restrict__ values,
                                                                const float *__restrict__ feat_bg,
                                                                float *__restrict__ out_feature)
{
    // A batch slot is 48 contiguous bytes: (x, y, conic a, conic b), (conic c, tau, opacity, r), (g, b, value, -):
    // one IMAD gives the slot's address and the loads take immediate offsets.  Every lane of a warp reads the same
    // slot, so the loads are broadcasts and the 48-byte stride costs no bank conflicts.  `value` is only staged (and
    // read) by FEAT.
    __shared__ __align__(16) float4 s_rec[BLEND_T * 3];
    // s_member[w][k]: slots 32k..32k+31 whose footprint mask has block w, bit-reversed (slot 32k + i is bit 31 - i)
    // so that the walk finds the next member with one clz
    __shared__ uint32_t s_member[8][BLEND_T / 32];
    if ((uint64_t)counters[0] > capacity) return;
    const int tile = (int)tile_order[blockIdx.x];
    const int tile_y = tile / gx, tile_x = tile - tile_y * gx;
    const int tid = threadIdx.x;
    const unsigned lane = tid & 31, wid = tid >> 5;
    const int tx0 = tile_x * SGR_TILE, ty0 = tile_y * SGR_TILE;
    const uint32_t pxi = tx0 + (wid & 1u) * 8 + (lane & 7u), pyi = ty0 + (wid >> 1) * 4 + (lane >> 3);
    const bool inside = pxi < (uint32_t)W && pyi < (uint32_t)H;
    const float pxf = (float)pxi, pyf = (float)pyi;
    const uint32_t lo = tile_start[tile], hi = tile_end[tile];  // the tile's live list (scatter)
    uint32_t done = inside ? 0u : 1u;  // 32-bit flag: a bool makes nvcc shuffle bytes (PRMT) in the hot loop
    float T = 1.0f, C0 = 0.f, C1 = 0.f, C2 = 0.f, C3 = 0.f;
    uint32_t last = 0;
    const uint32_t srec = smem_addr_pinned(s_rec);
    const uint32_t smem_put = smem_addr_pinned(&s_member[0][wid]), smem_get = smem_addr_pinned(&s_member[wid][0]);
    for (uint32_t b0 = lo; b0 < hi; b0 += BLEND_T) {
        if (__syncthreads_count(done != 0u) == BLEND_T) break;
        uint32_t mask = 0;
        if (b0 + tid < hi) {
            const uint32_t w = plist[b0 + tid];
            uint32_t id = w;
            if (packed) {
                id = w >> 8;
                mask = w & 0xffu;
            }
            if (!packed || mask) {
                const float4 *r = rec + (size_t)id * 3;
                const float4 r0 = __ldg(r), r1 = __ldg(r + 1), r2 = __ldg(r + 2);
                const float fv = FEAT ? __ldg(values + id) : 0.f;
                if (!packed) mask = block_mask_of_record(r0.x, r0.y, r0.z, r0.w, r1.x, r1.y, tx0, ty0);
                const uint32_t p = srec + (uint32_t)tid * 48u;
                sts128(p, r0.x, r0.y, r0.z, r0.w);
                sts128(p + 16, r1.x, r1.y, r1.z, r1.w);
                sts64(p + 32, r2.x, r2.y);
                if (FEAT) sts32(p + 40, __float_as_uint(fv));
            }
        }
#pragma unroll
        for (int blk = 0; blk < 8; blk++) {
            const uint32_t word = __ballot_sync(0xffffffffu, mask & (1u << blk));
            if (lane == 0) sts32(smem_put + blk * (BLEND_T / 32) * 4, __brev(word));
        }
        __syncthreads();
        const uint32_t base_pos = b0 - lo;
#ifdef SGR_BLEND_STATS
        if (tid == 0) FWD_STAT(6, min((uint32_t)BLEND_T, hi - b0));  // records staged
#endif
        if (!__all_sync(0xffffffffu, done != 0u)) {
#pragma unroll 1
            for (int k = 0; k < BLEND_T / 32; k++) {
                // every lane reads the same word: the OR over the warp is that word, but in a uniform register, so
                // ptxas knows the walk's branches are warp-uniform (no WARPSYNC in front of the votes) and runs the
                // walk's integer work on the uniform datapath
                uint32_t mw = __reduce_or_sync(0xffffffffu, lds32(smem_get + k * 4));
                const uint32_t wrec = srec + (uint32_t)k * (32u * 48u) + 31u * 48u;  // slot 32k + 31
                const uint32_t wlast = base_pos + (uint32_t)(k << 5) + 32u;       // n_contrib of slot 32k + 31
#pragma unroll 1
                while (mw) {
                    const uint32_t msb = 31 - __clz(mw);  // slot 32k + 31 - msb: the word's first member
                    mw &= low_mask(msb);
                    const uint32_t p = wrec - msb * 48u;
#ifdef SGR_BLEND_STATS
                    {
                        const float4 A = lds128(p);
                        const float4 B = lds128(p + 16);
                        const float power = splat_power(__fsub_rn(A.x, pxf), __fsub_rn(A.y, pyf), A.z, A.w, B.x);
                        const bool cand = !done && !(power > 0.0f || power < B.y);
                        const bool hit = cand && !(fminf(0.99f, __fmul_rn(B.z, expf(power))) < 1.0f / 255.0f);
                        const unsigned mc = __ballot_sync(0xffffffffu, cand), mh = __ballot_sync(0xffffffffu, hit);
                        const unsigned ml = __ballot_sync(0xffffffffu, !done);
                        if (lane == 0) {
                            FWD_STAT(0, 1);            // block-splat visits
                            FWD_STAT(1, mc != 0);      // ... with a lane that passes the power test
                            FWD_STAT(2, mh != 0);      // ... with a lane that contributes
                            FWD_STAT(3, __popc(mc));   // lanes passing the power test
                            FWD_STAT(4, __popc(mh));   // contributing (pixel, splat) pairs
                            FWD_STAT(5, __popc(ml));   // live lanes over all visits
                        }
                    }
#endif
                    const float4 A = lds128(p);
                    const float4 B = lds128(p + 16);
                    const float dx = __fsub_rn(A.x, pxf), dy = __fsub_rn(A.y, pyf);
                    const float power = splat_power(dx, dy, A.z, A.w, B.x);
                    const bool cand = (done == 0u) & !(power > 0.0f || power < B.y);
                    if (!__any_sync(0xffffffffu, cand)) continue;
                    // Every lane of a warp with a candidate evaluates the tail; selects (not products with 0) keep
                    // what a lane that does not contribute had, signed zeros and NaNs included.
                    float4 Cc;  // (g, b, value, -): one LDS.128 with FEAT, an LDS.64 of (g, b) without
                    if (FEAT) {
                        Cc = lds128(p + 32);
                    } else {
                        const float2 gb = lds64(p + 32);
                        Cc.x = gb.x;
                        Cc.y = gb.y;
                    }
                    const float alpha = fminf(0.99f, __fmul_rn(B.z, expf(power)));
                    const float test_T = __fmul_rn(T, __fsub_rn(1.0f, alpha));
                    const bool hit = cand && !(alpha < 1.0f / 255.0f);
                    const bool contrib = hit && !(test_T < 0.0001f);
                    done = (hit && test_T < 0.0001f) ? 1u : done;
                    const float n0 = __fmaf_rn(T, __fmul_rn(alpha, B.w), C0);
                    const float n1 = __fmaf_rn(T, __fmul_rn(alpha, Cc.x), C1);
                    const float n2 = __fmaf_rn(T, __fmul_rn(alpha, Cc.y), C2);
                    C0 = contrib ? n0 : C0;
                    C1 = contrib ? n1 : C1;
                    C2 = contrib ? n2 : C2;
                    if (FEAT) {
                        const float n3 = __fmaf_rn(T, __fmul_rn(alpha, Cc.z), C3);
                        C3 = contrib ? n3 : C3;
                    }
                    T = contrib ? test_T : T;
                    last = contrib ? wlast - msb : last;
                }
                if (__all_sync(0xffffffffu, done != 0u)) break;
            }
        }
    }
    if (inside) {
        const size_t pix = (size_t)pyi * W + pxi, plane = (size_t)H * W;
        final_T[pix] = T;
        n_contrib[pix] = last;
        out_color[pix] = __fmaf_rn(T, bg[0], C0);
        out_color[plane + pix] = __fmaf_rn(T, bg[1], C1);
        out_color[2 * plane + pix] = __fmaf_rn(T, bg[2], C2);
        if (FEAT) out_feature[pix] = __fmaf_rn(T, feat_bg[0], C3);
    }
}

#ifdef SGR_BLEND_STATS
int read_fwd_stats(unsigned long long *out, int reset)
{
    SGR_CUDA(cudaMemcpyFromSymbol(out, g_fwd_stats, sizeof(unsigned long long) * 8));
    if (reset) {
        unsigned long long z[8] = {};
        SGR_CUDA(cudaMemcpyToSymbol(g_fwd_stats, z, sizeof(z)));
    }
    return SGR_OK;
}
#endif

__global__ void mark_visible_kernel(int P, const float *__restrict__ means, const float *__restrict__ vm,
                                    uint8_t *__restrict__ present)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const float d = xf_row(vm, 2, means[3 * i], means[3 * i + 1], means[3 * i + 2]);
    present[i] = !(d <= 0.2f);
}

// ------------------------------------------------------------------------------------------------
// host orchestration
// ------------------------------------------------------------------------------------------------
// Host-side per-call state: one pinned word (the instance count's read-back) and one event.  Calls
// may overlap on one device (two streams / two threads), so every call takes its own slot from a small
// per-device pool and returns it when it is done.
struct CallSlot {
    uint32_t *pinned = nullptr;
    cudaEvent_t ev = nullptr;
};
struct DevicePool {
    std::mutex mu;
    std::vector<CallSlot> free_slots;
};
static DevicePool g_pools[SGR_MAX_DEVICES];

static int current_pool(DevicePool **out)
{
    int dev = 0;
    const int rc = current_device(&dev);
    if (rc) return rc;
    *out = &g_pools[dev];
    return SGR_OK;
}

static int acquire_slot(DevicePool *pool, CallSlot *slot)
{
    std::lock_guard<std::mutex> lock(pool->mu);
    if (!pool->free_slots.empty()) {
        *slot = pool->free_slots.back();
        pool->free_slots.pop_back();
        return SGR_OK;
    }
    SGR_CUDA(cudaHostAlloc((void **)&slot->pinned, 64, cudaHostAllocDefault));
    SGR_CUDA(cudaEventCreateWithFlags(&slot->ev, cudaEventDisableTiming));
    return SGR_OK;
}

struct SlotLease {  // returns the slot to its pool on every exit path
    DevicePool *pool = nullptr;
    CallSlot slot;
    ~SlotLease()
    {
        if (pool && slot.pinned) {
            std::lock_guard<std::mutex> lock(pool->mu);
            pool->free_slots.push_back(slot);
        }
    }
};

static int set_forward_attributes()
{
    SGR_CUDA(cudaFuncSetAttribute(preprocess_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    SGR_CUDA(cudaFuncSetAttribute(preprocess_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    SGR_CUDA(cudaFuncSetAttribute(tile_sort_merge_kernel<8192, 2048>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  8192 * 8));
    return SGR_OK;
}
static DeviceOnce g_forward_attributes;

static void launch_blend_forward(const ViewConsts &v, int P, const GeomState &geom, const ImageState &img,
                                 const BinState &bin, uint64_t capacity, float *out_color, const FeatureChannel *feat,
                                 cudaStream_t st)
{
    const bool packed = ids_packed(P);
    const auto kernel = feat ? (packed ? &blend_forward_kernel<true, true> : &blend_forward_kernel<false, true>)
                             : (packed ? &blend_forward_kernel<true, false> : &blend_forward_kernel<false, false>);
    kernel<<<v.gx * v.gy, BLEND_T, 0, st>>>(img.tile_order, img.tile_start, img.tile_cursor, bin.plist, geom.rec,
                                            img.counters, capacity, v.W, v.H, v.gx, v.bg, img.final_T, img.n_contrib,
                                            out_color, feat ? feat->values : nullptr, feat ? feat->bg : nullptr,
                                            feat ? feat->out : nullptr);
}

// scatter (into bin.inst_a, advancing `cursor` from tile_start) and the per-tile sorts of [tile_start, cursor)
// into bin.plist.  KEEP_DEAD: the full list of the reference instead of the live one.
template <bool KEEP_DEAD>
static int launch_scatter_and_sorts(int P, int gx, int T, const GeomState &geom, const uint32_t *tile_start,
                                    uint32_t *cursor, const uint32_t *counters, const BinState &bin, uint64_t capacity,
                                    cudaStream_t st)
{
    SGR_LAUNCH(K_SCATTER, st,
               scatter_kernel<KEEP_DEAD><<<(P + 255) / 256, 256, 0, st>>>(P, gx, geom.rect, geom.depth, geom.rec, cursor,
                                                                          counters, capacity, ids_packed(P) ? 1 : 0,
                                                                          bin.inst_a));
    sgr::prof_begin(K_SORT_SMEM, st);  // one timing bracket around the three size classes ...
    sgr::note_launches(2);             // ... but three launches
    const int slots = 2 * device_sm_count();
    const int small_grid = T < slots ? T : slots;  // 2 CTAs per SM, grid-stride over tiles
    tile_sort_merge_kernel<512, 0><<<T, 512 / SORT_VT, 512 * 8, st>>>(tile_start, cursor, counters, capacity, bin.inst_a,
                                                                      bin.plist, T);
    tile_sort_bucket_kernel<<<T, BK_T, 0, st>>>(tile_start, cursor, counters, capacity, bin.inst_a, bin.plist, T, 512);
    tile_sort_merge_kernel<8192, 2048><<<small_grid, 8192 / SORT_VT, 8192 * 8, st>>>(tile_start, cursor, counters,
                                                                                     capacity, bin.inst_a, bin.plist, T);
    sgr::prof_end(st);
    SGR_LAUNCH(K_SORT_GLOBAL, st,
               tile_sort_global_kernel<<<small_grid, GSORT_T, 0, st>>>(tile_start, cursor, counters, capacity,
                                                                       bin.inst_a, bin.inst_b, bin.plist, T));
    SGR_CUDA(cudaGetLastError());
    return SGR_OK;
}

static int launch_binning_and_blend(const ViewConsts &v, int P, const GeomState &geom, const ImageState &img,
                                    const BinState &bin, uint64_t capacity, float *out_color,
                                    const FeatureChannel *feat, cudaStream_t st)
{
    const int rc = launch_scatter_and_sorts<false>(P, v.gx, v.gx * v.gy, geom, img.tile_start, img.tile_cursor,
                                                   img.counters, bin, capacity, st);
    if (rc) return rc;
    // the blend reads the live ends scatter left in tile_cursor (same stream, after it)
    SGR_LAUNCH(K_BLEND_FWD, st, launch_blend_forward(v, P, geom, img, bin, capacity, out_color, feat, st));
    SGR_CUDA(cudaGetLastError());
    return SGR_OK;
}

// The reference's full per-tile list of a forward's state, dead instances included, into `full` (capacity
// num_rendered): tile_start[t + 1] ends each segment, `cursor` (T words) is scratch.  sgr_inspect_state.
int build_full_list(int P, int W, int H, const GeomState &geom, const ImageState &img, uint64_t num_rendered,
                    const BinState &full, uint32_t *cursor, cudaStream_t st)
{
    int rc = once_per_device(g_forward_attributes, set_forward_attributes);
    if (rc) return rc;
    const int gx = (W + SGR_TILE - 1) / SGR_TILE, T = gx * ((H + SGR_TILE - 1) / SGR_TILE);
    SGR_CUDA(cudaMemcpyAsync(cursor, img.tile_start, sizeof(uint32_t) * T, cudaMemcpyDeviceToDevice, st));
    return launch_scatter_and_sorts<true>(P, gx, T, geom, img.tile_start, cursor, img.counters, full, num_rendered, st);
}

int launch_forward(const SgrView *view, const SgrGaussians *g, SgrAlloc geom_alloc, void *geom_ctx,
                   SgrAlloc binning_alloc, void *binning_ctx, SgrAlloc image_alloc, void *image_ctx, float *out_color,
                   int32_t *radii, int64_t capacity_hint, int64_t *num_rendered, cudaStream_t st,
                   const FeatureChannel *feat)
{
    const int P = g->P, W = view->image_width, H = view->image_height;
    int rc = once_per_device(g_forward_attributes, set_forward_attributes);
    if (rc) return rc;
    SlotLease lease;
    rc = current_pool(&lease.pool);
    if (rc) return rc;
    rc = acquire_slot(lease.pool, &lease.slot);
    if (rc) return rc;
    CallSlot *slot = &lease.slot;

    const ViewConsts v = view_consts(view, g->M);
    const int T = v.gx * v.gy;

    void *geom_mem = geom_alloc(geom_ctx, sgr_geometry_bytes(P));
    void *img_mem = image_alloc(image_ctx, sgr_image_bytes(W, H));
    if (!geom_mem || !img_mem) {
        set_error("scratch allocator returned NULL");
        return SGR_ENOMEM;
    }
    Layout geom_l(geom_mem), img_l(img_mem);
    GeomState geom = GeomState::carve(geom_l, P);
    ImageState img = ImageState::carve(img_l, W, H);

    SGR_CUDA(cudaMemsetAsync(img.tile_count, 0, sizeof(uint32_t) * T, st));

    PreArgs a;
    a.P = P;
    a.means = g->means3D;
    a.scales = g->scales;
    a.rots = g->rotations;
    a.opac = g->opacities;
    a.shs = g->shs;
    a.sh_rest = g->sh_rest;
    const bool raw = g->activations != 0;
    a.colors = g->colors_precomp;
    a.cov_pre = g->cov3D_precomp;
    a.v = v;
    a.bulk_ok = aligned16(g->means3D) && aligned16(g->opacities) && (!g->scales || aligned16(g->scales)) &&
                (!g->rotations || aligned16(g->rotations)) && (!g->cov3D_precomp || aligned16(g->cov3D_precomp)) &&
                (!g->colors_precomp || aligned16(g->colors_precomp)) &&
                (!raw || !g->shs || (aligned16(g->shs) && (g->M == 1 || aligned16(g->sh_rest))));
    a.sh_stride = 0;
    a.sh_vec = 0;
    size_t dyn = 0;
    if (g->shs && raw) {
        dyn = (size_t)PRE_T * (g->M - 1) * 3 * sizeof(float) + 16;  // rows of the `rest` block, unpadded
    } else if (g->shs) {
        a.sh_stride = sh_row_stride(g->M, aligned16(g->shs), &a.sh_vec);
        dyn = (size_t)PRE_T * a.sh_stride * sizeof(float);
    }
    a.geom = geom;
    a.radii = radii;
    a.tile_count = img.tile_count;
    const auto preprocess = raw ? &preprocess_kernel<true> : &preprocess_kernel<false>;
    SGR_LAUNCH(K_PREPROCESS, st, preprocess<<<(P + PRE_T - 1) / PRE_T, PRE_T, dyn, st>>>(a));
    SGR_LAUNCH(K_TILE_SCAN, st,
               tile_scan_kernel<<<1, 1024, 0, st>>>(img.tile_count, img.tile_start, img.tile_cursor, img.tile_order,
                                                    img.counters, T, nullptr));
    SGR_CUDA(cudaGetLastError());
    SGR_CUDA(cudaMemcpyAsync(slot->pinned, img.counters, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    SGR_CUDA(cudaEventRecord(slot->ev, st));

    // Optimistic path: size the binning buffer from the caller's hint and enqueue everything
    // before looking at R; the device-side guard makes an overflowing attempt a no-op.
    bool launched = false;
    uint64_t capacity = 0;
    BinState bin;
    if (capacity_hint > 0) {
        capacity = (uint64_t)capacity_hint;
        void *bin_mem = binning_alloc(binning_ctx, sgr_binning_bytes((int64_t)capacity));
        if (!bin_mem) {
            set_error("binning allocator returned NULL");
            return SGR_ENOMEM;
        }
        Layout bin_l(bin_mem);
        bin = BinState::carve(bin_l, capacity);
        rc = launch_binning_and_blend(v, P, geom, img, bin, capacity, out_color, feat, st);
        if (rc) return rc;
        launched = true;
    }
    SGR_CUDA(cudaEventSynchronize(slot->ev));
    const uint64_t R = *slot->pinned;
    if (!launched || R > capacity) {
        capacity = R;
        void *bin_mem = binning_alloc(binning_ctx, sgr_binning_bytes((int64_t)capacity));
        if (!bin_mem) {
            set_error("binning allocator returned NULL");
            return SGR_ENOMEM;
        }
        Layout bin_l(bin_mem);
        bin = BinState::carve(bin_l, capacity);
        if (launched) {  // cursors were not advanced by the guarded attempt, but be explicit
            SGR_CUDA(cudaMemcpyAsync(img.tile_cursor, img.tile_start, sizeof(uint32_t) * T, cudaMemcpyDeviceToDevice, st));
        }
        rc = launch_binning_and_blend(v, P, geom, img, bin, capacity, out_color, feat, st);
        if (rc) return rc;
    }
    *num_rendered = (int64_t)R;
    if (view->debug) SGR_CUDA(cudaStreamSynchronize(st));
    return SGR_OK;
}

}  // namespace sgr
