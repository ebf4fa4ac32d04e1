// sgr_lpips.cu -- LPIPS (VGG16, v0.1) forward: the metric of metrics.py (gaussian_splatting/lpipsPyTorch), over a
// batch of 2N images -- the N renders x then the N ground truths y -- so every layer's weights are read once per pair.
//
//   conv1_1        lpips_conv1_kernel: z-score fused into its loads from the NCHW float32 images, K = 27 by FFMA
//   conv1_2..5_3   lpips_conv3x3_kernel: implicit GEMM over NHWC float32 activations, M = 2N*H*W pixels, N = Cout,
//                  K = 9*Cin in (r, s, c) order; TF32 mma.sync m16n8k8 with float32 accumulation, operands staged
//                  through a STAGES-deep cp.async pipeline (zero-filled outside the image = the conv's padding);
//                  A rounded to TF32 by cvt.rna at fragment load, B (the weights) rounded once when they are packed
//   taps 1..5      lpips_tap_kernel: one warp per 2x2 quad of pixels of one pair; both channel norms, the weighted
//                  squared difference of the normalised features, per-CTA sums in double; at taps 1-4 also the 2x2
//                  max pool (floors odd sizes) of x's and y's features for the next conv
//   result         lpips_reduce_kernel: per image and tap, the CTA sums in a fixed order (sgr_reduce.cuh), over H*W
//
// No float atomics anywhere: a result is bit-identical from run to run and independent of the batch it is in.
#include "sgr_internal.cuh"
#include "sgr_reduce.cuh"

namespace sgr {

constexpr int LP_TAPS = 5;
constexpr int LP_CONVS = 13;
constexpr int LP_CIN[LP_CONVS] = {3, 64, 64, 128, 128, 256, 256, 256, 512, 512, 512, 512, 512};
constexpr int LP_COUT[LP_CONVS] = {64, 64, 128, 128, 256, 256, 256, 512, 512, 512, 512, 512, 512};
constexpr int LP_TAP_C[LP_TAPS] = {64, 128, 256, 512, 512};

// ---------------------------------------------------------------------------------------------------------------
// conv1_1: 8 threads per output pixel, 8 output channels each (two float4 stores; a warp writes 4 pixels = 1 KB)
// ---------------------------------------------------------------------------------------------------------------
constexpr int C1_THREADS = 256, C1_PIX = C1_THREADS / 8;

__global__ void __launch_bounds__(C1_THREADS)
    lpips_conv1_kernel(int N, int H, int W, const float *__restrict__ x, const float *__restrict__ y,
                       const float *__restrict__ w, const float *__restrict__ bias, float *__restrict__ out)
{
    __shared__ float sw[27][64];  // [(r * 3 + s) * 3 + c][o]
    __shared__ float sb[64];
    const int tid = threadIdx.x;
    for (int i = tid; i < 64 * 27; i += C1_THREADS) sw[i % 27][i / 27] = w[i];
    if (tid < 64) sb[tid] = bias[tid];
    __syncthreads();
    const int HW = H * W;
    const int64_t p = (int64_t)blockIdx.x * C1_PIX + (tid >> 3);
    if (p >= 2 * (int64_t)N * HW) return;
    const int b = (int)(p / HW), q = (int)(p - (int64_t)b * HW), py = q / W, px = q - py * W;
    const float *img = b < N ? x + (size_t)b * 3 * HW : y + (size_t)(b - N) * 3 * HW;
    // the reference's z-score in float32, (v - mean) / std; the conv pads the z-scored image with zeros
    const float mean[3] = {-.030f, -.088f, -.188f}, stdv[3] = {.458f, .448f, .450f};
    float v[27];
#pragma unroll
    for (int r = 0; r < 3; r++) {
#pragma unroll
        for (int s = 0; s < 3; s++) {
            const int iy = py + r - 1, ix = px + s - 1;
            const bool in = iy >= 0 && iy < H && ix >= 0 && ix < W;
#pragma unroll
            for (int c = 0; c < 3; c++)
                v[(r * 3 + s) * 3 + c] = in ? __fdiv_rn(__ldg(img + (size_t)c * HW + iy * W + ix) - mean[c], stdv[c]) : 0.f;
        }
    }
    const int o0 = (tid & 7) * 8;
    float acc[8];
#pragma unroll
    for (int o = 0; o < 8; o++) acc[o] = 0.f;
#pragma unroll
    for (int k = 0; k < 27; k++) {
#pragma unroll
        for (int o = 0; o < 8; o++) acc[o] = fmaf(v[k], sw[k][o0 + o], acc[o]);
    }
    float4 *dst = (float4 *)(out + (size_t)p * 64 + o0);
    dst[0] = make_float4(fmaxf(acc[0] + sb[o0 + 0], 0.f), fmaxf(acc[1] + sb[o0 + 1], 0.f),
                         fmaxf(acc[2] + sb[o0 + 2], 0.f), fmaxf(acc[3] + sb[o0 + 3], 0.f));
    dst[1] = make_float4(fmaxf(acc[4] + sb[o0 + 4], 0.f), fmaxf(acc[5] + sb[o0 + 5], 0.f),
                         fmaxf(acc[6] + sb[o0 + 6], 0.f), fmaxf(acc[7] + sb[o0 + 7], 0.f));
}

// ---------------------------------------------------------------------------------------------------------------
// 3x3 conv + bias + ReLU as an implicit GEMM on the tensor cores
// ---------------------------------------------------------------------------------------------------------------
constexpr int CV_THREADS = 256, CV_BK = 32, CV_LDS = CV_BK + 4, CV_STAGES = 3;  // +4: conflict-free fragment loads

template <int BM, int BN>
constexpr size_t conv_smem_bytes()
{
    return (size_t)CV_STAGES * (BM + BN) * CV_LDS * sizeof(float);
}

// 16 bytes global -> shared; src_bytes = 0 zero-fills the destination (the conv's padding, rows past M)
__device__ __forceinline__ void cp_async16_zfill(uint32_t dst, const void *src, int src_bytes)
{
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}

__device__ __forceinline__ uint32_t tf32_rna(float v)
{
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;\n" : "=r"(r) : "f"(v));
    return r;
}

__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2])
{
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
                 "{%0,%1,%2,%3};\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

// One CTA computes a BM-pixel x BN-channel tile with 8 warps of 64 x 32 each.  in [M, CIN], wgt [Cout, 9 * CIN]
// (KRSC, TF32-rounded), out [M, Cout]; a 32-wide K tile lies inside one (r, s) tap because CIN % 32 == 0.
template <int CIN, int BM, int BN>
__global__ void __launch_bounds__(CV_THREADS, 2)
    lpips_conv3x3_kernel(int M, int H, int W, int Cout, const float *__restrict__ in, const float *__restrict__ wgt,
                         const float *__restrict__ bias, float *__restrict__ out)
{
    constexpr int WM = BM / 64, A_IT = BM * 8 / CV_THREADS, B_IT = BN * 8 / CV_THREADS;
    constexpr int K = 9 * CIN, KT = K / CV_BK;
    static_assert(WM * (BN / 32) == CV_THREADS / 32, "8 warps of 64 x 32");
    extern __shared__ float4 smem_f4[];
    float *As = (float *)smem_f4;                        // [STAGES][BM][LDS]
    float *Bs = As + CV_STAGES * BM * CV_LDS;            // [STAGES][BN][LDS]
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int wm = warp % WM, wn = warp / WM, g = lane >> 2, t = lane & 3;
    const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
    const int HW = H * W, col4 = (tid & 7) * 4;

    // the A rows this thread loads: pixel index and its (y, x); y = -4 marks a row past M (never in bounds)
    int a_m[A_IT], a_y[A_IT], a_x[A_IT];
#pragma unroll
    for (int j = 0; j < A_IT; j++) {
        const int m = m0 + (tid >> 3) + j * (CV_THREADS / 8);
        const int q = m % HW;
        a_m[j] = m;
        a_y[j] = m < M ? q / W : -4;
        a_x[j] = q % W;
    }
    const float *b_src = wgt + (size_t)(n0 + (tid >> 3)) * K + col4;

    auto load_stage = [&](int kt, int stage) {
        const int k0 = kt * CV_BK, rs = k0 / CIN, c0 = k0 - rs * CIN, dy = rs / 3 - 1, dx = rs % 3 - 1;
        float *as = As + stage * BM * CV_LDS;
#pragma unroll
        for (int j = 0; j < A_IT; j++) {
            const int iy = a_y[j] + dy, ix = a_x[j] + dx;
            const bool ok = iy >= 0 && iy < H && ix >= 0 && ix < W;
            const float *src = ok ? in + (size_t)(a_m[j] + dy * W + dx) * CIN + c0 + col4 : in;
            cp_async16_zfill(smem_u32(as + ((tid >> 3) + j * (CV_THREADS / 8)) * CV_LDS + col4), src, ok ? 16 : 0);
        }
        float *bs = Bs + stage * BN * CV_LDS;
#pragma unroll
        for (int j = 0; j < B_IT; j++)
            cp_async16_zfill(smem_u32(bs + ((tid >> 3) + j * (CV_THREADS / 8)) * CV_LDS + col4),
                       b_src + (size_t)j * (CV_THREADS / 8) * K + k0, 16);
    };

    float acc[4][4][4];
#pragma unroll
    for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 4; j++)
#pragma unroll
            for (int e = 0; e < 4; e++) acc[i][j][e] = 0.f;

#pragma unroll
    for (int s = 0; s < CV_STAGES - 1; s++) {
        if (s < KT) load_stage(s, s);
        cp_async_commit();
    }
    for (int kt = 0; kt < KT; kt++) {
        cp_async_wait<CV_STAGES - 2>();
        __syncthreads();  // stage kt landed for every thread; stage kt - 1 is free to overwrite
        if (kt + CV_STAGES - 1 < KT) load_stage(kt + CV_STAGES - 1, (kt + CV_STAGES - 1) % CV_STAGES);
        cp_async_commit();
        const float *as = As + (kt % CV_STAGES) * BM * CV_LDS + (wm * 64 + g) * CV_LDS + t;
        const float *bs = Bs + (kt % CV_STAGES) * BN * CV_LDS + (wn * 32 + g) * CV_LDS + t;
#pragma unroll
        for (int kk = 0; kk < CV_BK; kk += 8) {
            uint32_t bf[4][2];
#pragma unroll
            for (int j = 0; j < 4; j++) {
                bf[j][0] = __float_as_uint(bs[j * 8 * CV_LDS + kk]);
                bf[j][1] = __float_as_uint(bs[j * 8 * CV_LDS + kk + 4]);
            }
#pragma unroll
            for (int i = 0; i < 4; i++) {
                const float *a = as + i * 16 * CV_LDS + kk;
                const uint32_t af[4] = {tf32_rna(a[0]), tf32_rna(a[8 * CV_LDS]), tf32_rna(a[4]),
                                        tf32_rna(a[8 * CV_LDS + 4])};
#pragma unroll
                for (int j = 0; j < 4; j++) mma_tf32(acc[i][j], af, bf[j]);
            }
        }
    }
    cp_async_wait<0>();

#pragma unroll
    for (int j = 0; j < 4; j++) {
        const int n = n0 + wn * 32 + j * 8 + 2 * t;
        const float b0 = __ldg(bias + n), b1 = __ldg(bias + n + 1);
#pragma unroll
        for (int i = 0; i < 4; i++) {
            const int m = m0 + wm * 64 + i * 16 + g;
            if (m < M)
                *(float2 *)(out + (size_t)m * Cout + n) =
                    make_float2(fmaxf(acc[i][j][0] + b0, 0.f), fmaxf(acc[i][j][1] + b1, 0.f));
            if (m + 8 < M)
                *(float2 *)(out + (size_t)(m + 8) * Cout + n) =
                    make_float2(fmaxf(acc[i][j][2] + b0, 0.f), fmaxf(acc[i][j][3] + b1, 0.f));
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------
// taps: normalise, weighted squared difference, per-CTA sums; 2x2 max pool for the next block
// ---------------------------------------------------------------------------------------------------------------
constexpr int TAP_THREADS = 256, TAP_QPW = 4, TAP_QPC = TAP_QPW * TAP_THREADS / 32;  // quads per warp, per CTA

static int tap_blocks(int H, int W)
{
    const int64_t quads = (int64_t)((H + 1) / 2) * ((W + 1) / 2);
    return (int)((quads + TAP_QPC - 1) / TAP_QPC);
}

template <int VW>
__device__ __forceinline__ void load_vec(const float *p, float *v)
{
    if constexpr (VW == 4) {
        const float4 f = __ldg((const float4 *)p);
        v[0] = f.x, v[1] = f.y, v[2] = f.z, v[3] = f.w;
    } else {
        const float2 f = __ldg((const float2 *)p);
        v[0] = f.x, v[1] = f.y;
    }
}

template <int VW>
__device__ __forceinline__ void store_vec(float *p, const float *v)
{
    if constexpr (VW == 4)
        *(float4 *)p = make_float4(v[0], v[1], v[2], v[3]);
    else
        *(float2 *)p = make_float2(v[0], v[1]);
}

// feat [2N, H, W, C]: pair n is images n and N + n.  Lane l holds channels (j * 32 + l) * VW + e.
template <int C, bool POOL>
__global__ void __launch_bounds__(TAP_THREADS)
    lpips_tap_kernel(int N, int H, int W, const float *__restrict__ feat, const float *__restrict__ lin,
                     float *__restrict__ pooled, double *__restrict__ partials)
{
    constexpr int E = C / 32, VW = E >= 4 ? 4 : E, NV = E / VW;
    __shared__ double red[TAP_THREADS / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n = blockIdx.y;
    const int Wq = (W + 1) / 2, nq = ((H + 1) / 2) * Wq, Hp = H / 2, Wp = W / 2;
    const float *fx = feat + (size_t)n * H * W * C, *fy = feat + (size_t)(N + n) * H * W * C;
    float lw[E];
#pragma unroll
    for (int j = 0; j < NV; j++) load_vec<VW>(lin + (j * 32 + lane) * VW, lw + j * VW);
    double wsum = 0.0;
    for (int i = 0; i < TAP_QPW; i++) {
        const int qd = (blockIdx.x * (TAP_THREADS / 32) + warp) * TAP_QPW + i;
        if (qd >= nq) break;
        const int qy = qd / Wq, qx = qd - qy * Wq;
        float mx[E], my[E];
#pragma unroll
        for (int e = 0; e < E; e++) mx[e] = my[e] = -INFINITY;
#pragma unroll
        for (int d = 0; d < 4; d++) {
            const int py = 2 * qy + (d >> 1), px = 2 * qx + (d & 1);
            if (py >= H || px >= W) continue;
            const size_t o = ((size_t)py * W + px) * C;
            float ax[E], ay[E];
#pragma unroll
            for (int j = 0; j < NV; j++) {
                load_vec<VW>(fx + o + (j * 32 + lane) * VW, ax + j * VW);
                load_vec<VW>(fy + o + (j * 32 + lane) * VW, ay + j * VW);
            }
            float sx = 0.f, sy = 0.f;
#pragma unroll
            for (int e = 0; e < E; e++) {
                sx = fmaf(ax[e], ax[e], sx);
                sy = fmaf(ay[e], ay[e], sy);
            }
            // the reference's normalize_activation: eps outside the sqrt
            const float nx = sqrtf(warp_sum(sx)) + 1e-10f, ny = sqrtf(warp_sum(sy)) + 1e-10f;
            float dsum = 0.f;
#pragma unroll
            for (int e = 0; e < E; e++) {
                const float dd = ax[e] / nx - ay[e] / ny;
                dsum = fmaf(lw[e], dd * dd, dsum);
            }
            wsum += (double)warp_sum(dsum);
            if constexpr (POOL) {
#pragma unroll
                for (int e = 0; e < E; e++) {
                    mx[e] = fmaxf(mx[e], ax[e]);
                    my[e] = fmaxf(my[e], ay[e]);
                }
            }
        }
        if constexpr (POOL) {
            if (qy < Hp && qx < Wp) {
                const size_t o = ((size_t)qy * Wp + qx) * C;
                float *px_ = pooled + (size_t)n * Hp * Wp * C + o, *py_ = pooled + (size_t)(N + n) * Hp * Wp * C + o;
#pragma unroll
                for (int j = 0; j < NV; j++) {
                    store_vec<VW>(px_ + (j * 32 + lane) * VW, mx + j * VW);
                    store_vec<VW>(py_ + (j * 32 + lane) * VW, my + j * VW);
                }
            }
        }
    }
    const double s = cta_sum_by_warps<TAP_THREADS>(lane == 0 ? wsum : 0.0, red);
    if (threadIdx.x == 0) partials[(size_t)n * gridDim.x + blockIdx.x] = s;
}

// ---------------------------------------------------------------------------------------------------------------
// per image: each tap's CTA sums in a fixed order, over that tap's H*W; LPIPS = the sum of the five means
// ---------------------------------------------------------------------------------------------------------------
struct TapPlan {
    int H[LP_TAPS], W[LP_TAPS], blocks[LP_TAPS];
    size_t offset[LP_TAPS];  // doubles from the start of the partials, [N][blocks] per tap
    size_t total;
};

static TapPlan tap_plan(int N, int H, int W)
{
    TapPlan p;
    p.total = 0;
    for (int t = 0; t < LP_TAPS; t++) {
        p.H[t] = H >> t;
        p.W[t] = W >> t;
        p.blocks[t] = tap_blocks(p.H[t], p.W[t]);
        p.offset[t] = p.total;
        p.total += (size_t)N * p.blocks[t];
    }
    return p;
}

__global__ void __launch_bounds__(256)
    lpips_reduce_kernel(TapPlan plan, const double *__restrict__ partials, float *__restrict__ taps,
                        float *__restrict__ out)
{
    __shared__ double sh[256];
    const int n = blockIdx.x;
    double total = 0.0;
#pragma unroll
    for (int t = 0; t < LP_TAPS; t++) {
        const int nb = plan.blocks[t];
        const double s = cta_sum_partials<256>(nb, partials + plan.offset[t] + (size_t)n * nb, 1, sh);
        __syncthreads();  // sh is reused by the next tap
        const double mean = s / ((double)plan.H[t] * plan.W[t]);
        if (threadIdx.x == 0 && taps) taps[n * LP_TAPS + t] = (float)mean;
        total += mean;
    }
    if (threadIdx.x == 0) out[n] = (float)total;
}

// ---------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------
static size_t weight_floats()
{
    size_t n = 0;
    for (int l = 0; l < LP_CONVS; l++) n += (size_t)LP_COUT[l] * 9 * LP_CIN[l] + LP_COUT[l];
    for (int t = 0; t < LP_TAPS; t++) n += LP_TAP_C[t];
    return n;
}

static bool lpips_sizes_ok(int N, int H, int W, const char *who)
{
    if (N < 1 || H < 16 || W < 16 || 2 * (int64_t)N * H * W > INT32_MAX / 64) {
        set_error("%s: N=%d, H=%d, W=%d: LPIPS needs N >= 1, H, W >= 16 (the fifth tap is 1/16 of the size) and "
                  "2 N H W 64 < 2^31", who, N, H, W);
        return false;
    }
    return true;
}

struct LpipsCarve {
    float *act[2];
    double *partials;
};

static LpipsCarve lpips_carve(Layout &l, int N, int H, int W)
{
    LpipsCarve c;
    const size_t act = (size_t)2 * N * H * W * 64;  // the largest activation: conv1_x at full size
    c.act[0] = l.take<float>(act);
    c.act[1] = l.take<float>(act);
    c.partials = l.take<double>(tap_plan(N, H, W).total);
    return c;
}

template <int CIN, int BM, int BN>
static int launch_conv(int M, int H, int W, int Cout, const float *in, const float *w, const float *b, float *out,
                       cudaStream_t st)
{
    constexpr size_t smem = conv_smem_bytes<BM, BN>();
    static DeviceOnce attributes;
    const int rc = once_per_device(attributes, []() -> int {
        SGR_CUDA(cudaFuncSetAttribute(lpips_conv3x3_kernel<CIN, BM, BN>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (int)smem));
        return SGR_OK;
    });
    if (rc) return rc;
    const dim3 grid((unsigned)((M + BM - 1) / BM), (unsigned)(Cout / BN));
    SGR_LAUNCH(K_MISC, st,
               (lpips_conv3x3_kernel<CIN, BM, BN><<<grid, CV_THREADS, smem, st>>>(M, H, W, Cout, in, w, b, out)));
    SGR_CUDA(cudaGetLastError());
    return SGR_OK;
}

template <int CIN>
static int conv_cin(int M, int H, int W, int Cout, const float *in, const float *w, const float *b, float *out,
                    cudaStream_t st)
{
    if (Cout == 64) return launch_conv<CIN, 256, 64>(M, H, W, Cout, in, w, b, out, st);
    return launch_conv<CIN, 128, 128>(M, H, W, Cout, in, w, b, out, st);
}

template <int C>
static int launch_tap(int N, int H, int W, const float *feat, const float *lin, float *pooled, double *partials,
                      cudaStream_t st)
{
    const dim3 grid((unsigned)tap_blocks(H, W), (unsigned)N);
    if (pooled) {
        SGR_LAUNCH(K_MISC, st,
                   (lpips_tap_kernel<C, true><<<grid, TAP_THREADS, 0, st>>>(N, H, W, feat, lin, pooled, partials)));
    } else if constexpr (C == 512) {  // the fifth tap: pool5 never runs
        SGR_LAUNCH(K_MISC, st,
                   (lpips_tap_kernel<C, false><<<grid, TAP_THREADS, 0, st>>>(N, H, W, feat, lin, nullptr, partials)));
    }
    SGR_CUDA(cudaGetLastError());
    return SGR_OK;
}

}  // namespace sgr

using namespace sgr;

extern "C" {

size_t sgr_lpips_weight_floats(void) { return weight_floats(); }

int sgr_lpips_scratch_layout(int32_t N, int32_t H, int32_t W, const void *scratch, size_t *offsets)
{
    if (!lpips_sizes_ok(N, H, W, "sgr_lpips_scratch_layout")) return SGR_EINVAL;
    if (!offsets) {
        set_error("sgr_lpips_scratch_layout: null offsets");
        return SGR_EINVAL;
    }
    Layout l(scratch);
    const LpipsCarve c = lpips_carve(l, N, H, W);
    const TapPlan p = tap_plan(N, H, W);
    const char *base = (const char *)scratch;
    offsets[0] = (size_t)((const char *)c.act[0] - base);
    offsets[1] = (size_t)((const char *)c.act[1] - base);
    for (int t = 0; t < LP_TAPS; t++) offsets[2 + t] = (size_t)((const char *)(c.partials + p.offset[t]) - base);
    offsets[7] = l.bytes();
    return SGR_OK;
}

int sgr_lpips_conv1(int32_t N, int32_t H, int32_t W, const float *x, const float *y, const float *weight,
                    const float *bias, float *out, void *stream)
{
    if (N < 1 || H < 1 || W < 1 || 2 * (int64_t)N * H * W > INT32_MAX / 64) {
        set_error("sgr_lpips_conv1: bad sizes N=%d H=%d W=%d", N, H, W);
        return SGR_EINVAL;
    }
    if (!x || !y || !weight || !bias || !out || !aligned16(out)) {
        set_error("sgr_lpips_conv1: null pointer or `out` not 16-byte aligned");
        return SGR_EINVAL;
    }
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t M = 2 * (int64_t)N * H * W;
    SGR_LAUNCH(K_MISC, st,
               (lpips_conv1_kernel<<<(unsigned)((M + C1_PIX - 1) / C1_PIX), C1_THREADS, 0, st>>>(N, H, W, x, y, weight,
                                                                                                 bias, out)));
    SGR_CUDA(cudaGetLastError());
    return SGR_OK;
}

int sgr_lpips_conv3x3(int32_t B, int32_t H, int32_t W, int32_t Cin, int32_t Cout, const float *in,
                      const float *weight, const float *bias, float *out, void *stream)
{
    if (B < 1 || H < 1 || W < 1 || (int64_t)B * H * W * (Cin > Cout ? Cin : Cout) > INT32_MAX) {
        set_error("sgr_lpips_conv3x3: bad sizes B=%d H=%d W=%d", B, H, W);
        return SGR_EINVAL;
    }
    const auto vgg_width = [](int c) { return c == 64 || c == 128 || c == 256 || c == 512; };
    if (!vgg_width(Cin) || !vgg_width(Cout)) {
        set_error("sgr_lpips_conv3x3: Cin=%d, Cout=%d: each must be 64, 128, 256 or 512", Cin, Cout);
        return SGR_EINVAL;
    }
    if (!in || !weight || !bias || !out || !aligned16(in) || !aligned16(weight) || !aligned16(out)) {
        set_error("sgr_lpips_conv3x3: null pointer, or in / weight / out not 16-byte aligned");
        return SGR_EINVAL;
    }
    cudaStream_t st = (cudaStream_t)stream;
    const int M = B * H * W;
    switch (Cin) {
    case 64: return conv_cin<64>(M, H, W, Cout, in, weight, bias, out, st);
    case 128: return conv_cin<128>(M, H, W, Cout, in, weight, bias, out, st);
    case 256: return conv_cin<256>(M, H, W, Cout, in, weight, bias, out, st);
    default: return conv_cin<512>(M, H, W, Cout, in, weight, bias, out, st);
    }
}

int sgr_lpips_tap(int32_t N, int32_t H, int32_t W, int32_t C, const float *feat, const float *lin, float *pooled,
                  double *partials, void *stream)
{
    if (N < 1 || H < 1 || W < 1 || 2 * (int64_t)N * H * W > INT32_MAX) {
        set_error("sgr_lpips_tap: bad sizes N=%d H=%d W=%d", N, H, W);
        return SGR_EINVAL;
    }
    if (!feat || !lin || !partials || (!pooled && C != 512) || !aligned16(feat) || !aligned16(lin) ||
        (pooled && !aligned16(pooled))) {
        set_error("sgr_lpips_tap: null pointer (pooled may be NULL at C = 512 only), or feat / lin / pooled not "
                  "16-byte aligned");
        return SGR_EINVAL;
    }
    cudaStream_t st = (cudaStream_t)stream;
    switch (C) {
    case 64: return launch_tap<64>(N, H, W, feat, lin, pooled, partials, st);
    case 128: return launch_tap<128>(N, H, W, feat, lin, pooled, partials, st);
    case 256: return launch_tap<256>(N, H, W, feat, lin, pooled, partials, st);
    case 512: return launch_tap<512>(N, H, W, feat, lin, pooled, partials, st);
    default: set_error("sgr_lpips_tap: C=%d must be 64, 128, 256 or 512", C); return SGR_EINVAL;
    }
}

int sgr_lpips_reduce(int32_t N, int32_t H, int32_t W, const double *partials, float *taps, float *out, void *stream)
{
    if (!lpips_sizes_ok(N, H, W, "sgr_lpips_reduce")) return SGR_EINVAL;
    if (!partials || !out) {
        set_error("sgr_lpips_reduce: null pointer");
        return SGR_EINVAL;
    }
    cudaStream_t st = (cudaStream_t)stream;
    SGR_LAUNCH(K_MISC, st, (lpips_reduce_kernel<<<N, 256, 0, st>>>(tap_plan(N, H, W), partials, taps, out)));
    SGR_CUDA(cudaGetLastError());
    return SGR_OK;
}

}  // extern "C"
