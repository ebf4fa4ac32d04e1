// sgr_loss.cu -- the trainers' photometric loss, (1 - f) * L1 + f * (1 - SSIM), as one forward and one backward.
//
// Replaces the PyTorch chain of sugar_utils/loss_utils.py:17-62 (l1_loss, create_window, ssim, _ssim): five grouped
// 11x11 conv2d with zero padding, about fifteen elementwise temporaries and autograd through all of it.
//
// Forward, one CTA per 32x16 output tile of one (image, channel) plane:
//   stage x = img1, y = img2 with a 5-pixel halo (zero outside the image) -> horizontal 11-tap pass over the five
//   products x, y, x^2, y^2, xy -> vertical pass = the five windowed moments of each output pixel in registers ->
//   S, |x - y| and the three partial derivatives of S by the moments (d0 = dS/dmu1 with sigma1^2 and sigma12
//   expanded, d1 = dS/dE[x^2], d2 = dS/dE[xy]), which leave as the op's saved state (12 B per element); S and
//   |x - y| are summed over the CTA, one pair per CTA goes to scratch, and a second kernel sums each image's pairs
//   in a fixed order (no float atomics: the outputs are identical from run to run).
// Backward, same tiling: stage d0, d1, d2 with the halo, run the adjoint (flipped) separable passes, and combine
//   dL/dx_p = g_ssim / N * (conv(d0) + 2 x_p conv(d1) + y_p conv(d2)) + g_l1 / N * sign(x_p - y_p).
//
// The moments are accumulated in double.  sigma^2 = E[x^2] - mu^2 cancels: on a near-converged render (noise 0.01
// around 0.5) it keeps three of float's seven digits, which is what puts the reference's own float32 gradient 1e-4
// away from float64.  The passes read their double operands from shared memory once per tap, which (not HBM)
// bounds both kernels; DESIGN sections 3 and 9 have the numbers and the next steps.
#include "sgr_internal.cuh"

namespace sgr {

constexpr int LT_X = 32, LT_Y = 16, LR = 5;            // output tile, window radius
constexpr int LSX = LT_X + 2 * LR, LSY = LT_Y + 2 * LR;  // staged tile with halo: 42 x 26
constexpr int L_THREADS = 256;                          // 32 x 8: each thread owns rows ty and ty + 8

struct LossConsts {
    int C, H, W;
    double w[11];
    double c1, c2;
};

constexpr size_t LOSS_FWD_SMEM = (size_t)(2 * LSY * LSX + 5 * LSY * LT_X) * sizeof(double);

__device__ __forceinline__ double warp_sum_d(double v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

__global__ void __launch_bounds__(L_THREADS) loss_forward_kernel(const LossConsts k, const float *__restrict__ img1,
                                                                 const float *__restrict__ img2,
                                                                 float *__restrict__ dmaps, size_t n_total,
                                                                 double2 *__restrict__ partials)
{
    extern __shared__ double smem[];
    double *sx = smem, *sy = sx + LSY * LSX, *hs = sy + LSY * LSX;  // hs[5][LSY][LT_X]
    __shared__ double red[2][L_THREADS / 32];
    const int tx = threadIdx.x, ty = threadIdx.y, tid = ty * 32 + tx;
    const int x0 = blockIdx.x * LT_X, y0 = blockIdx.y * LT_Y;
    const int H = k.H, W = k.W;
    const size_t base = (size_t)blockIdx.z * H * W;
    const float *a = img1 + base, *b = img2 + base;
    for (int i = tid; i < LSY * LSX; i += L_THREADS) {
        const int r = i / LSX, c = i - r * LSX, gy = y0 - LR + r, gx = x0 - LR + c;
        float va = 0.f, vb = 0.f;
        if (gy >= 0 && gy < H && gx >= 0 && gx < W) {
            const size_t o = (size_t)gy * W + gx;
            va = __ldg(a + o);
            vb = __ldg(b + o);
        }
        sx[i] = va;
        sy[i] = vb;
    }
    __syncthreads();
    // horizontal pass: row r of the staged tile, output column c
    for (int i = tid; i < LSY * LT_X; i += L_THREADS) {
        const int r = i >> 5, c = i & 31;
        const double *px = sx + r * LSX + c, *py = sy + r * LSX + c;
        double m0 = 0, m1 = 0, m2 = 0, m3 = 0, m4 = 0;
#pragma unroll
        for (int j = 0; j < 11; j++) {
            const double u = px[j], v = py[j], wu = k.w[j] * u, wv = k.w[j] * v;
            m0 += wu;
            m1 += wv;
            m2 = fma(wu, u, m2);
            m3 = fma(wv, v, m3);
            m4 = fma(wu, v, m4);
        }
        hs[(0 * LSY + r) * LT_X + c] = m0;
        hs[(1 * LSY + r) * LT_X + c] = m1;
        hs[(2 * LSY + r) * LT_X + c] = m2;
        hs[(3 * LSY + r) * LT_X + c] = m3;
        hs[(4 * LSY + r) * LT_X + c] = m4;
    }
    __syncthreads();
    double sum_s = 0.0, sum_l1 = 0.0;
    const int gx = x0 + tx;
#pragma unroll
    for (int half = 0; half < 2; half++) {
        const int rr = ty + 8 * half, gy = y0 + rr;
        if (gy >= H || gx >= W) continue;
        double mu1 = 0, mu2 = 0, ex2 = 0, ey2 = 0, exy = 0;
#pragma unroll
        for (int j = 0; j < 11; j++) {
            const double w = k.w[j];
            const int o = (rr + j) * LT_X + tx;
            mu1 = fma(w, hs[0 * LSY * LT_X + o], mu1);
            mu2 = fma(w, hs[1 * LSY * LT_X + o], mu2);
            ex2 = fma(w, hs[2 * LSY * LT_X + o], ex2);
            ey2 = fma(w, hs[3 * LSY * LT_X + o], ey2);
            exy = fma(w, hs[4 * LSY * LT_X + o], exy);
        }
        const double mu11 = mu1 * mu1, mu22 = mu2 * mu2, mu12 = mu1 * mu2;
        const double A1 = 2.0 * mu12 + k.c1, A2 = 2.0 * (exy - mu12) + k.c2;
        const double B1 = mu11 + mu22 + k.c1, B2 = (ex2 - mu11) + (ey2 - mu22) + k.c2;
        const double inv = 1.0 / (B1 * B2);
        const double S = A1 * A2 * inv;
        const double d1 = -S * B1 * inv;       // -S / B2
        const double d2 = 2.0 * A1 * inv;
        const double d0 = 2.0 * mu2 * A2 * inv - 2.0 * mu1 * S * B2 * inv - 2.0 * mu1 * d1 - mu2 * d2;
        const size_t o = base + (size_t)gy * W + gx;
        dmaps[o] = (float)d0;
        dmaps[n_total + o] = (float)d1;
        dmaps[2 * n_total + o] = (float)d2;
        const int so = (rr + LR) * LSX + tx + LR;
        sum_s += S;
        sum_l1 += fabs(sx[so] - sy[so]);
    }
    sum_s = warp_sum_d(sum_s);
    sum_l1 = warp_sum_d(sum_l1);
    if (tx == 0) {
        red[0][ty] = sum_l1;
        red[1][ty] = sum_s;
    }
    __syncthreads();
    if (tid == 0) {
        double l = 0.0, s = 0.0;
        for (int w = 0; w < L_THREADS / 32; w++) {
            l += red[0][w];
            s += red[1][w];
        }
        const size_t tile = ((size_t)blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
        partials[tile] = make_double2(l, s);
    }
}

// one CTA per image: its C planes' CTA pairs, in a fixed order
__global__ void __launch_bounds__(256) loss_reduce_kernel(int pairs_per_image, double inv_n,
                                                          const double2 *__restrict__ partials, float *__restrict__ out)
{
    __shared__ double r0[256], r1[256];
    const int t = threadIdx.x;
    const double2 *p = partials + (size_t)blockIdx.x * pairs_per_image;
    double l = 0.0, s = 0.0;
    for (int i = t; i < pairs_per_image; i += 256) {
        const double2 v = p[i];
        l += v.x;
        s += v.y;
    }
    r0[t] = l;
    r1[t] = s;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if (t < o) {
            r0[t] += r0[t + o];
            r1[t] += r1[t + o];
        }
        __syncthreads();
    }
    if (t == 0) {
        out[2 * blockIdx.x] = (float)(r0[0] * inv_n);
        out[2 * blockIdx.x + 1] = (float)(r1[0] * inv_n);
    }
}

__global__ void __launch_bounds__(L_THREADS) loss_backward_kernel(const LossConsts k, const float *__restrict__ img1,
                                                                  const float *__restrict__ img2,
                                                                  const float *__restrict__ dmaps, size_t n_total,
                                                                  double inv_n, const float *__restrict__ g_l1,
                                                                  const float *__restrict__ g_ssim,
                                                                  float *__restrict__ grad)
{
    __shared__ double sd[3][LSY * LSX];
    __shared__ double hb[3][LSY * LT_X];
    const int tx = threadIdx.x, ty = threadIdx.y, tid = ty * 32 + tx;
    const int x0 = blockIdx.x * LT_X, y0 = blockIdx.y * LT_Y;
    const int H = k.H, W = k.W;
    const size_t base = (size_t)blockIdx.z * H * W;
    for (int i = tid; i < LSY * LSX; i += L_THREADS) {
        const int r = i / LSX, c = i - r * LSX, gy = y0 - LR + r, gx = x0 - LR + c;
        float v0 = 0.f, v1 = 0.f, v2 = 0.f;
        if (gy >= 0 && gy < H && gx >= 0 && gx < W) {
            const size_t o = base + (size_t)gy * W + gx;
            v0 = __ldg(dmaps + o);
            v1 = __ldg(dmaps + n_total + o);
            v2 = __ldg(dmaps + 2 * n_total + o);
        }
        sd[0][i] = v0;
        sd[1][i] = v1;
        sd[2][i] = v2;
    }
    __syncthreads();
    // adjoint of the zero-padded correlation = correlation with the flipped window
    for (int i = tid; i < LSY * LT_X; i += L_THREADS) {
        const int r = i >> 5, c = i & 31, o = r * LSX + c;
        double m0 = 0, m1 = 0, m2 = 0;
#pragma unroll
        for (int j = 0; j < 11; j++) {
            const double w = k.w[10 - j];
            m0 = fma(w, sd[0][o + j], m0);
            m1 = fma(w, sd[1][o + j], m1);
            m2 = fma(w, sd[2][o + j], m2);
        }
        hb[0][i] = m0;
        hb[1][i] = m1;
        hb[2][i] = m2;
    }
    __syncthreads();
    const int img = blockIdx.z / k.C;
    const double cs = (double)g_ssim[img] * inv_n, cl = (double)g_l1[img] * inv_n;
    const int gx = x0 + tx;
#pragma unroll
    for (int half = 0; half < 2; half++) {
        const int rr = ty + 8 * half, gy = y0 + rr;
        if (gy >= H || gx >= W) continue;
        double m0 = 0, m1 = 0, m2 = 0;
#pragma unroll
        for (int j = 0; j < 11; j++) {
            const double w = k.w[10 - j];
            const int o = (rr + j) * LT_X + tx;
            m0 = fma(w, hb[0][o], m0);
            m1 = fma(w, hb[1][o], m1);
            m2 = fma(w, hb[2][o], m2);
        }
        const size_t o = base + (size_t)gy * W + gx;
        const float xf = __ldg(img1 + o), yf = __ldg(img2 + o);
        const double x = xf, y = yf;
        const double sgn = (xf > yf) ? 1.0 : ((xf < yf) ? -1.0 : 0.0);  // torch's abs backward: sign(0) = 0
        grad[o] = (float)(cs * (m0 + 2.0 * x * m1 + y * m2) + cl * sgn);
    }
}

struct LossGrid {
    dim3 grid;
    int64_t n_image, n_total;
};

static int loss_check(const SgrSsimParams *p, LossGrid &g, const char *who)
{
    if (!p) {
        set_error("%s: null params", who);
        return SGR_EINVAL;
    }
    if (p->B <= 0 || p->C <= 0 || p->H <= 0 || p->W <= 0) {
        set_error("%s: bad sizes B=%d C=%d H=%d W=%d (every dimension must be >= 1)", who, p->B, p->C, p->H, p->W);
        return SGR_EINVAL;
    }
    g.n_image = (int64_t)p->C * p->H * p->W;
    g.n_total = g.n_image * p->B;
    if (g.n_total > INT32_MAX) {
        set_error("%s: %lld elements exceed 2^31 - 1", who, (long long)g.n_total);
        return SGR_EINVAL;
    }
    const int64_t planes = (int64_t)p->B * p->C, rows = (p->H + LT_Y - 1) / LT_Y;
    if (planes > 65535 || rows > 65535) {
        set_error("%s: B*C = %lld planes or %lld tile rows exceed the grid's 65535", who, (long long)planes,
                  (long long)rows);
        return SGR_EINVAL;
    }
    g.grid = dim3((unsigned)((p->W + LT_X - 1) / LT_X), (unsigned)rows, (unsigned)planes);
    return SGR_OK;
}

// the forward's per-(block, channel) partial sums, one per tile of every plane
static double2 *loss_partials(Layout &l, const LossGrid &g)
{
    return l.take<double2>((size_t)g.grid.x * g.grid.y * g.grid.z);
}

static LossConsts loss_consts(const SgrSsimParams *p)
{
    LossConsts k;
    k.C = p->C;
    k.H = p->H;
    k.W = p->W;
    for (int j = 0; j < 11; j++) k.w[j] = (double)p->window[j];
    k.c1 = (double)p->c1;
    k.c2 = (double)p->c2;
    return k;
}

}  // namespace sgr

using namespace sgr;

extern "C" {

size_t sgr_l1_ssim_scratch_bytes(int32_t B, int32_t C, int32_t H, int32_t W)
{
    SgrSsimParams p = {};
    p.B = B, p.C = C, p.H = H, p.W = W;
    LossGrid g;
    if (loss_check(&p, g, "sgr_l1_ssim_scratch_bytes")) return 0;
    return layout_bytes([&](Layout &l) { loss_partials(l, g); });
}

int sgr_l1_ssim_forward(const SgrSsimParams *p, const float *img1, const float *img2, float *partial_maps,
                        float *per_image_out, void *scratch, void *stream)
{
    LossGrid g;
    int rc = loss_check(p, g, "sgr_l1_ssim_forward");
    if (rc) return rc;
    if (!img1 || !img2 || !partial_maps || !per_image_out || !scratch) {
        set_error("sgr_l1_ssim_forward: null pointer");
        return SGR_EINVAL;
    }
    cudaStream_t st = (cudaStream_t)stream;
    const LossConsts k = loss_consts(p);
    Layout l(scratch);
    double2 *partials = loss_partials(l, g);
    static DeviceOnce attributes;
    rc = once_per_device(attributes, []() -> int {
        SGR_CUDA(cudaFuncSetAttribute(loss_forward_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (int)LOSS_FWD_SMEM));
        return SGR_OK;
    });
    if (rc) return rc;
    SGR_LAUNCH(K_LOSS_FWD, st,
               loss_forward_kernel<<<g.grid, dim3(32, L_THREADS / 32), LOSS_FWD_SMEM, st>>>(
                   k, img1, img2, partial_maps, (size_t)g.n_total, partials));
    const int pairs = (int)(g.grid.x * g.grid.y) * p->C;
    SGR_LAUNCH(K_LOSS_FWD, st,
               loss_reduce_kernel<<<p->B, 256, 0, st>>>(pairs, 1.0 / (double)g.n_image, partials, per_image_out));
    SGR_CUDA(cudaGetLastError());
    return SGR_OK;
}

int sgr_l1_ssim_backward(const SgrSsimParams *p, const float *img1, const float *img2, const float *partial_maps,
                         const float *g_l1, const float *g_ssim, float *grad_img1, void *stream)
{
    LossGrid g;
    int rc = loss_check(p, g, "sgr_l1_ssim_backward");
    if (rc) return rc;
    if (!img1 || !img2 || !partial_maps || !g_l1 || !g_ssim || !grad_img1) {
        set_error("sgr_l1_ssim_backward: null pointer");
        return SGR_EINVAL;
    }
    cudaStream_t st = (cudaStream_t)stream;
    const LossConsts k = loss_consts(p);
    SGR_LAUNCH(K_LOSS_BWD, st,
               loss_backward_kernel<<<g.grid, dim3(32, L_THREADS / 32), 0, st>>>(
                   k, img1, img2, partial_maps, (size_t)g.n_total, 1.0 / (double)g.n_image, g_l1, g_ssim, grad_img1));
    SGR_CUDA(cudaGetLastError());
    return SGR_OK;
}

}  // extern "C"
