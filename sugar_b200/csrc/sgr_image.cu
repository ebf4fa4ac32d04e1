// sgr_image.cu -- ground-truth image preparation (sugar_b200/dataset.py), byte for byte as the reference's Pillow and
// numpy lines prepare it (include/sugar_b200.h: sgr_image_prepare; oracle/imageprep_oracle.py restates each rule).
//
// One thread per output pixel, all of its channels.  Loads go through one of three source views:
//   RAW        the first NM channels of an NS-channel pixel (an RGB source, or the uint8 intermediate)
//   COMPOSITE  the float64 alpha composite of an RGBA pixel, from a per-CTA table of u / 255.0 (one division per
//              value instead of two per channel per tap), each product and sum rounded on its own (no FMA)
//   PREMUL     Pillow's rgbA2rgba of an RGBA pixel: c = MULDIV255(c, a)
// A pass (horizontal, vertical or none) sums Pillow's 22-bit fixed-point taps from 1 << 21 in int32 and clamps
// (libImaging/Resample.c); the last pass unpremultiplies a premultiplied pixel (rgba2rgbA) and writes u / 255.f.
#include "sgr_internal.cuh"

namespace sgr {

constexpr int IMG_BX = 32, IMG_BY = 8;
constexpr int IMG_PRECISION = 22;

enum ImgLoad { LOAD_RAW = 0, LOAD_COMPOSITE = 1, LOAD_PREMUL = 2 };
enum ImgAxis { AXIS_H = 0, AXIS_V = 1, AXIS_NONE = 2 };

__device__ __forceinline__ int clip8(int acc)
{
    if (acc >= (1 << IMG_PRECISION << 8)) return 255;
    if (acc <= 0) return 0;
    return acc >> IMG_PRECISION;
}

// numpy's trunc(((c/255) (a/255) + bg (1 - a/255)) 255), each operation rounded once
__device__ __forceinline__ int composite_byte(const double *norm, int c, int a, double bg)
{
    const double na = norm[a];
    const double arr = __dadd_rn(__dmul_rn(norm[c], na), __dmul_rn(bg, __dadd_rn(1.0, -na)));
    return (int)__dmul_rn(arr, 255.0);
}

template <int NS, int NM, int LOAD>
__device__ __forceinline__ void load_px(const uint8_t *__restrict__ src, size_t px, const double *norm, double bg,
                                        int v[NM])
{
    const uint8_t *p = src + px * NS;
    if constexpr (LOAD == LOAD_RAW) {
#pragma unroll
        for (int c = 0; c < NM; c++) v[c] = p[c];
    } else if constexpr (LOAD == LOAD_COMPOSITE) {
        const int a = p[3];
#pragma unroll
        for (int c = 0; c < 3; c++) v[c] = composite_byte(norm, p[c], a, bg);
    } else {
        const unsigned a = p[3];
#pragma unroll
        for (int c = 0; c < 3; c++) {
            const unsigned t = p[c] * a + 128u;
            v[c] = (int)(((t >> 8) + t) >> 8);
        }
        v[3] = (int)a;
    }
}

// NS source channels, NM channels carried through the passes (3, or 4 premultiplied), FINAL: write float32 planes
template <int AXIS, int NS, int NM, int LOAD, bool FINAL>
__device__ __forceinline__ void image_pass(int H_in, int W_in, int H_out, int W_out, int ksize,
                                           const int32_t *__restrict__ bounds, const int32_t *__restrict__ coeffs,
                                           const uint8_t *__restrict__ src, double bg, uint8_t *__restrict__ dst,
                                           float *__restrict__ out)
{
    __shared__ double norm[LOAD == LOAD_COMPOSITE ? 256 : 1];
    if constexpr (LOAD == LOAD_COMPOSITE) {
        for (int i = threadIdx.y * IMG_BX + threadIdx.x; i < 256; i += IMG_BX * IMG_BY)
            norm[i] = __ddiv_rn((double)i, 255.0);
        __syncthreads();
    }
    const int ox = blockIdx.x * IMG_BX + threadIdx.x, oy = blockIdx.y * IMG_BY + threadIdx.y;
    if (ox >= W_out || oy >= H_out) return;
    int v[NM];
    if constexpr (AXIS == AXIS_NONE) {
        load_px<NS, NM, LOAD>(src, (size_t)oy * W_in + ox, norm, bg, v);
    } else {
        const int o = AXIS == AXIS_H ? ox : oy;
        const int lo = bounds[2 * o], n = bounds[2 * o + 1];
        const int32_t *k = coeffs + (size_t)o * ksize;
        int acc[NM];
#pragma unroll
        for (int c = 0; c < NM; c++) acc[c] = 1 << (IMG_PRECISION - 1);
        for (int t = 0; t < n; t++) {
            const size_t px = AXIS == AXIS_H ? (size_t)oy * W_in + (lo + t) : (size_t)(lo + t) * W_in + ox;
            int s[NM];
            load_px<NS, NM, LOAD>(src, px, norm, bg, s);
            const int w = __ldg(k + t);
#pragma unroll
            for (int c = 0; c < NM; c++) acc[c] += s[c] * w;
        }
#pragma unroll
        for (int c = 0; c < NM; c++) v[c] = clip8(acc[c]);
    }
    const size_t q = (size_t)oy * W_out + ox;
    if constexpr (FINAL) {
        if constexpr (NM == 4) {   // rgba2rgbA
            const int a = v[3];
            if (a != 0 && a != 255) {
#pragma unroll
                for (int c = 0; c < 3; c++) v[c] = min(255 * v[c] / a, 255);
            }
        }
        const size_t plane = (size_t)H_out * W_out;
#pragma unroll
        for (int c = 0; c < 3; c++) out[c * plane + q] = __fdiv_rn((float)v[c], 255.0f);
    } else {
#pragma unroll
        for (int c = 0; c < NM; c++) dst[q * NM + c] = (uint8_t)v[c];
    }
}

// Three names for the profiler: the horizontal pass, the vertical pass and the pass of an unchanged size.
template <int NS, int NM, int LOAD, bool FINAL>
__global__ void __launch_bounds__(IMG_BX *IMG_BY)
    image_resample_h_kernel(int H_in, int W_in, int W_out, int ksize, const int32_t *__restrict__ bounds,
                            const int32_t *__restrict__ coeffs, const uint8_t *__restrict__ src, double bg,
                            uint8_t *__restrict__ dst, float *__restrict__ out)
{
    image_pass<AXIS_H, NS, NM, LOAD, FINAL>(H_in, W_in, H_in, W_out, ksize, bounds, coeffs, src, bg, dst, out);
}

template <int NS, int NM, int LOAD>
__global__ void __launch_bounds__(IMG_BX *IMG_BY)
    image_resample_v_kernel(int H_in, int W, int H_out, int ksize, const int32_t *__restrict__ bounds,
                            const int32_t *__restrict__ coeffs, const uint8_t *__restrict__ src, double bg,
                            float *__restrict__ out)
{
    image_pass<AXIS_V, NS, NM, LOAD, true>(H_in, W, H_out, W, ksize, bounds, coeffs, src, bg, nullptr, out);
}

template <int NS, int LOAD>
__global__ void __launch_bounds__(IMG_BX *IMG_BY)
    image_convert_kernel(int H, int W, const uint8_t *__restrict__ src, double bg, float *__restrict__ out)
{
    image_pass<AXIS_NONE, NS, 3, LOAD, true>(H, W, H, W, 0, nullptr, nullptr, src, bg, nullptr, out);
}

static dim3 img_grid(int W, int H) { return dim3((W + IMG_BX - 1) / IMG_BX, (H + IMG_BY - 1) / IMG_BY); }

// NS source channels, NM carried, LOAD the source view of the first pass
template <int NS, int NM, int LOAD>
static int image_prepare(int H_in, int W_in, double bg, int W_out, int kx, const int32_t *xb, const int32_t *xc, int H_out,
                  int ky, const int32_t *yb, const int32_t *yc, const uint8_t *src, uint8_t *tmp, float *out,
                  cudaStream_t st)
{
    const dim3 block(IMG_BX, IMG_BY);
    const bool h = W_out != W_in, v = H_out != H_in;
    if (h && v) {
        SGR_LAUNCH(K_MISC, st,
                   (image_resample_h_kernel<NS, NM, LOAD, false><<<img_grid(W_out, H_in), block, 0, st>>>(
                       H_in, W_in, W_out, kx, xb, xc, src, bg, tmp, nullptr)));
        SGR_LAUNCH(K_MISC, st,
                   (image_resample_v_kernel<NM, NM, LOAD_RAW><<<img_grid(W_out, H_out), block, 0, st>>>(
                       H_in, W_out, H_out, ky, yb, yc, tmp, bg, out)));
    } else if (h) {
        SGR_LAUNCH(K_MISC, st,
                   (image_resample_h_kernel<NS, NM, LOAD, true><<<img_grid(W_out, H_in), block, 0, st>>>(
                       H_in, W_in, W_out, kx, xb, xc, src, bg, nullptr, out)));
    } else if (v) {
        SGR_LAUNCH(K_MISC, st,
                   (image_resample_v_kernel<NS, NM, LOAD><<<img_grid(W_in, H_out), block, 0, st>>>(
                       H_in, W_in, H_out, ky, yb, yc, src, bg, out)));
    } else {
        if constexpr (LOAD == LOAD_PREMUL) {
            set_error("sgr_image_prepare: SGR_IMAGE_PREMULTIPLY needs a resize (Pillow copies an RGBA image of "
                      "unchanged size)");
            return SGR_EINVAL;
        } else {
            SGR_LAUNCH(K_MISC, st,
                       (image_convert_kernel<NS, LOAD><<<img_grid(W_in, H_in), block, 0, st>>>(H_in, W_in, src, bg,
                                                                                                out)));
        }
    }
    SGR_CUDA(cudaGetLastError());
    return SGR_OK;
}

}  // namespace sgr

using namespace sgr;

extern "C" int sgr_image_prepare(int32_t H_in, int32_t W_in, int32_t C, int32_t mode, int32_t white, int32_t W_out,
                                 int32_t kx, const int32_t *x_bounds, const int32_t *x_coeffs, int32_t H_out,
                                 int32_t ky, const int32_t *y_bounds, const int32_t *y_coeffs, const uint8_t *src,
                                 uint8_t *tmp, float *out, void *stream)
{
    const bool h = W_out != W_in, v = H_out != H_in;
    if (H_in < 1 || W_in < 1 || H_out < 1 || W_out < 1 || (C != 3 && C != 4) || (white != 0 && white != 1)) {
        set_error("sgr_image_prepare: bad sizes or channels (H_in=%d W_in=%d C=%d -> H_out=%d W_out=%d, white=%d)",
                  H_in, W_in, C, H_out, W_out, white);
        return SGR_EINVAL;
    }
    if ((mode == SGR_IMAGE_PLAIN && C == 4 && (h || v)) || (mode != SGR_IMAGE_PLAIN && C != 4) ||
        (mode == SGR_IMAGE_PREMULTIPLY && !h && !v) || mode < SGR_IMAGE_PLAIN || mode > SGR_IMAGE_PREMULTIPLY) {
        set_error("sgr_image_prepare: mode %d does not apply to C=%d at %dx%d -> %dx%d", mode, C, W_in, H_in, W_out,
                  H_out);
        return SGR_EINVAL;
    }
    if (!src || !out || (h && (kx < 1 || !x_bounds || !x_coeffs)) || (v && (ky < 1 || !y_bounds || !y_coeffs)) ||
        (h && v && !tmp)) {
        set_error("sgr_image_prepare: null pointer or empty resample table");
        return SGR_EINVAL;
    }
    const double bg = white ? 1.0 : 0.0;
    cudaStream_t st = (cudaStream_t)stream;
    if (mode == SGR_IMAGE_COMPOSITE)
        return image_prepare<4, 3, LOAD_COMPOSITE>(H_in, W_in, bg, W_out, kx, x_bounds, x_coeffs, H_out, ky, y_bounds,
                                                   y_coeffs, src, tmp, out, st);
    if (mode == SGR_IMAGE_PREMULTIPLY)
        return image_prepare<4, 4, LOAD_PREMUL>(H_in, W_in, bg, W_out, kx, x_bounds, x_coeffs, H_out, ky, y_bounds,
                                                y_coeffs, src, tmp, out, st);
    if (C == 4)
        return image_prepare<4, 3, LOAD_RAW>(H_in, W_in, bg, W_out, kx, x_bounds, x_coeffs, H_out, ky, y_bounds,
                                             y_coeffs, src, tmp, out, st);
    return image_prepare<3, 3, LOAD_RAW>(H_in, W_in, bg, W_out, kx, x_bounds, x_coeffs, H_out, ky, y_bounds, y_coeffs,
                                         src, tmp, out, st);
}
