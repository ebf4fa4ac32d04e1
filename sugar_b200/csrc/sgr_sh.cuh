// sgr_sh.cuh -- the rasterizer's spherical-harmonics colour (degree <= 3): its constants, view direction, basis,
// colour, direction Jacobian and the view-direction term of dL/dmean3D, and how the per-Gaussian passes lay SH rows
// out in shared memory.  The forward, the backward and the view-parallel finalize kernels all evaluate the basis here,
// so one Gaussian seen from one camera gets the same basis values, to the bit, in every kernel.
#pragma once
#include <type_traits>

#include "sgr_internal.cuh"

namespace sgr {

constexpr float SH_C0 = 0.28209479177387814f;
constexpr float SH_C1 = 0.4886025119029199f;
__device__ constexpr float SH_C2[5] = {1.0925484305920792f, -1.0925484305920792f, 0.31539156525252005f,
                                       -1.0925484305920792f, 0.5462742152960396f};
__device__ constexpr float SH_C3[7] = {-0.5900435899266435f, 2.890611442640554f, -0.4570457994644658f,
                                       0.3731763325901154f, -0.4570457994644658f, 1.445305721320277f,
                                       -0.5900435899266435f};

struct f3 {
    float x, y, z;
};

// The normalised view direction normalize(mean - campos) (forward.cu:20-71), in the forward's rounding chain: the
// forward is held bit-exact to the reference build, and every other kernel evaluates the basis at the same direction.
__device__ __forceinline__ f3 sh_dir(float mx, float my, float mz, float cx, float cy, float cz)
{
    const float dx = __fsub_rn(mx, cx), dy = __fsub_rn(my, cy), dz = __fsub_rn(mz, cz);
    const float len = __fsqrt_rn(__fmaf_rn(dz, dz, __fmaf_rn(dx, dx, __fmul_rn(dy, dy))));
    return {__fdiv_rn(dx, len), __fdiv_rn(dy, len), __fdiv_rn(dz, len)};
}

// Basis function K at the normalised direction d, rounded step by step as the reference build computes the colour
// (forward.cu:20-71).  The explicit roundings keep fp contraction from giving two kernels different bits.  Products
// no requested K uses are dead code.
template <int K> __device__ __forceinline__ float sh_basis(f3 d)
{
    static_assert(K >= 0 && K < 16, "degree 3 has 16 basis functions");
    const float x = d.x, y = d.y, z = d.z;
    const float xx = __fmul_rn(x, x), yy = __fmul_rn(y, y), zz = __fmul_rn(z, z);
    const float xy = __fmul_rn(x, y), yz = __fmul_rn(y, z), xz = __fmul_rn(x, z);
    const float zz2 = __fadd_rn(zz, zz), xx_yy = __fsub_rn(xx, yy);
    const float zz4_xx_yy = __fsub_rn(__fmaf_rn(zz, 4.0f, -xx), yy);
    if constexpr (K == 0) return SH_C0;
    else if constexpr (K == 1) return -__fmul_rn(y, SH_C1);
    else if constexpr (K == 2) return __fmul_rn(z, SH_C1);
    else if constexpr (K == 3) return -__fmul_rn(x, SH_C1);
    else if constexpr (K == 4) return __fmul_rn(xy, SH_C2[0]);
    else if constexpr (K == 5) return __fmul_rn(yz, SH_C2[1]);
    else if constexpr (K == 6) return __fmul_rn(__fsub_rn(__fsub_rn(zz2, xx), yy), SH_C2[2]);
    else if constexpr (K == 7) return __fmul_rn(xz, SH_C2[3]);
    else if constexpr (K == 8) return __fmul_rn(xx_yy, SH_C2[4]);
    else if constexpr (K == 9) return __fmul_rn(__fmul_rn(y, SH_C3[0]), __fmaf_rn(xx, 3.0f, -yy));
    else if constexpr (K == 10) return __fmul_rn(__fmul_rn(xy, SH_C3[1]), z);
    else if constexpr (K == 11) return __fmul_rn(__fmul_rn(y, SH_C3[2]), zz4_xx_yy);
    else if constexpr (K == 12) return __fmul_rn(__fmul_rn(z, SH_C3[3]), __fmaf_rn(yy, -3.0f, __fmaf_rn(xx, -3.0f, zz2)));
    else if constexpr (K == 13) return __fmul_rn(__fmul_rn(x, SH_C3[4]), zz4_xx_yy);
    else if constexpr (K == 14) return __fmul_rn(__fmul_rn(z, SH_C3[5]), xx_yy);
    else return __fmul_rn(__fmul_rn(x, SH_C3[6]), __fmaf_rn(yy, -3.0f, xx));
}

// f(std::integral_constant<int, K>{}) for K = K0 .. K1 - 1
template <int K0, int K1, class F> __device__ __forceinline__ void sh_for(F &&f)
{
    if constexpr (K0 < K1) {
        f(std::integral_constant<int, K0>{});
        sh_for<K0 + 1, K1>(f);
    }
}

// f(K) for the coefficients degree `deg` uses, K < (deg + 1)^2, one degree at a time.  Rows may hold fewer than 16
// coefficients, so nothing at or above (deg + 1)^2 may be touched.
template <class F> __device__ __forceinline__ void sh_for_active(int deg, F &&f)
{
    sh_for<0, 1>(f);
    if (deg > 0) {
        sh_for<1, 4>(f);
        if (deg > 1) {
            sh_for<4, 9>(f);
            if (deg > 2) sh_for<9, 16>(f);
        }
    }
}

// SH -> RGB for one channel (forward.cu:20-71), operation order as compiled for the reference: w_0 c_0, then
// fma(w_k, c_k, res).  `coef(k)` returns coefficient k of the channel.
template <class Coef> __device__ __forceinline__ float sh_channel(int deg, f3 d, Coef &&coef)
{
    float res = __fmul_rn(SH_C0, coef(0));
    sh_for_active(deg, [&](auto k) {
        constexpr int K = decltype(k)::value;
        if constexpr (K > 0) res = __fmaf_rn(sh_basis<K>(d), coef(K), res);
    });
    return res;
}

// dRGB/d(dir) for one channel: the three sums dRGBdx, dRGBdy, dRGBdz of backward.cu:36-128 (same terms, same
// grouping), from the coefficients sh_channel has just read.  `rest` points at coefficient 1 of the channel.
// The backward's view-direction term of dL/dmean3D is their dot product with dL/dRGB, so it needs these nine
// numbers per Gaussian instead of the whole SH row.
__device__ __forceinline__ void sh_channel_jacobian(int deg, const float *rest, float x, float y, float z, float &jx,
                                                    float &jy, float &jz)
{
#define SHK(k) rest[((k) - 1) * 3]
    jx = -SH_C1 * SHK(3);
    jy = -SH_C1 * SHK(1);
    jz = SH_C1 * SHK(2);
    if (deg > 1) {
        const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
        jx += SH_C2[0] * y * SHK(4) + SH_C2[2] * 2.f * -x * SHK(6) + SH_C2[3] * z * SHK(7) +
              SH_C2[4] * 2.f * x * SHK(8);
        jy += SH_C2[0] * x * SHK(4) + SH_C2[1] * z * SHK(5) + SH_C2[2] * 2.f * -y * SHK(6) +
              SH_C2[4] * 2.f * -y * SHK(8);
        jz += SH_C2[1] * y * SHK(5) + SH_C2[2] * 2.f * 2.f * z * SHK(6) + SH_C2[3] * x * SHK(7);
        if (deg > 2) {
            jx += SH_C3[0] * SHK(9) * 3.f * 2.f * xy + SH_C3[1] * SHK(10) * yz + SH_C3[2] * SHK(11) * -2.f * xy +
                  SH_C3[3] * SHK(12) * -3.f * 2.f * xz + SH_C3[4] * SHK(13) * (-3.f * xx + 4.f * zz - yy) +
                  SH_C3[5] * SHK(14) * 2.f * xz + SH_C3[6] * SHK(15) * 3.f * (xx - yy);
            jy += SH_C3[0] * SHK(9) * 3.f * (xx - yy) + SH_C3[1] * SHK(10) * xz +
                  SH_C3[2] * SHK(11) * (-3.f * yy + 4.f * zz - xx) + SH_C3[3] * SHK(12) * -3.f * 2.f * yz +
                  SH_C3[4] * SHK(13) * -2.f * xy + SH_C3[5] * SHK(14) * -2.f * yz +
                  SH_C3[6] * SHK(15) * -3.f * 2.f * xy;
            jz += SH_C3[1] * SHK(10) * xy + SH_C3[2] * SHK(11) * 4.f * 2.f * yz +
                  SH_C3[3] * SHK(12) * 3.f * (2.f * zz - xx - yy) + SH_C3[4] * SHK(13) * 4.f * 2.f * xz +
                  SH_C3[5] * SHK(14) * (xx - yy);
        }
    }
#undef SHK
}

// The view-direction term of dL/dmean3D (backward.cu:127-133): dL/ddir = (<dRGBdx, dL/dRGB>, <dRGBdy, ..>,
// <dRGBdz, ..>) from the Jacobian row `jac` the forward stored, then dnormvdv (auxiliary.h:107-117).
__device__ __forceinline__ f3 sh_dir_grad(const float *jac, f3 dRGB)
{
    return {jac[0] * dRGB.x + jac[1] * dRGB.y + jac[2] * dRGB.z, jac[3] * dRGB.x + jac[4] * dRGB.y + jac[5] * dRGB.z,
            jac[6] * dRGB.x + jac[7] * dRGB.y + jac[8] * dRGB.z};
}
__device__ __forceinline__ void add_dnormvdv(f3 o, f3 ddir, f3 &dmean)
{
    const float sum2 = o.x * o.x + o.y * o.y + o.z * o.z;
    const float invsum32 = 1.0f / sqrtf(sum2 * sum2 * sum2);
    dmean.x += ((+sum2 - o.x * o.x) * ddir.x - o.y * o.x * ddir.y - o.z * o.x * ddir.z) * invsum32;
    dmean.y += (-o.x * o.y * ddir.x + (sum2 - o.y * o.y) * ddir.y - o.z * o.y * ddir.z) * invsum32;
    dmean.z += (-o.x * o.z * ddir.x - o.y * o.z * ddir.y + (sum2 - o.z * o.z) * ddir.z) * invsum32;
}

// One view's SH gradient of one Gaussian, accumulated: acc[3k + c] += basis_k(d) * g_c (the dL_dsh part of
// backward.cu:20-139 is this outer product per view).
__device__ __forceinline__ void sh_accumulate(int deg, float *acc, f3 d, f3 g)
{
    sh_for_active(deg, [&](auto k) {
        constexpr int K = decltype(k)::value;
        const float w = sh_basis<K>(d);
        acc[K * 3] = fmaf(w, g.x, acc[K * 3]);
        acc[K * 3 + 1] = fmaf(w, g.y, acc[K * 3 + 1]);
        acc[K * 3 + 2] = fmaf(w, g.z, acc[K * 3 + 2]);
    });
}

// Row stride in floats of the per-Gaussian passes' shared-memory SH rows (M coefficients x 3): an odd number of
// 16-byte units when the rows can move as 16-byte copies (`vec_ok`: the global rows are 16-byte aligned), else an
// odd number of floats -- conflict-free either way.  *vec = 1 selects the 16-byte copies.
__host__ __device__ inline int sh_row_stride(int M, bool vec_ok, int *vec)
{
    const int row_f = M * 3;
    *vec = (row_f % 4) == 0 && vec_ok;
    if (*vec) {
        int s4 = row_f / 4;
        if ((s4 & 1) == 0) s4 += 1;
        return s4 * 4;
    }
    return (row_f & 1) ? row_f : row_f + 1;
}

// The n rows of row_f floats that are contiguous in global memory and `stride` floats apart in shared memory, walked
// by the CTA's T threads in units of W floats (4: 16-byte copies, see sh_row_stride): f(global offset, shared offset)
// per unit, in coalesced global order.  A thread's (row, unit) advances without divisions.
template <int T, int W, class F> __device__ __forceinline__ void sh_rows_walk(int n, int row_f, int stride, F &&f)
{
    const int row_w = row_f / W, total = n * row_w;
    int r = threadIdx.x / row_w, c = threadIdx.x - r * row_w;
    const int dr = T / row_w, dc = T - dr * row_w;
    for (int i = threadIdx.x; i < total; i += T) {
        f(i * W, r * stride + c * W);
        r += dr;
        c += dc;
        if (c >= row_w) {
            c -= row_w;
            r++;
        }
    }
}

}  // namespace sgr
